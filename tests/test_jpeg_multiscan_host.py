"""Host side of the multi-scan JPEG path: pg_jpeg_parse_multiscan against pg_jpeg_parse on every single-scan golden,
the frame and the scan scripts (restart intervals, segment counts, dependency levels) of tests/golden/jpeg_multiscan.npz
(tools/make_jpeg_multiscan_golden.py), each rejection's status and reason, the routing option of the pre-processor,
workspace sizing of mixed batches and the ctypes mirror of pg_jpeg_scan.  No GPU needed."""
import ctypes as C
import io
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def _load(name):
    G = np.load(os.path.join(GOLD, name))
    jo, po = G["jpg_off"], G["px_off"]
    out = []
    for k in range(int(G["count"])):
        d = dict(name=str(G["name"][k]), kind=str(G["kind"][k]), status=int(G["status"][k]),
                 data=G["jpg"][jo[k]:jo[k + 1]].tobytes(), shape=tuple(int(x) for x in G["shape"][k]),
                 px=G["px"][po[k]:po[k + 1]] if po[k + 1] > po[k] else None)
        if "reason" in G:
            d["reason"] = str(G["reason"][k])
            d["scans"] = G["scans"][G["scan_off"][k]:G["scan_off"][k + 1]].tolist()
        out.append(d)
    return out


@pytest.fixture(scope="module")
def multi():
    return _load("jpeg_multiscan.npz")


@pytest.fixture(scope="module")
def single():
    return _load("jpeg.npz")


def test_installed_pillow_reproduces_the_multiscan_goldens(multi):
    Image = pytest.importorskip("PIL.Image")
    n = 0
    for g in multi:
        if g["kind"] == "ok" and g["px"] is not None:
            px = np.asarray(Image.open(io.BytesIO(g["data"])).convert("RGB"))
            assert np.array_equal(px.reshape(-1), g["px"]), g["name"]
            n += 1
    assert n >= 150


def test_multiscan_parser_returns_the_single_scan_info_for_every_single_scan_file(single):
    from pigeon_b200 import jpeg
    n = 0
    for g in single:
        a, wa = jpeg.parse(g["data"])
        b, wb = jpeg.parse(g["data"], multiscan=True)
        if a.status == jpeg.OK:
            assert bytes(a) == bytes(b), g["name"]
            assert not jpeg.is_multiscan(b)
            n += 1
    assert n >= 300


def test_multiscan_frames_and_scripts(multi):
    from pigeon_b200 import jpeg
    n = 0
    for g in multi:
        if g["kind"] != "ok":
            continue
        info, why = jpeg.parse(g["data"], multiscan=True)
        assert info.status == jpeg.OK, (g["name"], why)
        assert jpeg.is_multiscan(info), g["name"]
        assert (info.height, info.width) == g["shape"][:2], g["name"]
        assert jpeg.parse(g["data"])[0].status == jpeg.UNSUPPORTED, g["name"]   # the default parser still refuses it
        got = [[s.components, *s.component, s.ss, s.se, s.ah, s.al, s.restart_interval, s.num_segments, s.level]
               for s in jpeg.scans(g["data"])]
        assert got == g["scans"], g["name"]
        assert info.num_segments == sum(r[9] for r in got), g["name"]
        assert info.restart_interval == got[0][8], g["name"]
        assert g["data"][info.scan_offset + info.scan_bytes:] == b"\xff\xd9", g["name"]
        n += 1
    assert n >= 150
    by = {g["name"]: g for g in multi}
    assert [s.level for s in jpeg.scans(by["420 progressive q75"]["data"])] == [1] * 5 + [2] * 4 + [3]
    assert {s.level for s in jpeg.scans(by["420 SOF0 non-interleaved Y Cb Cr"]["data"])} == {1}
    assert max(s.level for s in jpeg.scans(by["420 deep successive approximation"]["data"])) == 14
    assert jpeg.parse(by["420 SOF1 non-interleaved Y Cb Cr"]["data"], multiscan=True)[0].sof == 0xC1


def test_baseline_file_lists_one_scan(single):
    from pigeon_b200 import jpeg
    g = next(g for g in single if g["name"] == "444 restart blocks 3")
    info = jpeg.parse(g["data"])[0]
    (s,) = jpeg.scans(g["data"])
    assert (s.components, list(s.component), s.ss, s.se, s.ah, s.al, s.level) == (3, [0, 1, 2], 0, 63, 0, 0, 1)
    assert (s.restart_interval, s.num_segments) == (info.restart_interval, info.num_segments)


def test_every_rejection_carries_its_status_and_reason(multi):
    from pigeon_b200 import jpeg
    seen = 0
    for g in multi:
        if g["kind"] == "ok":
            continue
        info, why = jpeg.parse(g["data"], multiscan=True)
        if g["status"] == jpeg.BAD_CODE:                 # found by the decode kernel, not by the marker walk
            assert info.status == jpeg.OK, g["name"]
            continue
        assert info.status == g["status"], (g["name"], info.status, why)
        assert g["reason"] in why, (g["name"], why)
        if info.status != jpeg.OK:
            with pytest.raises(ValueError, match=g["reason"] or "."):
                jpeg.scans(g["data"])
        seen += 1
    assert seen >= 12


def test_single_scan_parser_rejections_are_unchanged_under_the_multiscan_parser(single):
    from pigeon_b200 import jpeg
    for name in ("CMYK", "SOF3 lossless", "12-bit", "4:4:0 sampling", "Adobe transform 0", "truncated header",
                 "not a JPEG", "truncated file", "wrong RST number"):
        g = next(g for g in single if g["name"] == name)
        a, wa = jpeg.parse(g["data"])
        b, wb = jpeg.parse(g["data"], multiscan=True)
        assert (a.status, wa) == (b.status, wb), name
    g = next(g for g in single if g["name"] == "progressive")
    assert jpeg.parse(g["data"], multiscan=True)[0].status == jpeg.OK


def test_routing_with_and_without_the_multiscan_option(multi, single):
    from pigeon_b200.preprocess import route_encoded
    by = {g["name"]: g for g in multi}
    for name in ("420 progressive q75", "gray progressive q5", "444 SOF0 non-interleaved Cr Y Cb"):
        assert route_encoded(by[name]["data"])[0] == "host", name
        assert route_encoded(by[name]["data"], multiscan=True)[0] == "gpu", name
    for name in ("incomplete progression", "bogus progression: wrong Ah", "too many scans"):
        assert route_encoded(by[name]["data"], multiscan=True)[0] == "host", name
    base = next(g for g in single if g["name"] == "420 photo q90")
    assert route_encoded(base["data"], multiscan=True)[0] == "gpu"
    with pytest.raises(ValueError, match="corrupt JPEG"):
        route_encoded(by["truncated progressive file"]["data"], multiscan=True)


def test_workspace_bytes_accepts_mixed_batches(multi, single):
    from pigeon_b200 import _lib, jpeg
    lib = _lib.load()
    files = [next(g for g in single if g["name"] == "420 photo q90")["data"]] + \
        [g["data"] for g in multi if g["name"] in ("420 progressive q75", "gray one scan per coefficient", "too many scans")]
    infos = [jpeg.parse(f, multiscan=True)[0] for f in files]
    arr = (_lib.JpegInfo * len(infos))(*infos)
    mixed = lib.pg_jpeg_workspace_bytes(arr, len(infos), sum(len(f) for f in files))
    base = lib.pg_jpeg_workspace_bytes(arr, 1, len(files[0]))
    assert mixed > base > 0


def test_jpeg_scan_mirror_matches_the_header_layout(tmp_path):
    from pigeon_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    cls = _lib.JpegScan
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "pigeon_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(pg_jpeg_scan));']
    lines += [f'  printf("{f} %zu\\n", offsetof(pg_jpeg_scan, {f}));' for f, _ in cls._fields_]
    lines += [f'  printf("MULTISCAN %d\\nMAX_SCANS %d\\n", PG_JPEG_MULTISCAN, PG_JPEG_MAX_SCANS);', "  return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    r = subprocess.run([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o",
                        str(tmp_path / "layout")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = dict(line.split() for line in subprocess.run([str(tmp_path / "layout")], capture_output=True,
                                                       text=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f
    from pigeon_b200 import jpeg
    assert (int(got["MULTISCAN"]), int(got["MAX_SCANS"])) == (jpeg.MULTISCAN, jpeg.MAX_SCANS)
