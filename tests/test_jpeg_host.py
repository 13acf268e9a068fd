"""Host side of the GPU JPEG decoder: the golden fixtures against the installed Pillow, the library's marker walk
(pg_jpeg_parse) against an independent Python walk, the rejection reasons, the ctypes mirror of pg_jpeg_info and the
pre-processor's routing of encoded files.  No GPU needed."""
import ctypes as C
import io
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "jpeg.npz")


def _load_gold():
    """tests/golden/jpeg.npz (tools/make_jpeg_golden.py) as one dict per case."""
    G = np.load(GOLD)
    jo, po = G["jpg_off"], G["px_off"]
    out = []
    for k in range(int(G["count"])):
        shape = tuple(int(x) for x in G["shape"][k])
        out.append(dict(name=str(G["name"][k]), kind=str(G["kind"][k]), status=int(G["status"][k]),
                        data=G["jpg"][jo[k]:jo[k + 1]].tobytes(),
                        px=G["px"][po[k]:po[k + 1]].reshape(shape) if po[k + 1] > po[k] else None,
                        sha=G[f"sha{k}"].tobytes() if f"sha{k}" in G else None,
                        sample=G[f"sample{k}"] if f"sample{k}" in G else None))
    return out


@pytest.fixture(scope="module")
def gold():
    return _load_gold()


def test_installed_pillow_reproduces_every_golden_decode(gold):
    import hashlib
    Image = pytest.importorskip("PIL.Image")
    n = 0
    for g in gold:
        if g["px"] is None and g["sha"] is None:
            continue
        px = np.asarray(Image.open(io.BytesIO(g["data"])).convert("RGB"))
        if g["px"] is not None:
            assert np.array_equal(px, g["px"]), g["name"]
        else:
            assert hashlib.sha256(px.tobytes()).digest() == g["sha"] and np.array_equal(px[::37, ::23], g["sample"]), g["name"]
        n += 1
    assert n >= 300


def _walk(b):
    """Independent marker walk (ITU T.81 B.2): frame, tables, DRI and the start of the entropy-coded data."""
    out = dict(qt={}, dc={}, ac={}, ri=0)
    p = 2
    while True:
        while b[p] == 0xFF and b[p + 1] == 0xFF:
            p += 1
        m, L = b[p + 1], b[p + 2] << 8 | b[p + 3]
        s = b[p + 4:p + 2 + L]
        if m in (0xC0, 0xC1):
            out.update(sof=m, precision=s[0], height=s[1] << 8 | s[2], width=s[3] << 8 | s[4], nf=s[5],
                       comps=[(s[6 + 3 * i], s[7 + 3 * i] >> 4, s[7 + 3 * i] & 15, s[8 + 3 * i]) for i in range(s[5])])
        elif m == 0xDB:
            o = 0
            while o < len(s):
                pq, tq = s[o] >> 4, s[o] & 15
                w = 2 if pq else 1
                out["qt"][tq] = [int.from_bytes(s[o + 1 + w * k:o + 1 + w * k + w], "big") for k in range(64)]
                o += 1 + 64 * w
        elif m == 0xC4:
            o = 0
            while o < len(s):
                tc, th = s[o] >> 4, s[o] & 15
                bits = list(s[o + 1:o + 17])
                (out["ac"] if tc else out["dc"])[th] = (bits, list(s[o + 17:o + 17 + sum(bits)]))
                o += 17 + sum(bits)
        elif m == 0xDD:
            out["ri"] = s[0] << 8 | s[1]
        elif m == 0xDA:
            out["scan"] = [(s[1 + 2 * i], s[2 + 2 * i] >> 4, s[2 + 2 * i] & 15) for i in range(s[0])]
            out["scan_offset"] = p + 2 + L
            return out
        p += 2 + L


def test_parser_agrees_with_a_python_marker_walk(gold):
    from pigeon_b200 import jpeg
    n = 0
    for g in gold:
        if g["kind"] != "ok":
            continue
        info, why = jpeg.parse(g["data"])
        assert info.status == 0, (g["name"], why)
        w = _walk(g["data"])
        name = g["name"]
        assert (info.sof, info.precision, info.height, info.width, info.components) == \
            (w["sof"], w["precision"], w["height"], w["width"], w["nf"]), name
        if g["px"] is not None:
            assert g["px"].shape == (info.height, info.width, 3), name
        assert info.restart_interval == w["ri"] and info.scan_offset == w["scan_offset"], name
        for c, (cid, h, v, tq) in enumerate(w["comps"]):
            assert (info.component_id[c], info.h_samp[c], info.v_samp[c], info.quant_table[c]) == (cid, h, v, tq), name
            assert list(info.qt[tq]) == w["qt"][tq], name
            _, td, ta = w["scan"][c]
            assert (info.dc_table[c], info.ac_table[c]) == (td, ta), name
            bits, vals = w["dc"][td]
            assert list(info.dc_bits[td]) == bits and list(info.dc_vals[td])[:len(vals)] == vals, name
            bits, vals = w["ac"][ta]
            assert list(info.ac_bits[ta]) == bits and list(info.ac_vals[ta])[:len(vals)] == vals, name
        mcus = -(-info.width // (8 * info.h_samp[0])) * -(-info.height // (8 * info.v_samp[0])) if info.components == 3 \
            else -(-info.width // 8) * -(-info.height // 8)
        assert info.num_segments == (-(-mcus // w["ri"]) if w["ri"] else 1), name
        assert g["data"][info.scan_offset + info.scan_bytes:] == b"\xff\xd9", name
        n += 1
    assert n >= 300
    assert any(jpeg.parse(g["data"])[0].sof == 0xC1 for g in gold if "16-bit" in g["name"])


EXPECTED_REASON = {"progressive": "progressive", "CMYK": "4 components", "SOF3 lossless": "lossless",
                   "SOF9 arithmetic": "arithmetic", "12-bit": "12-bit", "height 0 (DNL)": "DNL",
                   "4:4:0 sampling": "sampling", "two scans": "more than one scan", "Adobe transform 0": "RGB",
                   "component ids RGB": "RGB", "truncated header": "truncated", "not a JPEG": "SOI",
                   "truncated file": "EOI", "wrong RST number": "RST3"}


def test_parser_gives_the_reason_of_each_rejection(gold):
    from pigeon_b200 import jpeg
    seen = set()
    for g in gold:
        if g["kind"] == "ok":
            continue
        info, why = jpeg.parse(g["data"])
        if g["status"] in (jpeg.BAD_CODE, jpeg.OVERRUN):     # found by the decode kernel, not by the marker walk
            assert info.status == jpeg.OK, g["name"]
            continue
        assert info.status == g["status"], (g["name"], info.status, why)
        assert EXPECTED_REASON[g["name"]] in why, (g["name"], why)
        seen.add(g["name"])
    assert seen == set(EXPECTED_REASON)


def test_jpeg_info_mirror_matches_the_header_layout(tmp_path):
    from pigeon_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    cls = _lib.JpegInfo
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "pigeon_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(pg_jpeg_info));']
    lines += [f'  printf("{f} %zu\\n", offsetof(pg_jpeg_info, {f}));' for f, _ in cls._fields_]
    lines += ["  return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    r = subprocess.run([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"), "-o",
                        str(tmp_path / "layout")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = dict(line.split() for line in subprocess.run([str(tmp_path / "layout")], capture_output=True,
                                                       text=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(got[f]) == getattr(cls, f).offset, f


def test_processor_routes_encoded_files(gold):
    from pigeon_b200.preprocess import route_encoded
    by_name = {g["name"]: g for g in gold}
    for name in ("420 photo q90", "444 restart rows 1", "gray q75", "422 16-bit qtables", "420 4000x3000 q50"):
        assert route_encoded(by_name[name]["data"])[0] == "gpu", name
    for name in ("progressive", "CMYK", "SOF3 lossless", "12-bit", "Adobe transform 0", "two scans", "truncated header"):
        assert route_encoded(bytearray(by_name[name]["data"]))[0] == "host", name
    assert route_encoded(memoryview(b"\x89PNG\r\n\x1a\n" + b"\0" * 40))[0] == "host"
    for name in ("truncated file", "wrong RST number"):
        with pytest.raises(ValueError, match="corrupt JPEG"):
            route_encoded(by_name[name]["data"])
