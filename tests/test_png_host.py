"""PNG decoding without a GPU: the chunk walk (pg_png_parse) and routing of every golden in tests/golden/png.npz, the
device's inflate / unfilter / convert functions run on the CPU (pg_png_decode_host) against Pillow's pixels, the
inflate against `zlib.decompress` on a seeded matrix of streams and corruptions, the ctypes mirror of pg_png_info,
and the kernels' spill check."""
import hashlib
import os
import re
import shutil
import subprocess
import zlib

import numpy as np
import pytest

from pigeon_b200 import png

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "png.npz")


def _load():
    G = np.load(GOLD)
    off, po, so = G["png_off"], G["px_off"], G["sample_off"]
    out = []
    for k in range(int(G["count"])):
        out.append(dict(name=str(G["name"][k]), kind=str(G["kind"][k]), status=int(G["status"][k]),
                        data=G["png"][off[k]:off[k + 1]].tobytes(), shape=tuple(int(x) for x in G["shape"][k]),
                        px=G["px"][po[k]:po[k + 1]] if po[k + 1] > po[k] else None,
                        sha=G["sha"][k].tobytes() if so[k + 1] > so[k] else None,
                        sample=G["sample"][so[k]:so[k + 1]] if so[k + 1] > so[k] else None,
                        error=str(G["error"][k])))
    return out


@pytest.fixture(scope="module")
def gold():
    return _load()


def same(a, g):
    if g["shape"][0] == 0 or a.shape != g["shape"]:
        return False
    if g["px"] is not None:
        return np.array_equal(a.reshape(-1), g["px"])
    return hashlib.sha256(a.tobytes()).digest() == g["sha"] and np.array_equal(a[::37, ::23].reshape(-1), g["sample"])


def test_golden_covers_the_cases(gold):
    kinds = {}
    for g in gold:
        kinds[g["kind"]] = kinds.get(g["kind"], 0) + 1
    assert kinds["ok"] >= 300 and kinds["host"] >= 12 and kinds["fallback"] >= 14 and kinds["flip"] >= 40
    names = " ".join(g["name"] for g in gold)
    for ct, depths in ((0, (1, 2, 4, 8, 16)), (2, (8, 16)), (3, (1, 2, 4, 8)), (4, (8, 16)), (6, (8, 16))):
        for d in depths:
            for f in range(5):
                assert f"ct {ct} depth {d} 33x70 filter {f}" in names


def test_parse_status_and_route_of_every_golden(gold):
    from pigeon_b200.preprocess import route_encoded
    for g in gold:
        info, why = png.parse(g["data"])
        if g["kind"] == "host":
            assert info.status == g["status"] and why, g["name"]
            assert route_encoded(g["data"], png=True)[0] == "host", g["name"]
        else:
            assert info.status == png.OK and why == "", (g["name"], why)
            assert route_encoded(g["data"], png=True)[0] == "gpu", g["name"]
        # without the option every PNG goes to Pillow, as before
        assert route_encoded(g["data"])[0] == "host", g["name"]


def test_reasons_name_what_was_refused(gold):
    why = {g["name"]: png.parse(g["data"])[1] for g in gold if g["kind"] == "host"}
    assert "interlaced" in why["Adam7 interlaced"] and "APNG" in why["APNG"]
    assert "CRC" in why["bad CRC in tEXt before IDAT"] and "not consecutive" in why["IDAT runs split by a tEXt chunk"]
    assert "MAX_TEXT_CHUNK" in why["zTXt above MAX_TEXT_CHUNK"]


def test_more_pixels_than_max_image_pixels_go_to_pillow(gold, monkeypatch):
    from PIL import Image
    g = next(g for g in gold if g["name"] == "pillow RGB 7x13 level 6")
    monkeypatch.setattr(Image, "MAX_IMAGE_PIXELS", 90)
    info, why = png.parse(g["data"])
    assert info.status == png.UNSUPPORTED and "MAX_IMAGE_PIXELS" in why
    monkeypatch.setattr(Image, "MAX_IMAGE_PIXELS", None)
    assert png.parse(g["data"])[0].status == png.OK


def test_host_decode_equals_pillow_on_every_gpu_route_golden(gold):
    cases = [g for g in gold if g["kind"] != "host"]
    out, status = png.decode_host([g["data"] for g in cases])
    for g, a, st in zip(cases, out, status):
        if g["kind"] == "ok":
            assert st == png.OK and same(a, g), g["name"]
        elif g["kind"] == "fallback":
            assert st == g["status"], (g["name"], st)
        elif st == png.OK:                    # a bit flip the stream survives: then Pillow decodes the same pixels
            assert same(a, g), g["name"]


def _streams():
    """Seeded zlib streams over every level, strategy and window size, of 2 B to 1 MB: (raw, stream).  Each raw starts
    with a 0 byte, so that it is one PNG row with filter type None."""
    rng = np.random.default_rng(11)
    strategies = [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED]
    out = []
    for k, size in enumerate((2, 3, 17, 259, 1000, 32768, 32770, 70000, 300000, 1 << 20)):
        if k % 3 == 0:
            body = rng.integers(0, 256, size - 1, dtype=np.uint8).tobytes()
        elif k % 3 == 1:
            body = np.repeat(rng.integers(0, 4, size // 50 + 1, dtype=np.uint8), 50)[:size - 1].tobytes()
        else:
            body = (np.arange(size - 1) // 7 % 256).astype(np.uint8).tobytes()
        raw = b"\0" + body
        for level in range(10):
            c = zlib.compressobj(level, zlib.DEFLATED, 9 + (k + level) % 7, 8, strategies[(k + level) % 5])
            out.append((raw, c.compress(raw) + c.flush()))
    return out


def _inflate_as_png(stream, raw_len):
    """pg_png_decode_host on a one-row 8-bit grey PNG of raw_len - 1 pixels whose IDAT is `stream`: (status, the row's
    bytes or None)."""
    import struct

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)
    f = png.SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", raw_len - 1, 1, 8, 0, 0, 0, 0)) + \
        chunk(b"IDAT", stream) + chunk(b"IEND", b"")
    out, status = png.decode_host([f])
    return int(status[0]), (None if out[0] is None else out[0][0, :, 0].tobytes())


def test_host_inflate_equals_zlib_on_a_seeded_matrix():
    streams = _streams()
    assert len(streams) == 100
    for raw, stream in streams:
        assert zlib.decompress(stream) == raw
        st, got = _inflate_as_png(stream, len(raw))
        assert st == png.OK and got == raw[1:], (len(raw), st)


def test_host_inflate_is_never_more_lenient_than_zlib():
    """Seeded bit flips and truncations: never OK where zlib raises, never OK with other bytes than zlib's."""
    rng = np.random.default_rng(5)
    verdicts = set()
    for raw, good in _streams()[:80:3]:
        for _ in range(12):
            bad = bytearray(good)
            for _ in range(int(rng.integers(1, 4))):
                p = int(rng.integers(0, len(bad)))
                bad[p] ^= 1 << int(rng.integers(0, 8))
            if rng.integers(0, 4) == 0:
                bad = bad[:int(rng.integers(0, len(bad)))]
            bad = bytes(bad)
            try:
                ref = zlib.decompress(bad)
            except zlib.error:
                ref = None
            st, got = _inflate_as_png(bad, len(raw))
            verdicts.add(st)
            if st == png.OK:
                assert ref is not None, "OK where zlib raises"
                assert ref[:len(raw)] == b"\0" + got, "OK with other bytes than zlib's"
    assert len(verdicts) >= 3


def test_png_info_ctypes_mirror_matches_the_header_layout(tmp_path):
    import ctypes as C
    from pigeon_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    cls = _lib.PngInfo
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "pigeon_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(pg_png_info));']
    lines += [f'  printf("{f} %zu\\n", offsetof(pg_png_info, {f}));' for f, _ in cls._fields_]
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


def test_png_kernels_do_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    from pigeon_b200 import _build
    r = subprocess.run([nvcc, *_build._flags(), "-Xptxas", "-v", "-I", os.path.join(ROOT, "include"), "-c",
                        os.path.join(ROOT, "pigeon_b200", "csrc", "png.cu"), "-o", str(tmp_path / "png.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for kernel in ("png_inflate_kernel", "png_unfilter_kernel", "png_rgb_kernel"):
        m = re.search(rf"Compiling entry function '\S*{kernel}\S*'.*?\n(.*?spill stores.*?)\n", r.stderr, re.S)
        assert m, r.stderr
        assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", m.group(1)), m.group(1)
