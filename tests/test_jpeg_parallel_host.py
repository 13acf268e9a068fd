"""The chunked, self-synchronising Huffman decoder of csrc/jpeg.cu on the CPU, through pg_jpeg_entropy_host (the same
__host__ __device__ chunk functions as chunked_kernel, in its order of rounds): coefficients and per-image status equal
the one-thread-per-segment decoder's at every chunk size, on the goldens, on Pillow-encoded photos of every subsampling
and on seeded corruptions of the entropy-coded data.  Plus the new kernel's spill check.  No GPU needed."""
import io
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from pigeon_b200 import jpeg, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CHUNKS = [1, 2, 3, 5, 8, 13, 64, 1024, -1]           # forced sizes in de-stuffed bytes; -1 = the automatic size


def _block_ranges(files):
    """[start, end) of each file's blocks in entropy_host's coefficient array, None for a file it does not decode."""
    out, b = [], 0
    for f in files:
        info = jpeg.parse(f)[0]
        if info.status != jpeg.OK:
            out.append(None)
            continue
        three = info.components == 3
        hmax, vmax = (info.h_samp[0], info.v_samp[0]) if three else (1, 1)
        mcus = -(-info.width // (8 * hmax)) * -(-info.height // (8 * vmax))
        n = mcus * (sum(info.h_samp[c] * info.v_samp[c] for c in range(3)) if three else 1)
        out.append((b, b + n))
        b += n
    return out


def _check_same(files, chunks=CHUNKS):
    """Every chunk size gives the sequential decoder's status, and its coefficients wherever the status is OK."""
    ref_coef, ref_st, ref_rounds = jpeg.entropy_host(files, 0)
    assert (ref_rounds == 0).all()
    ranges = _block_ranges(files)
    for cb in chunks:
        coef, st, rounds = jpeg.entropy_host(files, cb)
        assert st.tolist() == ref_st.tolist(), cb
        for i, r in enumerate(ranges):
            if r is not None and st[i] == jpeg.OK:
                assert np.array_equal(coef[r[0]:r[1]], ref_coef[r[0]:r[1]]), (cb, i)
                assert rounds[i] >= 1
    return ref_st


def _encode(img, q=90, subsampling=2, optimize=False, gray=False, **kw):
    from PIL import Image
    f = io.BytesIO()
    im = Image.fromarray(img).convert("L") if gray else Image.fromarray(img)
    if gray:
        im.save(f, "JPEG", quality=q, optimize=optimize, **kw)
    else:
        im.save(f, "JPEG", quality=q, subsampling=subsampling, optimize=optimize, **kw)
    return f.getvalue()


def test_jpeg_goldens_ok_and_corrupt():
    G = np.load(os.path.join(GOLD, "jpeg.npz"))
    jo = G["jpg_off"]
    kinds = [str(k) for k in G["kind"]]
    files = [G["jpg"][jo[k]:jo[k + 1]].tobytes() for k in range(int(G["count"])) if kinds[k] in ("ok", "corrupt")]
    expect = [int(G["status"][k]) for k in range(int(G["count"])) if kinds[k] in ("ok", "corrupt")]
    st = _check_same(files)
    assert st.tolist() == expect
    assert {jpeg.OVERRUN, jpeg.BAD_CODE} <= set(st.tolist())


def test_benchmark_golden_baseline_jpegs():
    B = np.load(os.path.join(GOLD, "benchmark.npz"))
    off = B["off"]
    files = [B["data"][off[k]:off[k + 1]].tobytes() for k in range(int(B["count"])) if str(B["route"][k]) == "gpu"]
    assert len(files) >= 10
    assert (_check_same(files) == jpeg.OK).all()


@pytest.mark.parametrize("layout", ["444", "422", "420", "gray"])
@pytest.mark.parametrize("optimize", [False, True])
def test_pillow_photos_every_subsampling_and_size(layout, optimize):
    pytest.importorskip("PIL")
    sizes = [(1, 1), (1, 37), (29, 1), (7, 13), (17, 33), (63, 65), (121, 250), (480, 641)]
    sub = {"444": 0, "422": 1, "420": 2, "gray": 0}[layout]
    files = [_encode(synthetic.synthetic_photo(h, w, seed=h * 7 + w), q=85, subsampling=sub, optimize=optimize,
                     gray=layout == "gray") for h, w in sizes]
    assert (_check_same(files) == jpeg.OK).all()


@pytest.mark.parametrize("layout", ["444", "420", "gray"])
def test_large_photos(layout):
    pytest.importorskip("PIL")
    sub = {"444": 0, "420": 2, "gray": 0}[layout]
    files = [_encode(synthetic.synthetic_photo(1536, 2048, seed=5), q=90, subsampling=sub, gray=layout == "gray"),
             _encode(synthetic.synthetic_photo(771, 1029, seed=6), q=75, subsampling=sub, optimize=True,
                     gray=layout == "gray")]
    _, _, rounds = jpeg.entropy_host(files, -1)
    assert (rounds >= 1).all() and (rounds <= 256).all()
    assert (_check_same(files, [1, 13, 64, -1]) == jpeg.OK).all()


def test_dense_stuffing_on_and_around_chunk_boundaries():
    pytest.importorskip("PIL")
    rng = np.random.default_rng(3)
    noise = rng.integers(0, 256, size=(96, 160, 3), dtype=np.uint8)
    sat = np.zeros((64, 128, 3), dtype=np.uint8)
    sat[:, ::2] = 255                                  # saturated stripes: large DC / AC values at q100
    files = [_encode(noise, q=100, subsampling=0), _encode(noise, q=100, subsampling=2, optimize=True),
             _encode(sat, q=100, subsampling=0), _encode(noise, q=100, gray=True)]
    for f in files:
        assert f.count(b"\xff\x00") >= 40             # stuffed bytes land on and beside many chunk boundaries
    assert (_check_same(files, [1, 2, 3, 4, 5, 7, 8, 13, 64, 1024, -1]) == jpeg.OK).all()


def _scan_range(f):
    info = jpeg.parse(f)[0]
    assert info.status == jpeg.OK
    return int(info.scan_offset), int(info.scan_offset + info.scan_bytes)


def test_seeded_corruptions_of_the_entropy_data():
    pytest.importorskip("PIL")
    base = [_encode(synthetic.synthetic_photo(120, 200, seed=11), q=90, subsampling=2),
            _encode(synthetic.synthetic_photo(90, 131, seed=12), q=80, subsampling=0, optimize=True),
            _encode(synthetic.synthetic_photo(77, 150, seed=13), q=95, gray=True),
            _encode(synthetic.synthetic_photo(64, 200, seed=14), q=90, subsampling=1)]
    rng = np.random.default_rng(2024)
    files = []
    for seed in range(60):
        f = bytearray(base[seed % len(base)])
        a, b = _scan_range(bytes(f))
        kind = seed % 3
        if kind == 0:                                  # bit flips
            for _ in range(1 + seed % 4):
                p = int(rng.integers(a, b))
                f[p] ^= 1 << int(rng.integers(0, 8))
        elif kind == 1:                                # a run of random bytes
            p = int(rng.integers(a, b - 1))
            k = int(rng.integers(1, min(40, b - p)))
            f[p:p + k] = rng.integers(0, 256, size=k, dtype=np.uint8).tobytes()
        else:                                          # the scan cut short before EOI
            p = int(rng.integers(a, b))
            f = f[:p] + b"\xff\xd9"
        files.append(bytes(f))
    st = _check_same(files, [1, 3, 8, 64, -1])
    # the batch exercises every entropy-data outcome the decoders report
    assert {jpeg.OK, jpeg.BAD_CODE, jpeg.OVERRUN} <= set(st.tolist())


def test_multiscan_info_is_refused():
    pytest.importorskip("PIL")
    from pigeon_b200 import _lib
    f = _encode(synthetic.synthetic_photo(32, 32), progressive=True)
    info = jpeg.parse(f, multiscan=True)[0]
    assert jpeg.is_multiscan(info)
    lib = _lib.load()
    packed = np.frombuffer(f, dtype=np.uint8)
    offsets = np.array([0, len(f)], dtype=np.int64)
    status = np.zeros(1, dtype=np.int32)
    assert lib.pg_jpeg_entropy_host(packed.ctypes.data, offsets.ctypes.data, (_lib.JpegInfo * 1)(info), 1, 0, None,
                                    status.ctypes.data, None) == -1
    assert b"multi-scan" in lib.pg_last_error()


def test_schedule_switch_rejects_bad_arguments():
    from pigeon_b200 import _lib
    lib = _lib.load()
    assert lib.pg_jpeg_set_schedule(3, 0) == 1 and lib.pg_jpeg_set_schedule(-1, 0) == 1
    assert lib.pg_jpeg_set_schedule(0, -5) == 1
    assert lib.pg_jpeg_set_schedule(0, 0) == 0


def test_chunked_kernel_does_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    from pigeon_b200 import _build
    r = subprocess.run([nvcc, *_build._flags(), "-Xptxas", "-v", "-I", os.path.join(ROOT, "include"), "-c",
                        os.path.join(ROOT, "pigeon_b200", "csrc", "jpeg.cu"), "-o", str(tmp_path / "jpeg.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    m = re.search(r"Compiling entry function '\S*chunked_kernel\S*'.*?\n(.*?spill stores.*?)\n", r.stderr, re.S)
    assert m, r.stderr
    assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", m.group(1)), m.group(1)
