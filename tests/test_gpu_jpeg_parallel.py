"""Chunked, self-synchronising Huffman decoding on the GPU (csrc/jpeg.cu chunked_kernel): under every schedule of
pg_jpeg_set_schedule the decoder gives Pillow's bytes and the golden statuses, large marker-less photos of every
subsampling decode identically under schedules 0, 1 and 2, a mixed batch keeps every image to itself, and the
pre-processor on such files equals the pre-processor on Pillow's pixels."""
import io
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "jpeg.npz")


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from pigeon_b200 import jpeg
    yield torch.device("cuda:0")
    jpeg.set_schedule(0, 0)


@pytest.fixture(scope="module")
def gold():
    import hashlib
    G = np.load(GOLD)
    jo, po = G["jpg_off"], G["px_off"]
    out = {}
    for k in range(int(G["count"])):
        shape = tuple(int(x) for x in G["shape"][k])
        out[str(G["name"][k])] = dict(kind=str(G["kind"][k]), status=int(G["status"][k]),
                                      data=G["jpg"][jo[k]:jo[k + 1]].tobytes(),
                                      px=G["px"][po[k]:po[k + 1]].reshape(shape) if po[k + 1] > po[k] else None,
                                      sha=G[f"sha{k}"].tobytes() if f"sha{k}" in G else None,
                                      sample=G[f"sample{k}"] if f"sample{k}" in G else None)
    out["_same"] = lambda a, g: (np.array_equal(a, g["px"]) if g["px"] is not None else
                                 hashlib.sha256(a.tobytes()).digest() == g["sha"] and
                                 np.array_equal(a[::37, ::23], g["sample"]))
    return out


def _photo(h, w, layout, seed, q=90, restart=False, progressive=False):
    from PIL import Image
    from pigeon_b200 import synthetic
    im = Image.fromarray(synthetic.synthetic_photo(h, w, seed=seed))
    kw = dict(quality=q)
    if layout == "gray":
        im = im.convert("L")
    else:
        kw["subsampling"] = {"444": 0, "422": 1, "420": 2}[layout]
    if restart:
        kw["restart_marker_rows"] = 1
    if progressive:
        kw["progressive"] = True
    f = io.BytesIO()
    im.save(f, "JPEG", **kw)
    return f.getvalue()


def _pillow(data):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


SCHEDULES = [(2, 1), (2, 7), (2, 64), (2, 0), (0, 0), (1, 0)]


@pytest.mark.parametrize("mode,chunk", SCHEDULES)
def test_goldens_under_every_schedule(cuda, gold, mode, chunk):
    from pigeon_b200 import jpeg
    jpeg.set_schedule(mode, chunk)
    try:
        dec = jpeg.JpegDecoder(cuda)
        ok = [k for k, g in gold.items() if k != "_same" and g["kind"] == "ok"]
        imgs = dec.decode([gold[k]["data"] for k in ok])
        for k, t in zip(ok, imgs):
            assert gold["_same"](t.cpu().numpy(), gold[k]), (mode, chunk, k)
        bad = [k for k, g in gold.items() if k != "_same" and g["kind"] == "corrupt"]
        with pytest.raises(jpeg.JpegDecodeError):
            dec.decode([gold[k]["data"] for k in bad])
        for k in bad:                                  # one per call: the status of each file on its own
            with pytest.raises(jpeg.JpegDecodeError) as e:
                dec.decode([gold[k]["data"]])
            if gold[k]["status"] in (jpeg.BAD_CODE, jpeg.OVERRUN):    # the others fail in the host marker walk
                assert e.value.failed[0] == jpeg.STATUS_TEXT[gold[k]["status"]], (mode, chunk, k)
    finally:
        jpeg.set_schedule(0, 0)


@pytest.mark.parametrize("layout", ["444", "422", "420", "gray"])
def test_large_markerless_photos_identical_under_every_schedule(cuda, layout):
    from pigeon_b200 import jpeg
    files = [_photo(640, 640, layout, 1), _photo(1536, 2048, layout, 2, q=85), _photo(3000, 4000, layout, 3, q=80),
             _photo(769, 1023, layout, 4, q=95)]
    ref = [_pillow(f) for f in files]
    dec = jpeg.JpegDecoder(cuda)
    try:
        for mode in (0, 1, 2):
            jpeg.set_schedule(mode, 0)
            out = dec.decode(files)
            for i, (t, r) in enumerate(zip(out, ref)):
                assert np.array_equal(t.cpu().numpy(), r), (mode, i)
    finally:
        jpeg.set_schedule(0, 0)


def test_mixed_batch_keeps_each_image_to_itself(cuda, gold):
    from pigeon_b200 import _lib, jpeg
    lib = _lib.load()
    good = [_photo(1200, 1600, "420", 21), _photo(480, 640, "420", 22, restart=True), _photo(700, 900, "444", 23),
            _photo(600, 800, "420", 24, progressive=True), _photo(333, 500, "gray", 25)]
    trunc = bytearray(good[0])
    info0 = jpeg.parse(bytes(trunc))[0]
    cut = int(info0.scan_offset + info0.scan_bytes // 2)
    trunc = bytes(trunc[:cut]) + b"\xff\xd9"                         # a long segment that overruns
    files = [gold["all-ones code"]["data"], good[0], trunc, good[1], good[2], good[3], gold["truncated scan + EOI"]["data"],
             good[4], trunc]
    expect_fail = {0: jpeg.BAD_CODE, 2: jpeg.OVERRUN, 6: jpeg.OVERRUN, 8: jpeg.OVERRUN}
    infos = [jpeg.parse(f, multiscan=True)[0] for f in files]
    assert all(i.status == jpeg.OK for i in infos) and jpeg.is_multiscan(infos[5])
    n, pad, guard = len(files), 7, 4096
    strides = [3 * i.width + pad for i in infos]
    sizes = [s * i.height for s, i in zip(strides, infos)]
    starts = np.cumsum([guard] + [s + guard for s in sizes])[:-1]
    packed = np.frombuffer(b"".join(files), dtype=np.uint8).copy()
    offsets = np.concatenate([[0], np.cumsum([len(f) for f in files])]).astype(np.int64)
    info_arr = (_lib.JpegInfo * n)(*infos)
    try:
        for mode, chunk in ((0, 0), (2, 0), (2, 7), (1, 0)):
            jpeg.set_schedule(mode, chunk)
            buf = torch.full((int(starts[-1] + sizes[-1] + guard),), 0xA5, dtype=torch.uint8, device=cuda)
            desc = (_lib.Image * n)(*[_lib.Image(buf.data_ptr() + int(st), i.height, i.width, s)
                                      for st, i, s in zip(starts, infos, strides)])
            ws = torch.empty(int(lib.pg_jpeg_workspace_bytes(info_arr, n, int(offsets[-1]))), dtype=torch.uint8,
                             device=cuda)
            status = torch.full((n,), -1, dtype=torch.int32, device=cuda)
            _lib.check(lib.pg_jpeg_decode(packed.ctypes.data, offsets.ctypes.data, info_arr, n, desc, ws.data_ptr(),
                                          ws.numel(), status.data_ptr(), _lib.current_stream_ptr()), "pg_jpeg_decode")
            st = status.tolist()
            assert st == [expect_fail.get(i, 0) for i in range(n)], (mode, chunk, st)
            host = buf.cpu().numpy()
            mask = np.ones(host.shape, dtype=bool)
            for i, (s0, info, s) in enumerate(zip(starts, infos, strides)):
                rows = host[s0:s0 + s * info.height].reshape(info.height, s)
                if i not in expect_fail:
                    assert np.array_equal(rows[:, :3 * info.width].reshape(info.height, info.width, 3),
                                          _pillow(files[i])), (mode, chunk, i)
                for r in range(info.height):
                    mask[s0 + r * s:s0 + r * s + 3 * info.width] = False
            assert (host[mask] == 0xA5).all(), (mode, chunk)
    finally:
        jpeg.set_schedule(0, 0)


def test_processor_on_large_markerless_files_equals_processor_on_pixels(cuda):
    from pigeon_b200.preprocess import ClipImageProcessor
    files = [_photo(1024, 768, "420", 31), _photo(900, 1400, "444", 32), _photo(2000, 1500, "gray", 33, q=85)]
    proc = ClipImageProcessor(device=cuda, dtype=torch.float32)
    a = proc(images=files)["pixel_values"]
    assert proc.gpu_decoded == len(files)
    b = ClipImageProcessor(device=cuda, dtype=torch.float32)(images=[_pillow(f) for f in files])["pixel_values"]
    assert torch.equal(a, b)
