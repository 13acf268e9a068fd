"""GPU PNG decoding (csrc/png.cu) against Pillow's decodes stored in tests/golden/png.npz: byte-identical pixels one
file per call and in one batch with guard bytes and per-image statuses, large photos, and the encoded-bytes paths of
ClipImageProcessor(png=True) (against the default route on every golden), square_crop, CLIPEmbedding and
`run.py embed --png`."""
import io
import re

import numpy as np
import pytest
import torch

from test_png_host import _load, same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _keep_global_rng():
    """The towers built here draw from torch's global generators: leave them as this module found them."""
    with torch.random.fork_rng(devices=range(torch.cuda.device_count())):
        yield


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def gold():
    return _load()


def test_every_gpu_route_golden_decodes_byte_identical_one_per_call_and_batched(cuda, gold):
    from pigeon_b200.png import PngDecoder
    dec = PngDecoder(cuda)
    ok = [g for g in gold if g["kind"] == "ok"]
    for g in ok:
        assert same(dec.decode([g["data"]])[0].cpu().numpy(), g), g["name"]
    first = [t.clone() for t in dec.decode([g["data"] for g in ok])]
    for g, t in zip(ok, first):
        assert same(t.cpu().numpy(), g), g["name"]
    again = dec.decode([g["data"] for g in ok])
    assert all(torch.equal(a, b) for a, b in zip(first, again))


def test_mixed_batch_statuses_and_guard_bytes(cuda, gold):
    from pigeon_b200 import _lib, png
    lib = _lib.load()
    cases = [g for g in gold if g["kind"] in ("fallback", "flip", "host")] + [g for g in gold if g["kind"] == "ok"][::9]
    files = [g["data"] for g in cases]
    infos = [png.parse(f)[0] for f in files]
    _, host_status = png.decode_host(files)
    n, pad, guard = len(files), 5, 4096
    strides = [3 * max(i.width, 1) + pad for i in infos]
    sizes = [s * max(i.height, 1) if i.status == 0 else 0 for s, i in zip(strides, infos)]
    starts = np.cumsum([guard] + [s + guard for s in sizes])[:-1]
    buf = torch.full((int(starts[-1] + sizes[-1] + guard),), 0xA5, dtype=torch.uint8, device=cuda)
    desc = (_lib.Image * n)(*[_lib.Image(buf.data_ptr() + int(st), i.height, i.width, s) if i.status == 0 else _lib.Image()
                              for st, i, s in zip(starts, infos, strides)])
    packed = np.frombuffer(b"".join(files), dtype=np.uint8).copy()
    offsets = np.concatenate([[0], np.cumsum([len(f) for f in files])]).astype(np.int64)
    info_arr = (_lib.PngInfo * n)(*infos)
    ws = torch.empty(int(lib.pg_png_workspace_bytes(info_arr, n, int(offsets[-1]))), dtype=torch.uint8, device=cuda)
    status = torch.full((n,), -1, dtype=torch.int32, device=cuda)
    _lib.check(lib.pg_png_decode(packed.ctypes.data, offsets.ctypes.data, info_arr, n, desc, ws.data_ptr(), ws.numel(),
                                 status.data_ptr(), _lib.current_stream_ptr()), "pg_png_decode")
    st = status.cpu().numpy()
    assert st.tolist() == host_status.tolist()
    for g, s in zip(cases, st):
        if g["kind"] == "ok":
            assert s == 0, g["name"]
        elif g["kind"] in ("fallback", "host"):
            assert s == g["status"], g["name"]
    host = buf.cpu().numpy()
    mask = np.ones(host.shape, dtype=bool)
    for g, s0, i, s, code in zip(cases, starts, infos, strides, st):
        if code:
            continue
        rows = host[s0:s0 + s * i.height].reshape(i.height, s)
        assert same(np.ascontiguousarray(rows[:, :3 * i.width]).reshape(i.height, i.width, 3), g), g["name"]
        for r in range(i.height):
            mask[s0 + r * s:s0 + r * s + 3 * i.width] = False
    assert (host[mask] == 0xA5).all()
    with pytest.raises(png.PngDecodeError) as err:
        png.PngDecoder(cuda).decode(files)
    assert sorted(err.value.failed) == [k for k, s in enumerate(st) if s]


@pytest.mark.parametrize("h,w", [(768, 1024), (3000, 4000)])
def test_large_photos(cuda, h, w):
    from PIL import Image
    from pigeon_b200 import synthetic
    from pigeon_b200.png import decode_png
    photo = synthetic.synthetic_photo(h, w, seed=h)
    files = []
    for mode, kw in (("RGB", {}), ("RGBA", dict(compress_level=1)), ("L", dict(compress_level=9))):
        f = io.BytesIO()
        Image.fromarray(photo).convert(mode).save(f, "PNG", **kw)
        files.append(f.getvalue())
    for f, t in zip(files, decode_png(files, cuda)):
        assert np.array_equal(t.cpu().numpy(), np.asarray(Image.open(io.BytesIO(f)).convert("RGB")))


def _run(proc, images, **kw):
    try:
        return proc(images=images, **kw)["pixel_values"], None
    except Exception as e:  # noqa: BLE001 - the exception is compared
        return None, (type(e), re.sub(r"0x[0-9a-fA-F]+", "0x?", str(e)))


def test_processor_with_png_equals_the_default_route_on_every_golden(cuda, gold):
    from pigeon_b200.preprocess import ClipImageProcessor
    a, b = ClipImageProcessor(device=cuda, png=True), ClipImageProcessor(device=cuda)
    for g in gold:
        pa, ea = _run(a, [g["data"]])
        pb, eb = _run(b, [g["data"]])
        assert ea == eb, g["name"]
        if ea is None:
            assert torch.equal(pa, pb), g["name"]
    assert b.gpu_decoded == 0
    ok = sum(g["kind"] == "ok" for g in gold)
    assert a.gpu_decoded >= ok and a.gpu_decoded + a.host_decoded == b.host_decoded   # encoded files that Image.open took


def test_mixed_jpeg_png_and_host_batch(cuda, gold):
    from PIL import Image
    from pigeon_b200 import synthetic
    from pigeon_b200.preprocess import ClipImageProcessor
    photo = synthetic.synthetic_photo(90, 120, seed=3)
    jpg, prog = io.BytesIO(), io.BytesIO()
    Image.fromarray(photo).save(jpg, "JPEG", quality=90)
    Image.fromarray(photo).save(prog, "JPEG", quality=90, progressive=True)
    by = {g["name"]: g["data"] for g in gold}
    batch = [jpg.getvalue(), by["pillow RGBA 500x333 level 6"], prog.getvalue(), by["Adam7 interlaced"],
             by["bad Adler-32 after trailing image data"], photo, by["ct 3 depth 4 33x70 mixed filters"],
             by["pillow 1 29x1 optimize"]]
    for crop in (False, True):
        a = ClipImageProcessor(device=cuda, png=True)
        pa = a(images=batch, square_crop=crop)["pixel_values"]
        b = ClipImageProcessor(device=cuda)
        pb = b(images=batch, square_crop=crop)["pixel_values"]
        assert torch.equal(pa, pb)
        assert (a.gpu_decoded, a.host_decoded) == (4, 3) and (b.gpu_decoded, b.host_decoded) == (1, 6)


def _embedder(processor=None):
    from pigeon_b200 import CLIPEmbedding, synthetic
    from pigeon_b200.super_guessr import CLIPVisionTower
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims(image_size=336, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=6, std=0.05), strict=True)
    return CLIPEmbedding("unused", device="cuda", clip_model=tower, processor=processor)


NAMES = ["pillow RGB 500x333 optimize", "pillow P 7x13 level 9", "ct 0 depth 16 33x70 filter 4",
         "ct 6 depth 16 33x70 mixed filters"]


def _pixels(g):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(g["data"])).convert("RGB"))


def test_embedding_from_png_bytes_equals_embedding_from_pixels(cuda, gold):
    from pigeon_b200.preprocess import ClipImageProcessor
    by = {g["name"]: g for g in gold}
    proc = ClipImageProcessor(device=cuda, dtype=torch.float16, png=True)
    model = _embedder(proc)
    ref = model([_pixels(by[k]) for k in NAMES]).cpu().numpy()
    assert np.array_equal(model([by[k]["data"] for k in NAMES]).cpu().numpy(), ref)
    assert proc.gpu_decoded == len(NAMES) and proc.host_decoded == 0


def test_run_embed_with_png_decodes_png_files_on_the_gpu(cuda, gold, tmp_path, monkeypatch):
    datasets = pytest.importorskip("datasets")
    import run
    by = {g["name"]: g for g in gold}
    ref = _embedder()([_pixels(by[k]) for k in NAMES]).cpu().numpy()
    made = []

    def fake(*a, **k):
        made.append(k.get("processor"))
        return _embedder(k.get("processor"))
    feats = datasets.Features({"image": datasets.Image(), "index": datasets.Value("int64")})
    ds = datasets.Dataset.from_dict({"image": [{"bytes": by[k]["data"], "path": None} for k in NAMES],
                                     "index": [5, 6, 7, 8]}, features=feats)
    datasets.DatasetDict({"train": ds}).save_to_disk(str(tmp_path / "ds"))
    monkeypatch.setattr(run, "CLIPEmbedding", fake)
    monkeypatch.chdir(tmp_path)
    run.main(["embed", "unused", "-l", str(tmp_path / "ds"), "--png"])
    out = tmp_path / "data" / "landmark_embeddings"
    assert np.load(out / "train.npy").tobytes() == ref.tobytes()
    assert np.load(out / "train_indices.npy").tolist() == [5, 6, 7, 8]
    assert made[0].png and made[0].gpu_decoded == len(NAMES) and made[0].host_decoded == 0
