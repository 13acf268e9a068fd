"""GPU JPEG decoder (csrc/jpeg.cu) against Pillow's decodes stored in tests/golden/jpeg.npz: byte-identical pixels, one
file per call and in one mixed batch, guard bytes, per-image error status, and the encoded-bytes paths of
ClipImageProcessor, CLIPEmbedding, embed_images and `run.py embed`.  Reads only the goldens: Pillow is not needed except
by the test of the host route, which is Pillow."""
import hashlib
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
    return torch.device("cuda:0")


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
    return {g["name"]: g for g in _load_gold()}


def _same(img, g):
    a = img.cpu().numpy()
    if g["px"] is not None:
        return np.array_equal(a, g["px"])
    return hashlib.sha256(a.tobytes()).digest() == g["sha"] and np.array_equal(a[::37, ::23], g["sample"])


def test_every_supported_golden_decodes_byte_identical(cuda, gold):
    from pigeon_b200.jpeg import JpegDecoder
    dec = JpegDecoder(cuda)
    ok = {k: g for k, g in gold.items() if g["kind"] == "ok"}
    assert len(ok) >= 300
    for name, g in ok.items():                                         # one file per call
        assert _same(dec.decode([g["data"]])[0], g), name
    names = list(ok)
    first = dec.decode([ok[k]["data"] for k in names])                 # one mixed batch
    first = [t.clone() for t in first]
    for name, t in zip(names, first):
        assert _same(t, ok[name]), name
    again = dec.decode([ok[k]["data"] for k in names])
    assert all(torch.equal(a, b) for a, b in zip(first, again))


def test_guard_bytes_around_the_destinations_are_unchanged(cuda, gold):
    from pigeon_b200 import _lib, jpeg
    lib = _lib.load()
    names = ["420 13x17 q90", "422 1x300", "444 photo q100", "gray 9x13", "420 restart rows 1", "422 saturated edges q100"]
    files = [gold[k]["data"] for k in names]
    infos = [jpeg.parse(f)[0] for f in files]
    n, pad, guard = len(files), 13, 4096
    strides = [3 * i.width + pad for i in infos]
    sizes = [s * i.height for s, i in zip(strides, infos)]
    starts = np.cumsum([guard] + [s + guard for s in sizes])[:-1]
    buf = torch.full((int(starts[-1] + sizes[-1] + guard),), 0xA5, dtype=torch.uint8, device=cuda)
    desc = (_lib.Image * n)(*[_lib.Image(buf.data_ptr() + int(st), i.height, i.width, s)
                              for st, i, s in zip(starts, infos, strides)])
    packed = np.frombuffer(b"".join(files), dtype=np.uint8).copy()
    offsets = np.concatenate([[0], np.cumsum([len(f) for f in files])]).astype(np.int64)
    info_arr = (_lib.JpegInfo * n)(*infos)
    ws = torch.empty(int(lib.pg_jpeg_workspace_bytes(info_arr, n, int(offsets[-1]))), dtype=torch.uint8, device=cuda)
    status = torch.full((n,), -1, dtype=torch.int32, device=cuda)
    _lib.check(lib.pg_jpeg_decode(packed.ctypes.data, offsets.ctypes.data, info_arr, n, desc, ws.data_ptr(), ws.numel(),
                                  status.data_ptr(), _lib.current_stream_ptr()), "pg_jpeg_decode")
    assert status.tolist() == [0] * n
    host = buf.cpu().numpy()
    mask = np.ones(host.shape, dtype=bool)
    for name, st, i, s in zip(names, starts, infos, strides):
        rows = host[st:st + s * i.height].reshape(i.height, s)
        assert np.array_equal(rows[:, :3 * i.width].reshape(i.height, i.width, 3), gold[name]["px"]), name
        for r in range(i.height):
            mask[st + r * s:st + r * s + 3 * i.width] = False
    assert (host[mask] == 0xA5).all()


def test_a_corrupt_file_fails_alone(cuda, gold):
    from pigeon_b200.jpeg import STATUS_TEXT, JpegDecodeError, JpegDecoder, BAD_CODE, OVERRUN
    batch = ["420 photo q90", "truncated scan + EOI", "444 restart blocks 3", "all-ones code", "gray q75",
             "wrong RST number", "422 133x251", "truncated file", "420 4000x3000 q50"]
    with pytest.raises(JpegDecodeError) as e:
        JpegDecoder(cuda).decode([gold[k]["data"] for k in batch])
    err = e.value
    assert sorted(err.failed) == [1, 3, 5, 7]
    assert err.failed[1] == STATUS_TEXT[OVERRUN] and err.failed[3] == STATUS_TEXT[BAD_CODE]
    assert "RST" in err.failed[5] and "EOI" in err.failed[7]
    for i, name in enumerate(batch):
        if i in err.failed:
            assert err.images[i] is None
        else:
            assert _same(err.images[i], gold[name]), name


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_processor_on_encoded_bytes_equals_the_processor_on_pixels(cuda, gold, dtype):
    from pigeon_b200.preprocess import ClipImageProcessor
    names = ["420 noise q100", "444 photo q90", "422 saturated edges q100", "gray q75", "420 17x6 q75", "420 restart rows 1",
             "444 16-bit qtables"]
    proc = ClipImageProcessor(device=cuda, dtype=dtype)
    a = proc(images=[gold[k]["data"] for k in names])["pixel_values"]
    assert proc.gpu_decoded == len(names) and proc.host_decoded == 0
    b = ClipImageProcessor(device=cuda, dtype=dtype)(images=[gold[k]["px"] for k in names])["pixel_values"]
    assert torch.equal(a, b)


def test_progressive_file_goes_through_the_host_route(cuda, gold):
    pytest.importorskip("PIL")
    from pigeon_b200.preprocess import ClipImageProcessor
    names = ["420 photo q75", "progressive", "gray 9x13"]
    proc = ClipImageProcessor(device=cuda)
    a = proc(images=[gold[k]["data"] for k in names])["pixel_values"]
    assert proc.gpu_decoded == 2 and proc.host_decoded == 1
    b = ClipImageProcessor(device=cuda)(images=[gold[k]["px"] for k in names])["pixel_values"]
    assert torch.equal(a, b)


def _embedder(cuda):
    from pigeon_b200 import CLIPEmbedding, synthetic
    from pigeon_b200.super_guessr import CLIPVisionTower
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims(image_size=336, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=6, std=0.05), strict=True)
    return CLIPEmbedding("unused", device="cuda", clip_model=tower)


EMBED = ["420 noise q100", "444 photo q90", "gray q75", "422 restart rows 1", "420 640x640 q90"]


def test_embedding_from_bytes_equals_embedding_from_pixels(cuda, gold, tmp_path):
    from pigeon_b200.loops import embed_images, encoded_image_collate
    model = _embedder(cuda)
    files = [gold[k]["data"] for k in EMBED]
    pixels = [gold[k]["px"] if gold[k]["px"] is not None else None for k in EMBED]
    from pigeon_b200.jpeg import decode_jpeg
    pixels[-1] = decode_jpeg([files[-1]], cuda)[0].cpu().numpy()       # 640x640: checked against its SHA-256 first
    assert _same(torch.from_numpy(pixels[-1]), gold[EMBED[-1]])
    ref = model(pixels).cpu().numpy()
    assert np.array_equal(model(files).cpu().numpy(), ref)
    rows = [{"image": {"bytes": f, "path": None}, "index": i} for i, f in enumerate(files)]
    path = tmp_path / "on_disk.jpg"
    path.write_bytes(files[0])
    rows[0]["image"] = {"bytes": None, "path": str(path)}                # `path` is read when `bytes` is None

    class DS(torch.utils.data.Dataset):
        def __len__(self):
            return len(rows)

        def __getitem__(self, i):
            return rows[i]

    embed_images(model, {"train": DS()}, save_dir=str(tmp_path), collate_fn=encoded_image_collate)
    assert np.load(tmp_path / "train.npy").tobytes() == ref.tobytes()
    assert np.load(tmp_path / "train_indices.npy").tolist() == list(range(len(files)))


def test_run_embed_reads_the_reference_image_dataset(cuda, gold, tmp_path, monkeypatch):
    datasets = pytest.importorskip("datasets")
    import run
    model = _embedder(cuda)
    files = [gold[k]["data"] for k in EMBED[:4]]
    ref = model([gold[k]["px"] for k in EMBED[:4]]).cpu().numpy()
    feats = datasets.Features({"image": datasets.Image(), "index": datasets.Value("int64")})
    ds = datasets.Dataset.from_dict({"image": [{"bytes": f, "path": None} for f in files], "index": [10, 11, 12, 13]},
                                    features=feats)
    datasets.DatasetDict({"train": ds, "val": ds.select([2, 0])}).save_to_disk(str(tmp_path / "ds"))
    monkeypatch.setattr(run, "CLIPEmbedding", lambda *a, **k: model)
    monkeypatch.chdir(tmp_path)
    run.main(["embed", "unused", "-l", str(tmp_path / "ds")])
    out = tmp_path / "data" / "landmark_embeddings"
    assert np.load(out / "train.npy").tobytes() == ref.tobytes()
    assert np.load(out / "train_indices.npy").tolist() == [10, 11, 12, 13]
    assert np.load(out / "val.npy").tobytes() == model([gold[EMBED[2]]["px"], gold[EMBED[0]]["px"]]).cpu().numpy().tobytes()
    assert np.load(out / "val_indices.npy").tolist() == [12, 10]
