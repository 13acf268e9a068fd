"""GPU decoding of progressive and multi-scan JPEGs (csrc/jpeg.cu multiscan_kernel) against Pillow's decodes stored in
tests/golden/jpeg_multiscan.npz: byte-identical pixels one file per call and in one batch, a mixed batch of baseline,
progressive, refused and corrupt files with guard bytes, baseline files through either parser, and the encoded-bytes
paths of ClipImageProcessor(jpeg_multiscan=True), CLIPEmbedding and `run.py embed --jpeg-multiscan`."""
import hashlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.dirname(__file__) + "/golden/"


@pytest.fixture(scope="module", autouse=True)
def _keep_global_rng():
    """The towers built here draw from torch's global generators, which later modules' unseeded initialisations also
    use: leave them as this module found them."""
    with torch.random.fork_rng(devices=range(torch.cuda.device_count())):
        yield


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _load(name):
    G = np.load(GOLD + name)
    jo, po = G["jpg_off"], G["px_off"]
    out = {}
    for k in range(int(G["count"])):
        shape = tuple(int(x) for x in G["shape"][k])
        out[str(G["name"][k])] = dict(kind=str(G["kind"][k]), status=int(G["status"][k]),
                                      data=G["jpg"][jo[k]:jo[k + 1]].tobytes(),
                                      px=G["px"][po[k]:po[k + 1]].reshape(shape) if po[k + 1] > po[k] else None,
                                      sha=G[f"sha{k}"].tobytes() if f"sha{k}" in G else None,
                                      sample=G[f"sample{k}"] if f"sample{k}" in G else None)
    return out


@pytest.fixture(scope="module")
def multi():
    return _load("jpeg_multiscan.npz")


@pytest.fixture(scope="module")
def single():
    return _load("jpeg.npz")


def _same(img, g):
    a = img.cpu().numpy()
    if g["px"] is not None:
        return np.array_equal(a, g["px"])
    return hashlib.sha256(a.tobytes()).digest() == g["sha"] and np.array_equal(a[::37, ::23], g["sample"])


def test_every_multiscan_golden_decodes_byte_identical(cuda, multi):
    from pigeon_b200.jpeg import JpegDecoder
    dec = JpegDecoder(cuda)
    ok = {k: g for k, g in multi.items() if g["kind"] == "ok"}
    assert len(ok) >= 150
    for name, g in ok.items():
        assert _same(dec.decode([g["data"]], multiscan=True)[0], g), name
    names = list(ok)
    first = [t.clone() for t in dec.decode([ok[k]["data"] for k in names], multiscan=True)]
    for name, t in zip(names, first):
        assert _same(t, ok[name]), name
    again = dec.decode([ok[k]["data"] for k in names], multiscan=True)
    assert all(torch.equal(a, b) for a, b in zip(first, again))


def test_the_progressive_single_scan_golden_decodes_to_its_pillow_pixels(cuda, single):
    from pigeon_b200.jpeg import decode_jpeg
    g = single["progressive"]
    assert _same(decode_jpeg([g["data"]], cuda, multiscan=True)[0], g)


def test_mixed_batch_fails_alone_and_keeps_the_guard_bytes(cuda, multi, single):
    from pigeon_b200 import _lib, jpeg
    lib = _lib.load()
    batch = [(single, "420 photo q90"), (multi, "420 progressive q90"), (multi, "incomplete progression"),
             (multi, "gray one scan per coefficient"), (multi, "bad code in an AC refinement scan"),
             (single, "444 restart blocks 3"), (multi, "422 SOF0 non-interleaved Cr Y Cb"),
             (multi, "truncated progressive file"), (multi, "420 DRI changed and removed between scans"),
             (single, "all-ones code"), (multi, "marker inside a DC scan"), (multi, "420 deep successive approximation")]
    files = [src[k]["data"] for src, k in batch]
    parsed = [jpeg.parse(f, multiscan=True) for f in files]
    infos = [p[0] for p in parsed]
    n, pad, guard = len(files), 7, 4096
    strides = [3 * max(i.width, 1) + pad for i in infos]
    sizes = [s * max(i.height, 1) for s, i in zip(strides, infos)]
    starts = np.cumsum([guard] + [s + guard for s in sizes])[:-1]
    buf = torch.full((int(starts[-1] + sizes[-1] + guard),), 0xA5, dtype=torch.uint8, device=cuda)
    desc = (_lib.Image * n)(*[_lib.Image(buf.data_ptr() + int(st), i.height, i.width, s) if i.status == 0 else _lib.Image()
                              for st, i, s in zip(starts, infos, strides)])
    packed = np.frombuffer(b"".join(files), dtype=np.uint8).copy()
    offsets = np.concatenate([[0], np.cumsum([len(f) for f in files])]).astype(np.int64)
    info_arr = (_lib.JpegInfo * n)(*infos)
    ws = torch.empty(int(lib.pg_jpeg_workspace_bytes(info_arr, n, int(offsets[-1]))), dtype=torch.uint8, device=cuda)
    status = torch.full((n,), -1, dtype=torch.int32, device=cuda)
    _lib.check(lib.pg_jpeg_decode(packed.ctypes.data, offsets.ctypes.data, info_arr, n, desc, ws.data_ptr(), ws.numel(),
                                  status.data_ptr(), _lib.current_stream_ptr()), "pg_jpeg_decode")
    expect = [0, 0, jpeg.UNSUPPORTED, 0, jpeg.BAD_CODE, 0, 0, jpeg.NO_EOI, 0, jpeg.BAD_CODE, jpeg.BAD_RST, 0]
    assert status.tolist() == expect
    host = buf.cpu().numpy()
    mask = np.ones(host.shape, dtype=bool)
    for (src, name), st, i, s, e in zip(batch, starts, infos, strides, expect):
        if e:
            continue
        rows = host[st:st + s * i.height].reshape(i.height, s)
        assert _same(torch.from_numpy(np.ascontiguousarray(rows[:, :3 * i.width]).reshape(i.height, i.width, 3)),
                     src[name]), name
        for r in range(i.height):
            mask[st + r * s:st + r * s + 3 * i.width] = False
    assert (host[mask] == 0xA5).all()
    from pigeon_b200.jpeg import JpegDecodeError, JpegDecoder
    with pytest.raises(JpegDecodeError) as err:
        JpegDecoder(cuda).decode(files, multiscan=True)
    assert sorted(err.value.failed) == [i for i, e in enumerate(expect) if e]
    assert "incomplete progression" in err.value.failed[2] and "EOI" in err.value.failed[7]
    assert err.value.failed[4] == jpeg.STATUS_TEXT[jpeg.BAD_CODE]


def test_baseline_files_decode_the_same_through_either_parser(cuda, single):
    from pigeon_b200 import jpeg
    dec = jpeg.JpegDecoder(cuda)
    names = [k for k, g in single.items() if g["kind"] == "ok"][::7]
    files = [single[k]["data"] for k in names]
    a = [t.clone() for t in dec.decode(files)]
    b = dec.decode(files, multiscan=True)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


PROC = ["420 progressive q90", "444 progressive restart rows 1", "gray progressive q75", "422 SOF1 non-interleaved Y Cb Cr",
        "420 flat long EOB runs restart 5", "420 progressive 7x13"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_processor_on_encoded_progressive_files_equals_the_processor_on_pixels(cuda, multi, dtype):
    from pigeon_b200.preprocess import ClipImageProcessor
    proc = ClipImageProcessor(device=cuda, dtype=dtype, jpeg_multiscan=True)
    a = proc(images=[multi[k]["data"] for k in PROC])["pixel_values"]
    assert proc.gpu_decoded == len(PROC) and proc.host_decoded == 0
    b = ClipImageProcessor(device=cuda, dtype=dtype)(images=[multi[k]["px"] for k in PROC])["pixel_values"]
    assert torch.equal(a, b)


def _embedder(processor=None):
    from pigeon_b200 import CLIPEmbedding, synthetic
    from pigeon_b200.super_guessr import CLIPVisionTower
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims(image_size=336, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=6, std=0.05), strict=True)
    return CLIPEmbedding("unused", device="cuda", clip_model=tower, processor=processor)


def test_embedding_from_progressive_bytes_equals_embedding_from_pixels(cuda, multi):
    from pigeon_b200.preprocess import ClipImageProcessor
    proc = ClipImageProcessor(device=cuda, dtype=torch.float16, jpeg_multiscan=True)
    model = _embedder(proc)
    ref = model([multi[k]["px"] for k in PROC]).cpu().numpy()
    assert np.array_equal(model([multi[k]["data"] for k in PROC]).cpu().numpy(), ref)
    assert proc.gpu_decoded == len(PROC) and proc.host_decoded == 0


def test_run_embed_with_jpeg_multiscan_decodes_progressive_files_on_the_gpu(cuda, multi, tmp_path, monkeypatch):
    datasets = pytest.importorskip("datasets")
    import run
    names = PROC[:4]
    ref = _embedder()([multi[k]["px"] for k in names]).cpu().numpy()
    made = []

    def fake(*a, **k):
        made.append(k.get("processor"))
        return _embedder(k.get("processor"))
    feats = datasets.Features({"image": datasets.Image(), "index": datasets.Value("int64")})
    ds = datasets.Dataset.from_dict({"image": [{"bytes": multi[k]["data"], "path": None} for k in names],
                                     "index": [5, 6, 7, 8]}, features=feats)
    datasets.DatasetDict({"train": ds}).save_to_disk(str(tmp_path / "ds"))
    monkeypatch.setattr(run, "CLIPEmbedding", fake)
    monkeypatch.chdir(tmp_path)
    run.main(["embed", "unused", "-l", str(tmp_path / "ds"), "--jpeg-multiscan"])
    out = tmp_path / "data" / "landmark_embeddings"
    assert np.load(out / "train.npy").tobytes() == ref.tobytes()
    assert np.load(out / "train_indices.npy").tolist() == [5, 6, 7, 8]
    assert made[0].jpeg_multiscan and made[0].gpu_decoded == len(names) and made[0].host_decoded == 0
