"""Benchmark and holdout evaluation from encoded image files on the GPU (pigeon_b200.benchmark, the `square_crop`
keyword of ClipImageProcessor, evaluate_model's encoded route, `run.py evaluate -l NAME`):
  * pixel_values bit-identical to tests/golden/benchmark.npz (the reference's per-item CPU path) through
    BenchmarkDataset[i] and through one mixed batch of GPU- and host-decoded files;
  * without `square_crop` the processor gives the oracle's uncropped pixels, as before;
  * evaluate_model on a 37-image benchmark (and on four-view EvalDataset rows) gives the bits of evaluate_model on the
    same images' pixel_values computed on the CPU and passed the way pre-processed datasets are, with and without a
    refiner."""
import hashlib
import io
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
GOLD = os.path.join(ROOT, "tests", "golden", "benchmark.npz")
C = 200                      # geocells of the synthetic head


@pytest.fixture(scope="module", autouse=True)
def _keep_global_rng():
    """The heads built here draw from torch's global generators, which later modules' unseeded initialisations also
    use: leave them as this module found them."""
    with torch.random.fork_rng(devices=range(torch.cuda.device_count())):
        yield


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def gold():
    G = np.load(GOLD)
    off = G["off"]
    return [dict(name=str(G["name"][k]), route=str(G["route"][k]), data=G["data"][off[k]:off[k + 1]].tobytes(),
                 sha=G[f"sha{k}"].tobytes(), sample=G[f"sample{k}"]) for k in range(int(G["count"]))]


def _same(px, g):
    a = px.detach().cpu().numpy()
    return hashlib.sha256(a.tobytes()).digest() == g["sha"] and np.array_equal(a[:, ::17, ::13], g["sample"])


def _write_benchmark(tmp_path, gold, n):
    """benchmarks.json naming one benchmark of n images (the goldens, cycled) under an image-folder prefix."""
    rng = np.random.default_rng(5)
    img = tmp_path / "images"
    img.mkdir(exist_ok=True)
    names = []
    for i in range(n):
        names.append(f"{i:04d}_{gold[i % len(gold)]['name'].replace(' ', '_')}")
        (img / names[-1]).write_bytes(gold[i % len(gold)]["data"])
    import pandas as pd
    pd.DataFrame(dict(image=names, lng=rng.uniform(-180, 180, n), lat=rng.uniform(-60, 70, n),
                      geocell_idx_yfcc=rng.integers(0, C, n))).to_csv(tmp_path / "meta.csv", index=False)
    j = tmp_path / "benchmarks.json"
    j.write_text(json.dumps({"tiny": {"meta": str(tmp_path / "meta.csv"), "images": str(img) + os.sep}}))
    return str(j)


def test_pixel_values_are_the_goldens_per_item_and_batched(cuda, gold, tmp_path, monkeypatch):
    from pigeon_b200 import benchmark, config, loops
    from pigeon_b200.preprocess import ClipImageProcessor
    monkeypatch.setattr(config, "BENCHMARKS", _write_benchmark(tmp_path, gold, len(gold)))
    ds = benchmark.BenchmarkDataset("tiny")
    for i, g in enumerate(gold):
        item = ds[i]
        assert tuple(item["pixel_values"].shape) == (1, 3, 336, 336) and item["pixel_values"].is_cuda
        assert _same(item["pixel_values"][0], g), g["name"]
    proc = ClipImageProcessor(device=cuda)
    rows = ds.encoded()
    batch = loops.encoded_pixel_values(loops.encoded_eval_collate([rows[i] for i in range(len(gold))]), proc)
    assert proc.gpu_decoded == sum(g["route"] == "gpu" for g in gold) and proc.host_decoded == len(gold) - proc.gpu_decoded
    assert proc.host_decoded >= 5 and proc.gpu_decoded >= 10
    for px, g in zip(batch["pixel_values"], gold):
        assert _same(px, g), g["name"]


def test_without_square_crop_the_processor_is_unchanged(cuda, gold):
    from PIL import Image
    from oracle.preprocess import clip_preprocess
    from pigeon_b200.preprocess import ClipImageProcessor
    picks = [g for g in gold if g["name"] in ("420 q90 333x500", "png p 101x77", "420 q90 57x1", "444 q90 241x338")]
    proc = ClipImageProcessor(device=cuda)
    px = proc(images=[g["data"] for g in picks])["pixel_values"].cpu().numpy()
    assert np.array_equal(px, proc(images=[g["data"] for g in picks], square_crop=False)["pixel_values"].cpu().numpy())
    for p, g in zip(px, picks):
        ref = clip_preprocess(np.asarray(Image.open(io.BytesIO(g["data"])).convert("RGB")))
        assert np.array_equal(p, ref), g["name"]


def _model(panorama):
    from pigeon_b200 import SuperGuessr, synthetic
    from pigeon_b200.super_guessr import CLIPVisionTower
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims(layers=1)
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=11, std=0.05))
    torch.manual_seed(12)
    return SuperGuessr(tower, panorama=panorama, freeze_base=True, num_candidates=10,
                       geocells=synthetic.synthetic_geocells(C, 3)).to("cuda").eval()


def _refiner():
    from pigeon_b200 import ProtoRefiner, synthetic
    bank = synthetic.synthetic_bank(C, 1500, 1024, seed=4, members_mean=3.0, empty_cells=2)
    return ProtoRefiner(topk=5, max_refinement=1000, temperature=1.6, protos=bank).eval()


class Precomputed(torch.utils.data.Dataset):
    """Rows of pixel_values computed on the CPU, shaped as a pre-processed dataset yields them."""

    def __init__(self, px, labels, labels_clf):
        self.px, self.labels, self.labels_clf = px, labels, labels_clf

    def __len__(self):
        return len(self.px)

    def __getitem__(self, i):
        if i == "labels":
            return self.labels.numpy()
        if i == "labels_clf":
            return self.labels_clf.numpy()
        return dict(pixel_values=self.px[i], labels=self.labels[i], labels_clf=self.labels_clf[i])


def _same_eval(a, b):
    for k in ("preds", "preds_geocell", "top_geocells"):
        assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), k
    assert a["Geocell_accuracy"] == b["Geocell_accuracy"] and a["loss"] == b["loss"]


@pytest.mark.parametrize("refine", [False, True])
def test_evaluate_benchmark_equals_precomputed_pixels(cuda, gold, tmp_path, monkeypatch, refine):
    import make_benchmark_golden as M
    from pigeon_b200 import benchmark, config, loops
    from pigeon_b200.preprocess import ClipImageProcessor
    monkeypatch.setattr(config, "BENCHMARKS", _write_benchmark(tmp_path, gold, 37))
    ds = benchmark.BenchmarkDataset("tiny")
    cpu = {g["name"]: torch.from_numpy(M.reference_pixel_values(g["data"])) for g in gold}
    px = torch.stack([cpu[gold[i % len(gold)]["name"]] for i in range(37)]).unsqueeze(1)      # [37, 1, 3, 336, 336]
    pre = Precomputed(px, torch.from_numpy(ds["labels"]), torch.from_numpy(ds["labels_clf"]))
    args = SimpleNamespace(per_device_eval_batch_size=16)
    model = _model(panorama=False)
    refiner = _refiner() if refine else None
    want = loops.evaluate_model(model, pre, None, args, refiner)
    got = loops.evaluate_model(model, ds.encoded(), None, args, refiner, collate_fn=loops.encoded_eval_collate,
                               processor=ClipImageProcessor(device=cuda))
    _same_eval(got, want)
    assert len(got["preds"]) == 37


@pytest.mark.parametrize("refine", [False, True])
def test_evaluate_raw_four_view_split_equals_its_preprocessed_rows(cuda, gold, tmp_path, refine):
    datasets = pytest.importorskip("datasets")
    from PIL import Image
    from oracle.preprocess import clip_preprocess
    from pigeon_b200 import benchmark, loops
    from pigeon_b200.preprocess import ClipImageProcessor
    n, cols = 7, ["image", "image_2", "image_3", "image_4"]
    rng = np.random.default_rng(9)
    pick = [[gold[(5 * r + 3 * v) % len(gold)] for v in range(4)] for r in range(n)]
    raw = {c: [] for c in cols}
    for r in range(n):
        for v, c in enumerate(cols):
            if (r + v) % 3 == 0:                                  # some views read from their path
                p = tmp_path / f"{c}_{r}.bin"
                p.write_bytes(pick[r][v]["data"])
                raw[c].append({"bytes": None, "path": str(p)})
            else:
                raw[c].append({"bytes": pick[r][v]["data"], "path": None})
    labels, labels_clf = rng.uniform(-60, 60, (n, 2)).tolist(), rng.integers(0, C, n).tolist()
    feats = {c: datasets.Image() for c in cols}
    feats.update(labels=datasets.Sequence(datasets.Value("float32")), labels_clf=datasets.Value("int64"))
    split = datasets.Dataset.from_dict(dict(raw, labels=labels, labels_clf=labels_clf),
                                       features=datasets.Features(feats)).with_format("torch")
    views = {}
    for g in gold:
        views[g["name"]] = clip_preprocess(np.asarray(Image.open(io.BytesIO(g["data"])).convert("RGB")))
    px = np.stack([np.concatenate([views[pick[r][v]["name"]] for v in range(4)]) for r in range(n)])
    pre = datasets.Dataset.from_dict(
        dict(pixel_values=px, labels=labels, labels_clf=labels_clf),
        features=datasets.Features(dict(pixel_values=datasets.Array3D((12, 336, 336), "float32"),
                                        labels=datasets.Sequence(datasets.Value("float32")),
                                        labels_clf=datasets.Value("int64")))).with_format("torch")
    args = SimpleNamespace(per_device_eval_batch_size=3)
    model = _model(panorama=True)
    refiner = _refiner() if refine else None
    want = loops.evaluate_model(model, pre, None, args, refiner)
    ev = benchmark.EvalDataset(split)
    got = loops.evaluate_model(model, ev.encoded(), None, args, refiner, collate_fn=loops.encoded_eval_collate,
                               processor=ClipImageProcessor(device=cuda))
    _same_eval(got, want)
    assert torch.equal(ev[2]["pixel_values"].cpu(), torch.from_numpy(px[2:3]))


def test_run_evaluate_benchmark_by_name(cuda, gold, tmp_path, monkeypatch):
    import types
    import make_benchmark_golden as M
    import run
    from pigeon_b200 import benchmark, config, loops
    monkeypatch.setattr(config, "BENCHMARKS", _write_benchmark(tmp_path, gold, 21))
    model, refiner, made, results = _model(panorama=False), _refiner(), [], []
    model.load_state = lambda path: None                          # no checkpoints: the synthetic head stays

    def fake_guessr(base, **kw):
        made.append(kw)
        return model
    real = loops.evaluate_model

    def spy(*a, **kw):
        results.append(real(*a, **kw))
        return results[-1]
    # run.evaluate imports CLIPVisionModel for -b; a stand-in module keeps the real transformers (which would import
    # torchvision and change how `datasets` formats columns for every later test) out of sys.modules
    fake_transformers = types.ModuleType("transformers")
    fake_transformers.CLIPVisionModel = SimpleNamespace(from_pretrained=lambda *a, **k: None)
    monkeypatch.setitem(sys.modules, "transformers", fake_transformers)
    monkeypatch.setattr(run, "SuperGuessr", fake_guessr)
    monkeypatch.setattr(run, "ProtoRefiner", lambda *a, **kw: refiner)
    monkeypatch.setattr(run, "evaluate_model", spy)
    monkeypatch.chdir(tmp_path)
    os.makedirs("saved_models/refiner")
    run.main(["evaluate", "head.model", "-l", "tiny", "-b", config.CLIP_MODEL, "--yfcc"])
    assert made[0]["panorama"] is False and made[0]["yfcc"] is True
    ds = benchmark.BenchmarkDataset("tiny")
    px = torch.stack([torch.from_numpy(M.reference_pixel_values(gold[i % len(gold)]["data"])) for i in range(21)])
    want = real(model, Precomputed(px.unsqueeze(1), torch.from_numpy(ds["labels"]), torch.from_numpy(ds["labels_clf"])),
                None, None, refiner)
    _same_eval(results[0], want)
