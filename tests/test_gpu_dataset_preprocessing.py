"""pigeon_b200.dataset_preprocessing on the GPU: `labels_clf` from `CountryIndex.locate` over the geocell polygons equals
the unmodified reference's (tests/golden/dataset_preprocessing.npz) element for element in every split and both
branches; a seeded stress set of 10^5 points, a third of them snapped onto edges and vertices, equals the exact oracle
(tests/metrics_oracle.py) in cell id and fallback flag; and the datasets `preprocess` makes are read by their consumers:
the embedding branch trains an epoch through `finetune_on_embeddings`, feeds `python -m pigeon_b200.prototypes` and
loads into `ProtoRefiner(dataset_path=...)`, and the raw branch takes a `run.py finetune -l` step from its image files."""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
datasets = pytest.importorskip("datasets")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dataset_preprocessing_data as data  # noqa: E402
import metrics_oracle as mo  # noqa: E402

from pigeon_b200 import config  # noqa: E402
from pigeon_b200 import dataset_preprocessing as dp  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "dataset_preprocessing.npz"))


@pytest.fixture(autouse=True)
def _rows_without_torchvision(monkeypatch):
    """datasets' torch formatter imports torchvision.io.VideoReader whenever torchvision is loaded (an earlier test's
    transformers import loads it), and this torchvision has none: format the rows as a process without it does."""
    monkeypatch.delitem(sys.modules, "torchvision", raising=False)


@pytest.fixture(scope="module", autouse=True)
def _keep_global_rng():
    with torch.random.fork_rng(devices=range(torch.cuda.device_count())):
        yield


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _write_inputs(tmp_path, monkeypatch, embeds_by_split):
    monkeypatch.chdir(tmp_path)
    os.makedirs(os.path.dirname(config.GEOCELL_PATH), exist_ok=True)
    with open(config.GEOCELL_PATH, "wb") as f:
        f.write(GOLDEN["geocells_csv"].tobytes())
    os.makedirs("emb", exist_ok=True)
    for s, (e, i) in embeds_by_split.items():
        np.save(f"emb/{s}.npy", e)
        np.save(f"emb/{s}_indices.npy", i)


def _golden_inputs():
    return {s: {k[len(f"in/{s}/"):]: GOLDEN[k] for k in GOLDEN.files
                if k.startswith(f"in/{s}/") and not k.endswith(("embeds", "indices"))} for s in data.SPLITS}


@pytest.mark.parametrize("name", ["emb_mt", "raw"])
def test_labels_clf_equal_the_reference(cuda, tmp_path, monkeypatch, name):
    _write_inputs(tmp_path, monkeypatch, {s: (GOLDEN[f"in/{s}/embeds"], GOLDEN[f"in/{s}/indices"]) for s in data.SPLITS})
    emb, mt = bool(GOLDEN[f"{name}/args"][1]), bool(GOLDEN[f"{name}/args"][2])
    out = dp.preprocess(data.raw_dataset(_golden_inputs()), config.GEOCELL_PATH, embedder=True if emb else None,
                        multi_task=mt, embeddings_dir="emb")
    for s in data.SPLITS:
        table = out[s].with_format("arrow")[:]
        assert out[s].column_names == GOLDEN[f"{name}/{s}/columns"].tolist()
        got = table.column("labels_clf").to_numpy()
        assert got.dtype == np.int64 and np.array_equal(got, GOLDEN[f"{name}/{s}/labels_clf"]), s
        assert np.array_equal(np.asarray(table.column("labels").to_pylist()), GOLDEN[f"{name}/{s}/labels"])


def test_locate_stress_equals_exact_oracle(cuda, tmp_path):
    """10^5 seeded points over the synthetic cells (a third exactly on vertices or on edges at parameters k / 16, the
    rest uniform over the cells' extent and beyond) against the exact oracle: cell ids and fallback flags."""
    (csr, lnglat) = dp.parse_geocells(data.geocell_frame())
    data.geocell_frame().to_csv(tmp_path / "cells.csv", index=False)
    index, cells_lnglat = dp.load_geocells(str(tmp_path / "cells.csv"))
    assert np.array_equal(cells_lnglat, lnglat)
    geoms = mo.geometries_from_csr(*csr)
    rng = np.random.default_rng(5)
    N = 100_000
    verts, ring_off = csr[0], csr[1]
    starts = np.concatenate([np.arange(ring_off[r], ring_off[r + 1] - 1) for r in range(len(ring_off) - 1)])
    k = N // 3
    e = rng.choice(starts, k)
    t = rng.integers(0, 17, k)[:, None] / 16.0
    snapped = verts[e] + t * (verts[e + 1] - verts[e])
    uniform = np.concatenate([rng.uniform([-70, -50], [35, 35], (N - k - 4000, 2)), rng.uniform([-180, -90], [180, 90], (4000, 2))])
    pts = np.concatenate([snapped, uniform])
    pts = pts[rng.permutation(N)]
    country, flags, _ = index.locate(pts)
    torch.cuda.synchronize()
    want_c, want_f, _ = mo.locate(geoms, pts, pts)
    got_c, got_f = country.cpu().numpy(), flags.cpu().numpy()
    assert got_c.dtype == np.int32 and np.array_equal(got_c, want_c)
    assert np.array_equal(got_f, want_f)
    assert 0.02 < want_f.mean() < 0.9 and len(np.unique(want_c)) == len(geoms)



def _e2e_inputs(seed):
    """Larger splits for the consumers: points in clumps inside the cells, so that every cell gets prototypes."""
    rng = np.random.default_rng(seed)
    out = {}
    centres = np.asarray([[2, 2], [13, 1], [2.5, 14], [8, 14], [22, 22], [28, 28], [-40, -30], [175, 85], [-175, -85],
                          [4, 4]], np.float64)
    for k, (s, n) in enumerate(zip(data.SPLITS, (120, 24, 12))):
        c = data.inputs(s, seed + k)
        pts = centres[rng.integers(0, len(centres), n)] + rng.normal(0, 0.3, (n, 2))
        pts = np.clip(pts, [-180, -90], [180, 90])
        extra = {key: np.resize(v, n) for key, v in c.items()}
        extra["lng"], extra["lat"] = pts[:, 0], pts[:, 1]
        extra["index"] = np.arange(n, dtype=np.int64) * 3 + 1000 * k
        extra["labels_climate"] = rng.dirichlet(np.ones(28), n).astype(np.float32)   # the climate head's soft targets
        extra["labels_month"] = rng.integers(0, 12, n).astype(np.int64)
        out[s] = extra
    return out


def _e2e_embeddings(inputs, seed):
    rng = np.random.default_rng(seed)
    files = {}
    for s, c in inputs.items():
        order = rng.permutation(len(c["index"]))
        files[s] = (rng.standard_normal((len(order), config.CLIP_EMBED_DIM)).astype(np.float32), c["index"][order])
    return files


def test_embedding_dataset_trains_feeds_prototypes_and_refiner(cuda, tmp_path, monkeypatch):
    import pandas as pd
    from pigeon_b200 import ProtoRefiner, training
    inputs = _e2e_inputs(40)
    files = _e2e_embeddings(inputs, 41)
    _write_inputs(tmp_path, monkeypatch, files)
    raw = data.raw_dataset(inputs)
    raw.save_to_disk("raw")
    r = subprocess.run([sys.executable, "-m", "pigeon_b200.dataset_preprocessing", "raw", config.GEOCELL_PATH, "out",
                        "--embeddings", "emb", "--multitask"], cwd=str(tmp_path), capture_output=True, text=True,
                       env=dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", "")))
    assert r.returncode == 0, r.stderr[-3000:]
    ds = datasets.DatasetDict.load_from_disk("out")
    train = ds["train"].with_format("arrow")[:]
    emb = np.asarray(train.column("embedding").to_pylist(), np.float32)
    e, idx = files["train"]
    assert np.array_equal(emb, e[np.argsort(idx)])                    # row i: the embedding of the i-th index value
    _, lnglat = dp.parse_geocells(config.GEOCELL_PATH)

    args = SimpleNamespace(learning_rate=1e-3, per_device_train_batch_size=32, per_device_eval_batch_size=16,
                           num_train_epochs=1, gradient_accumulation_steps=1)
    torch.manual_seed(0)
    model = training.finetune_on_embeddings(ds.with_format("torch"), multi_task=True, heading=False, yfcc=False,
                                            train_args=args, geocells=lnglat, num_candidates=5)
    assert len(model.train_history) == 1 and np.isfinite(model.train_history).all()

    pd.DataFrame(dict(lng=inputs["train"]["lng"], lat=inputs["train"]["lat"], selection="train")).to_csv("meta.csv",
                                                                                                          index=False)
    r = subprocess.run([sys.executable, "-m", "pigeon_b200.prototypes", "meta.csv", "out", "protos.csv",
                        "--min-samples", "3"], cwd=str(tmp_path), capture_output=True, text=True,
                       env=dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", "")))
    assert r.returncode == 0, r.stderr[-3000:]
    protos = pd.read_csv("protos.csv")
    cells = np.unique(protos["geocell_idx"].astype(int))
    assert len(protos) > 0 and set(cells) <= set(train.column("labels_clf").to_numpy().tolist())
    refiner = ProtoRefiner(topk=1, max_refinement=1000, temperature=1.6, proto_path="protos.csv",
                           dataset_path="out").eval()
    B = 3
    cand = torch.tensor(np.resize(cells, (B, 1)), dtype=torch.int64)
    _, ll, cell = refiner(torch.randn(B, config.CLIP_EMBED_DIM), initial_preds=torch.zeros(B, 2), candidate_cells=cand,
                          candidate_probs=torch.ones(B, 1))
    torch.cuda.synchronize()
    assert cell.cpu().tolist() == cand[:, 0].tolist() and torch.isfinite(ll).all()


def test_raw_dataset_takes_a_finetune_step_from_files(cuda, tmp_path, monkeypatch):
    import run
    from pigeon_b200 import SuperGuessr, synthetic, training
    from pigeon_b200.super_guessr import CLIPVisionTower
    from pigeon_b200.vit_engine import VitDims
    inputs = _e2e_inputs(50)
    inputs = {s: {k: v[:8] for k, v in c.items()} for s, c in inputs.items()}
    _write_inputs(tmp_path, monkeypatch, {})
    out = dp.preprocess(data.raw_dataset(inputs), config.GEOCELL_PATH, multi_task=True)
    out.save_to_disk("pre")
    assert run.is_raw_split(out["train"])
    _, lnglat = dp.parse_geocells(config.GEOCELL_PATH)
    seen = {}

    def finetune_model(name, ds, multi_task, heading, yfcc, metrics=None, **kw):
        dims = VitDims(image_size=336, patch_size=14, hidden=256, heads=4, intermediate=512, layers=2)
        tower = CLIPVisionTower(dims)
        tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=3, std=0.05), strict=True)
        torch.manual_seed(3)
        sg = SuperGuessr(tower, panorama=True, multi_task=multi_task, should_smooth_labels=True, num_candidates=5,
                         freeze_base=True, geocells=lnglat).to("cuda")
        args = SimpleNamespace(learning_rate=1e-3, per_device_train_batch_size=8, per_device_eval_batch_size=8,
                               num_train_epochs=1, gradient_accumulation_steps=1)
        before = sg.cell_layer.weight.detach().clone()
        training.train_model(sg, ds, False, yfcc, args, metrics, **kw)
        seen.update(history=sg.train_history, moved=not torch.equal(before, sg.cell_layer.weight.detach()),
                    proc=kw["processor"])

    monkeypatch.setattr(training, "finetune_model", finetune_model)
    run.main(["finetune", config.CLIP_MODEL, "-l", "pre", "-m"])
    assert len(seen["history"]) == 1 and np.isfinite(seen["history"]).all() and seen["moved"]
    assert seen["proc"].host_decoded + seen["proc"].gpu_decoded >= 4 * 8
