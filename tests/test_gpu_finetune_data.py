"""`run.py` without -l on the GPU, from a metadata CSV and a folder of seeded synthetic JPEG and PNG files: `embed` writes
the embedding files, saves a dataset whose `embedding` rows equal CLIPEmbedding on the same files decoded by Pillow and
whose `labels_clf` equal `preprocess` on a hand-built raw split, and trains the head on it; `finetune` takes a step from
the image files; `evaluate -t` evaluates the `test` split.  The towers are small random ones: one layer of the
ViT-L width for the embedder (the embedding files must be config.CLIP_EMBED_DIM wide), and the tower of
tests/test_gpu_dataset_preprocessing.py for fine-tuning and evaluation."""
import io
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
datasets = pytest.importorskip("datasets")
pd = pytest.importorskip("pandas")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dataset_preprocessing_data as cells_data  # noqa: E402

from pigeon_b200 import config  # noqa: E402
from pigeon_b200 import dataset_preprocessing as dp  # noqa: E402

VIEWS = ("image", "image_2", "image_3", "image_4")
CENTRES = [[2, 2], [13, 1], [2.5, 14], [8, 14], [22, 22], [28, 28], [-40, -30], [175, 85], [-175, -85], [4, 4]]
SELECTION = ["train"] * 9 + ["val"] * 3 + ["holdout"] + ["test"] * 4
CLIMATES = ["Tropical, savannah", "Polar, frost", "Arid, desert, hot", "Temperate, no dry season, warm summer"]


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


def _encode(a, fmt):
    from PIL import Image
    f = io.BytesIO()
    Image.fromarray(a).save(f, fmt, **({"quality": 90} if fmt == "JPEG" else {}))
    return f.getvalue()


@pytest.fixture
def corpus(tmp_path, monkeypatch):
    """The metadata CSV (four views per row, every third file a PNG), the image folder and the geocell CSV, with the
    working directory and config.METADATA_PATH / IMAGE_PATH pointed at them."""
    from pigeon_b200 import synthetic
    monkeypatch.chdir(tmp_path)
    os.makedirs("imgs")
    rng = np.random.default_rng(11)
    n = len(SELECTION)
    names = {v: [] for v in VIEWS}
    for r in range(n):
        for j, v in enumerate(VIEWS):
            k = 4 * r + j
            fmt = "PNG" if k % 3 == 0 else "JPEG"
            name = f"r{r}_{j}.{'png' if fmt == 'PNG' else 'jpg'}"
            h, w = 40 + 7 * (k % 9), 48 + 5 * (k % 11)
            with open(os.path.join("imgs", name), "wb") as f:
                f.write(_encode(synthetic.synthetic_photo(h, w, seed=100 + k), fmt))
            names[v].append(name)
    pts = np.asarray(CENTRES, np.float64)[np.arange(n) % len(CENTRES)] + rng.normal(0, 0.2, (n, 2))
    frame = pd.DataFrame(dict(**names, lng=pts[:, 0], lat=np.clip(pts[:, 1], -90, 90)))
    for j, c in enumerate(dp.MULTI_TASK_COLUMNS):
        frame[f"{c}_reg"] = rng.normal(j, 1, n)
    frame["climate"] = [CLIMATES[k % len(CLIMATES)] for k in range(n)]
    frame["heading"] = rng.uniform(0, 360, n)
    frame["month"] = rng.integers(1, 13, n)
    frame["selection"] = SELECTION
    frame["geo_area"] = "Area"
    frame.to_csv("meta.csv", index=False)
    monkeypatch.setattr(config, "METADATA_PATH", "meta.csv")
    monkeypatch.setattr(config, "IMAGE_PATH", "imgs")
    os.makedirs(os.path.dirname(config.GEOCELL_PATH), exist_ok=True)
    cells_data.geocell_frame().to_csv(config.GEOCELL_PATH, index=False)
    _, lnglat = dp.parse_geocells(config.GEOCELL_PATH)
    return SimpleNamespace(frame=frame, lnglat=lnglat)


def _tower(dims, seed):
    from pigeon_b200 import synthetic
    from pigeon_b200.super_guessr import CLIPVisionTower
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=seed, std=0.05), strict=True)
    return tower


def _small_dims():
    from pigeon_b200.vit_engine import VitDims
    return VitDims(image_size=336, patch_size=14, hidden=256, heads=4, intermediate=512, layers=2)


def _rows(frame, split):
    return frame[frame["selection"] == split]


def _train_args():
    return SimpleNamespace(learning_rate=1e-3, per_device_train_batch_size=8, per_device_eval_batch_size=8,
                           num_train_epochs=1, gradient_accumulation_steps=1)


@pytest.mark.parametrize("sample", [None, "12"])
def test_embed_without_load_writes_embeddings_labels_and_trains(cuda, corpus, monkeypatch, sample):
    """With -s the drawn rows are a seeded subset (torch seed 0 leaves every split non-empty); every saved row must
    still get its own image's embedding."""
    import run
    from PIL import Image
    from pigeon_b200 import CLIPEmbedding, SuperGuessr, training
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims(image_size=336, patch_size=14, hidden=config.CLIP_EMBED_DIM, heads=16, intermediate=1024, layers=1)
    model = CLIPEmbedding("unused", device="cuda", clip_model=_tower(dims, 5))
    made, seen = [], {}

    def embedder(*a, **kw):
        made.append((a, kw))
        return model

    def finetune_on_embeddings(dataset, multi_task, heading, yfcc, metrics=None, **kw):
        torch.manual_seed(3)
        sg = SuperGuessr(base_model=None, panorama=not yfcc, multi_task=multi_task, heading=heading, freeze_base=True,
                         should_smooth_labels=True, yfcc=yfcc, geocells=corpus.lnglat, num_candidates=5).to("cuda")
        before = sg.cell_layer.weight.detach().clone()
        training.train_model(sg, dataset, True, yfcc, _train_args(), metrics)
        seen.update(history=sg.train_history, moved=not torch.equal(before, sg.cell_layer.weight.detach()))

    monkeypatch.setattr(run, "CLIPEmbedding", embedder)
    monkeypatch.setattr(training, "finetune_on_embeddings", finetune_on_embeddings)
    torch.manual_seed(0)
    run.main(["embed", "clip.model"] + ([] if sample is None else ["-s", sample]))
    assert made == [(("clip.model",), dict(load_checkpoint=True, panorama=True))]
    assert len(seen["history"]) == 1 and np.isfinite(seen["history"]).all() and seen["moved"]

    saved = datasets.DatasetDict.load_from_disk("data/hf_new_VIT" if sample is None else f"data/hf_dataset_{sample}")
    all_cells, drawn = [], 0
    for split in ("train", "val", "test"):
        index = saved[split].with_format("arrow")[:].column("index").to_numpy().tolist()
        rows = corpus.frame.loc[index]
        assert len(rows) > 0 and (rows["selection"] == split).all() and index == sorted(index)
        if sample is None:
            assert index == _rows(corpus.frame, split).index.tolist()
        drawn += len(rows)
        idx = np.load(f"data/landmark_embeddings/{split}_indices.npy")
        assert idx.tolist() == index
        pixels = [np.asarray(Image.open(os.path.join("imgs", f)).convert("RGB")) for f in rows["image"]]
        want = model(pixels).cpu().numpy()
        assert np.load(f"data/landmark_embeddings/{split}.npy").tobytes() == want.tobytes()
        table = saved[split].with_format("arrow")[:]
        assert not set(VIEWS) & set(saved[split].column_names)
        assert np.asarray(table.column("embedding").to_pylist(), np.float32).tobytes() == want.tobytes()
        cols = {v: [os.path.join("imgs", f) for f in rows[v]] for v in VIEWS}
        cols.update(lng=rows["lng"].to_numpy(), lat=rows["lat"].to_numpy(), index=rows.index.to_numpy(),
                    heading=rows["heading"].to_numpy())
        cols.update((c, rows[f"{c}_reg"].to_numpy()) for c in dp.MULTI_TASK_COLUMNS)
        raw = datasets.Dataset.from_dict(cols, features=datasets.Features(
            {**{v: datasets.Image() for v in VIEWS}, **{k: datasets.Value("int64" if k == "index" else "float64")
                                                        for k in cols if k not in VIEWS}}))
        got_cells = table.column("labels_clf").to_numpy()
        want_cells = dp.preprocess(datasets.DatasetDict({split: raw}), config.GEOCELL_PATH)[split]
        assert np.array_equal(got_cells, want_cells.with_format("arrow")[:].column("labels_clf").to_numpy())
        all_cells += got_cells.tolist()
    assert len(set(all_cells)) > 1
    holdout = int((corpus.frame["selection"] == "holdout").sum())
    assert drawn == len(corpus.frame) - holdout if sample is None else int(sample) - holdout <= drawn <= int(sample)


def test_finetune_without_load_takes_a_step_from_files(cuda, corpus, monkeypatch):
    import run
    from pigeon_b200 import SuperGuessr, training
    seen = {}

    def finetune_model(name, ds, multi_task, heading, yfcc, metrics=None, **kw):
        torch.manual_seed(3)
        sg = SuperGuessr(_tower(_small_dims(), 3), panorama=True, multi_task=multi_task, should_smooth_labels=True,
                         num_candidates=5, freeze_base=True, geocells=corpus.lnglat).to("cuda")
        before = sg.cell_layer.weight.detach().clone()
        training.train_model(sg, ds, False, yfcc, _train_args(), metrics, **kw)
        seen.update(history=sg.train_history, moved=not torch.equal(before, sg.cell_layer.weight.detach()),
                    proc=kw["processor"], n=len(ds["train"]))

    monkeypatch.setattr(training, "finetune_model", finetune_model)
    run.main(["finetune", config.CLIP_MODEL])
    assert len(seen["history"]) == 1 and np.isfinite(seen["history"]).all() and seen["moved"]
    assert seen["n"] == len(_rows(corpus.frame, "train"))
    assert seen["proc"].host_decoded + seen["proc"].gpu_decoded >= 4 * seen["n"] and seen["proc"].gpu_decoded > 0
    assert run.is_raw_split(datasets.DatasetDict.load_from_disk("data/hf_new_VIT")["train"])


def test_evaluate_without_load_takes_test_with_t(cuda, corpus, monkeypatch):
    import run
    from pigeon_b200 import SuperGuessr
    from pigeon_b200.benchmark import EvalDataset
    from pigeon_b200.loops import encoded_eval_collate, evaluate_model
    from pigeon_b200.preprocess import ClipImageProcessor
    out = []

    def evaluate(name, split, yfcc, landmarks=False, base_model=None, **kw):
        assert isinstance(split, EvalDataset) and base_model == "base.model"
        torch.manual_seed(3)
        sg = SuperGuessr(_tower(_small_dims(), 3), panorama=split.panorama, freeze_base=True, num_candidates=5,
                         geocells=corpus.lnglat).to("cuda")
        out.append(evaluate_model(sg, split.encoded(), None, None, None, collate_fn=encoded_eval_collate,
                                  processor=ClipImageProcessor()))

    monkeypatch.setattr(run, "evaluate", evaluate)
    run.main(["evaluate", "head.model", "-b", "base.model", "-t"])
    test = datasets.DatasetDict.load_from_disk("data/hf_new_VIT")["test"].with_format("arrow")[:]
    assert len(out[0]["preds"]) == len(_rows(corpus.frame, "test")) == test.num_rows
    assert np.isfinite(out[0]["loss"]) and 0 <= out[0]["Geocell_accuracy"] <= 1
    assert out[0]["preds_geocell"].shape == (test.num_rows,)
