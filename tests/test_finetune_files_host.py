"""Host side of fine-tuning from the image files of raw splits: the encoded collate carries every label column
`SuperGuessr.forward` takes (with the dtype and shape the pixel_values route's default collate gives it) and only
those the split has, evaluation batches keep their keys, `train_model` takes `collate_fn` and `processor` together
only, both routes draw the same batches from the same torch seed, and `run.py finetune` picks the encoded route for
raw splits.  No GPU: pixel_values come from a stand-in processor here."""
import os
import sys

import numpy as np
import pytest
import torch

datasets = pytest.importorskip("datasets")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "benchmark.npz")
VIEWS = ["image", "image_2", "image_3", "image_4"]
OPTIONAL = ["labels_multi_task", "labels_climate", "labels_month", "heading"]


@pytest.fixture(autouse=True)
def _rows_without_torchvision(monkeypatch):
    """datasets' torch formatter imports torchvision.io.VideoReader whenever torchvision is loaded (an earlier test's
    transformers import loads it), and this torchvision has none: format the rows as a process without it does."""
    monkeypatch.delitem(sys.modules, "torchvision", raising=False)


def _files(n):
    G = np.load(GOLD)
    off = G["off"]
    return [G["data"][off[k % int(G["count"])]:off[k % int(G["count"]) + 1]].tobytes() for k in range(n)]


def _columns(n, optional=True, seed=0):
    rng = np.random.default_rng(seed)
    cols = dict(labels=rng.uniform(-60, 60, (n, 2)).tolist(), labels_clf=rng.integers(0, 50, n).tolist())
    feats = dict(labels=datasets.Sequence(datasets.Value("float64")), labels_clf=datasets.Value("int64"))
    if optional:
        cols.update(labels_multi_task=rng.normal(size=(n, 6)).tolist(),
                    labels_climate=rng.dirichlet(np.ones(28), n).tolist(),                    # soft targets
                    labels_month=rng.integers(0, 12, n).tolist(), heading=rng.uniform(0, 360, (n, 4)).tolist())
        feats.update(labels_multi_task=datasets.Sequence(datasets.Value("float32")),
                     labels_climate=datasets.Sequence(datasets.Value("float32")), labels_month=datasets.Value("int64"),
                     heading=datasets.Sequence(datasets.Value("float32")))
    return cols, feats


def raw_split(n, optional=True, seed=0):
    """A raw four-view split (encoded `image`..`image_4`) and its twin with a pixel_values column instead."""
    cols, feats = _columns(n, optional, seed)
    files = _files(4 * n)
    raw = dict(cols, **{c: [{"bytes": files[4 * r + v], "path": None} for r in range(n)] for v, c in enumerate(VIEWS)})
    rf = dict(feats, **{c: datasets.Image() for c in VIEWS})
    px = np.arange(n, dtype=np.float32).reshape(n, 1, 1, 1) * np.ones((1, 12, 2, 2), np.float32)
    twin = dict(cols, pixel_values=px)
    tf = dict(feats, pixel_values=datasets.Array3D((12, 2, 2), "float32"))
    return (datasets.Dataset.from_dict(raw, features=datasets.Features(rf)).with_format("torch"),
            datasets.Dataset.from_dict(twin, features=datasets.Features(tf)).with_format("torch"))


class FakeProcessor:
    """Stands in for ClipImageProcessor: returns a [n, 3, 336, 336] tensor numbering the files."""

    def __call__(self, images=None, square_crop=False, **kw):
        n = len(images)
        return {"pixel_values": torch.arange(n, dtype=torch.float32).view(n, 1, 1, 1).expand(n, 3, 336, 336).clone()}


@pytest.mark.parametrize("optional", [True, False])
def test_collate_carries_the_label_columns_the_split_has(optional):
    from pigeon_b200 import benchmark, loops
    raw, twin = raw_split(5, optional)
    rows = benchmark.EvalDataset(raw).encoded()
    idx = [3, 0, 4]
    got = loops.encoded_eval_collate([rows[i] for i in idx])
    want = torch.utils.data.default_collate([twin[i] for i in idx])       # what the pixel_values route's loader yields
    keys = ["labels", "labels_clf"] + (OPTIONAL if optional else [])
    assert sorted(k for k in got if k in loops.LABEL_COLUMNS) == sorted(keys)
    for k in keys:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape and torch.equal(got[k], want[k]), k
    assert got["labels_multi_task" if optional else "labels"].shape == ((3, 6) if optional else (3, 2))
    assert got["files"] == [rows[i]["images"][v]["bytes"] for i in idx for v in range(4)] and got["views"] == 4
    out = loops.encoded_pixel_values(got, FakeProcessor())
    assert sorted(out) == sorted(keys + ["pixel_values"]) and tuple(out["pixel_values"].shape) == (3, 12, 336, 336)
    for k in keys:
        assert out[k] is got[k]


def test_evaluation_batches_keep_their_keys(tmp_path, monkeypatch):
    """A benchmark (no optional columns by construction) and a raw split without them: labels and labels_clf only."""
    import json
    import pandas as pd
    from pigeon_b200 import benchmark, config, loops
    (tmp_path / "imgs").mkdir()
    for i, f in enumerate(_files(3)):
        (tmp_path / "imgs" / f"{i}.bin").write_bytes(f)
    pd.DataFrame(dict(image=[f"{i}.bin" for i in range(3)], lng=[1.0, 2.0, 3.0], lat=[4.0, 5.0, 6.0],
                      geocell_idx_yfcc=[7, 8, 9])).to_csv(tmp_path / "meta.csv", index=False)
    (tmp_path / "b.json").write_text(json.dumps({"t": {"meta": str(tmp_path / "meta.csv"),
                                                      "images": str(tmp_path / "imgs") + os.sep}}))
    monkeypatch.setattr(config, "BENCHMARKS", str(tmp_path / "b.json"))
    rows = benchmark.BenchmarkDataset("t").encoded()
    batch = loops.encoded_eval_collate([rows[i] for i in range(3)])
    assert sorted(batch) == ["files", "labels", "labels_clf", "square_crop", "views"]
    assert batch["labels"].dtype == torch.float64 and batch["labels_clf"].dtype == torch.int64
    assert sorted(loops.encoded_pixel_values(batch, FakeProcessor())) == ["labels", "labels_clf", "pixel_values"]
    raw, _ = raw_split(3, optional=False)
    row = benchmark.EvalDataset(raw).encoded()[1]
    assert sorted(row) == ["images", "labels", "labels_clf", "square_crop"]


def test_train_model_takes_collate_and_processor_together():
    from pigeon_b200 import loops, training
    with pytest.raises(ValueError, match="go together"):
        training.train_model(None, {}, False, False, None, None, collate_fn=loops.encoded_eval_collate)
    with pytest.raises(ValueError, match="go together"):
        training.train_model(None, {}, False, False, None, None, processor=FakeProcessor())


def test_both_routes_draw_the_same_batches():
    """The loaders train_model builds for the two routes, from the same seed: the same rows in the same order, and the
    global generator left in the same state."""
    from pigeon_b200 import benchmark, loops
    raw, twin = raw_split(11)
    rows = benchmark.EvalDataset(raw).encoded()
    seen = []
    for ds, kw in ((twin, {}), (rows, dict(collate_fn=loops.encoded_eval_collate))):
        torch.manual_seed(3)
        dl = torch.utils.data.DataLoader(ds, 4, shuffle=True, **kw)
        order = [b["labels_clf"].tolist() for epoch in range(2) for b in dl]
        seen.append((order, torch.rand(3)))
    assert seen[0][0] == seen[1][0] and torch.equal(seen[0][1], seen[1][1])
    assert sorted(sum(seen[0][0][:3], [])) == sorted(np.asarray(twin["labels_clf"]).tolist())


def test_run_finetune_routes_raw_and_pixel_splits(tmp_path, monkeypatch):
    import run
    from pigeon_b200 import benchmark, loops, preprocess, training
    calls, procs = [], []

    class Proc:
        def __init__(self, **kw):
            procs.append(kw)

    monkeypatch.setattr(training, "finetune_model", lambda name, ds, **kw: calls.append((name, ds, kw)))
    monkeypatch.setattr(preprocess, "ClipImageProcessor", Proc)
    raw, twin = raw_split(3)
    datasets.DatasetDict(train=raw, val=raw).save_to_disk(str(tmp_path / "raw"))
    datasets.DatasetDict(train=twin, val=twin).save_to_disk(str(tmp_path / "pre"))
    name = "openai/clip-vit-large-patch14-336"
    run.main(["finetune", name, "-l", str(tmp_path / "raw"), "--png", "-w", "3", "-m"])
    _, ds, kw = calls[-1]
    assert sorted(ds) == ["train", "val"] and all(isinstance(v, benchmark.EncodedRows) for v in ds.values())
    assert isinstance(ds["train"].dataset, benchmark.EvalDataset) and len(ds["train"]) == 3 and ds["train"].panorama
    assert kw["collate_fn"] is loops.encoded_eval_collate and isinstance(kw["processor"], Proc)
    assert procs[-1] == dict(jpeg_multiscan=False, png=True)
    assert kw["num_workers"] == 3 and kw["multi_task"] is True
    run.main(["finetune", name, "-l", str(tmp_path / "raw"), "--jpeg-multiscan"])
    assert procs[-1] == dict(jpeg_multiscan=True, png=False) and calls[-1][2]["num_workers"] == 0
    run.main(["finetune", name, "-l", str(tmp_path / "pre")])
    _, ds, kw = calls[-1]
    assert isinstance(ds, datasets.DatasetDict) and "pixel_values" in ds["train"].column_names
    assert "collate_fn" not in kw and "processor" not in kw and len(procs) == 2
    args = run.build_parser().parse_args(["finetune", name, "-l", "d", "--png", "--jpeg-multiscan", "-w", "2"])
    assert args.png and args.jpeg_multiscan and args.workers == 2
    assert run.is_raw_split(raw) and not run.is_raw_split(twin) and not run.is_raw_split(object())


GLOO_WORKER = """
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, %r)
sys.path.insert(0, %r)
import test_finetune_files_host as H
from pigeon_b200 import benchmark, loops
rank = int(sys.argv[1])
os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=sys.argv[2], RANK=str(rank), WORLD_SIZE="2")
dist.init_process_group("gloo", rank=rank, world_size=2)
raw, twin = H.raw_split(11)
rows = benchmark.EvalDataset(raw).encoded()
seen = []
for ds, kw in ((twin, {}), (rows, dict(collate_fn=loops.encoded_eval_collate))):
    torch.manual_seed(3)
    sampler = torch.utils.data.distributed.DistributedSampler(ds, shuffle=True)      # as train_model builds it
    dl = torch.utils.data.DataLoader(ds, 2, sampler=sampler, **kw)
    order = []
    for epoch in range(2):
        sampler.set_epoch(epoch)
        for b in dl:
            order.append(b["labels_clf"])
            assert b["labels_multi_task"].shape == (len(b["labels_clf"]), 6)
    seen.append(torch.cat(order))
assert torch.equal(seen[0], seen[1])
both = [torch.empty_like(seen[1]) for _ in range(2)]
dist.all_gather(both, seen[1])
assert len(seen[1]) == 2 * 6                                # per rank and epoch: ceil(11 / 2) rows
for e in range(2):
    rows_e = torch.cat([both[0][6 * e:6 * e + 6], both[1][6 * e:6 * e + 6]]).tolist()
    assert set(rows_e) == set(torch.as_tensor(twin["labels_clf"]).tolist())
dist.destroy_process_group()
print("rank", rank, "ok")
"""


def test_distributed_sampler_and_collate_gloo_world2(tmp_path):
    """Under torch.distributed (gloo, world size 2) each rank draws the same rows on both routes, and the ranks
    together cover the split every epoch."""
    import subprocess
    script = tmp_path / "w.py"
    script.write_text(GLOO_WORKER % (ROOT, os.path.join(ROOT, "tests")))
    port = str(31000 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), str(r), port], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
             for r in range(2)]
    outs = [p.communicate(timeout=300)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o[-3000:]
