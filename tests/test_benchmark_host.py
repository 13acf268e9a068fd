"""Host side of pigeon_b200.benchmark (BenchmarkDataset, EvalDataset, the encoded-file collate) and of `run.py evaluate`
routing: tests/golden/benchmark.npz against Pillow, the uint8 -> float32 / 255 -> uint8 round trip the reference's
CLIPProcessor call makes, the square-crop rule, the benchmarks.json lookup, string indexing, key filtering and the
collate reading bytes and paths.  No GPU: pixel_values come from a stand-in processor here."""
import hashlib
import io
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
GOLD = os.path.join(ROOT, "tests", "golden", "benchmark.npz")


def golden():
    G = np.load(GOLD)
    off = G["off"]
    return [dict(name=str(G["name"][k]), route=str(G["route"][k]), size=tuple(int(x) for x in G["size"][k]),
                 data=G["data"][off[k]:off[k + 1]].tobytes(), sha=G[f"sha{k}"].tobytes(), sample=G[f"sample{k}"])
            for k in range(int(G["count"]))]


def test_goldens_match_pillow_and_the_reference_crop():
    import make_benchmark_golden as M
    from PIL import Image
    cases = golden()
    assert os.path.getsize(GOLD) < 1 << 20
    for g in cases:
        im = Image.open(io.BytesIO(g["data"]))
        assert im.size[::-1] == g["size"], g["name"]
        px = M.reference_pixel_values(g["data"])
        assert px.shape == (3, 336, 336) and px.dtype == np.float32
        assert hashlib.sha256(px.tobytes()).digest() == g["sha"], g["name"]
        assert np.array_equal(px[:, ::17, ::13], g["sample"]), g["name"]
    sizes = [g["size"] for g in cases]
    assert (1, 1) in sizes and any(h == 1 and w > 1 for h, w in sizes) and any(w == 1 and h > 1 for h, w in sizes)
    assert any(int((w - min(h, w)) / 2) % 2 == 1 for h, w in sizes)              # an odd w0: rows not 4-byte aligned
    assert any(min(h, w) < 336 for h, w in sizes) and any(min(h, w) > 336 for h, w in sizes)
    assert {"P", "RGBA", "L", "CMYK"} <= {Image.open(io.BytesIO(g["data"])).mode for g in cases}


def test_goldens_route_as_labelled():
    from pigeon_b200.preprocess import route_encoded
    for g in golden():
        assert route_encoded(g["data"])[0] == g["route"], g["name"]


def test_float32_round_trip_is_the_identity():
    """_load_jpg divides by 255 in float32; transformers 4.23.1 to_pil_image multiplies by 255 and truncates."""
    v = np.arange(256, dtype=np.uint8)
    back = ((v.astype(np.float32) / 255) * 255).astype(np.uint8)
    assert np.array_equal(back, v)
    img = np.random.default_rng(0).integers(0, 256, (7, 9, 3), dtype=np.uint8)
    assert np.array_equal(((np.asarray(img, dtype=np.float32) / 255) * 255).astype(np.uint8), img)


def _reference_crop(image):
    s = np.min(image.shape[:2])
    h_start = int((image.shape[0] - s) / 2)
    w_start = int((image.shape[1] - s) / 2)
    return image[h_start: h_start + s, w_start:w_start + s]


@pytest.mark.parametrize("h,w", [(1, 1), (1, 2), (2, 1), (1, 57), (57, 1), (333, 500), (500, 333), (336, 337),
                                 (337, 336), (100, 103), (103, 100), (768, 1024), (4, 4)])
def test_square_crop_matches_the_reference(h, w):
    from pigeon_b200.preprocess import _square, square_crop_box
    img = np.arange(h * w * 3, dtype=np.int64).reshape(h, w, 3)
    h0, w0, s = square_crop_box(h, w)
    assert np.array_equal(img[h0:h0 + s, w0:w0 + s], _reference_crop(img))
    assert np.array_equal(_square(img), _reference_crop(img))
    t = torch.from_numpy(img.astype(np.uint8))
    v = _square(t)
    assert v.stride(2) == 1 and v.stride(1) == 3 and v.data_ptr() == t.data_ptr() + (h0 * w + w0) * 3


class FakeProcessor:
    """Stands in for ClipImageProcessor: records its calls, returns a [n, 3, 336, 336] tensor numbering the files."""

    def __init__(self):
        self.calls = []

    def __call__(self, images=None, square_crop=False, **kw):
        self.calls.append((list(images), square_crop))
        n = len(images)
        return {"pixel_values": torch.arange(n, dtype=torch.float32).view(n, 1, 1, 1).expand(n, 3, 336, 336).clone()}


@pytest.fixture
def bench(tmp_path, monkeypatch):
    """A two-benchmark benchmarks.json with one CSV and an image folder given as a prefix (no trailing separator)."""
    from pigeon_b200 import benchmark, config
    (tmp_path / "imgs").mkdir()
    files = {}
    for i, g in enumerate(golden()[:5]):
        name = f"{i:03d}.bin"
        (tmp_path / "imgs" / f"pre_{name}").write_bytes(g["data"])
        files[name] = g["data"]
    import pandas as pd
    df = pd.DataFrame(dict(image=list(files), lng=[10.5, -3.25, 0.0, 179.9, -120.0], lat=[1.0, 2.0, -45.5, 60.0, 0.5],
                           geocell_idx_yfcc=[3, 1, 4, 1, 5], extra=list("abcde")))
    df.to_csv(tmp_path / "meta.csv", index=False)
    j = tmp_path / "benchmarks.json"
    j.write_text(json.dumps({"tiny": {"meta": str(tmp_path / "meta.csv"), "images": str(tmp_path / "imgs" / "pre_")},
                             "other": {"meta": "missing.csv", "images": "x"}}))
    monkeypatch.setattr(config, "BENCHMARKS", str(j))
    proc = FakeProcessor()
    monkeypatch.setattr(benchmark, "_processor", proc)
    return benchmark, files, proc


def test_benchmark_lookup_and_string_indexing(bench):
    benchmark, files, proc = bench
    ds = benchmark.BenchmarkDataset("tiny")
    assert ds.name == "tiny" and len(ds) == 5 and ds.panorama is False and ds.multi_task is False
    lab = ds["labels"]
    assert lab.dtype == np.float64 and lab.shape == (5, 2) and lab[1].tolist() == [-3.25, 2.0]
    assert ds["labels_clf"].tolist() == [3, 1, 4, 1, 5]
    assert ds["extra"].tolist() == list("abcde")
    assert ds.image_path("000.bin").endswith(os.path.join("imgs", "pre_000.bin"))       # concatenation, not join
    item = ds[1]
    assert proc.calls == [([files["001.bin"]], True)]
    assert tuple(item["pixel_values"].shape) == (1, 3, 336, 336)
    assert item["labels"].dtype == torch.float64 and item["labels"].tolist() == [-3.25, 2.0]
    assert item["labels_clf"].dtype == torch.int64 and int(item["labels_clf"]) == 1
    with pytest.raises(AssertionError, match="nope is not a valid benchmark"):
        benchmark.BenchmarkDataset("nope")


def test_encoded_rows_and_collate_read_paths(bench):
    from pigeon_b200 import loops
    benchmark, files, proc = bench
    rows = benchmark.BenchmarkDataset("tiny").encoded()
    assert len(rows) == 5 and rows.panorama is False and rows["labels_clf"].tolist() == [3, 1, 4, 1, 5]
    batch = loops.encoded_eval_collate([rows[i] for i in (4, 0, 2)])
    assert batch["files"] == [files["004.bin"], files["000.bin"], files["002.bin"]]
    assert batch["views"] == 1 and batch["square_crop"] is True
    assert batch["labels"].dtype == torch.float64 and batch["labels"].tolist() == [[-120.0, 0.5], [10.5, 1.0], [0.0, -45.5]]
    assert batch["labels_clf"].dtype == torch.int64 and batch["labels_clf"].tolist() == [5, 3, 4]
    out = loops.encoded_pixel_values(batch, proc)
    assert proc.calls[-1] == (batch["files"], True)
    assert tuple(out["pixel_values"].shape) == (3, 3, 336, 336) and sorted(out) == ["labels", "labels_clf", "pixel_values"]
    # the collate is what DataLoader workers run
    dl = torch.utils.data.DataLoader(rows, 2, collate_fn=loops.encoded_eval_collate)
    assert [b["labels_clf"].tolist() for b in dl] == [[3, 1], [4, 1], [5]]


def _raw_split(views: int, n: int = 3, path_dir=None):
    datasets = pytest.importorskip("datasets")
    G = golden()
    cols = ["image"] + [f"image_{i}" for i in range(2, views + 1)]
    data = {}
    for v, c in enumerate(cols):
        vals = []
        for r in range(n):
            b = G[(r * views + v) % len(G)]["data"]
            if path_dir is not None and (r + v) % 2:
                p = os.path.join(path_dir, f"{c}_{r}.bin")
                with open(p, "wb") as f:
                    f.write(b)
                vals.append({"bytes": None, "path": p})
            else:
                vals.append({"bytes": b, "path": None})
        data[c] = vals
    data["labels"] = [[float(r), -float(r)] for r in range(n)]
    data["labels_clf"] = list(range(10, 10 + n))
    feats = {c: datasets.Image() for c in cols}
    feats.update(labels=datasets.Sequence(datasets.Value("float64")), labels_clf=datasets.Value("int64"))
    return datasets.Dataset.from_dict(data, features=datasets.Features(feats)).with_format("torch"), data


def test_eval_dataset_filters_image_keys_and_concatenates_views(bench, tmp_path):
    benchmark, _, proc = bench
    split, data = _raw_split(4, path_dir=str(tmp_path))
    ds = benchmark.EvalDataset(split)
    assert len(ds) == 3 and ds.views == ["image", "image_2", "image_3", "image_4"] and ds.panorama
    item = ds[1]
    assert sorted(item) == ["labels", "labels_clf", "pixel_values"]
    assert tuple(item["pixel_values"].shape) == (1, 12, 336, 336) and proc.calls[-1][1] is False
    want = [benchmark.read_encoded(data[c][1]) for c in ds.views]
    assert proc.calls[-1][0] == want
    sl = ds[0:2]
    assert sorted(sl) == ["labels", "labels_clf", "pixel_values"] and tuple(sl["pixel_values"].shape) == (2, 12, 336, 336)
    assert proc.calls[-1][0] == [benchmark.read_encoded(data[c][r]) for r in range(2) for c in ds.views]
    assert np.asarray(ds["labels_clf"]).tolist() == [10, 11, 12]                          # passes through
    from pigeon_b200 import loops
    rows = ds.encoded()
    batch = loops.encoded_eval_collate([rows[i] for i in range(3)])
    assert batch["views"] == 4 and batch["square_crop"] is False and len(batch["files"]) == 12
    assert batch["files"] == [benchmark.read_encoded(data[c][r]) for r in range(3) for c in ds.views]
    assert batch["labels_clf"].tolist() == [10, 11, 12] and batch["labels"].tolist() == [[0, 0], [1, -1], [2, -2]]
    assert tuple(loops.encoded_pixel_values(batch, proc)["pixel_values"].shape) == (3, 12, 336, 336)
    one = benchmark.EvalDataset(_raw_split(1)[0])
    assert one.views == ["image"] and not one.panorama and tuple(one[0]["pixel_values"].shape) == (1, 3, 336, 336)
    datasets = pytest.importorskip("datasets")
    dd = benchmark.EvalDataset.transform(datasets.DatasetDict(train=split, val=split, test=split))
    assert isinstance(dd, datasets.DatasetDict) and all(isinstance(v, benchmark.EvalDataset) for v in dd.values())


def test_evaluate_model_takes_collate_and_processor_together():
    from pigeon_b200 import loops
    with pytest.raises(ValueError, match="go together"):
        loops.evaluate_model(None, [], None, collate_fn=loops.encoded_eval_collate)


def test_run_routes_names_directories_and_raw_splits(bench, tmp_path, monkeypatch):
    datasets = pytest.importorskip("datasets")
    import run
    benchmark = bench[0]
    seen = []
    monkeypatch.setattr(run, "evaluate", lambda name, ds, *a, **kw: seen.append((name, ds, kw)))
    run.main(["evaluate", "head.model", "-l", "tiny", "-b", "base", "-w", "3"])
    assert isinstance(seen[-1][1], benchmark.BenchmarkDataset) and seen[-1][1].name == "tiny"
    assert seen[-1][2]["num_workers"] == 3 and seen[-1][2]["base_model"] == "base"
    split, _ = _raw_split(4)
    datasets.DatasetDict(test=split).save_to_disk(str(tmp_path / "raw"))
    run.main(["evaluate", "head.model", "-l", str(tmp_path / "raw")])
    assert isinstance(seen[-1][1], benchmark.EvalDataset) and len(seen[-1][1]) == 3
    pre = datasets.Dataset.from_dict({"pixel_values": [[0.0]], "labels": [[0.0, 0.0]], "labels_clf": [0]})
    datasets.DatasetDict(test=pre).save_to_disk(str(tmp_path / "pre"))
    run.main(["evaluate", "head.model", "-l", str(tmp_path / "pre")])
    assert isinstance(seen[-1][1], datasets.Dataset) and not isinstance(seen[-1][1], benchmark.EvalDataset)
    assert seen[-1][1].column_names == ["pixel_values", "labels", "labels_clf"]


def test_evaluate_needs_a_base_model_for_images(bench):
    import run
    with pytest.raises(ValueError, match="base model"):
        run.evaluate("head.model", bench[0].BenchmarkDataset("tiny"), yfcc=True)
