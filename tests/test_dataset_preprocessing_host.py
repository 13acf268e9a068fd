"""Host side of pigeon_b200.dataset_preprocessing: the WKT reader against hand-built CSR arrays and its rejections, the
heading and multi-task columns bit for bit against the reference (tests/golden/dataset_preprocessing.npz, from
tools/make_dataset_preprocessing_golden.py), whole `preprocess` runs with the device locator replaced by
tests/metrics_oracle.py's exact one (every column, its order and its torch dtype against the reference's), the
embedding join and its errors, and the command line."""
import os
import sys

import numpy as np
import pytest

datasets = pytest.importorskip("datasets")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dataset_preprocessing_data as data  # noqa: E402
import metrics_oracle as mo  # noqa: E402

from pigeon_b200 import config  # noqa: E402
from pigeon_b200 import dataset_preprocessing as dp  # noqa: E402

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dataset_preprocessing.npz"))
CONFIGS = ["emb", "emb_mt", "raw", "raw_mt", "emb_other"]


def golden_inputs():
    return {s: {k[len(f"in/{s}/"):]: GOLDEN[k] for k in GOLDEN.files
                if k.startswith(f"in/{s}/") and not k.endswith(("embeds", "indices"))} for s in data.SPLITS}


@pytest.fixture(autouse=True)
def _rows_without_torchvision(monkeypatch):
    """datasets' torch formatter imports torchvision.io.VideoReader whenever torchvision is loaded (an earlier test's
    transformers import loads it), and this torchvision has none: format the rows as a process without it does."""
    monkeypatch.delitem(sys.modules, "torchvision", raising=False)


class OracleIndex:
    """metrics.CountryIndex's constructor and `locate`, on the host with the exact oracle."""
    calls = []

    def __init__(self, verts, ring_off, part_ring_off, geom_part_off, device=None):
        self.geoms = mo.geometries_from_csr(verts, ring_off, part_ring_off, geom_part_off)

    def locate(self, labels, preds=None):
        import torch
        labels = np.asarray(labels, dtype=np.float64)
        OracleIndex.calls.append(len(labels))
        c, f, _ = mo.locate(self.geoms, labels, labels)
        return torch.from_numpy(c), torch.from_numpy(f), None


@pytest.fixture
def oracle(monkeypatch):
    OracleIndex.calls = []
    monkeypatch.setattr(dp, "CountryIndex", OracleIndex)
    return OracleIndex


def test_wkt_reader_builds_the_csr_layout():
    text = ("MULTIPOLYGON Z (((0 0 1, 10 0 1, 10 10 1, 0 10 1, 0 0 1), (3 3 0, 3 5 0, 5 5 0, 5 3 0, 3 3 0)), "
            "((12 0 7, 14 0 7, 14 2 7, 12 0 7)))")
    parts = dp.parse_wkt(text)
    poly = dp.parse_wkt("polygon((-180 -90, 180 -90, 180 90, -180 -90))")
    verts, ring_off, part_ring_off, geom_part_off = dp.geometries_to_csr([parts, poly])
    want = np.asarray([[0, 0], [10, 0], [10, 10], [0, 10], [0, 0], [3, 3], [3, 5], [5, 5], [5, 3], [3, 3],
                       [12, 0], [14, 0], [14, 2], [12, 0], [-180, -90], [180, -90], [180, 90], [-180, -90]], np.float64)
    assert verts.dtype == np.float64 and np.array_equal(verts, want)
    assert ring_off.tolist() == [0, 5, 10, 14, 18]
    assert part_ring_off.tolist() == [0, 2, 3, 4] and geom_part_off.tolist() == [0, 2, 3]
    assert all(o.dtype == np.int64 for o in (ring_off, part_ring_off, geom_part_off))
    # correctly rounded like GEOS's reader; Z and M positions keep x and y
    x = dp.parse_wkt("POLYGON ZM ((0.1 1e-320 5 6, 2.675 -0 5 6, 0.3 0.7 5 6, 0.1 1e-320 5 6))")[0][0]
    assert x[0, 1] == 1e-320 and x[1, 0] == 2.675 and np.signbit(x[1, 1]) and x[2, 0] == 0.3
    assert dp.parse_wkt("POLYGON M ((0 0 9, 1 0 9, 1 1 9, 0 0 9))")[0][0].shape == (4, 2)


@pytest.mark.parametrize("text, match", [
    ("POLYGON EMPTY", "empty"), ("MULTIPOLYGON EMPTY", "empty"), ("POLYGON Z EMPTY", "empty"),
    ("GEOMETRYCOLLECTION (POLYGON ((0 0, 1 0, 1 1, 0 0)))", "POLYGON or MULTIPOLYGON"),
    ("POINT (1 2)", "POLYGON or MULTIPOLYGON"), ("LINESTRING (0 0, 1 1)", "POLYGON or MULTIPOLYGON"),
    ("POLYGON ((0 0, 1 0, 1 1, 0 1))", "not closed"), ("POLYGON ((0 0, 1 0, 0 0))", "at least 4"),
    ("POLYGON ((0 0, 1 0, 1 1, 0 0), (0 0, 1 0, 0 0))", "at least 4"),
    ("POLYGON ((0 0, nan 0, 1 1, 0 0))", "non-finite"), ("POLYGON ((0 0, 1 0, 1 inf, 0 0))", "non-finite"),
    ("POLYGON ((0 0, 1 0, 1 1, 0 0)", "malformed"), ("POLYGON ((0 0, 1 0, 1 1, 0 0))) x", "malformed"),
    ("POLYGON ((0 0, 1_0 0, 1 1, 0 0))", "not a number"), ("POLYGON ((0, 1 0, 1 1, 0))", "2 to 4"), ("", "nothing"),
])
def test_wkt_reader_rejects(text, match):
    with pytest.raises(ValueError, match=match) as e:
        dp.parse_wkt(text, "geocell row 7")
    assert "geocell row 7" in str(e.value)


def test_geocell_csv_rows_are_named_and_match_the_golden(tmp_path):
    (csr, lnglat) = dp.parse_geocells(data.geocell_frame())
    path = tmp_path / "cells.csv"
    path.write_bytes(GOLDEN["geocells_csv"].tobytes())
    csr2, lnglat2 = dp.parse_geocells(str(path))
    assert all(np.array_equal(a, b) for a, b in zip(csr, csr2)) and np.array_equal(lnglat, lnglat2)
    geoms = mo.geometries_from_csr(*csr)
    assert len(geoms) == len(data.cells()) and lnglat.dtype == np.float64 and lnglat.shape == (len(geoms), 2)
    df = data.geocell_frame()
    df.loc[3, "polygon"] = "POLYGON EMPTY"
    with pytest.raises(ValueError, match="geocell row 3"):
        dp.parse_geocells(df)
    with pytest.raises(ValueError, match="polygon"):
        dp.parse_geocells(df.drop(columns=["polygon"]))


@pytest.mark.parametrize("split", data.SPLITS)
def test_heading_and_multi_task_columns_equal_the_reference(split):
    inp = golden_inputs()[split]
    h = dp.heading_features(inp["heading"])
    assert h.dtype == np.float64 and h.shape == (len(inp["heading"]), 4, 2)
    assert np.array_equal(h, GOLDEN[f"emb/{split}/heading"])
    mt = dp.multi_task_labels([inp[c] for c in data.MT])
    assert mt.dtype == np.float64 and np.array_equal(mt, GOLDEN[f"emb_mt/{split}/labels_multi_task"])
    assert dp.multi_task_labels([np.arange(3)] * 6).dtype == np.int64            # np.array of six ints


def _run(name, tmp_path, monkeypatch, inputs=None, **kw):
    emb, path_is_default = bool(GOLDEN[f"{name}/args"][1]), bool(GOLDEN[f"{name}/args"][0])
    mt = bool(GOLDEN[f"{name}/args"][2])
    monkeypatch.chdir(tmp_path)
    path = config.GEOCELL_PATH if path_is_default else "cells/other.csv"
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(GOLDEN["geocells_csv"].tobytes())
    for s in data.SPLITS:
        os.makedirs("emb", exist_ok=True)
        np.save(f"emb/{s}.npy", GOLDEN[f"in/{s}/embeds"])
        np.save(f"emb/{s}_indices.npy", GOLDEN[f"in/{s}/indices"])
    ds = data.raw_dataset(inputs or golden_inputs())
    return ds, dp.preprocess(ds, path, embedder=object() if emb else None, multi_task=mt, embeddings_dir="emb", **kw)


@pytest.mark.parametrize("name", CONFIGS)
def test_preprocess_columns_and_dtypes_equal_the_reference(name, tmp_path, monkeypatch, oracle):
    raw, out = _run(name, tmp_path, monkeypatch)
    assert sorted(out) == sorted(data.SPLITS) and oracle.calls == [len(raw[s]) for s in out]   # one locate per split
    for s in data.SPLITS:
        split = out[s]
        cols = GOLDEN[f"{name}/{s}/columns"].tolist()
        assert split.column_names == cols
        assert split.format["type"] == "torch"
        row = split[:2]
        assert [str(row[c].dtype) if hasattr(row[c], "dtype") else "-" for c in cols] == \
            GOLDEN[f"{name}/{s}/torch_dtypes"].tolist()
        table = split.with_format("arrow")[:]
        for c in cols:
            if c.startswith("image"):
                assert table.column(c).to_pylist() == raw[s].with_format("arrow")[:].column(c).to_pylist()
                continue
            got = np.asarray(table.column(c).to_pylist())
            want = GOLDEN[f"{name}/{s}/{c}"]
            assert got.shape == want.shape and np.array_equal(got, want), (s, c)
        assert split.features["labels"].feature.dtype == "float64"
        assert split.features["labels_clf"].dtype == "int64"


def test_embedding_join_order_and_errors(tmp_path, monkeypatch, oracle):
    idx = np.asarray([30, 10, 40, 20, 10])                     # file order of the dataset's index values, one padding row
    embeds = np.arange(5, dtype=np.float32)[:, None] * np.ones((1, config.CLIP_EMBED_DIM), np.float32)
    got = dp.join_embeddings(4, embeds, idx)
    assert got[:, 0].tolist() == [1, 3, 0, 2] and got.dtype == np.float32          # argsort(indices[:4])
    assert dp.join_embeddings(3, embeds, idx.reshape(-1, 1))[:, 0].tolist() == [1, 0, 2]
    with pytest.raises(ValueError, match="D = 512"):
        dp.join_embeddings(4, np.zeros((5, 512), np.float32), idx)
    with pytest.raises(ValueError, match="2-D"):
        dp.join_embeddings(4, np.zeros(5 * 1024, np.float32), idx)
    with pytest.raises(ValueError, match="for 6 rows"):
        dp.join_embeddings(6, embeds, idx)
    # a wrong D in the files, and a split that lacks a column the reference removes, fail before any work is done
    inputs = golden_inputs()
    del inputs["val"]["temp_diff"]
    with pytest.raises(ValueError, match="'val'.*temp_diff"):
        _run("emb", tmp_path, monkeypatch, inputs)
    assert oracle.calls == []
    inputs = golden_inputs()
    del inputs["test"]["lat"]
    with pytest.raises(ValueError, match="'test'.*lat"):
        _run("raw", tmp_path, monkeypatch, inputs)
    np.save(tmp_path / "emb" / "val.npy", np.zeros((40, 768), np.float32))
    ds = data.raw_dataset(golden_inputs())
    with pytest.raises(ValueError, match="D = 768"):
        dp.preprocess(ds, config.GEOCELL_PATH, embedder=True, embeddings_dir="emb")


def test_embedding_branch_needs_the_image_columns(tmp_path, monkeypatch, oracle):
    ds = data.raw_dataset(golden_inputs())
    ds["train"] = ds["train"].remove_columns(["image_3"])
    monkeypatch.chdir(tmp_path)
    (tmp_path / "data").mkdir()
    (tmp_path / config.GEOCELL_PATH).write_bytes(GOLDEN["geocells_csv"].tobytes())
    with pytest.raises(ValueError, match="'train'.*image_3"):
        dp.preprocess(ds, config.GEOCELL_PATH, embedder=True)
    out = dp.preprocess(ds, config.GEOCELL_PATH)                 # the raw branch keeps whatever views the split has
    assert "image_3" not in out["train"].column_names and "image_3" in out["val"].column_names


def test_cli_arguments(monkeypatch):
    a = dp.build_parser().parse_args(["raw", "cells.csv", "out"])
    assert (a.raw_dataset_dir, a.geocell_csv, a.output_dir, a.embeddings, a.multitask) == ("raw", "cells.csv", "out", None, False)
    a = dp.build_parser().parse_args(["raw", "cells.csv", "out", "--embeddings", "e", "--multitask"])
    assert a.embeddings == "e" and a.multitask
    with pytest.raises(SystemExit):
        dp.build_parser().parse_args(["raw", "cells.csv"])
    seen = {}

    class Saved:
        def save_to_disk(self, path):
            seen["saved"] = path

    monkeypatch.setattr(datasets.DatasetDict, "load_from_disk", staticmethod(lambda p: seen.setdefault("loaded", p)))
    monkeypatch.setattr(dp, "preprocess", lambda ds, path, **kw: seen.update(args=(ds, path, kw)) or Saved())
    dp.main(["raw", "cells.csv", "out", "--embeddings", "e", "--multitask"])
    assert seen["args"] == ("raw", "cells.csv", dict(multi_task=True, embedder=True, embeddings_dir="e"))
    assert seen["saved"] == "out"
    dp.main(["raw", "cells.csv", "out"])
    assert seen["args"] == ("raw", "cells.csv", dict(multi_task=False))
