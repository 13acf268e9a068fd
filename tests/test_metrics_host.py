"""CPU tests of the GeoGuessr metrics: GeoJSON parsing, the exact oracle and the numpy restatement against the reference
golden (tests/golden/metrics.npz, tools/make_metrics_golden.py), the host multi-task keys and the run.py wiring."""
import copy
import json
import os

import numpy as np
import pytest

import metrics_oracle as mo
from pigeon_b200 import config, metrics

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "metrics.npz")
CASES = ("f32_1d_month", "f64_2d_yfcc", "f64_1d_no_mt")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def world(g):
    return json.loads(g["world"].tobytes().decode())


def case(g, name):
    p = f"{name}/in/"
    return {k[len(p):]: v for k, v in g.items() if k.startswith(p)}


def test_parse_matches_golden_csr(golden):
    verts, ring_off, part_ring_off, geom_part_off, names = metrics.parse_geojson(world(golden))
    for a, k in ((verts, "verts"), (ring_off, "ring_off"), (part_ring_off, "part_ring_off"), (geom_part_off, "geom_part_off")):
        np.testing.assert_array_equal(a, golden[k])
    assert names[:3] == ["Concavia", "Holland", "Enclave"] and len(names) == 8
    assert ring_off.dtype == np.int64 and verts.dtype == np.float64


def test_parse_keeps_two_coordinates_and_reads_files(golden, tmp_path):
    w = world(golden)
    w3 = copy.deepcopy(w)
    for f in w3["features"]:
        c = f["geometry"]["coordinates"]
        polys = c if f["geometry"]["type"] == "MultiPolygon" else [c]
        for poly in polys:
            for ring in poly:
                for pos in ring:
                    pos.append(123.0)
    path = tmp_path / "c.geojson"
    path.write_text(json.dumps(w3))
    for a, b in zip(metrics.parse_geojson(str(path))[:4], metrics.parse_geojson(w)[:4]):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("mutate, message", [
    (lambda f: f.update(geometry=None), "got null"),
    (lambda f: f.update(geometry={"type": "Point", "coordinates": [0, 0]}), "got Point"),
    (lambda f: f["geometry"]["coordinates"][0].pop(), "not closed"),
    (lambda f: f["geometry"].update(coordinates=[[[0, 0], [1, 0], [0, 0]]]), "at least 4"),
    (lambda f: f["geometry"]["coordinates"][0][1].__setitem__(0, float("nan")), "non-finite"),
    (lambda f: f["geometry"]["coordinates"][0][1].__setitem__(1, float("inf")), "non-finite"),
])
def test_parse_rejects_naming_the_feature(golden, mutate, message):
    w = world(golden)
    mutate(w["features"][1])
    with pytest.raises(ValueError, match=rf"feature 1 \(Holland\).*{message}"):
        metrics.parse_geojson(w)


def test_missing_country_file_names_the_path(tmp_path, monkeypatch):
    path = str(tmp_path / "nowhere" / "countries.geojson")
    with pytest.raises(FileNotFoundError, match="nowhere/countries.geojson"):
        metrics.CountryIndex.from_geojson(path)
    monkeypatch.setattr(config, "COUNTRY_PATH", path)
    monkeypatch.setattr(metrics, "_DEFAULT", None)
    with pytest.raises(FileNotFoundError, match="nowhere/countries.geojson"):
        metrics.default_countries()


@pytest.mark.parametrize("name", CASES)
def test_oracle_locate_matches_golden(golden, name):
    c = case(golden, name)
    geoms = mo.geometries_from_csr(golden["verts"], golden["ring_off"], golden["part_ring_off"], golden["geom_part_off"])
    country, flags, inside = mo.locate(geoms, c["labels"], np.asarray(c["predictions"], dtype=np.float64))
    np.testing.assert_array_equal(country, golden[f"{name}/country"])
    np.testing.assert_array_equal(inside, golden[f"{name}/pred_inside"])
    assert flags.sum() >= 2   # the two labels outside every country take the nearest one


@pytest.mark.parametrize("name", CASES)
def test_numpy_restatement_matches_golden(golden, name):
    c = case(golden, name)
    keys = list(golden[f"{name}/keys"])
    cell_labels = c["cell_labels"] if c["cell_labels"].ndim == 1 else np.argmax(c["cell_labels"], -1)
    out, d = mo.metrics(c["predictions"], c["labels"], c["cell_preds"], cell_labels, c["top5"], golden[f"{name}/pred_inside"])
    assert d.dtype == np.float64
    np.testing.assert_array_equal(d, golden[f"{name}/distances"])
    assert list(out) == keys[:len(out)]
    np.testing.assert_array_equal(np.asarray(list(out.values())), golden[f"{name}/values"][:len(out)])


def _write_scalers(golden, tmp_path, monkeypatch):
    import joblib
    from sklearn.preprocessing import StandardScaler
    for which, attr in (("main", "SCALER_PATH"), ("yfcc", "SCALER_PATH_YFCC")):
        ms = golden[f"scaler_{which}"]
        sc = StandardScaler()
        sc.mean_, sc.scale_, sc.var_, sc.n_features_in_ = ms[:6], ms[6:], ms[6:] ** 2, 6
        path = str(tmp_path / f"{which}.scaler")
        joblib.dump(sc, path)
        monkeypatch.setattr(config, attr, path)


@pytest.mark.parametrize("name", ("f32_1d_month", "f64_2d_yfcc"))
def test_multitask_keys_match_golden(golden, name, tmp_path, monkeypatch):
    _write_scalers(golden, tmp_path, monkeypatch)
    c = case(golden, name)
    out = metrics.multitask_metrics(c["preds_mt"], c["labels_mt"], c["preds_climate"], c["labels_climate"],
                                    c.get("preds_month"), c.get("labels_month"))
    keys = list(golden[f"{name}/keys"])
    assert list(out) == keys[16:]
    np.testing.assert_array_equal(np.asarray(list(out.values())), golden[f"{name}/values"][16:])


def test_golden_key_order():
    g = np.load(GOLDEN)
    keys = list(g["f32_1d_month/keys"])
    assert keys[:2] == ["Mean_km_error", "Median_km_error"]
    assert keys[2:12] == [f"Under_{km}_km" for km in metrics.KM_THRESHOLDS]
    assert keys[12:16] == ["Country_accuracy", "Geoguessr_score", "Geocell_accuracy", "Geocell_top5_accuracy"]
    assert "Month_accuracy" not in list(g["f64_2d_yfcc/keys"]) and len(g["f64_1d_no_mt/keys"]) == 16


def test_run_metrics_flag():
    import run
    args = run.build_parser().parse_args(["evaluate", "head.model", "-l", "d", "--metrics"])
    assert run.metrics_fn(args) is metrics.compute_geoguessr_metrics
    args = run.build_parser().parse_args(["finetune", "m", "-l", "d"])
    assert run.metrics_fn(args) is None


def test_run_passes_metrics_to_evaluate_and_finetune(monkeypatch):
    import sys
    import types
    import run
    seen = {}
    ds = types.ModuleType("datasets")

    class DD(dict):
        @staticmethod
        def load_from_disk(path):
            split = types.SimpleNamespace(with_format=lambda f: "split")
            return DD(test=split, **{"with_format": None})

        def with_format(self, f):
            return self
    ds.DatasetDict = DD
    monkeypatch.setitem(sys.modules, "datasets", ds)
    monkeypatch.setattr(run, "evaluate", lambda *a, **kw: seen.setdefault("evaluate", kw["metrics"]))
    training = types.ModuleType("pigeon_b200.training")
    training.finetune_model = lambda *a, **kw: seen.setdefault("finetune", kw["metrics"])
    training.finetune_on_embeddings = lambda *a, **kw: seen.setdefault("embeddings", kw["metrics"])
    monkeypatch.setitem(sys.modules, "pigeon_b200.training", training)
    run.main(["evaluate", "h", "-l", "d", "--metrics"])
    run.main(["finetune", "m", "-l", "d", "--metrics"])
    run.main(["finetune", "-", "-l", "d", "--embeddings"])
    assert seen == {"evaluate": metrics.compute_geoguessr_metrics, "finetune": metrics.compute_geoguessr_metrics,
                    "embeddings": None}
