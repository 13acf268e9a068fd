"""Generate tests/golden/metrics.npz by running the UNMODIFIED reference evaluation/metrics.py
(`compute_geoguessr_metrics`) on seeded synthetic samples and one synthetic country file.

Authoring-time only: it needs the reference checkout (PIGEON_REFERENCE, default /root/reference) and is never run by tests.
Around the unmodified module:
  - oracle/reference_shim.py provides its `config` and `preprocessing` (haversine_np);
  - `geopandas` and `shapely.geometry` are stub modules built on tests/metrics_oracle.py's exact point location and GEOS
    point-to-segment distance: `read_file`, `set_crs`, `sindex.query(point, predicate='covered_by')` (covering
    geometries, ascending), `sindex.nearest(point, return_all=False)` (lowest index on ties), `points_from_xy` and
    `contains`; `buffer(0)` returns the geometry unchanged;
  - the joblib scalers are StandardScalers fitted on synthetic data, written where config.SCALER_PATH(_YFCC) point;
  - the run happens in a scratch directory holding data/geocells/countries.geojson.
The stubs record which geometry find_country returned for every label, so the file pins the country control flow too.

    python tools/make_metrics_golden.py
"""
from __future__ import annotations

import contextlib
import importlib.util
import io
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "metrics.npz")


def world():
    """A small country file: a concave country, one with an enclave (a hole filled by another country), an island
    MultiPolygon, two neighbours sharing a border vertex for vertex, and an overlapping pair."""
    sq = lambda x0, y0, x1, y1: [[x0, y0], [x1, y0], [x1, y1], [x0, y1], [x0, y0]]
    feats = [
        ("Concavia", "Polygon", [[[0, 0], [10, 0], [10, 10], [5, 4], [0, 10], [0, 0]]]),
        ("Holland", "Polygon", [sq(12, 0, 20, 8), sq(14, 2, 16, 4)[::-1]]),
        ("Enclave", "Polygon", [sq(14, 2, 16, 4)]),
        ("Islands", "MultiPolygon", [[sq(-10, -10, -8, -8)], [sq(-6, -10, -4, -7)], [[[-10, -5], [-7, -5], [-8.5, -2], [-10, -5]]]]),
        ("West", "Polygon", [[[0, 12], [5, 12], [5.5, 14], [5, 16], [0, 16], [0, 12]]]),
        ("East", "Polygon", [[[5, 12], [10, 12], [10, 16], [5, 16], [5.5, 14], [5, 12]]]),
        ("OverlapA", "Polygon", [sq(20, 20, 26, 26)]),
        ("OverlapB", "Polygon", [sq(24, 24, 30, 30)]),
    ]
    return {"type": "FeatureCollection",
            "features": [{"type": "Feature", "properties": {"name": n},
                          "geometry": {"type": t, "coordinates": c}} for n, t, c in feats]}


def samples(rng, n, f32, one_hot, month, mt=True):
    labels = np.concatenate([rng.uniform([-12, -12], [32, 32], (n - 6, 2)),
                             [[5, 4], [10, 5], [14, 3], [5, 14], [-20, 40], [11, 11]]])  # vertex, edge, hole edge, ...
    scale = rng.choice([0.001, 0.01, 0.05, 0.2, 1, 4, 10, 40], n)
    preds = labels + rng.normal(0, 1, (n, 2)) * scale[:, None]
    preds[:5] = labels[:5]
    preds = preds.astype(np.float32) if f32 else preds
    C = 50
    cell_labels = rng.integers(0, C, n)
    cell_preds = np.where(rng.random(n) < 0.4, cell_labels, rng.integers(0, C, n))
    top5 = np.stack([rng.permutation(C)[:5] for _ in range(n)])
    hit = rng.random(n) < 0.5
    top5[hit, rng.integers(0, 5, hit.sum())] = cell_labels[hit]
    lab_cells = np.eye(C)[cell_labels] if one_hot else cell_labels
    case = dict(predictions=preds, cell_preds=cell_preds, top5=top5, labels=labels, cell_labels=lab_cells)
    if mt:
        case.update(preds_mt=rng.normal(0, 1, (n, 6)), labels_mt=rng.normal(0, 1, (n, 6)),
                    preds_climate=rng.normal(0, 1, (n, 7)), labels_climate=rng.integers(0, 7, n))
        if month:
            case.update(preds_month=rng.normal(0, 1, (n, 12)), labels_month=rng.integers(0, 12, n))
    return case


CASES = [("f32_1d_month", 11, True, False, True, True), ("f64_2d_yfcc", 12, False, True, False, True),
         ("f64_1d_no_mt", 13, False, False, True, False)]


def stubs(geoms, record):
    class Pt:
        def __init__(self, x, y):
            self.x, self.y = float(x), float(y)

        def __repr__(self):
            return f"POINT ({self.x} {self.y})"

    class Geom:
        def __init__(self, q):
            self.q = q

        def buffer(self, d):
            return self

        def contains(self, p):
            cov, bnd = geoms[self.q].locate(p.x, p.y)
            record["contains"].append(cov and not bnd)
            return cov and not bnd

    class SIndex:
        def query(self, p, predicate=None):
            assert predicate == "covered_by"
            return np.asarray([q for q, g in enumerate(geoms) if g.locate(p.x, p.y)[0]], dtype=np.int64)

        def nearest(self, p, return_all=True):
            d = [g.distance(p.x, p.y) for g in geoms]
            return np.asarray([[0], [int(np.argmin(d))]])

    class GeoSeries(list):
        sindex = SIndex()

        def apply(self, f):
            return GeoSeries(f(x) for x in self)

        @property
        def values(self):
            return list(self)

    class Row(dict):
        pass

    class ILoc:
        def __init__(self, df):
            self.df = df

        def __getitem__(self, i):
            record["country"].append(int(i))
            return Row(geometry=self.df.cols["geometry"][int(i)])

    class GeoDataFrame:
        def __init__(self, n):
            self.cols = {"geometry": GeoSeries(Geom(q) for q in range(n))}
            self.iloc = ILoc(self)

        def set_crs(self, crs):
            return self

        def __getitem__(self, k):
            return self.cols[k]

        def __setitem__(self, k, v):
            self.cols[k] = v if isinstance(v, GeoSeries) else GeoSeries(v)

    gpd = types.ModuleType("geopandas")
    gpd.read_file = lambda path: GeoDataFrame(len(json.load(open(path))["features"]))
    gpd.points_from_xy = lambda x, y, crs=None: [Pt(a, b) for a, b in zip(x, y)]
    shp = types.ModuleType("shapely")
    shp.__path__ = []
    geo = types.ModuleType("shapely.geometry")
    geo.Point, geo.MultiPolygon = Pt, Geom
    shp.geometry = geo
    return {"geopandas": gpd, "shapely": shp, "shapely.geometry": geo}


def main():
    import joblib
    from sklearn.preprocessing import StandardScaler
    from oracle import reference_shim
    import metrics_oracle as mo
    from pigeon_b200.metrics import parse_geojson
    reference_shim.install()
    cfg = sys.modules["config"]
    w = world()
    verts, ring_off, part_ring_off, geom_part_off, names = parse_geojson(w)
    geoms = mo.geometries_from_csr(verts, ring_off, part_ring_off, geom_part_off)
    record = {"country": [], "contains": []}
    sys.modules.update(stubs(geoms, record))
    out = dict(verts=verts, ring_off=ring_off, part_ring_off=part_ring_off, geom_part_off=geom_part_off,
               world=np.frombuffer(json.dumps(w).encode(), dtype=np.uint8))
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            os.makedirs(os.path.dirname(cfg.COUNTRY_PATH))
            json.dump(w, open(cfg.COUNTRY_PATH, "w"))
            rng = np.random.default_rng(0)
            for path, shift in ((cfg.SCALER_PATH, 0.0), (cfg.SCALER_PATH_YFCC, 0.5)):
                os.makedirs(os.path.dirname(path), exist_ok=True)
                sc = StandardScaler().fit(rng.normal([6.5, 4, 12, 2.5, 4, 3], [0.5, 1, 8, 0.4, 0.8, 0.5], (500, 6)) + shift)
                joblib.dump(sc, path)
                out[f"scaler_{'yfcc' if shift else 'main'}"] = np.concatenate([sc.mean_, sc.scale_])
            spec = importlib.util.spec_from_file_location("ref_metrics", os.path.join(reference_shim.REF, "evaluation", "metrics.py"))
            ref = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(ref)
            for name, seed, f32, one_hot, month, mt in CASES:
                case = samples(np.random.default_rng(seed), 400, f32, one_hot, month, mt)
                g = case.get
                results = (g("predictions"), g("cell_preds"), g("preds_mt"), g("preds_climate"), g("preds_month"),
                           g("top5"), g("labels"), g("cell_labels"), g("labels_mt"), g("labels_climate"), g("labels_month"))
                record["country"].clear()
                record["contains"].clear()
                with contextlib.redirect_stdout(io.StringIO()):
                    res = ref.compute_geoguessr_metrics(results)
                for k, v in case.items():
                    out[f"{name}/in/{k}"] = np.asarray(v)
                out[f"{name}/keys"] = np.asarray(list(res.keys()))
                out[f"{name}/values"] = np.asarray([float(v) for v in res.values()], dtype=np.float64)
                out[f"{name}/types"] = np.asarray([type(v).__name__ for v in res.values()])
                out[f"{name}/country"] = np.asarray(record["country"], dtype=np.int32)
                out[f"{name}/pred_inside"] = np.asarray(record["contains"], dtype=np.uint8)
                out[f"{name}/distances"] = ref.haversine_np(g("predictions"), g("labels"))
        finally:
            os.chdir(cwd)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
