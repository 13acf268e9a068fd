"""GeoGuessr evaluation metrics: reference evaluation/metrics.py with the per-sample work on the GPU
(csrc/geo_metrics.cu).

`compute_geoguessr_metrics(results)` returns the reference's dict, keys in the same order: mean / median km error, the
Under_*_km shares, Country_accuracy, Geoguessr_score, Geocell top-1 / top-5 accuracy and, with multi-task outputs, the
six regression errors and climate / month accuracy.  Country_accuracy locates every label in the country file
(`config.COUNTRY_PATH`, a GeoJSON FeatureCollection of Polygon / MultiPolygon features) with exact point-in-polygon
predicates (`CountryIndex`, `pg_country_locate`); the distance metrics are one fused kernel (`pg_geo_metrics`) and an exact
device median.  The multi-task keys run on the host with numpy, as the reference does.  Deviations (DESIGN.md §1): no
`buffer(0)` of the geometry, the lowest-index country wins where countries overlap, 1-D `cell_labels` are used as they are
(the reference one-hot encodes them through 2076 columns and fails above that), and labels are taken in float64.
"""
from __future__ import annotations

import json
import os
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import config
from ._lib import PgCountries, PigeonB200Error, check, current_stream_ptr, load, ptr

KM_THRESHOLDS = (1, 5, 10, 25, 50, 100, 200, 750, 1000, 2500)
_RESULTS = 16      # PG_GEO_NUM_RESULTS; slots as in include/pigeon_b200.h


# ------------------------------------------------------------------------------------------------------------ countries
def _ring(coords, where: str) -> np.ndarray:
    try:
        a = np.asarray([(float(c[0]), float(c[1])) for c in coords], dtype=np.float64).reshape(-1, 2)
    except (TypeError, ValueError, IndexError) as e:
        raise ValueError(f"{where}: a ring must be a list of [lng, lat] positions") from e
    if len(a) < 4:
        raise ValueError(f"{where}: a ring needs at least 4 positions (got {len(a)})")
    if not np.isfinite(a).all():
        raise ValueError(f"{where}: non-finite coordinate")
    if not np.array_equal(a[0], a[-1]):
        raise ValueError(f"{where}: ring is not closed (first position {a[0].tolist()} != last {a[-1].tolist()})")
    return a


def parse_geojson(obj) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, List[str]]:
    """FeatureCollection (a dict, or a path to read with `json`) -> CSR arrays in feature order:
    (verts f64 [V, 2], ring_off i64 [R + 1], part_ring_off i64 [P + 1], geom_part_off i64 [G + 1], names).
    Polygon and MultiPolygon only; 3-D positions keep their first two coordinates.  A null or other geometry, a ring
    that is not closed or has fewer than 4 positions, and a non-finite coordinate raise ValueError naming the feature."""
    if not isinstance(obj, dict):
        with open(obj) as f:
            obj = json.load(f)
    if obj.get("type") != "FeatureCollection" or not isinstance(obj.get("features"), list):
        raise ValueError("countries: expected a GeoJSON FeatureCollection")
    verts, ring_off, part_ring_off, geom_part_off, names = [], [0], [0], [0], []
    for k, feat in enumerate(obj["features"]):
        props = (feat or {}).get("properties") or {}
        name = next((str(props[key]) for key in ("name", "NAME", "ADMIN", "iso_a3", "ISO_A3") if key in props), "")
        where = f"feature {k}" + (f" ({name})" if name else "")
        geom = (feat or {}).get("geometry")
        kind = geom.get("type") if isinstance(geom, dict) else None
        if kind == "Polygon":
            polys = [geom.get("coordinates")]
        elif kind == "MultiPolygon":
            polys = geom.get("coordinates")
        else:
            raise ValueError(f"{where}: geometry must be a Polygon or MultiPolygon (got {kind if geom else 'null'})")
        if not isinstance(polys, list) or not polys:
            raise ValueError(f"{where}: empty geometry")
        for poly in polys:
            if not isinstance(poly, list) or not poly:
                raise ValueError(f"{where}: a polygon needs a shell")
            for ring in poly:
                a = _ring(ring, where)
                verts.append(a)
                ring_off.append(ring_off[-1] + len(a))
            part_ring_off.append(len(ring_off) - 1)
        geom_part_off.append(len(part_ring_off) - 1)
        names.append(name)
    if not names:
        raise ValueError("countries: the FeatureCollection has no features")
    i64 = lambda x: np.asarray(x, dtype=np.int64)
    return np.concatenate(verts), i64(ring_off), i64(part_ring_off), i64(geom_part_off), names


class CountryIndex:
    """Country geometries on the device with their locate index (bounding boxes and latitude bands of edges), built once.
    `locate(labels, preds)` -> (country i32, flags u8, pred_inside u8) device tensors; see pg_country_locate."""

    def __init__(self, verts, ring_off, part_ring_off, geom_part_off, names: Optional[List[str]] = None, device=None):
        import torch
        if not torch.cuda.is_available():
            raise PigeonB200Error("CountryIndex needs a CUDA device (there is no CPU path)")
        verts = np.ascontiguousarray(np.asarray(verts, dtype=np.float64).reshape(-1, 2))
        offs = [np.ascontiguousarray(np.asarray(o, dtype=np.int64)) for o in (ring_off, part_ring_off, geom_part_off)]
        for o, top, what in zip(offs, (len(verts), len(offs[0]) - 1, len(offs[1]) - 1), ("ring", "part", "geometry")):
            if len(o) < 2 or o[0] != 0 or o[-1] != top or np.any(np.diff(o) < 1):
                raise ValueError(f"CountryIndex: {what} offsets must rise strictly from 0 to {top}")
        if not np.isfinite(verts).all():
            raise ValueError("CountryIndex: coordinates must be finite")
        self.names = list(names) if names is not None else [str(q) for q in range(len(offs[2]) - 1)]
        lib = load()
        dev = device or torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        self._verts = torch.from_numpy(verts).to(dev)
        self._offs = [torch.from_numpy(o).to(dev) for o in offs]
        V, R, P, G = len(verts), len(offs[0]) - 1, len(offs[1]) - 1, len(offs[2]) - 1
        self.num_geoms = G
        self._index = torch.zeros(int(lib.pg_country_index_bytes(V, P, G)), dtype=torch.uint8, device=dev)
        self._c = PgCountries(ptr(self._verts), ptr(self._offs[0]), ptr(self._offs[1]), ptr(self._offs[2]), V, R, P, G,
                              ptr(self._index), self._index.numel(), None, 0)
        total = torch.empty(1, dtype=torch.int64, device=dev)
        check(lib.pg_country_index_build(self._c, ptr(total), current_stream_ptr()), "pg_country_index_build")
        n = int(total.item())                                        # one sync per index build, none per locate
        self._entries = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        self._c.entries, self._c.num_entries = ptr(self._entries), n
        check(lib.pg_country_index_fill(self._c, current_stream_ptr()), "pg_country_index_fill")

    @classmethod
    def from_geojson(cls, path, device=None) -> "CountryIndex":
        if not isinstance(path, dict) and not os.path.exists(path):
            raise FileNotFoundError(f"country file not found: {path}")
        return cls(*parse_geojson(path), device=device)

    def locate(self, labels, preds=None):
        import torch
        lib = load()
        lab = _lnglat_f64(labels, "labels").to(self.device)
        pr = None if preds is None else _lnglat_f64(preds, "predictions").to(self.device)
        N = lab.shape[0]
        if pr is not None and pr.shape[0] != N:
            raise ValueError(f"locate: {N} labels but {pr.shape[0]} predictions")
        country = torch.empty(N, dtype=torch.int32, device=self.device)
        flags = torch.empty(N, dtype=torch.uint8, device=self.device)
        inside = None if pr is None else torch.empty(N, dtype=torch.uint8, device=self.device)
        check(lib.pg_country_locate(self._c, ptr(lab), ptr(pr), N, ptr(country), ptr(flags), ptr(inside),
                                    current_stream_ptr()), "pg_country_locate")
        return country, flags, inside


def _lnglat_f64(x, what: str):
    import torch
    t = torch.as_tensor(x)
    if t.ndim != 2 or t.shape[1] != 2:
        raise ValueError(f"{what} must have shape [N, 2] (got {tuple(t.shape)})")
    t = t.to(torch.float64).contiguous()
    if not bool(torch.isfinite(t).all()):
        raise ValueError(f"{what} must be finite")
    return t


_DEFAULT: Optional[CountryIndex] = None


def default_countries() -> CountryIndex:
    """The index of config.COUNTRY_PATH, loaded on first use and cached (the reference loads it at import time)."""
    global _DEFAULT
    if _DEFAULT is None:
        _DEFAULT = CountryIndex.from_geojson(config.COUNTRY_PATH)
    return _DEFAULT


# ------------------------------------------------------------------------------------------------------- the metrics
def mae(labels: np.ndarray, preds: np.ndarray) -> float:
    """metrics.py:22-27."""
    error = np.mean(np.abs(labels - preds))
    if type(error) == tuple:
        return error[0]
    return error


def recover_regression_values(values: np.ndarray, yfcc: bool = False) -> np.ndarray:
    """metrics.py:29-57: inverse of the joblib StandardScaler, exp of the log-transformed columns, minus the offsets."""
    import joblib
    scaler = joblib.load(config.SCALER_PATH_YFCC if yfcc else config.SCALER_PATH)
    vals = scaler.inverse_transform(values)
    vals[:, :2] = np.exp(vals[:, :2])
    vals[:, 3:] = np.exp(vals[:, 3:])
    offset_val = 416 if yfcc else 408
    return vals - np.array([offset_val, 1, 0, 1, 1, 1]).transpose()


def find_country(point, countries: Optional[CountryIndex] = None) -> int:
    """metrics.py:59-72 for one (lng, lat) point -> the index of its country (the covering geometry of lowest index, else
    the nearest one).  The reference returns the geometry; `countries.names[i]` names it."""
    idx = countries or default_countries()
    c, _, _ = idx.locate(np.asarray(point, dtype=np.float64).reshape(1, 2))
    return int(c.item())


def country_accuracy(predictions: np.ndarray, labels: np.ndarray, countries: Optional[CountryIndex] = None) -> float:
    """metrics.py:74-88: share of samples whose prediction lies inside (interior) the label's country."""
    _, _, inside = (countries or default_countries()).locate(labels, _lnglat_f64(predictions, "predictions"))
    return np.float64(inside.double().mean().item()) if inside.numel() else np.float64("nan")


def percentage_within_radius(distances: np.ndarray, km: float) -> float:
    """metrics.py:90-101."""
    return (distances < km).sum() / len(distances)


def geoguessr_score(distances: np.ndarray) -> float:
    """metrics.py:103-115: mean of round(5000 exp(-d / DECAY_CONSTANT))."""
    return np.mean(np.round(5000 * np.exp(-distances / config.DECAY_CONSTANT)))


def topk_geocell_accuracy(cell_labels: np.ndarray, topk_preds: np.ndarray) -> float:
    """metrics.py:117-137."""
    num_correct = sum(1 for label, top in zip(cell_labels, topk_preds) if label in top)
    return num_correct / len(cell_labels)


def geo_metrics(predictions, labels, cell_preds, cell_labels, topk, countries: CountryIndex):
    """The GPU part of compute_geoguessr_metrics -> (results f64 [16] on the host, distances f64 [N] on the device,
    (country, flags, pred_inside) of the labels).  `predictions` keep their dtype (float32 or float64: numpy's dtype
    rules in haversine_np depend on it); everything else is validated and converted here."""
    import torch
    lib = load()
    dev = countries.device
    p = torch.as_tensor(np.asarray(predictions) if not isinstance(predictions, torch.Tensor) else predictions)
    if p.ndim != 2 or p.shape[1] != 2:
        raise ValueError(f"predictions must have shape [N, 2] (got {tuple(p.shape)})")
    if not bool(torch.isfinite(p).all()):
        raise ValueError("predictions must be finite")
    f32 = p.dtype == torch.float32
    p = p.to(dev, torch.float32 if f32 else torch.float64).contiguous()
    lab = _lnglat_f64(labels, "labels").to(dev)
    N = p.shape[0]
    as_i64 = lambda x: torch.as_tensor(np.asarray(x)).to(dev, torch.int64).contiguous()
    cp, cl, tk = as_i64(cell_preds).reshape(-1), as_i64(cell_labels).reshape(-1), as_i64(topk)
    if tk.ndim == 1:
        tk = tk.reshape(N, -1) if N else tk.reshape(0, 1)
    if N < 1 or lab.shape[0] != N or cp.numel() != N or cl.numel() != N or tk.ndim != 2 or tk.shape[0] != N or tk.shape[1] < 1:
        raise ValueError(f"geo_metrics: inconsistent shapes (predictions {tuple(p.shape)}, labels {tuple(lab.shape)}, "
                         f"cell preds {tuple(cp.shape)}, cell labels {tuple(cl.shape)}, top-k {tuple(tk.shape)})")
    country, flags, inside = countries.locate(lab, p.double())
    dist = torch.empty(N, dtype=torch.float64, device=dev)
    res = torch.empty(_RESULTS, dtype=torch.float64, device=dev)
    ws = torch.empty(int(lib.pg_geo_metrics_workspace_bytes(N)), dtype=torch.uint8, device=dev)
    check(lib.pg_geo_metrics(ptr(p), int(f32), ptr(lab), N, ptr(cp), ptr(cl), ptr(tk), tk.shape[1], ptr(inside), ptr(ws),
                             ws.numel(), ptr(dist), ptr(res), current_stream_ptr()), "pg_geo_metrics")
    return res.cpu().numpy(), dist, (country, flags, inside)


def multitask_metrics(preds_mt, labels_mt, preds_climate, labels_climate, preds_month, labels_month) -> Dict:
    """metrics.py:184-200 on the host: the six regression errors, Climate_accuracy and, unless labels_month is None
    (YFCC), Month_accuracy.  Labels are recovered with the non-YFCC scaler whatever the data set, as the reference does."""
    from sklearn.metrics import accuracy_score
    yfcc = labels_month is None
    preds_mt = recover_regression_values(np.asarray(preds_mt), yfcc)
    labels_mt = recover_regression_values(np.asarray(labels_mt))    # metrics.py:186: always yfcc=False
    out = {}
    for col, name in enumerate(('elevation', 'population', 'temperature', 'temp_diff', 'precipitation', 'prec_diff')):
        out[f'Mean_{name}_error'] = mae(labels_mt[:, col], preds_mt[:, col])
    out['Climate_accuracy'] = accuracy_score(labels_climate, np.argmax(preds_climate, axis=-1))
    if not yfcc:
        out['Month_accuracy'] = accuracy_score(labels_month, np.argmax(preds_month, axis=-1))
    return out


def compute_geoguessr_metrics(results, countries: Optional[CountryIndex] = None) -> Dict:
    """metrics.py:139-202 on the 11-tuple evaluate_model passes: (predictions, cell_preds, preds_mt, preds_climate,
    preds_month, top5_geocells, labels, cell_labels, labels_mt, labels_climate, labels_month)."""
    (predictions, cell_preds, preds_mt, preds_climate, preds_month, top5_geocells,
     labels, cell_labels, labels_mt, labels_climate, labels_month) = results
    cell_labels = np.asarray(cell_labels)
    if cell_labels.ndim != 1:                                        # the 1-D one-hot round trip is the identity
        cell_labels = np.argmax(cell_labels, axis=-1)
    res, _, _ = geo_metrics(predictions, labels, cell_preds, cell_labels, top5_geocells, countries or default_countries())
    f = lambda i: np.float64(res[i])
    eval_dict = {'Mean_km_error': f(0), 'Median_km_error': f(1)}
    for t, km in enumerate(KM_THRESHOLDS):
        eval_dict[f'Under_{km}_km'] = f(2 + t)
    eval_dict.update({'Country_accuracy': f(12), 'Geoguessr_score': f(13), 'Geocell_accuracy': float(res[14]),
                      'Geocell_top5_accuracy': float(res[15])})
    if labels_mt is not None:
        eval_dict.update(multitask_metrics(preds_mt, labels_mt, preds_climate, labels_climate, preds_month, labels_month))
    print(eval_dict)
    return eval_dict
