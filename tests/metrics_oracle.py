"""Host oracle for the GeoGuessr metrics (pigeon_b200.metrics, csrc/geo_metrics.cu).

- Point location with GEOS semantics in the (lng, lat) plane: RayCrossingCounter's crossing rule with an exact
  orientation sign (an fp64 filter, then `fractions.Fraction`); boundary = exactly on an edge of any ring; covered =
  boundary or an odd crossing count over some part; contains = covered and not boundary.
- GEOS Distance::pointToSegment in numpy float64, elementwise, same operation order, for the nearest-country fallback.
- The reference's haversine_np and metrics restated in numpy, with per-sample decision margins: the relative distance to
  each km threshold and the distance of 5000 exp(-d / 1492.7) to its nearest .5.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

KM = (1, 5, 10, 25, 50, 100, 200, 750, 1000, 2500)
DECAY = 1492.7


def orient(ax, ay, bx, by, cx, cy) -> int:
    """Exact sign of (a - c) x (b - c)."""
    l = (ax - cx) * (by - cy)
    r = (ay - cy) * (bx - cx)
    det = l - r
    bound = 3.3306690738754716e-16 * (abs(l) + abs(r))
    if det > bound:
        return 1
    if -det > bound:
        return -1
    F = Fraction
    e = (F(ax) - F(cx)) * (F(by) - F(cy)) - (F(ay) - F(cy)) * (F(bx) - F(cx))
    return (e > 0) - (e < 0)


class Geometry:
    """One Polygon / MultiPolygon as parts = [[ring f64 [n, 2], ...], ...] (shell first, then holes)."""

    def __init__(self, parts):
        self.parts = [[np.asarray(r, dtype=np.float64) for r in part] for part in parts]
        allv = np.concatenate([r for p in self.parts for r in p])
        self.box = (allv[:, 0].min(), allv[:, 1].min(), allv[:, 0].max(), allv[:, 1].max())

    def locate(self, x: float, y: float):
        """-> (covered, boundary).  RayCrossingCounter over every edge, vectorised; only orientations the fp64 filter
        cannot decide go to `orient`'s exact Fraction path."""
        x, y = float(x), float(y)
        b = self.box
        if not (b[0] <= x <= b[2] and b[1] <= y <= b[3]):
            return False, False
        inside = False
        for part in self.parts:
            cross = 0
            for ring in part:
                x1, y1, x2, y2 = ring[:-1, 0], ring[:-1, 1], ring[1:, 0], ring[1:, 1]
                live = ~((x1 < x) & (x2 < x))
                if np.any(live & (x == x2) & (y == y2)):
                    return True, True
                horiz = live & (y1 == y) & (y2 == y)
                if np.any(horiz & (np.minimum(x1, x2) <= x) & (x <= np.maximum(x1, x2))):
                    return True, True
                cand = live & ~horiz & (((y1 > y) & (y2 <= y)) | ((y2 > y) & (y1 <= y)))
                cx1, cy1, cx2, cy2 = x1[cand], y1[cand], x2[cand], y2[cand]
                l = (cx1 - x) * (cy2 - y)
                r = (cy1 - y) * (cx2 - x)
                det = l - r
                bound = 3.3306690738754716e-16 * (np.abs(l) + np.abs(r))
                o = np.where(det > bound, 1, np.where(-det > bound, -1, 0))
                for k in np.flatnonzero(o == 0):
                    o[k] = orient(cx1[k], cy1[k], cx2[k], cy2[k], x, y)
                if np.any(o == 0):
                    return True, True
                o = np.where(cy2 < cy1, -o, o)
                cross += int(np.sum(o > 0))
            inside |= bool(cross & 1)
        return inside, False

    def distance(self, x: float, y: float) -> float:
        """min over edges of GEOS Distance::pointToSegment (float64, same operation order)."""
        return min(float(np.min(segment_distances(x, y, ring[:-1], ring[1:]))) for part in self.parts for ring in part)


def segment_distances(x, y, a, b):
    """GEOS Distance::pointToSegment of (x, y) to every segment a[i] -> b[i], elementwise in float64."""
    px, py = np.float64(x), np.float64(y)
    ax, ay, bx, by = a[:, 0], a[:, 1], b[:, 0], b[:, 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        len2 = (bx - ax) * (bx - ax) + (by - ay) * (by - ay)
        r = ((px - ax) * (bx - ax) + (py - ay) * (by - ay)) / len2
        s = ((ay - py) * (bx - ax) - (ax - px) * (by - ay)) / len2
        mid = np.abs(s) * np.sqrt(len2)
    da, db = _pdist(px, py, ax, ay), _pdist(px, py, bx, by)
    same = (ax == bx) & (ay == by)
    return np.where(same | (r <= 0.0), da, np.where(r >= 1.0, db, mid))


def _pdist(px, py, ax, ay):
    dx, dy = px - ax, py - ay
    return np.sqrt(dx * dx + dy * dy)


def locate(geoms, labels, preds):
    """-> country i32 [N], flags u8 [N] (1 = nearest fallback), pred_inside u8 [N], as pg_country_locate."""
    N = len(labels)
    country, flags, inside = np.zeros(N, np.int32), np.zeros(N, np.uint8), np.zeros(N, np.uint8)
    for n in range(N):
        lx, ly = labels[n]
        c = next((q for q, g in enumerate(geoms) if g.locate(lx, ly)[0]), -1)
        if c < 0:
            d = [g.distance(lx, ly) for g in geoms]
            c, flags[n] = int(np.argmin(d)), 1          # argmin: lowest index on exact ties
        country[n] = c
        cov, bnd = geoms[c].locate(*preds[n])
        inside[n] = cov and not bnd
    return country, flags, inside


def geometries_from_csr(verts, ring_off, part_ring_off, geom_part_off):
    out = []
    for q in range(len(geom_part_off) - 1):
        parts = []
        for p in range(geom_part_off[q], geom_part_off[q + 1]):
            parts.append([verts[ring_off[r]:ring_off[r + 1]] for r in range(part_ring_off[p], part_ring_off[p + 1])])
        out.append(Geometry(parts))
    return out


def haversine_np(x, y):
    """preprocessing/geo_utils.py haversine_np (x = predictions, y = labels), numpy dtype rules included."""
    x_rad, y_rad = map(np.radians, [x, y])
    delta = y_rad - x_rad
    a = np.sin(delta[:, 1] / 2) ** 2 + np.cos(x_rad[:, 1]) * np.cos(y_rad[:, 1]) * np.sin(delta[:, 0] / 2) ** 2
    c = 2 * np.arcsin(np.sqrt(a))
    return (np.float64(6378137.0) * c) / 1000


def haversine_a(x, y):
    """The haversine term `a` of haversine_np, whose conditioning bounds how far two implementations' distances may
    differ: d = 2 R asin(sqrt(a)) has relative condition number sqrt(a) / (2 sqrt(1 - a) asin(sqrt(a))) in a."""
    x_rad, y_rad = map(np.radians, [x, y])
    delta = y_rad - x_rad
    return np.sin(delta[:, 1] / 2) ** 2 + np.cos(x_rad[:, 1]) * np.cos(y_rad[:, 1]) * np.sin(delta[:, 0] / 2) ** 2


def scores(d):
    return np.round(5000 * np.exp(-d / DECAY))


def margins(d):
    """Per-sample relative decision margin: distance to the nearest km threshold and of the unrounded score to its
    nearest .5, both relative."""
    d = np.asarray(d, dtype=np.float64)
    km = np.min(np.abs(d[:, None] - np.asarray(KM, dtype=np.float64)[None, :]) / np.asarray(KM)[None, :], axis=1)
    raw = 5000 * np.exp(-d / DECAY)
    half = np.abs(raw - np.floor(raw) - 0.5) / np.maximum(raw, 1.0)
    return np.minimum(km, half)


def metrics(predictions, labels, cell_preds, cell_labels, topk, pred_inside):
    """The GPU part of compute_geoguessr_metrics in numpy: dict in the reference's key order."""
    d = haversine_np(predictions, np.asarray(labels, dtype=np.float64))
    out = {'Mean_km_error': np.mean(d), 'Median_km_error': np.median(d)}
    for km in KM:
        out[f'Under_{km}_km'] = (d < km).sum() / len(d)
    out['Country_accuracy'] = np.mean(np.asarray(pred_inside, dtype=int))
    out['Geoguessr_score'] = np.mean(scores(d))
    out['Geocell_accuracy'] = float(np.mean(np.asarray(cell_preds) == np.asarray(cell_labels)))
    out['Geocell_top5_accuracy'] = sum(1 for l, t in zip(cell_labels, topk) if l in t) / len(cell_labels)
    return out, d
