"""numpy restatement of per-geocell OPTICS-xi (test infrastructure): the distance matrix of reference
dataset_creation/prototype/prototype.py:121-133 (`_compute_distances` over preprocessing/geo_utils.py:77-93
`haversine_matrix_np`), scikit-learn's `compute_optics_graph` for a precomputed matrix with max_eps = inf
(sklearn/cluster/_optics.py: `_compute_core_distances_`, the main loop and `_set_reach_dist`) and `cluster_optics_xi`
(`_xi_cluster`, `_extend_region`, `_update_filter_sdas`, `_correct_predecessor`, `_extract_xi_labels`).

Rows of the matrix are computed when needed, so a 20 000-point cell needs no 3 GB matrix.  `optics_graph` also
reports decision margins: the smallest relative gap, over all ordering steps, between the chosen reachability and the
next distinct candidate, and the smallest relative distance of a reachability ratio from the xi thresholds.
"""
from __future__ import annotations

import numpy as np

RAD_M = np.float64(6378137.0)   # geo_utils.py:7


def prepare(lnglat):
    rad = np.deg2rad(np.asarray(lnglat, dtype=np.float64).reshape(-1, 2))
    return rad, np.cos(rad[:, 1])


def rows(rad, cos, idx):
    """Rows idx of the reference's distance matrix (km, exact zeros as 1e-5), numpy's operation order."""
    idx = np.atleast_1d(idx)
    dlng = rad[idx, 0][:, None] - rad[None, :, 0]
    dlat = rad[idx, 1][:, None] - rad[None, :, 1]
    p = cos[idx][:, None] * cos[None, :]
    a = np.sin(dlat / 2) ** 2 + p * np.sin(dlng / 2) ** 2
    km = (RAD_M * (2 * np.arcsin(np.sqrt(a)))) / 1000
    return np.where(km == 0, 1e-5, km)


def core_distances(rad, cos, m, chunk=256):
    n = len(cos)
    core = np.empty(n)
    for s in range(0, n, chunk):
        r = rows(rad, cos, np.arange(s, min(n, s + chunk)))
        core[s:s + len(r)] = np.partition(r, m - 1, axis=1)[:, m - 1]
    return np.around(core, 15)


def optics_graph(lnglat, m):
    """-> ordering, core, reach, pred (sklearn's ordering_, core_distances_, reachability_, predecessor_) and the
    smallest relative ordering gap."""
    rad, cos = prepare(lnglat)
    n = len(cos)
    core = core_distances(rad, cos, m)
    reach = np.full(n, np.inf)
    pred = np.full(n, -1, dtype=np.int64)
    done = np.zeros(n, dtype=bool)
    ordering = np.zeros(n, dtype=np.int64)
    gap = np.inf
    for k in range(n):
        un = np.flatnonzero(~done)
        r_un = reach[un]
        p = un[np.argmin(r_un)]          # lowest index on ties, inf included
        v0 = reach[p]
        if np.isfinite(v0):
            above = r_un[r_un > v0]
            if above.size:
                gap = min(gap, (above.min() - v0) / v0)
        done[p] = True
        ordering[k] = p
        un = np.flatnonzero(~done)
        if not un.size:
            break
        r = np.around(np.maximum(rows(rad, cos, p)[0, un], core[p]), 15)
        better = r < reach[un]
        reach[un[better]] = r[better]
        pred[un[better]] = p
    return ordering, core, reach, pred, gap


def _ratios(reach_plot):
    r = np.hstack((reach_plot, np.inf))
    with np.errstate(invalid="ignore", divide="ignore"):
        return r[:-1] / r[1:], r


def xi_margin(reach, ordering, xi):
    """Smallest relative distance of a finite reachability ratio from 1 - xi and 1 / (1 - xi)."""
    q, _ = _ratios(reach[ordering])
    xc = 1 - xi
    q = q[np.isfinite(q) & (q > 0)]
    if not q.size:
        return np.inf
    return float(min(np.min(np.abs(q - xc) / xc), np.min(np.abs(q - 1 / xc) * xc)))


def _extend(steep, xward, start, m):
    non, end, index = 0, start, start
    while index < len(steep):
        if steep[index]:
            non, end = 0, index
        elif not xward[index]:
            non += 1
            if non > m:
                break
        else:
            return end
        index += 1
    return end


def xi_labels(reach, pred, ordering, m, xi):
    """cluster_optics_xi(min_cluster_size=m, predecessor_correction=True) labels."""
    ratio, r = _ratios(reach[ordering])
    pp = pred[ordering]
    pos = np.empty(len(ordering), dtype=np.int64)
    pos[ordering] = np.arange(len(ordering))
    xc = 1 - xi
    s_up, s_down, down, up = ratio <= xc, ratio >= 1 / xc, ratio > 1, ratio < 1
    sdas, clusters, index, mib = [], [], 0, 0.0

    def filt(sdas, mib):
        if np.isinf(mib):
            return []
        kept = [d for d in sdas if mib <= r[d[0]] * xc]
        for d in kept:
            d[2] = max(d[2], mib)
        return kept

    for s in np.flatnonzero(s_up | s_down):
        if s < index:
            continue
        mib = max(mib, np.max(r[index:s + 1]))
        sdas = filt(sdas, mib)
        if s_down[s]:
            end = _extend(s_down, up, s, m)
            sdas.append([s, end, 0.0])
            index = end + 1
            mib = r[index]
            continue
        u_end = _extend(s_up, down, s, m)
        index = u_end + 1
        mib = r[index]
        found = []
        for d in sdas:
            cs, ce = d[0], u_end
            if r[ce + 1] * xc < d[2]:
                continue
            dmax = r[d[0]]
            if dmax * xc >= r[ce + 1]:
                while r[cs + 1] > r[ce + 1] and cs < d[1]:
                    cs += 1
            elif r[ce + 1] * xc >= dmax:
                while r[ce - 1] > dmax and ce > s:
                    ce -= 1
            while cs < ce:                       # _correct_predecessor
                if r[cs] > r[ce] or (pp[ce] >= 0 and cs <= pos[pp[ce]] < ce):
                    break
                ce -= 1
            else:
                continue
            if ce - cs + 1 < m or cs > d[1] or ce < s:
                continue
            found.append((cs, ce))
        clusters.extend(reversed(found))
    lab = np.full(len(ordering), -1, dtype=np.int64)
    label = 0
    for cs, ce in clusters:
        if not np.any(lab[cs:ce + 1] != -1):
            lab[cs:ce + 1] = label
            label += 1
    out = np.empty_like(lab)
    out[ordering] = lab
    return out


def optics_xi(lnglat, m, xi):
    """-> dict(labels, ordering, core, reach, pred, order_gap, xi_gap) for one cell; a cell below m gets labels 0
    (prototype.py:144-145) and no graph."""
    n = len(np.asarray(lnglat).reshape(-1, 2))
    if n < m:
        return dict(labels=np.zeros(n, dtype=np.int64), ordering=None, core=None, reach=None, pred=None,
                    order_gap=np.inf, xi_gap=np.inf)
    ordering, core, reach, pred, gap = optics_graph(lnglat, m)
    return dict(labels=xi_labels(reach, pred, ordering, m, xi), ordering=ordering, core=core, reach=reach, pred=pred,
                order_gap=gap, xi_gap=xi_margin(reach, ordering, xi))
