"""Benchmark of the GeoGuessr metrics (pigeon_b200.metrics) on a synthetic admin-0-sized world.

World: 250 countries tiling lng [-180, 180] x lat [-80, 80] (25 x 10), every border a fractal polyline shared vertex for
vertex by its two countries, one country in ten with a square enclave (a hole filled by one of 25 enclave countries), and
one in twenty-five with an island part north of 80°; the polar caps are left to the nearest-country fallback.
About 2 M vertices in total, the order of a detailed admin-0 file.  N = 26 000 (YFCC26k) and 1 000 000 samples.

Reported separately: GeoJSON parse, upload + index build, the locate kernel, the metrics kernels (fused pass, median,
finalise) and end-to-end compute_geoguessr_metrics; CUDA events after warm-up, median of the repeats.  For context, a
vectorised numpy fp64 crossing-number test on a CPU subsample (bounding-box prefilter, no exact predicates).

    python tools/metrics_bench.py [--points 2048] [--repeats 20]
"""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def fractal(a, b, n, amp, rng):
    """Polyline of n + 1 points from a to b by midpoint displacement perpendicular to a -> b (endpoints pinned)."""
    t = np.linspace(0, 1, n + 1)
    off = np.zeros(n + 1)
    step, scale = n, amp
    while step > 1:
        half = step // 2
        idx = np.arange(half, n, step)
        off[idx] = (off[idx - half] + off[idx + half]) / 2 + rng.uniform(-scale, scale, len(idx))
        step, scale = half, scale * 0.6
    d = np.asarray(b, float) - np.asarray(a, float)
    nrm = np.array([-d[1], d[0]]) / np.hypot(*d)
    return np.asarray(a, float) + t[:, None] * d + off[:, None] * nrm


def world(points: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    nx, ny = 25, 10
    xs, ys = np.linspace(-180, 180, nx + 1), np.linspace(-80, 80, ny + 1)
    cw, ch = xs[1] - xs[0], ys[1] - ys[0]
    h = {(i, j): fractal((xs[i], ys[j]), (xs[i + 1], ys[j]), points, 0.15 * ch, rng) for i in range(nx) for j in range(ny + 1)}
    v = {(i, j): fractal((xs[i], ys[j]), (xs[i], ys[j + 1]), points, 0.15 * cw, rng) for i in range(nx + 1) for j in range(ny)}
    feats, enclaves = [], []
    for j in range(ny):
        for i in range(nx):
            shell = np.concatenate([h[i, j][:-1], v[i + 1, j][:-1], h[i, j + 1][::-1][:-1], v[i, j][::-1]])
            rings = [shell.tolist()]
            k = j * nx + i
            if k % 10 == 3:
                cx, cy = (xs[i] + xs[i + 1]) / 2, (ys[j] + ys[j + 1]) / 2
                sq = [[cx - 2, cy - 2], [cx + 2, cy - 2], [cx + 2, cy + 2], [cx - 2, cy + 2], [cx - 2, cy - 2]]
                rings.append(sq[::-1])
                enclaves.append(sq)
            geom = {"type": "Polygon", "coordinates": rings}
            if k % 25 == 7:
                isl = [[xs[i] + 1, 82], [xs[i] + 4, 82], [xs[i] + 3, 85], [xs[i] + 1, 82]]
                geom = {"type": "MultiPolygon", "coordinates": [rings, [isl]]}
            feats.append({"type": "Feature", "properties": {"name": f"C{k}"}, "geometry": geom})
    for e, sq in enumerate(enclaves):
        feats.append({"type": "Feature", "properties": {"name": f"E{e}"}, "geometry": {"type": "Polygon", "coordinates": [sq]}})
    return {"type": "FeatureCollection", "features": feats}


def numpy_crossing(csr, pts):
    """fp64 crossing number per point against every geometry whose box holds it (first hit wins), numpy-vectorised."""
    verts, ring_off, part_ring_off, geom_part_off = csr[:4]
    G = len(geom_part_off) - 1
    boxes, segs = [], []
    for q in range(G):
        r0, r1 = part_ring_off[geom_part_off[q]], part_ring_off[geom_part_off[q + 1]]
        vv = verts[ring_off[r0]:ring_off[r1]]
        boxes.append((vv[:, 0].min(), vv[:, 1].min(), vv[:, 0].max(), vv[:, 1].max()))
        a = np.concatenate([verts[ring_off[r]:ring_off[r + 1] - 1] for r in range(r0, r1)])
        b = np.concatenate([verts[ring_off[r] + 1:ring_off[r + 1]] for r in range(r0, r1)])
        segs.append((a, b))
    out = np.full(len(pts), -1)
    for n, (x, y) in enumerate(pts):
        for q in range(G):
            bx = boxes[q]
            if not (bx[0] <= x <= bx[2] and bx[1] <= y <= bx[3]):
                continue
            a, b = segs[q]
            c = ((a[:, 1] > y) != (b[:, 1] > y))
            xi = a[c, 0] + (y - a[c, 1]) * (b[c, 0] - a[c, 0]) / (b[c, 1] - a[c, 1])
            if np.count_nonzero(xi > x) & 1:
                out[n] = q
                break
    return out


def gpu_info():
    import torch
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - report, do not fail the measurement
        power = f"unknown ({e})"
    return name, power


def timed(fn, repeats):
    import torch
    times = []
    for _ in range(repeats):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        times.append(s.elapsed_time(e))
    return float(np.median(times))


def main():
    import torch
    from pigeon_b200 import metrics
    from pigeon_b200._lib import check, current_stream_ptr, load, ptr
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=2048, help="segments per border")
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--sizes", default="26000,1000000")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("metrics_bench needs a CUDA device")
    card, power = gpu_info()
    w = world(args.points)
    report = dict(card=card, power_limit=power)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "countries.geojson")
        with open(path, "w") as f:
            json.dump(w, f)
        t0 = time.perf_counter()
        csr = metrics.parse_geojson(path)
        report["parse_s"] = time.perf_counter() - t0
    report.update(geometries=len(csr[3]) - 1, parts=len(csr[2]) - 1, rings=len(csr[1]) - 1, vertices=len(csr[0]))
    metrics.CountryIndex(*csr)                                              # warm-up (module load)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    idx = metrics.CountryIndex(*csr)
    torch.cuda.synchronize()
    report["upload_and_index_build_ms"] = (time.perf_counter() - t0) * 1e3
    report["index_entries"] = int(idx._c.num_entries)
    lib = load()
    for N in [int(s) for s in args.sizes.split(",")]:
        rng = np.random.default_rng(N)
        labels = np.stack([rng.uniform(-180, 180, N), np.degrees(np.arcsin(rng.uniform(-1, 1, N)))], 1)
        preds = (labels + rng.normal(0, 1, (N, 2)) * rng.choice([0.01, 0.1, 1, 5, 20], N)[:, None]).astype(np.float32)
        preds[:, 1] = np.clip(preds[:, 1], -90, 90)
        C = 2076
        cl = rng.integers(0, C, N)
        cp = np.where(rng.random(N) < 0.3, cl, rng.integers(0, C, N))
        top5 = rng.integers(0, C, (N, 5))
        dev = idx.device
        lab = torch.from_numpy(labels).to(dev)
        pr = torch.from_numpy(preds).to(dev)
        pr64 = pr.double()
        country = torch.empty(N, dtype=torch.int32, device=dev)
        flags = torch.empty(N, dtype=torch.uint8, device=dev)
        inside = torch.empty(N, dtype=torch.uint8, device=dev)
        cpt, clt, tk = (torch.from_numpy(a).to(dev) for a in (cp, cl, top5))
        dist = torch.empty(N, dtype=torch.float64, device=dev)
        res = torch.empty(16, dtype=torch.float64, device=dev)
        ws = torch.empty(int(lib.pg_geo_metrics_workspace_bytes(N)), dtype=torch.uint8, device=dev)

        def locate():
            check(lib.pg_country_locate(idx._c, ptr(lab), ptr(pr64), N, ptr(country), ptr(flags), ptr(inside),
                                        current_stream_ptr()), "locate")

        def kernels():
            check(lib.pg_geo_metrics(ptr(pr), 1, ptr(lab), N, ptr(cpt), ptr(clt), ptr(tk), 5, ptr(inside), ptr(ws),
                                     ws.numel(), ptr(dist), ptr(res), current_stream_ptr()), "metrics")

        results = (preds, cp, None, None, None, top5, labels, cl, None, None, None)

        def end_to_end():
            with contextlib.redirect_stdout(io.StringIO()):
                metrics.compute_geoguessr_metrics(results, countries=idx)

        for fn in (locate, kernels, end_to_end):
            fn()
        torch.cuda.synchronize()
        r = dict(locate_ms=timed(locate, args.repeats), metrics_kernels_ms=timed(kernels, args.repeats),
                 end_to_end_ms=timed(end_to_end, max(3, args.repeats // 4)),
                 nearest_fallback_share=float(flags.double().mean().item()),
                 country_accuracy=float(res[12].item()))
        report[f"N={N}"] = r
    sub = np.stack([np.random.default_rng(1).uniform(-180, 180, 200), np.random.default_rng(2).uniform(-80, 80, 200)], 1)
    t0 = time.perf_counter()
    numpy_crossing(csr, sub)
    report["cpu_numpy_fp64_crossing_ms_per_point (CPU, 200-point subsample, not exact)"] = \
        (time.perf_counter() - t0) * 1e3 / len(sub)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
