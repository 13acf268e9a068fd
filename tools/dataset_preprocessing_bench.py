"""Benchmark of geocell labelling in pigeon_b200.dataset_preprocessing on a synthetic world of about 2 000 geocells.

Geocells: a 50 x 40 grid over lng [-180, 180] x lat [-90, 90], every inner border a fractal polyline (256 segments)
shared vertex for vertex by its two cells, one cell in seven with a square hole, and one in thirty-three left out as
sea; about 2 M vertices in total, written as the WKT geocell CSV `preprocess` reads.  Points: 1 M and 5 M uniform over
the world (about 3 % of them at sea or in a hole, so they take the nearest-cell fallback).

Reported: WKT parse of the CSV (`parse_geocells`), upload + index build (`CountryIndex`), `locate` on the device
(CUDA events after warm-up, median of the repeats) and `preprocess` end to end on a raw DatasetDict of one split with
the reference's non-image columns (heading features, labels, multi-task labels), with the card name and power limit.

    python tools/dataset_preprocessing_bench.py [--points 1000000,5000000] [--repeats 5]
"""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from metrics_bench import fractal, gpu_info, timed  # noqa: E402


def geocell_frame(seg: int = 256, seed: int = 0):
    import pandas as pd
    rng = np.random.default_rng(seed)
    nx, ny = 50, 40
    xs, ys = np.linspace(-180, 180, nx + 1), np.linspace(-90, 90, ny + 1)
    cw, ch = xs[1] - xs[0], ys[1] - ys[0]
    h = {(i, j): fractal((xs[i], ys[j]), (xs[i + 1], ys[j]), seg, 0.15 * ch * (0 < j < ny), rng)
         for i in range(nx) for j in range(ny + 1)}
    v = {(i, j): fractal((xs[i], ys[j]), (xs[i], ys[j + 1]), seg, 0.15 * cw * (0 < i < nx), rng)
         for i in range(nx + 1) for j in range(ny)}
    ring = lambda r: "(" + ", ".join(f"{x!r} {y!r}" for x, y in r.tolist()) + ")"
    rows = []
    for j in range(ny):
        for i in range(nx):
            k = j * nx + i
            if k % 33 == 5:
                continue
            shell = np.concatenate([h[i, j][:-1], v[i + 1, j][:-1], h[i, j + 1][::-1][:-1], v[i, j][::-1]])
            rings = [ring(shell)]
            cx, cy = (xs[i] + xs[i + 1]) / 2, (ys[j] + ys[j + 1]) / 2
            if k % 7 == 2:
                a, b = cw / 8, ch / 8
                rings.append(ring(np.asarray([[cx - a, cy - b], [cx - a, cy + b], [cx + a, cy + b], [cx + a, cy - b],
                                              [cx - a, cy - b]])))
            rows.append((cx, cy, "POLYGON (" + ", ".join(rings) + ")"))
    return pd.DataFrame(rows, columns=["lng", "lat", "polygon"])


def raw_dataset(n: int, seed: int = 1):
    import datasets
    rng = np.random.default_rng(seed)
    cols = dict(lng=rng.uniform(-180, 180, n), lat=rng.uniform(-90, 90, n), heading=rng.uniform(0, 360, n),
                index=np.arange(n, dtype=np.int64), labels_climate=rng.integers(0, 28, n))
    for j, c in enumerate(("elevation", "population", "temp_avg", "temp_diff", "prec_avg", "prec_diff")):
        cols[c] = rng.normal(j, 1, n)
    return datasets.DatasetDict(train=datasets.Dataset.from_dict(cols))


def main():
    import torch
    from pigeon_b200 import config
    from pigeon_b200 import dataset_preprocessing as dp
    from pigeon_b200.metrics import CountryIndex
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", default="1000000,5000000")
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    card, power = gpu_info()
    report = dict(card=card, power_limit=power)
    t = time.perf_counter()
    frame = geocell_frame()
    report["world_s"] = time.perf_counter() - t
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, config.GEOCELL_PATH)
        os.makedirs(os.path.dirname(path))
        frame.to_csv(path, index=False)
        report["csv_mb"] = os.path.getsize(path) / 1e6
        t = time.perf_counter()
        csr, lnglat = dp.parse_geocells(path)
        report["parse_wkt_s"] = time.perf_counter() - t
        report["cells"], report["vertices"] = len(lnglat), len(csr[0])
        CountryIndex(*csr)                                                         # module load, allocator warm-up
        torch.cuda.synchronize()
        t = time.perf_counter()
        index = CountryIndex(*csr)
        torch.cuda.synchronize()
        report["index_build_s"] = time.perf_counter() - t
        for n in (int(x) for x in a.points.split(",")):
            rng = np.random.default_rng(n)
            pts = torch.from_numpy(np.stack([rng.uniform(-180, 180, n), rng.uniform(-90, 90, n)], 1)).cuda()
            index.locate(pts)
            ms = timed(lambda: index.locate(pts), a.repeats)
            _, flags, _ = index.locate(pts)
            row = dict(locate_ms=ms, fallback_share=float(flags.double().mean().item()))
            ds = raw_dataset(n)
            cwd = os.getcwd()
            os.chdir(tmp)
            try:
                with contextlib.redirect_stderr(io.StringIO()):
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    out = dp.preprocess(ds, config.GEOCELL_PATH, multi_task=True)
                    torch.cuda.synchronize()
                row["preprocess_s"] = time.perf_counter() - t
            finally:
                os.chdir(cwd)
            assert out["train"].num_rows == n
            report[f"n={n}"] = row
            print(json.dumps({f"n={n}": row}), flush=True)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
