"""Time the prototype builder (pg_optics_xi) at MP-16 scale: ~2 000 geocells with log-normal sizes (median 1 700,
sigma 0.8, mean ~2 350) and one 30 000-point cell, ~4.7 M points in all, seeded.  Reports, after a warm-up call:
  - the whole pg_optics_xi call (CUDA events), and per kernel (core distances, ordering, xi) from torch.profiler in a
    separate pass;
  - the largest cell's call on its own (its ordering loop is the critical path of the whole launch);
  - fp64 haversine evaluations: sum n^2 per radix pass of the core selection plus sum n^2 / 2 for the ordering;
  - ProtoDataset.generate() end to end (host groupby, upload, clustering, aggregation, CSV);
  - sklearn OPTICS on one 2 000-point cell on this host's CPU, for context (--sklearn-sizes 2000 8000 adds more).
The card name and power limit are read in the same run.

    python tools/prototype_bench.py [--cells 2000] [--sklearn-sizes 2000]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from clip_train_bench import card  # noqa: E402
from pigeon_b200 import prototypes as P  # noqa: E402


def workload(cells: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    sizes = np.maximum(1, rng.lognormal(np.log(1700), 0.8, cells).astype(np.int64))
    sizes[np.argmax(sizes)] = max(int(sizes.max()), 30000)
    pts = []
    for n in sizes:
        centre = rng.uniform([-170, -60], [170, 70])
        k = int(rng.integers(1, 12))
        sub = centre + rng.normal(0, 0.3, (k, 2))
        pts.append(sub[rng.integers(0, k, n)] + rng.normal(0, 0.02, (n, 2)))
    return np.concatenate(pts), np.repeat(np.arange(cells), sizes), sizes


def timed_call(x, off, m, xi, reps=1):
    P.optics_xi_csr(x, off, m, xi)   # warm-up
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        s.record()
        P.optics_xi_csr(x, off, m, xi)   # includes the upload of x / off and the download of the labels
        e.record()
        torch.cuda.synchronize()
        ms.append(s.elapsed_time(e))
    return min(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=2000)
    ap.add_argument("--min-samples", type=int, default=100)
    ap.add_argument("--xi", type=float, default=0.1)
    ap.add_argument("--sklearn-sizes", type=int, nargs="*", default=[2000])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prototype_bench: no CUDA device")
    x, cells, sizes = workload(a.cells)
    order, _, off = P.group_by_cell(cells)
    x = x[order]
    res = dict(card=card(), cells=int(a.cells), points=int(len(x)), max_cell=int(sizes.max()),
               median_cell=float(np.median(sizes)))
    res["call_ms"] = timed_call(x, off, a.min_samples, a.xi)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        P.optics_xi_csr(x, off, a.min_samples, a.xi)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        for k in ("prep_kernel", "cell_order_kernel", "core_kernel", "ordering_kernel", "xi_kernel"):
            if k in ev.key:
                per[k] = per.get(k, 0.0) + ev.device_time_total / 1e3
    res["kernel_ms"] = per

    big = int(np.argmax(sizes))
    xb = x[off[big]:off[big + 1]]
    res["largest_cell_call_ms"] = timed_call(xb, [0, len(xb)], a.min_samples, a.xi)

    n2 = float(np.sum(sizes.astype(np.float64) ** 2))
    res["haversine_core_per_pass"] = n2
    res["haversine_ordering"] = n2 / 2
    if "ordering_kernel" in per:
        res["ordering_haversine_per_s"] = n2 / 2 / (per["ordering_kernel"] / 1e3)
    if "core_kernel" in per:
        res["core_haversine_per_s_per_pass"] = n2 / (per["core_kernel"] / 1e3)

    import pandas as pd
    from datasets import Dataset, DatasetDict
    with tempfile.TemporaryDirectory() as tmp:
        DatasetDict(train=Dataset.from_dict({"labels_clf": [0]})).save_to_disk(os.path.join(tmp, "emb"))
        df = pd.DataFrame(dict(lng=x[:, 0], lat=x[:, 1], geocell_idx=cells[order], selection="train"))
        t = time.perf_counter()
        P.ProtoDataset(df, os.path.join(tmp, "emb"), os.path.join(tmp, "protos.csv"),
                       (a.min_samples, a.xi)).generate()
        res["generate_s"] = time.perf_counter() - t
        res["prototypes"] = int(sum(1 for _ in open(os.path.join(tmp, "protos.csv")))) - 1

    from sklearn.cluster import OPTICS
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import optics_oracle as O
    sk = {}
    for n in a.sklearn_sizes:
        xs, _, _ = workload(1, seed=n)
        xs = xs[:n]
        rad, cos = O.prepare(xs)
        t = time.perf_counter()
        D = O.rows(rad, cos, np.arange(len(xs)))
        OPTICS(min_samples=a.min_samples, xi=a.xi, metric="precomputed").fit_predict(D)
        sk[str(n)] = time.perf_counter() - t
    res["sklearn_cpu_s"] = sk
    res["cpu_count"] = os.cpu_count()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
