#!/usr/bin/env python
"""Throughput of benchmark evaluation from image files (`run.py evaluate -l NAME`'s path) on one GPU, with the card
name and its power limit read in the same run.

Corpus: a seeded Flickr-like benchmark written to a temporary directory: --images JPEGs from 500x375 to 1024x768 in
both orientations, q85-95, mostly 4:2:0 without restart markers, about 4 % progressive and 2 % PNG (those go to Pillow
on the host), with a metadata CSV and a benchmarks.json.  Model: ViT-L/14-336 (24 layers, random weights) + a
2 000-cell geocell head + a ProtoRefiner over a synthetic 20 000-prototype bank; metrics: Geocell accuracy.

Measured:
  * `evaluate`: evaluate_model over BenchmarkDataset.encoded() end to end (file reads on DataLoader workers, GPU JPEG
    decode + square crop + pre-processing, tower, head, refiner, metrics), images/s;
  * `decode_gpu`: the decode + crop + pre-processing step alone (ClipImageProcessor(square_crop=True) on batches of
    files already in memory), images/s, and its share of the evaluate time;
  * `decode_host`: the host route for the same step: Pillow decode + convert('RGB') + crop on --threads threads, then
    the same GPU pre-processing, images/s.
Prints one JSON line per measurement.

    python tools/benchmark_eval_bench.py [--images 3000] [--batch 256] [--workers 4] [--threads 8] [--out DIR]
"""
import argparse
import io
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(375, 500), (500, 375), (480, 640), (640, 480), (600, 800), (800, 600), (768, 1024), (1024, 768)]
CELLS = 2000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0]) if r.returncode == 0 else None
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        power = None
    return name, power


def corpus(n, seed=0, distinct=96):
    """n (name, bytes, kind): `distinct` seeded encodes, repeated under different names."""
    from PIL import Image
    from pigeon_b200 import synthetic
    rng = np.random.default_rng(seed)
    pool = []
    for k in range(distinct):
        h, w = SIZES[k % len(SIZES)]
        img = Image.fromarray(synthetic.synthetic_photo(h, w, seed * 1000 + k))
        f = io.BytesIO()
        r = rng.random()
        if r < 0.02:
            img.save(f, "PNG")
            kind = "png"
        else:
            img.save(f, "JPEG", quality=int(rng.integers(85, 96)), subsampling=2 if rng.random() < 0.9 else 0,
                     progressive=bool(r < 0.06))
            kind = "progressive" if r < 0.06 else "baseline"
        pool.append((f.getvalue(), kind))
    order = rng.integers(0, distinct, n)
    return [(f"{i:05d}.{'png' if pool[j][1] == 'png' else 'jpg'}", pool[j][0], pool[j][1]) for i, j in enumerate(order)]


def model_and_refiner():
    from pigeon_b200 import ProtoRefiner, SuperGuessr, synthetic
    from pigeon_b200.super_guessr import CLIPVisionTower
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims()
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=0))
    torch.manual_seed(1)
    model = SuperGuessr(tower, panorama=False, freeze_base=True, num_candidates=50,
                        geocells=synthetic.synthetic_geocells(CELLS, 2)).to("cuda").eval()
    bank = synthetic.synthetic_bank(CELLS, 20000, dims.hidden, seed=3, members_mean=3.0)
    refiner = ProtoRefiner(topk=40, max_refinement=100000, temperature=0.6, protos=bank).eval()
    return model, refiner


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--images", type=int, default=3000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--png", action="store_true", help="also measure ClipImageProcessor(png=True)")
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/benchmark_eval_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmark_eval_bench: no CUDA device")
    gpu, power = card()
    base = dict(gpu=gpu, power_limit_w=power, images=args.images, batch=args.batch, host_threads=args.threads)
    lines = []

    def emit(d):
        d = dict(base, **d)
        lines.append(d)
        print(json.dumps(d), flush=True)

    files = corpus(args.images)
    tmp = tempfile.mkdtemp(prefix="benchmark_eval_bench_")
    try:
        run(args, files, tmp, emit)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "benchmark_eval_bench.jsonl"), "w") as f:
            f.write("".join(json.dumps(d) + "\n" for d in lines))


def run(args, files, tmp, emit):
    from PIL import Image
    from pigeon_b200 import benchmark, config, loops
    from pigeon_b200.preprocess import ClipImageProcessor, _square
    kinds = {k: sum(f[2] == k for f in files) for k in ("baseline", "progressive", "png")}
    os.makedirs(os.path.join(tmp, "img"))
    for name, data, _ in files:
        with open(os.path.join(tmp, "img", name), "wb") as f:
            f.write(data)
    rng = np.random.default_rng(7)
    import pandas as pd
    pd.DataFrame(dict(image=[f[0] for f in files], lng=rng.uniform(-180, 180, len(files)),
                      lat=rng.uniform(-60, 70, len(files)),
                      geocell_idx_yfcc=rng.integers(0, CELLS, len(files)))).to_csv(os.path.join(tmp, "meta.csv"), index=False)
    with open(os.path.join(tmp, "benchmarks.json"), "w") as f:
        json.dump({"synthetic": {"meta": os.path.join(tmp, "meta.csv"), "images": os.path.join(tmp, "img") + os.sep}}, f)
    config.BENCHMARKS = os.path.join(tmp, "benchmarks.json")
    ds = benchmark.BenchmarkDataset("synthetic")
    mb = sum(len(f[1]) for f in files) / 1e6

    model, refiner = model_and_refiner()
    procs = {"default": ClipImageProcessor()}
    if args.png:
        procs["png"] = ClipImageProcessor(png=True)
    proc = procs["default"]
    train_args = SimpleNamespace(per_device_eval_batch_size=args.batch)

    def evaluate(p):
        return loops.evaluate_model(model, ds.encoded(), None, train_args, refiner, num_workers=args.workers,
                                    collate_fn=loops.encoded_eval_collate, processor=p)

    for p in procs.values():
        evaluate(p)                                               # warm-up: modules, workspaces, allocator
    times = {r: [] for r in procs}
    for _ in range(args.repeats):
        for r, p in procs.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            evaluate(p)
            torch.cuda.synchronize()
            times[r].append(time.perf_counter() - t)
    t_evals = {r: float(np.median(ts)) for r, ts in times.items()}
    for r, ts in times.items():
        emit(dict(measure="evaluate", route=r, images_per_s=round(len(files) / t_evals[r], 1),
                  seconds=[round(x, 3) for x in ts], corpus_mb=round(mb, 1), kinds=kinds, workers=args.workers,
                  refiner=True, metrics="Geocell_accuracy"))

    batches = [[f[1] for f in files[i:i + args.batch]] for i in range(0, len(files), args.batch)]

    def gpu_route(p=proc):
        for b in batches:
            p(images=b, square_crop=True)
        torch.cuda.synchronize()

    pool = ThreadPoolExecutor(args.threads)

    def host_decode(data):
        a = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))
        return np.ascontiguousarray(_square(a))

    def host_route():
        for b in batches:
            proc(images=list(pool.map(host_decode, b)))
        torch.cuda.synchronize()

    arms = [("decode_gpu", r, (lambda p=p: gpu_route(p))) for r, p in procs.items()] + [("decode_host", None, host_route)]
    for name, r, fn in arms:
        fn()
        ts = []
        for _ in range(args.repeats):
            t = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t)
        t_dec = float(np.median(ts))
        d = dict(measure=name, images_per_s=round(len(files) / t_dec, 1), seconds=[round(x, 3) for x in ts])
        if r is not None:
            d["route"] = r
            d["share_of_evaluate"] = round(t_dec / t_evals[r], 3)
        emit(d)
    pool.shutdown()


if __name__ == "__main__":
    main()
