#!/usr/bin/env python
"""GPU PNG decoding throughput on one GPU, with the card name and its power limit read in the same run.

Corpora (seeded, Pillow-saved at the default level): 640x640 and 1024x768 synthetic photos, and a flat, screenshot-like
1024x768 corpus (flat panels, text-like strokes) where matches dominate.  For each corpus and 1, 4, 64, 256 and 1 024
files per call:
  * `gpu_decode`: PngDecoder.decode, ms per call and images/s;
  * `gpu_decode_preprocess`: ClipImageProcessor(png=True) on the encoded files (decode + pg_preprocess_clip);
  * `host_decode_preprocess`: Pillow decode + convert('RGB') on --threads threads, then the same pre-processing;
  * `kernels`: per-kernel ms of one gpu_decode call (png_inflate, png_unfilter, png_rgb; CUDA events).
Prints one JSON line per measurement and writes them to --out/png_bench.jsonl.

    python tools/png_bench.py [--iters 5] [--warmup 2] [--threads 8] [--out DIR]
"""
import argparse
import ctypes as C
import io
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCHES = [1, 4, 64, 256, 1024]
DISTINCT = 16


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0]) if r.returncode == 0 else None
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        power = None
    return name, power


def flat(h, w, seed):
    """Screenshot-like: flat panels, borders and rows of text-like strokes on a light background."""
    rng = np.random.default_rng(seed)
    img = np.full((h, w, 3), 242, dtype=np.uint8)
    for _ in range(12):
        y0, x0 = int(rng.integers(0, h - 40)), int(rng.integers(0, w - 40))
        y1, x1 = y0 + int(rng.integers(30, h // 2)), x0 + int(rng.integers(30, w // 2))
        img[y0:y1, x0:x1] = rng.integers(0, 256, 3)
        img[y0:y1, x0] = img[y0, x0:x1] = 40
    for y in range(20, h - 12, 18):                      # "text": short dark strokes on a baseline grid
        xs = np.cumsum(rng.integers(4, 12, w // 6))
        for x in xs[xs < w - 3][::2]:
            img[y:y + 9, x:x + 2] = 30
    return img


def corpora():
    from PIL import Image
    from pigeon_b200 import synthetic
    out = {}
    for name, make in (("photo 640x640", lambda s: synthetic.synthetic_photo(640, 640, seed=s)),
                       ("photo 1024x768", lambda s: synthetic.synthetic_photo(768, 1024, seed=s)),
                       ("flat 1024x768", lambda s: flat(768, 1024, s))):
        files = []
        for s in range(DISTINCT):
            f = io.BytesIO()
            Image.fromarray(make(s)).save(f, "PNG")
            files.append(f.getvalue())
        out[name] = files
    return out


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def stage_ms(fn):
    from pigeon_b200 import _lib
    lib = _lib.load()
    torch.cuda.synchronize()
    lib.pg_profile_begin()
    fn()
    torch.cuda.synchronize()
    n = lib.pg_profile_end()
    names, ms, counts = (C.c_char_p * n)(), (C.c_float * n)(), (C.c_int32 * n)()
    lib.pg_profile_read(names, ms, counts, n)
    return {names[i].decode(): round(float(ms[i]), 4) for i in range(n)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/png_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("png_bench needs a CUDA device")
    from PIL import Image
    from pigeon_b200.png import PngDecoder
    from pigeon_b200.preprocess import ClipImageProcessor
    gpu, power = card()
    base = dict(gpu=gpu, power_limit_w=power, host_threads=args.threads, iters=args.iters)
    lines = []

    def emit(d):
        d = dict(base, **d)
        lines.append(d)
        print(json.dumps(d), flush=True)

    dec = PngDecoder("cuda")
    proc = ClipImageProcessor(png=True)
    pool = ThreadPoolExecutor(args.threads)

    def host(data):
        return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))

    for cname, pool_files in corpora().items():
        mb = sum(len(f) for f in pool_files) / len(pool_files) / 1e6
        for n in BATCHES:
            files = [pool_files[i % DISTINCT] for i in range(n)]
            iters = args.iters if n < 1024 else max(2, args.iters // 2)
            for measure, fn in (("gpu_decode", lambda: dec.decode(files)),
                                ("gpu_decode_preprocess", lambda: proc(images=files)),
                                ("host_decode_preprocess", lambda: proc(images=list(pool.map(host, files))))):
                t = timed(fn, iters, args.warmup)
                emit(dict(corpus=cname, mean_file_mb=round(mb, 3), files=n, measure=measure, ms_per_call=round(t * 1e3, 3),
                          images_per_s=round(n / t, 1)))
            emit(dict(corpus=cname, files=n, measure="kernels", ms=stage_ms(lambda: dec.decode(files))))
    pool.shutdown()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "png_bench.jsonl"), "w") as f:
            f.write("".join(json.dumps(d) + "\n" for d in lines))


if __name__ == "__main__":
    main()
