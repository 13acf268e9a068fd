#!/usr/bin/env python
"""GPU JPEG decoding throughput on one GPU, with the card name and its power limit read in the same run.

Corpora: 640x640 4:2:0 q90 (Street-View-like) and 1024x768 4:2:0 q85 (YFCC-like), each without restart markers and
with one restart interval per MCU row, at 1 and 4 files per call (latency) and 64, 256 and 1024 (throughput; 16
distinct synthetic photos, repeated).  For each, under the entropy-kernel schedules of pg_jpeg_set_schedule in
alternation (1 = one thread per segment, 0 = automatic, 2 = chunked everywhere; `--reps` times): images/s and MB/s of
compressed input for decode alone and for decode + pg_preprocess_clip, the per-stage kernel times (CUDA events around
each launch: jpeg_entropy for one thread per segment, jpeg_entropy_chunked for the chunked kernel), and the
host-to-device bytes.  Per corpus, the chunked decoder's synchronisation rounds (maximum and mean over the files).  For context: Pillow decoding on every
host core followed by the same GPU pre-processing, and a CLIPEmbedding (ViT-L/14-336) pass from bytes against the same
pass from pre-decoded host pixels.  Prints one JSON line per measurement.

`--multiscan` measures instead the progressive versions of the two corpora (Pillow's progressive=True, libjpeg's
10-scan script, no restart markers) through the multi-scan path (`jpeg_multiscan=True`), with the kernel time of each
dependency level, against the host route (Pillow on every host core + the same GPU pre-processing).

    python tools/jpeg_bench.py [--multiscan] [--iters 10] [--warmup 3] [--reps 2] [--out DIR]
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


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0]) if r.returncode == 0 else None
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        power = None
    return name, power


def corpus(h, w, q, restart, distinct=16, progressive=False):
    from PIL import Image, ImageFile
    from pigeon_b200 import synthetic
    ImageFile.MAXBLOCK = max(ImageFile.MAXBLOCK, 1 << 24)      # Pillow's progressive encoder buffers the whole file
    out = []
    for i in range(distinct):
        f = io.BytesIO()
        kw = dict(restart_marker_rows=1) if restart else {}
        if progressive:
            kw["progressive"] = True
        Image.fromarray(synthetic.synthetic_photo(h, w, seed=1000 + i)).save(f, "JPEG", quality=q, subsampling=2, **kw)
        out.append(f.getvalue())
    return out


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


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
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/jpeg_bench.jsonl")
    ap.add_argument("--multiscan", action="store_true", help="progressive corpora through the multi-scan path")
    ap.add_argument("--reps", type=int, default=2, help="alternations of the entropy-kernel schedules per workload")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("jpeg_bench needs a CUDA device")
    from PIL import Image
    from pigeon_b200.jpeg import JpegDecoder, entropy_host, set_schedule
    from pigeon_b200.preprocess import ClipImageProcessor
    dev = torch.device("cuda:0")
    gpu, power = card()
    cores = os.cpu_count()
    base = dict(gpu=gpu, power_limit_w=power, host_cores=cores, iters=args.iters, warmup=args.warmup)
    lines = []

    def emit(d):
        d = dict(base, **d)
        lines.append(d)
        print(json.dumps(d), flush=True)

    dec = JpegDecoder(dev)
    proc = ClipImageProcessor(device=dev, dtype=torch.float16)
    corpora = {"640x640 q90": (640, 640, 90), "1024x768 q85": (768, 1024, 85)}
    if args.multiscan:
        multiscan(args, dec, corpora, emit)
    for cname, (h, w, q) in (corpora.items() if not args.multiscan else ()):
        for restart in (False, True):
            distinct = corpus(h, w, q, restart)
            # synchronisation rounds of the chunked decoder at its automatic chunk size, from the host entry that runs
            # the kernel's chunk functions in its order of rounds (the counts do not depend on the device)
            _, _, rounds = entropy_host(distinct, -1)
            emit(dict(corpus=cname, restart_rows=restart, files=len(distinct), sync_rounds_max=int(rounds.max()),
                      sync_rounds_mean=round(float(rounds.mean()), 2),
                      note="rounds per file: the most any of its segments took"))
            for n in (1, 4, 64, 256, 1024):
                files = [distinct[i % len(distinct)] for i in range(n)]
                mb = sum(len(f) for f in files) / 1e6
                iters = args.iters * (10 if n <= 4 else 1)
                # the schedules alternate within the job: 1 = one thread per segment (the previous decoder),
                # 0 = automatic, 2 = chunked for every segment
                for rep in range(args.reps):
                    for sched in (1, 0, 2):
                        set_schedule(sched, 0)
                        t_dec = timed(lambda: dec.decode(files), iters, args.warmup)
                        t_pre = timed(lambda: proc(images=files), iters, args.warmup)
                        stages = stage_ms(lambda: dec.decode(files))
                        emit(dict(corpus=cname, restart_rows=restart, images=n, schedule=sched, rep=rep,
                                  compressed_mb=round(mb, 3), h2d_bytes=sum(len(f) for f in files),
                                  decode_ms=round(t_dec * 1e3, 3), decode_img_s=round(n / t_dec, 1),
                                  decode_mb_s=round(mb / t_dec, 1), decode_pre_ms=round(t_pre * 1e3, 3),
                                  decode_pre_img_s=round(n / t_pre, 1), decode_pre_mb_s=round(mb / t_pre, 1),
                                  stage_ms=stages))
                set_schedule(0, 0)
            # Pillow on every host core, then the same GPU pre-processing (one call of 256 files)
            files = [distinct[i % len(distinct)] for i in range(256)]
            pool = ThreadPoolExecutor(cores)

            def pillow_then_gpu():
                px = list(pool.map(lambda b: np.asarray(Image.open(io.BytesIO(b)).convert("RGB")), files))
                return proc(images=px)

            t = timed(pillow_then_gpu, max(2, args.iters // 3), 1)
            pool.shutdown()
            emit(dict(corpus=cname, restart_rows=restart, images=256, pillow_threads=cores,
                      pillow_decode_pre_ms=round(t * 1e3, 3), pillow_decode_pre_img_s=round(256 / t, 1)))

    if not args.multiscan:
        embedding(args, emit)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        name = "jpeg_bench_multiscan.jsonl" if args.multiscan else "jpeg_bench.jsonl"
        with open(os.path.join(args.out, name), "w") as f:
            f.write("".join(json.dumps(d) + "\n" for d in lines))


def multiscan(args, dec, corpora, emit):
    from PIL import Image
    from pigeon_b200.preprocess import ClipImageProcessor
    proc = ClipImageProcessor(device=dec.device, dtype=torch.float16, jpeg_multiscan=True)
    cores = os.cpu_count()
    for cname, (h, w, q) in corpora.items():
        distinct = corpus(h, w, q, False, progressive=True)
        for n in (64, 256, 1024):
            files = [distinct[i % len(distinct)] for i in range(n)]
            mb = sum(len(f) for f in files) / 1e6
            t_dec = timed(lambda: dec.decode(files, multiscan=True), args.iters, args.warmup)
            t_pre = timed(lambda: proc(images=files), args.iters, args.warmup)
            stages = stage_ms(lambda: dec.decode(files, multiscan=True))
            emit(dict(corpus=cname + " progressive", images=n, compressed_mb=round(mb, 3),
                      decode_ms=round(t_dec * 1e3, 3), decode_img_s=round(n / t_dec, 1),
                      decode_pre_ms=round(t_pre * 1e3, 3), decode_pre_img_s=round(n / t_pre, 1), stage_ms=stages))
            pool = ThreadPoolExecutor(cores)
            host = ClipImageProcessor(device=dec.device, dtype=torch.float16)

            def pillow_then_gpu():
                px = list(pool.map(lambda b: np.asarray(Image.open(io.BytesIO(b)).convert("RGB")), files))
                return host(images=px)

            t = timed(pillow_then_gpu, max(2, args.iters // 3), 1)
            pool.shutdown()
            emit(dict(corpus=cname + " progressive", images=n, pillow_threads=cores,
                      pillow_decode_pre_ms=round(t * 1e3, 3), pillow_decode_pre_img_s=round(n / t, 1)))


def embedding(args, emit):
    # CLIPEmbedding (ViT-L/14-336, random weights) from bytes against from pre-decoded host pixels, batch 64
    from PIL import Image
    from pigeon_b200 import CLIPEmbedding, synthetic
    from pigeon_b200.super_guessr import CLIPVisionTower
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims()
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=0), strict=True)
    model = CLIPEmbedding("unused", device="cuda", clip_model=tower)
    distinct = corpus(640, 640, 90, False)
    files = [distinct[i % len(distinct)] for i in range(64)]
    pixels = [np.asarray(Image.open(io.BytesIO(b)).convert("RGB")) for b in files]
    a = model(files)
    b = model(pixels)
    same = bool(torch.equal(a, b))
    t_bytes = timed(lambda: model(files), args.iters, args.warmup)
    t_px = timed(lambda: model(pixels), args.iters, args.warmup)
    emit(dict(workload="CLIPEmbedding ViT-L/14-336 batch 64, 640x640 q90", embeddings_identical=same,
              from_bytes_ms=round(t_bytes * 1e3, 3), from_host_pixels_ms=round(t_px * 1e3, 3)))


if __name__ == "__main__":
    main()
