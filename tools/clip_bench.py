"""Timing of the CLIPModel forward pieces on one GPU (CUDA events after warm-up), with algorithmic FLOPs from the shapes.

    text features   1000 captions at S = 77, and a mixed-length batch (lengths 5 ... 60, padded to the longest)
    image features  CLIPModel.get_image_features against CLIPEmbedding (token mean) on 1024 views: the CLS copy,
                    post_layernorm and visual_projection are the only extra work
    logits          1024 images x 1000 captions (normalise, scaled dot products, softmax, argmax)

Random-init CLIP-L/14-336 weights (timings do not depend on the values).  Prints one JSON line per measurement, with the
card name and its power limit read in the same run.

    python tools/clip_bench.py [--iters 10] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

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


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(iters):
        start.record()
        fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    times.sort()
    return times[len(times) // 2]


def text_flops(td, lengths_padded_to):
    """GEMMs (qkv, out_proj, fc1, fc2) + causal attention (half of QK^T and PV) over the padded batch, plus nothing for
    the memory-bound embedding / LayerNorm / pooling kernels."""
    n, S = lengths_padded_to
    h, f = td.hidden, td.intermediate
    gemm = 2 * n * S * (4 * h * h + 2 * h * f)
    attn = 2 * 2 * n * td.heads * 64 * S * (S + 1) / 2
    return td.layers * (gemm + attn)


def vit_flops(vd, n):
    T, h, f = vd.tokens, vd.hidden, vd.intermediate
    per_layer = 2 * T * (4 * h * h + 2 * h * f) + 2 * 2 * T * T * h
    return n * (vd.layers * per_layer + 2 * (T - 1) * h * vd.patch_k)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from pigeon_b200 import CLIPEmbedding, CLIPModel, TextDims, VitDims, synthetic
    dev = torch.device("cuda:0")
    name, power = card()
    td, vd = TextDims(), VitDims()
    model = CLIPModel(td, vd)
    model.load_state_dict(synthetic.random_clip_state_dict(td, vd, seed=0))
    model = model.to(dev).eval()
    model.text_tower.max_texts_per_pass = 1000
    g = torch.Generator().manual_seed(0)
    base = dict(gpu=name, power_limit_w=power, iters=args.iters, warmup=args.warmup)

    def report(what, ms, flops=None, **extra):
        rec = dict(base, what=what, ms=round(ms, 4), **extra)
        if flops:
            rec["tflops"] = round(flops / (ms * 1e-3) / 1e12, 1)
        print(json.dumps(rec), flush=True)

    # text features: full length
    n = 1000
    ids = torch.randint(0, td.vocab - 2, (n, 77), generator=g)
    ids[:, 0], ids[:, -1] = td.vocab - 2, td.vocab - 1
    ids = ids.to(dev)
    ms = time_ms(lambda: model.get_text_features(ids), args.iters, args.warmup)
    report("text_features_1000x77", ms, text_flops(td, (n, 77)), captions=n, seq=77)
    # text features: mixed lengths, padded to the longest like CLIPProcessor(padding=True)
    lengths = torch.randint(5, 61, (n,), generator=g)
    S = int(lengths.max())
    mids = torch.full((n, S), td.vocab - 1, dtype=torch.int64)
    mask = torch.zeros((n, S), dtype=torch.int64)
    for b, L in enumerate(lengths.tolist()):
        mids[b, 0] = td.vocab - 2
        mids[b, 1:L - 1] = torch.randint(0, td.vocab - 2, (L - 2,), generator=g)
        mask[b, :L] = 1
    mids, mask = mids.to(dev), mask.to(dev)
    ms = time_ms(lambda: model.get_text_features(mids, mask), args.iters, args.warmup)
    report("text_features_1000_mixed", ms, text_flops(td, (n, S)), captions=n, seq=S,
           mean_length=round(float(lengths.float().mean()), 1))

    # image features against the token-mean embedder on the same tower
    nv = 1024
    px = torch.randn(nv, 3, vd.image_size, vd.image_size, generator=g).half().to(dev)
    emb = CLIPEmbedding("", device="cuda", clip_model=model.vision_tower)
    ms_emb = time_ms(lambda: emb(px), args.iters, args.warmup)
    report("clip_embedding_1024", ms_emb, vit_flops(vd, nv), views=nv)
    proj = 2 * nv * vd.hidden * 3 * model.projection_dim
    ms_img = time_ms(lambda: model.get_image_features(px), args.iters, args.warmup)
    report("image_features_1024", ms_img, vit_flops(vd, nv) + proj, views=nv,
           extra_over_clip_embedding_ms=round(ms_img - ms_emb, 4))

    # logits 1024 x 1000
    img = torch.randn(nv, model.projection_dim, generator=g).to(dev)
    txt = torch.randn(n, model.projection_dim, generator=g).to(dev)
    ms = time_ms(lambda: model.logits(img, txt, per_text=True, probs=True, pred=True), args.iters, args.warmup)
    report("logits_1024x1000", ms, 2 * nv * n * model.projection_dim, images=nv, captions=n)
    ms = time_ms(lambda: model.logits(img[:n], txt, per_text=True, loss=True), args.iters, args.warmup)
    report("logits_loss_1000x1000", ms, 2 * n * n * model.projection_dim, images=n, captions=n)


if __name__ == "__main__":
    main()
