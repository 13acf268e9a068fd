"""Time one CLIPModel contrastive training step (`forward_train` + `backward`) on the GPU at the reference's per-device
batch: 32 images at 336 x 336 and 32 captions at S = 77 (mixed lengths), CLIP-L/14-336 (ViT-L/14 + the 12 x 768 text tower),
every parameter trainable.  Prints the card name and power limit of the same run and the median of CUDA-event times.

    python tools/clip_train_bench.py [--n 32] [--steps 10] [--warmup 3]
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
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=32)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clip_train_bench: no CUDA device")
    from pigeon_b200 import CLIPModel, TextDims, VitDims, synthetic
    dev = torch.device("cuda:0")
    td, vd = TextDims(), VitDims()
    m = CLIPModel(td, vd, projection_dim=768)
    m.load_state_dict(synthetic.random_clip_state_dict(td, vd, seed=0, std=0.02, projection_dim=768))
    m = m.to(dev)
    g = torch.Generator().manual_seed(1)
    n, S = a.n, td.max_positions
    ids = torch.full((n, S), td.vocab - 1, dtype=torch.int64)
    mask = torch.zeros((n, S), dtype=torch.int64)
    for b in range(n):
        L = int(torch.randint(3, S + 1, (1,), generator=g))
        ids[b, 0] = td.vocab - 2
        ids[b, 1:L - 1] = torch.randint(0, td.vocab - 2, (L - 2,), generator=g)
        mask[b, :L] = 1
    ids, mask = ids.to(dev), mask.to(dev)
    px = torch.randn(n, 3, vd.image_size, vd.image_size, generator=g).to(dev)
    times = []
    for i in range(a.warmup + a.steps):
        m.zero_grad(set_to_none=True)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        out = m.forward_train(ids, px, mask)
        m.backward()
        t1.record()
        torch.cuda.synchronize()
        if i >= a.warmup:
            times.append(t0.elapsed_time(t1))
    times.sort()
    print(json.dumps({"card": card(), "n": n, "S": S, "step_ms_median": times[len(times) // 2], "step_ms_min": times[0],
                      "step_ms_max": times[-1], "loss": out.loss.item(),
                      "peak_mem_gb": torch.cuda.max_memory_allocated() / 1e9}))


if __name__ == "__main__":
    main()
