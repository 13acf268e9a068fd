"""Cost of the hierarchical panorama head (SuperGuessr(hierarchical=True): positional encoding + view self-attention, CLS row
to the cell layer) against the view mean, on one GPU, timed with CUDA events after warm-up:

  head      the head forward on embeddings, N = 256 panoramas, E = 1024, C = 2076 geocells, top-5, loss
  train     a head-only training step on embeddings: forward, backward(), AdamW step
  eval      the ViT-L/14-336 evaluation step: 1024 views through the tower, then the head (random tower weights)

Each pair is timed alternately (mean, hierarchical, mean, ...) so that both see the same clocks.  Prints the card's name
and power limit, then one JSON line per workload with the milliseconds of both heads and the FLOPs counted from the shapes.

    python tools/hierarchical_bench.py [--iters 20] [--warmup 5] [--rounds 3] [--no-tower]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

N, E, C, K = 256, 1024, 2076, 5


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = (s.strip() for s in out[0].split(",")) if out else (torch.cuda.get_device_name(), "?", "?")
    return dict(card=name, power_limit=power, max_sm_clock=clock)


def flops() -> dict:
    """Multiply-adds x 2 from the shapes.  The split GEMM runs every projection with K = 3E (x3 on the tensor cores)."""
    attn_fwd = 2 * N * E * E + 2 * 4 * N * 2 * E * E + 2 * N * E * E + 2 * 2 * N * E * 4   # q0, k v, out_proj, core
    attn_bwd = 2 * (2 * N * E * E) + 2 * (2 * 4 * N * 3 * E * E)                           # out_proj dW, dX; in_proj dW, dX
    head_fwd = 2 * N * C * E
    d, t, L, inter = 1024, 577, 24, 4096                                                   # ViT-L/14 at 336 px
    tower = 4 * N * (2 * 576 * d * 588 + L * (2 * t * d * (3 * d + d + 2 * inter) + 2 * 2 * t * t * d))
    return dict(attention_forward=attn_fwd, attention_forward_tensor_core=3 * (attn_fwd - 2 * 2 * N * E * 4),
                attention_backward_fp32=attn_bwd, cell_layer_forward=head_fwd, tower_forward=tower)


def timed(fn, warmup: int, iters: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def compare(name: str, fns: dict, args) -> dict:
    ms = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, fn in fns.items():
            ms[k].append(timed(fn, args.warmup, args.iters))
    res = {"workload": name}
    for k, v in ms.items():
        res[f"{k}_ms"] = round(min(v), 4)
        res[f"{k}_ms_rounds"] = [round(x, 4) for x in v]
    res["added_ms"] = round(res["hierarchical_ms"] - res["mean_ms"], 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-tower", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hierarchical_bench: no CUDA device")
    from pigeon_b200 import CLIPVisionTower, SuperGuessr, VitDims, synthetic
    from pigeon_b200.training import AdamW
    dev = torch.device("cuda:0")
    print(json.dumps(dict(card(), N=N, E=E, C=C, flops=flops())))
    cells = synthetic.synthetic_geocells(C, 0)
    g = torch.Generator().manual_seed(0)
    emb = (torch.randn(N, 4, E, generator=g) * 0.3).to(dev)
    labels_clf = (torch.arange(N) % C).to(dev)

    def head(hier, base=None):
        torch.manual_seed(0)
        return SuperGuessr(base, panorama=True, hierarchical=hier, freeze_base=base is not None, num_candidates=K,
                           embed_dim=E, geocells=cells).to(dev)

    models = {"mean": head(False), "hierarchical": head(True)}
    for m in models.values():
        m.eval()
    print(json.dumps(compare("head", {k: (lambda m=m: m(embedding=emb, labels_clf=labels_clf)) for k, m in models.items()},
                             args)))

    def train_step(m, opt):
        out = m(embedding=emb, labels_clf=labels_clf)
        m.backward(out.loss)
        opt.step()
        opt.zero_grad()

    steps = {}
    for k, m in models.items():
        m.train()
        opt = AdamW(m.parameters(), lr=1e-5)
        steps[k] = lambda m=m, opt=opt: train_step(m, opt)
    print(json.dumps(compare("train", steps, args)))

    if args.no_tower:
        return
    dims = VitDims()
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=0))
    tower.max_views_per_pass = 4 * N
    px = torch.randn(N, 12, dims.image_size, dims.image_size, generator=g).half().to(dev)
    towered = {"mean": head(False, tower).eval(), "hierarchical": head(True, tower).eval()}
    tower_args = argparse.Namespace(rounds=args.rounds, warmup=2, iters=max(3, args.iters // 4))
    print(json.dumps(compare("eval", {k: (lambda m=m: m(pixel_values=px, labels_clf=labels_clf)) for k, m in towered.items()},
                             tower_args)))


if __name__ == "__main__":
    main()
