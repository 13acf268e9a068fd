"""Time one optimizer step of CLIP pretraining at the reference's PRETAIN_ARGS shape: 32 image-caption pairs per micro-batch
(336 x 336, S = 77 with mixed caption lengths), gradient accumulation 8, CLIP-L/14-336 from random init with every one of
its ~428 M parameters trainable.  Reports, per optimizer step: the micro-steps (`forward_train` + `backward`), the global
norm + clip coefficient (pg_grad_norm_clip), the HF AdamW update (pg_adamw_hf_step per tensor), under torchrun the summing
all-reduce of the flat gradient, and peak memory, with the card name and power limit read in the same run.

    python tools/clip_pretrain_bench.py [--steps 3] [--warmup 1]
    python -m torch.distributed.run --nproc-per-node 2 tools/clip_pretrain_bench.py
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from clip_train_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=32)
    ap.add_argument("--acc", type=int, default=8)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clip_pretrain_bench: no CUDA device")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        torch.distributed.init_process_group("nccl")
    rank = torch.distributed.get_rank() if world > 1 else 0
    import clip_pretrain_oracle as O
    from pigeon_b200 import CLIPModel, TextDims, VitDims, synthetic
    from pigeon_b200.pretrain import CLIPCollator, CLIPPretrainer
    dev = torch.device("cuda", torch.cuda.current_device())
    td, vd = TextDims(), VitDims()
    m = CLIPModel(td, vd, projection_dim=768)
    m.load_state_dict(synthetic.random_clip_state_dict(td, vd, seed=0, std=0.02, projection_dim=768))
    m = m.to(dev)
    n_params = sum(p.numel() for p in m.parameters())
    rows = O.golden_rows(a.n * a.acc, vd.image_size, td.vocab, td.max_positions, 1 + rank)
    args = SimpleNamespace(output_dir="/nonexistent", per_device_train_batch_size=a.n, gradient_accumulation_steps=a.acc,
                           num_train_epochs=1, max_steps=a.steps + a.warmup, learning_rate=1e-6, adam_beta1=0.9,
                           adam_beta2=0.98, adam_epsilon=1e-6, weight_decay=0.001, max_grad_norm=1.0, warmup_ratio=0.2,
                           lr_scheduler_type="linear", logging_steps=1, evaluation_strategy="no", save_strategy="no", seed=42)
    tr = CLIPPretrainer(m, args, rows, None)
    # the loop's pieces, timed separately with CUDA events over the same work the loop does per optimizer step
    tr._setup(args.max_steps, 0)
    batches = [CLIPCollator()(rows[i * a.n:(i + 1) * a.n]) for i in range(a.acc)]
    batches = [{k: v.to(dev) for k, v in b.items()} for b in batches]
    from pigeon_b200.ops import grad_norm_clip
    ws = torch.empty(0, dtype=torch.uint8, device=dev)
    times = {"micro_steps": [], "allreduce": [], "norm_clip": [], "optimizer": []}
    torch.cuda.reset_peak_memory_stats()
    for it in range(a.warmup + a.steps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        ev[0].record()
        for b in batches:
            m.forward_train(b["input_ids"], b["pixel_values"], b["attention_mask"])
            m.backward()
        ev[1].record()
        if world > 1:
            torch.distributed.all_reduce(tr._flat)
        ev[2].record()
        scale = 1.0 / (a.acc * world)
        _, coef = grad_norm_clip(tr._flat, 1.0, scale, ws)
        ev[3].record()
        tr.optimizer.step(clip_coef=coef, grad_scale=scale)
        tr.lr_scheduler.step()
        ev[4].record()
        tr._flat.zero_()
        torch.cuda.synchronize()
        if it >= a.warmup:
            for k, (i, j) in zip(times, ((0, 1), (1, 2), (2, 3), (3, 4))):
                times[k].append(ev[i].elapsed_time(ev[j]))
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    flat_gb = tr._flat.numel() * 4 / 1e9
    if rank == 0:
        res = {k: round(statistics.median(v), 3) for k, v in times.items()}
        res.update(card=card(), world=world, pairs_per_micro_batch=a.n, acc=a.acc, parameters=n_params,
                   flat_gradient_gb=round(flat_gb, 3), peak_memory_gib=round(peak, 2), steps=a.steps,
                   # norm reads the gradient (4 B); the update reads p, g, m, v and writes p, m, v (28 B)
                   norm_gbps=round(tr._flat.numel() * 4 / (res["norm_clip"] * 1e6), 1),
                   optimizer_gbps=round(n_params * 28 / (res["optimizer"] * 1e6), 1))
        print(json.dumps(res), flush=True)
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
