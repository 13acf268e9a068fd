"""Generate tests/golden/clip_pretrain.npz: six optimizer steps of the HF Trainer (transformers 4.23.1 loop, restated in
tests/clip_pretrain_oracle.py) around HF `CLIPModel` fp32 autograd on the CPU, for `pigeon_b200.pretrain.CLIPPretrainer`.
Needs no reference checkout and no GPU.

Geometry: the `mid` towers of clip_train.npz (2-layer text and vision towers of width 256, captions up to S = 77), 4 pairs
per micro-batch, 7 micro-batches per epoch, gradient accumulation 2 and 2 epochs: 3 updates per epoch, T = 6, W = 2, and
the seventh micro-batch of epoch 0 carries into the first update of epoch 1.  Weights come from
`synthetic.random_clip_state_dict(seed)`, rows from `clip_pretrain_oracle.golden_rows(seed)`; only the results are stored:
  log/<key>         per update: loss, learning_rate, grad_norm, epoch (6 entries); eval/loss at every eval_steps
  sub/<k>/<name>    every STRIDE-th element of each parameter after update k (k = 1 and 6), norm/<k>/<name> its L2 norm
  meta              the settings (json)

    python tools/make_clip_pretrain_golden.py
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import clip_pretrain_oracle as O  # noqa: E402
from make_clip_golden import hf_clip  # noqa: E402
from make_clip_train_golden import GEOMETRIES  # noqa: E402
from pigeon_b200 import synthetic  # noqa: E402
from pigeon_b200.pretrain import CLIPCollator  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "clip_pretrain.npz")
STRIDE = 53
SNAPSHOTS = (1, 6)
SETTINGS = dict(batch=4, eval_batch=4, acc=2, epochs=2, lr=2e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.1,
                max_grad_norm=4.6, warmup_ratio=0.2, eval_steps=2, seed=42)
DATA = dict(n_train=28, n_eval=8, train_seed=51, eval_seed=52, weight_seed=31, std=0.05)


def setup():
    g = GEOMETRIES["mid"]
    td, vd, P = g["text"], g["vision"], g["projection"]
    sd = synthetic.random_clip_state_dict(td, vd, seed=DATA["weight_seed"], std=DATA["std"], projection_dim=P)
    train_rows = O.golden_rows(DATA["n_train"], vd.image_size, td.vocab, td.max_positions, DATA["train_seed"])
    eval_rows = O.golden_rows(DATA["n_eval"], vd.image_size, td.vocab, td.max_positions, DATA["eval_seed"])
    return td, vd, P, sd, train_rows, eval_rows, CLIPCollator(pad_token_id=td.vocab - 1)


def run():
    td, vd, P, sd, train_rows, eval_rows, collate = setup()
    torch.manual_seed(0)
    m = hf_clip(td, vd, P, sd)
    snaps = {}

    def on_step(k):
        if k in SNAPSHOTS:
            snaps[k] = {n: p.detach().clone() for n, p in m.named_parameters()}

    log = O.train(m, train_rows, eval_rows, collate, on_step=on_step, **SETTINGS)
    return log, snaps


def main():
    log, snaps = run()
    steps = [e for e in log if "loss" in e]
    evals = [e for e in log if "eval_loss" in e]
    norms = [e["grad_norm"] for e in steps]
    print("grad norms", norms, "max_grad_norm", SETTINGS["max_grad_norm"])
    assert len(steps) == 6, len(steps)
    assert any(n > SETTINGS["max_grad_norm"] for n in norms) and any(n < SETTINGS["max_grad_norm"] for n in norms), \
        "max_grad_norm must clip some updates and not others"
    out = {f"log/{k}": np.array([e[k] for e in steps], np.float64) for k in ("loss", "learning_rate", "grad_norm", "epoch")}
    out["eval/loss"] = np.array([e["eval_loss"] for e in evals], np.float64)
    out["eval/step"] = np.array([e["step"] for e in evals], np.int64)
    for k, ps in snaps.items():
        for n, p in ps.items():
            flat = p.reshape(-1)
            out[f"sub/{k}/{n}"] = flat[::STRIDE].numpy().astype(np.float32)
            out[f"norm/{k}/{n}"] = np.float64(flat.double().norm().item())
    out["meta"] = np.array(json.dumps(dict(settings=SETTINGS, data=DATA, stride=STRIDE, snapshots=SNAPSHOTS)))
    np.savez_compressed(OUT, **out)
    print({k: v.tolist() for k, v in out.items() if k.startswith(("log/", "eval/"))})
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
