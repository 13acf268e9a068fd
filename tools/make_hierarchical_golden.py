"""Generate tests/golden/hierarchical.npz from the UNMODIFIED reference SuperGuessr(panorama=True, hierarchical=True)
(behind oracle/reference_shim.py; the hierarchical path needs no CUDA, so it runs on the CPU).

    python tools/make_hierarchical_golden.py

Inputs are never stored: embeddings, labels and weights are regenerated from the recorded seeds (torch CPU generators,
tests/hierarchical_oracle.py), and of a gradient or parameter with more than 4096 elements only every 37th is kept
(`hierarchical_oracle.sample`), so the file stays small.  Cases:
  eval_a   E = 1024, N = 9, index labels                       eval_b  E = 256, N = 37, smoothed labels, multi_task
  eval_c   E = 256, N = 1000 (the positional-encoding limit)   serve   E = 256, N = 37, serving=True, multi_task
  grad     E = 128, N = 24, smoothed labels, multi_task: d loss / d every trainable parameter and d embedding
  adam     E = 128, N = 24, index labels: 3 torch.optim.AdamW steps (train_eval_loop.py:187 defaults, lr 1e-3)
  state    E = 32: the seeded initial state_dict (construction order decides which random draws each module gets)
  tower    a 1-layer 336 px tower (hidden 256) under the hierarchical head, every parameter trainable: loss and gradients
The eval cases take the first seed for which every sample's top-1 / top-2 probability margin exceeds 1e-5; the margins
are stored.  Training cases set both dropouts to p = 0 on the instance (pos_encoder.dropout.p, self_attn.dropout).
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

import numpy as np
import pandas as pd
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import reference_shim as rs  # noqa: E402
from pigeon_b200 import synthetic  # noqa: E402
from pigeon_b200.vit_engine import VitDims  # noqa: E402
import hierarchical_oracle as ho  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "hierarchical.npz")
C = 1000
MARGIN = 1e-5
EVAL_CASES = {"eval_a": dict(E=1024, N=9, smooth=False, mt=False, serving=False),
              "eval_b": dict(E=256, N=37, smooth=True, mt=True, serving=False),
              "eval_c": dict(E=256, N=1000, smooth=False, mt=False, serving=False),
              "serve": dict(E=256, N=37, smooth=False, mt=True, serving=True)}


def reference_model(tmp, seed, E, base_model=None, **kw):
    from models.super_guessr import SuperGuessr
    with rs.chdir(tmp):
        torch.manual_seed(seed)
        sg = SuperGuessr(base_model, panorama=True, hierarchical=True, embed_dim=E, num_candidates=5, **kw)
    with torch.no_grad():
        for k, v in ho.synthetic_params(sg.hidden_size, C, seed).items():
            sg.state_dict()[k].copy_(v)
    return sg


def no_dropout(sg):
    sg.pos_encoder.dropout.p = 0.0
    sg.self_attn.dropout = 0.0


def eval_case(tmp, name, E, N, smooth, mt, serving):
    for seed in range(100, 200):
        sg = reference_model(tmp, seed, E, should_smooth_labels=smooth, multi_task=mt, serving=serving).eval()
        emb = ho.embeddings(N, E, seed)
        labels, labels_clf, lmt, lcl, lmo = ho.labels(N, seed)
        kw = dict(labels_multi_task=lmt, labels_climate=lcl, labels_month=lmo) if mt else {}
        with torch.no_grad():
            o = sg(embedding=emb, labels=labels, labels_clf=labels_clf, **kw)
        topk = o[1] if serving else o.top5_geocells
        margin = (topk.values[:, 0] - topk.values[:, 1]).numpy()
        if margin.min() > MARGIN:
            break
    else:
        raise RuntimeError(f"{name}: no seed clears the margin")
    out = {f"{name}_seed": np.asarray(seed), f"{name}_margin": margin, f"{name}_topk_val": topk.values.numpy(),
           f"{name}_topk_idx": topk.indices.numpy()}
    if serving:
        out.update({f"{name}_preds_LLH": o[0].numpy(), f"{name}_preds_mt": o[2].numpy()})
        assert torch.equal(o[3], emb)
        return out
    out.update({f"{name}_preds_LLH": o.preds_LLH.numpy(), f"{name}_preds_geocell": o.preds_geocell.numpy(),
                f"{name}_loss": o.loss.detach().numpy(), f"{name}_loss_clf": o.loss_clf.detach().numpy()})
    if mt:
        out.update({f"{name}_preds_mt": o.preds_mt.numpy(), f"{name}_preds_climate": o.preds_climate.numpy(),
                    f"{name}_preds_month": o.preds_month.numpy()})
    assert torch.equal(o.embedding, emb)
    return out


def grad_case(tmp, seed=300, E=128, N=24):
    sg = reference_model(tmp, seed, E, should_smooth_labels=True, multi_task=True).train()
    no_dropout(sg)
    emb = ho.embeddings(N, E, seed).requires_grad_(True)
    labels, labels_clf, lmt, lcl, lmo = ho.labels(N, seed)
    o = sg(embedding=emb, labels=labels, labels_clf=labels_clf, labels_multi_task=lmt, labels_climate=lcl,
           labels_month=lmo)
    o.loss.backward()
    out = {"grad_seed": np.asarray(seed), "grad_loss": o.loss.detach().numpy(),
           "grad/embedding": ho.sample(emb.grad).numpy().copy()}
    for k, p in sg.named_parameters():
        if p.grad is not None:
            out["grad/" + k] = ho.sample(p.grad).numpy().copy()
    return out


def adam_case(tmp, seed=400, E=128, N=24, steps=3, lr=1e-3):
    sg = reference_model(tmp, seed, E).train()
    no_dropout(sg)
    opt = torch.optim.AdamW(sg.parameters(), lr=lr)
    losses = []
    for i in range(steps):
        labels, labels_clf, *_ = ho.labels(N, seed + i)
        o = sg(embedding=ho.embeddings(N, E, seed + i), labels=labels, labels_clf=labels_clf)
        o.loss.backward()
        opt.step()
        opt.zero_grad()
        losses.append(float(o.loss.detach()))
    out = {"adam_seed": np.asarray(seed), "adam_steps": np.asarray(steps), "adam_lr": np.asarray(lr),
           "adam_losses": np.asarray(losses)}
    for k in ho.ATTN_KEYS + ("cell_layer.weight", "cell_layer.bias"):
        out["adam/" + k] = ho.sample(sg.state_dict()[k]).numpy().copy()
    return out


def state_case(tmp, seed=5, E=32):
    from models.super_guessr import SuperGuessr
    with rs.chdir(tmp):
        torch.manual_seed(seed)
        sg = SuperGuessr(None, panorama=True, hierarchical=True, embed_dim=E, multi_task=True)
    out = {"state_seed": np.asarray(seed), "state_E": np.asarray(E),
           "state_shapes": json.dumps({k: list(v.shape) for k, v in sg.state_dict().items()})}
    for k, v in sg.state_dict().items():
        out["state/" + k] = ho.sample(v).numpy().copy()
    return out


def tower_case(tmp, seed=600, N=2):
    from oracle.make_golden import hf_model
    dims = VitDims(image_size=336, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    sd = synthetic.random_vit_state_dict(dims, seed=seed, std=0.05)
    hf = hf_model(dims, sd)
    sg = reference_model(tmp, seed, dims.hidden, base_model=hf.base_model, should_smooth_labels=True).train()
    no_dropout(sg)
    for p in sg.parameters():
        p.requires_grad_(p.dtype == torch.float32)
    sg.lla_geocells.requires_grad_(False)
    sg.pos_encoder.pos_encoding.requires_grad_(False)
    px = torch.randn(N, 12, 336, 336, generator=torch.Generator().manual_seed(seed + 1))
    labels, labels_clf, *_ = ho.labels(N, seed)
    o = sg(pixel_values=px, labels=labels, labels_clf=labels_clf)
    o.loss.backward()
    out = {"tower_meta": json.dumps(dict(dims=dims.__dict__, seed=seed, std=0.05, N=N)),
           "tower_loss": o.loss.detach().numpy()}
    for k, p in sg.named_parameters():
        if p.grad is not None:
            g = p.grad.detach().reshape(-1).double()
            out["tower_norm/" + k] = np.asarray(float(g.norm()))
            out["tower_sub/" + k] = ho.sample(g).float().numpy()
    return out


def main():
    tmp = tempfile.mkdtemp(prefix="pigeon_golden_")
    os.makedirs(os.path.join(tmp, "data"))
    cells = synthetic.synthetic_geocells(C, 0)
    pd.DataFrame({"lng": cells[:, 0], "lat": cells[:, 1]}).to_csv(os.path.join(tmp, "data", "geocells_2203.csv"), index=False)
    rs.install()
    torch.set_num_threads(os.cpu_count())
    out = {}
    for name, kw in EVAL_CASES.items():
        out.update(eval_case(tmp, name, **kw))
    out.update(grad_case(tmp))
    out.update(adam_case(tmp))
    out.update(state_case(tmp))
    out.update(tower_case(tmp))
    with rs.chdir(tmp):
        from models.super_guessr import SuperGuessr
        out["centroids"] = SuperGuessr(None, panorama=True, embed_dim=32).lla_geocells.detach().numpy().copy()
    out["meta"] = json.dumps(dict(C=C, margin=MARGIN, cases=EVAL_CASES))
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
