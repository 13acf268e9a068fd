"""Generate tests/golden/clip_train.npz: the loss and every parameter gradient of one HF `CLIPModel` contrastive step
(`model(input_ids, pixel_values, attention_mask, return_loss=True).loss.backward()`, the installed `transformers`, eager
attention, fp32 autograd on the CPU), for the CLIPModel training step of pigeon_b200.  Needs no reference checkout and no GPU.

Weights, captions and pixels come from the seeded helpers of tools/make_clip_golden.py (only the inputs and the sampled
gradients are stored).  Two geometries:
  tiny  the tiny weights of clip.npz: 2-layer towers of width 256, 3 images x 3 captions, S = 12;
  mid   2-layer towers of width 256, 8 images x 8 captions, S = 77 with mixed caption lengths, so that the causal tiles of
        the attention backward cross a 64-row block.
Per parameter (HF name) `<geom>/norm/<name>` is the gradient's L2 norm and `<geom>/sub/<name>` every STRIDE-th element of the
flattened gradient (the train_tower_* layout).  For text_model.embeddings.token_embedding.weight only the rows of the ids
that occur are sampled: `<geom>/tok_ids` (sorted, unique), and the sub / norm of `grad[tok_ids]`.

    python tools/make_clip_train_golden.py
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

from make_clip_golden import GEOMETRIES as FORWARD_GEOMETRIES, captions, hf_clip, pixels  # noqa: E402
from pigeon_b200 import synthetic  # noqa: E402
from pigeon_b200.clip_text import TextDims  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "clip_train.npz")
STRIDE = 53
TOKEN = "text_model.embeddings.token_embedding.weight"

_tiny = FORWARD_GEOMETRIES["tiny"]
GEOMETRIES = {
    "tiny": dict(_tiny),
    "mid": dict(text=TextDims(vocab=1000, max_positions=77, hidden=256, heads=4, intermediate=512, layers=2),
                vision=_tiny["vision"], projection=256, n_images=8, lengths=[77, 5, 20, 41, 64, 66, 12, 70], seed=31,
                px_seed=32, ids_seed=33, std=0.05),
}


def geometry(name, g):
    td, vd = g["text"], g["vision"]
    sd = synthetic.random_clip_state_dict(td, vd, seed=g["seed"], std=g["std"], projection_dim=g["projection"])
    ids, mask = captions(g["lengths"], td.vocab, g["ids_seed"])
    assert ids.shape[0] == g["n_images"]
    px = pixels(g["n_images"], vd.image_size, g["px_seed"])
    m = hf_clip(td, vd, g["projection"], sd)
    o = m(input_ids=ids, attention_mask=mask, pixel_values=px, return_loss=True)
    o.loss.backward()
    tok_ids = torch.unique(ids)
    out = {"input_ids": ids.numpy(), "attention_mask": mask.numpy(), "loss": np.float64(o.loss.item()),
           "tok_ids": tok_ids.numpy()}
    for key, p in m.named_parameters():
        gr = p.grad.detach()
        if key == TOKEN:
            gr = gr[tok_ids]
        flat = gr.reshape(-1)
        out["norm/" + key] = np.float64(flat.double().norm().item())
        out["sub/" + key] = flat[::STRIDE].numpy().astype(np.float32)
    meta = dict(text=vars(td), vision=vars(vd), projection=g["projection"], seed=g["seed"], std=g["std"],
                px_seed=g["px_seed"], stride=STRIDE)
    out["meta"] = np.array(json.dumps(meta))
    return {f"{name}/{k}": v for k, v in out.items()}


def main():
    torch.manual_seed(0)
    arrays = {}
    for name, g in GEOMETRIES.items():
        arrays.update(geometry(name, g))
        print(name, "done", flush=True)
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
