"""Generate tests/golden/clip.npz: HF `CLIPModel` (the installed `transformers`, eager attention) on seeded weights and
inputs, for the CLIP text tower / CLIPModel forward of pigeon_b200.  Needs no reference checkout and no GPU.

Weights are `pigeon_b200.synthetic.random_clip_state_dict(text_dims, vision_dims, seed, std)` and pixels
`torch.randn(..., generator=manual_seed(px_seed))`: both are regenerated from the stored seeds, only the small inputs and
outputs are stored.  Two geometries:
  tiny  2-layer towers of width 256, 3 images x 3 captions (S = 12, right-padded), with the loss;
  large the real text tower (12 x 768, 77 positions, vocab 49408) and ViT-L/14-336, 2 images x 4 captions of lengths
        77, 3, 20, 41 (right-padded with attention_mask), plus the loss of the first two captions.

Captions are built as CLIP's tokenizer builds them: BOS (vocab - 2) first, EOS (vocab - 1) last, padded with EOS — so
the first-EOS pooling of transformers >= 4.31 and the `input_ids.argmax(-1)` pooling of 4.23.1 pick the same row.

    python tools/make_clip_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pigeon_b200 import synthetic  # noqa: E402
from pigeon_b200.clip_text import TextDims  # noqa: E402
from pigeon_b200.vit_engine import VitDims  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "clip.npz")

GEOMETRIES = {
    "tiny": dict(text=TextDims(vocab=1000, max_positions=16, hidden=256, heads=4, intermediate=512, layers=2),
                 vision=VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=2),
                 projection=256, n_images=3, lengths=[12, 5, 9], seed=11, px_seed=12, ids_seed=13, std=0.05),
    "large": dict(text=TextDims(), vision=VitDims(), projection=768, n_images=2, lengths=[77, 3, 20, 41], seed=21,
                  px_seed=22, ids_seed=23, std=0.02),
}
SAMPLED_POSITIONS = 3   # last_hidden_state rows kept per caption in the large geometry: first, middle, last token


def captions(lengths, vocab, seed):
    """input_ids / attention_mask [n, max(lengths)] i64 the way CLIPProcessor(text=..., padding=True) lays them out."""
    g = torch.Generator().manual_seed(seed)
    S = max(lengths)
    ids = torch.full((len(lengths), S), vocab - 1, dtype=torch.int64)
    mask = torch.zeros((len(lengths), S), dtype=torch.int64)
    for b, L in enumerate(lengths):
        ids[b, 0] = vocab - 2
        if L > 2:
            ids[b, 1:L - 1] = torch.randint(0, vocab - 2, (L - 2,), generator=g)
        mask[b, :L] = 1
    return ids, mask


def pixels(n, size, seed):
    return torch.randn(n, 3, size, size, generator=torch.Generator().manual_seed(seed))


def hf_clip(td: TextDims, vd: VitDims, projection: int, sd):
    from transformers import CLIPConfig, CLIPModel
    cfg = CLIPConfig(
        text_config=dict(vocab_size=td.vocab, hidden_size=td.hidden, intermediate_size=td.intermediate,
                         num_hidden_layers=td.layers, num_attention_heads=td.heads, max_position_embeddings=td.max_positions,
                         hidden_act="quick_gelu", layer_norm_eps=td.ln_eps, bos_token_id=td.vocab - 2,
                         eos_token_id=td.vocab - 1, pad_token_id=1),
        vision_config=dict(hidden_size=vd.hidden, intermediate_size=vd.intermediate, num_hidden_layers=vd.layers,
                           num_attention_heads=vd.heads, image_size=vd.image_size, patch_size=vd.patch_size,
                           hidden_act="quick_gelu", layer_norm_eps=vd.ln_eps),
        projection_dim=projection)
    cfg._attn_implementation = "eager"
    cfg.text_config._attn_implementation = "eager"
    cfg.vision_config._attn_implementation = "eager"
    m = CLIPModel(cfg).eval()
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return m


def geometry(name, g):
    from transformers.models.clip.modeling_clip import clip_loss
    td, vd = g["text"], g["vision"]
    sd = synthetic.random_clip_state_dict(td, vd, seed=g["seed"], std=g["std"], projection_dim=g["projection"])
    ids, mask = captions(g["lengths"], td.vocab, g["ids_seed"])
    px = pixels(g["n_images"], vd.image_size, g["px_seed"])
    m = hf_clip(td, vd, g["projection"], sd)
    with torch.no_grad():
        o = m(input_ids=ids, attention_mask=mask, pixel_values=px, return_loss=ids.shape[0] == px.shape[0])
        lhs = o.text_model_output.last_hidden_state
        n_loss = min(ids.shape[0], px.shape[0])
        loss = clip_loss(o.logits_per_text[:n_loss, :n_loss])
    out = {"input_ids": ids.numpy(), "attention_mask": mask.numpy(), "text_embeds": o.text_embeds.numpy(),
           "image_embeds": o.image_embeds.numpy(), "logits_per_image": o.logits_per_image.numpy(),
           "logits_per_text": o.logits_per_text.numpy(), "loss": np.float32(loss), "n_loss": np.int64(n_loss),
           "config": np.array([g["seed"], g["px_seed"], g["projection"]], np.int64), "std": np.float32(g["std"])}
    if name == "tiny":
        out["last_hidden_state"] = lhs.numpy()
    else:
        pos = np.array([[0, (L - 1) // 2, L - 1] for L in g["lengths"]], np.int64)
        out["lhs_positions"] = pos
        out["last_hidden_state_rows"] = np.stack([lhs[b, pos[b]].numpy() for b in range(len(g["lengths"]))])
    return {f"{name}_{k}": v for k, v in out.items()}


def main():
    arrays = {}
    for name, g in GEOMETRIES.items():
        arrays.update(geometry(name, g))
        print(name, "done", flush=True)
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
