"""clip_loss of HF `CLIPModel.forward` (transformers 4.23.1) with autograd enabled, built from the fp32 restatements in
tests/clip_oracle.py (text side) and oracle/vit.py (image side) — the checker of the CLIPModel training step at the real
geometry.  Those functions are decorated with torch.no_grad(); their undecorated bodies (`__wrapped__`) are called here.

The text side runs on the CPU (clip_oracle.text_forward builds its masks there), the image side and the logits on the device
of pixel_values; autograd carries the pooled rows across.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import clip_oracle
from oracle import vit as ovit


def clip_loss_autograd(sd, input_ids, pixel_values, attention_mask=None, *, text_heads: int, text_layers: int, patch: int,
                       vision_heads: int, vision_layers: int, eps: float = 1e-5):
    """sd: HF-named fp32 leaves with requires_grad set (`text_model.*` on the CPU, every other tensor on the device of
    pixel_values); input_ids / attention_mask on the CPU -> clip_loss (a graph node: call .backward())."""
    with torch.enable_grad():
        _, pooled = clip_oracle.text_forward.__wrapped__(sd, input_ids, attention_mask, heads=text_heads, layers=text_layers,
                                                         eps=eps)
        tf = pooled.to(pixel_values.device) @ sd["text_projection.weight"].T
        hs = ovit.vit_last_hidden_state.__wrapped__(sd, pixel_values, patch=patch, heads=vision_heads, layers=vision_layers,
                                                    eps=eps)
        cls = F.layer_norm(hs[:, 0], (hs.shape[-1],), sd["vision_model.post_layernorm.weight"],
                           sd["vision_model.post_layernorm.bias"], eps)
        imf = cls @ sd["visual_projection.weight"].T
        te = tf / tf.norm(p=2, dim=-1, keepdim=True)
        ie = imf / imf.norm(p=2, dim=-1, keepdim=True)
        lpt = te @ ie.T * sd["logit_scale"].exp()
        t = torch.arange(lpt.shape[0], device=lpt.device)
        return (F.cross_entropy(lpt, t) + F.cross_entropy(lpt.T, t)) / 2
