"""fp32 restatement of HF `CLIPTextTransformer` and `CLIPModel.forward` (transformers 4.23.1 `models/clip/modeling_clip.py`,
the version the reference pins in env.yml:60) — test infrastructure, the checker of pigeon_b200.CLIPModel.  The image side
is oracle/vit.py.

  CLIPTextEmbeddings.forward: token_embedding(input_ids) + position_embedding(position_ids[:, :S]); no pre-LayerNorm
  CLIPTextTransformer.forward: _build_causal_attention_mask (finfo.min above the diagonal) + _expand_mask(attention_mask)
                               (finfo.min where the key's mask is 0), the same pre-LN CLIPEncoderLayer stack as the vision
                               tower, final_layer_norm, pooled_output = last_hidden_state[arange(n), input_ids.argmax(-1)]
  CLIPModel.get_image_features: visual_projection(post_layernorm(vision last_hidden_state[:, 0]))
  CLIPModel.get_text_features:  text_projection(pooled_output)
  CLIPModel.forward: embeds / norm, logits_per_text = text @ image.T * logit_scale.exp(), logits_per_image = .T,
                     clip_loss = (CE(logits_per_text, arange) + CE(logits_per_image, arange)) / 2
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import vit as ovit


def _text_sd(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    return {k[len("text_model."):] if k.startswith("text_model.") else k: v for k, v in sd.items()}


@torch.no_grad()
def text_forward(sd: Dict[str, torch.Tensor], input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None, *,
                 heads: int, layers: int, eps: float = 1e-5):
    """input_ids [n, S] -> (last_hidden_state [n, S, hidden] after final_layer_norm, pooled_output [n, hidden]), fp32."""
    sd = _text_sd(sd)
    n, S = input_ids.shape
    tok = sd["embeddings.token_embedding.weight"].float()
    pos = sd["embeddings.position_embedding.weight"].float()
    if S > pos.shape[0]:
        raise ValueError(f"sequence length {S} > max_position_embeddings {pos.shape[0]}")
    h = tok[input_ids] + pos[:S].unsqueeze(0)
    hidden = h.shape[-1]
    hd = hidden // heads
    neg = torch.finfo(torch.float32).min
    causal = torch.full((S, S), neg).triu(1)[None, None]                       # _build_causal_attention_mask
    if attention_mask is not None:                                             # _expand_mask
        pad = (1.0 - attention_mask.float())[:, None, None, :].expand(n, 1, S, S)
        pad = pad.masked_fill(pad.bool(), neg)
    else:
        pad = torch.zeros(n, 1, S, S)
    for i in range(layers):
        p = f"encoder.layers.{i}."
        r = h
        y = F.layer_norm(h, (hidden,), sd[p + "layer_norm1.weight"].float(), sd[p + "layer_norm1.bias"].float(), eps)
        q = F.linear(y, sd[p + "self_attn.q_proj.weight"].float(), sd[p + "self_attn.q_proj.bias"].float()) * hd ** -0.5
        k = F.linear(y, sd[p + "self_attn.k_proj.weight"].float(), sd[p + "self_attn.k_proj.bias"].float())
        v = F.linear(y, sd[p + "self_attn.v_proj.weight"].float(), sd[p + "self_attn.v_proj.bias"].float())
        q, k, v = (t.view(n, S, heads, hd).transpose(1, 2) for t in (q, k, v))
        w = q @ k.transpose(-1, -2)
        w = w + causal                                                          # CLIPAttention: causal mask, then padding
        w = w + pad
        o = (torch.softmax(w, dim=-1) @ v).transpose(1, 2).reshape(n, S, hidden)
        h = r + F.linear(o, sd[p + "self_attn.out_proj.weight"].float(), sd[p + "self_attn.out_proj.bias"].float())
        r = h
        y = F.layer_norm(h, (hidden,), sd[p + "layer_norm2.weight"].float(), sd[p + "layer_norm2.bias"].float(), eps)
        y = F.linear(y, sd[p + "mlp.fc1.weight"].float(), sd[p + "mlp.fc1.bias"].float())
        y = y * torch.sigmoid(1.702 * y)
        h = r + F.linear(y, sd[p + "mlp.fc2.weight"].float(), sd[p + "mlp.fc2.bias"].float())
    h = F.layer_norm(h, (hidden,), sd["final_layer_norm.weight"].float(), sd["final_layer_norm.bias"].float(), eps)
    pooled = h[torch.arange(n), input_ids.to(torch.int64).argmax(dim=-1)]
    return h, pooled


@torch.no_grad()
def image_features(sd, pixel_values, *, patch: int, heads: int, layers: int, eps: float = 1e-5):
    hs = ovit.vit_last_hidden_state(sd, pixel_values, patch=patch, heads=heads, layers=layers, eps=eps)
    hidden = hs.shape[-1]
    cls = F.layer_norm(hs[:, 0], (hidden,), sd["vision_model.post_layernorm.weight"].float(),
                       sd["vision_model.post_layernorm.bias"].float(), eps)
    return cls @ sd["visual_projection.weight"].float().T


@torch.no_grad()
def clip_forward(sd, input_ids, pixel_values, attention_mask=None, *, text_heads: int, text_layers: int, patch: int,
                 vision_heads: int, vision_layers: int, eps: float = 1e-5, return_loss: bool = False):
    """-> dict(text_embeds, image_embeds (normalised), logits_per_text, logits_per_image, loss (or None),
    last_hidden_state (text), text_features, image_features (projected, not normalised))."""
    lhs, pooled = text_forward(sd, input_ids, attention_mask, heads=text_heads, layers=text_layers, eps=eps)
    tf = pooled @ sd["text_projection.weight"].float().T
    imf = image_features(sd, pixel_values, patch=patch, heads=vision_heads, layers=vision_layers, eps=eps)
    te = tf / tf.norm(p=2, dim=-1, keepdim=True)
    ie = imf / imf.norm(p=2, dim=-1, keepdim=True)
    lpt = te @ ie.T * sd["logit_scale"].float().exp()
    lpi = lpt.T
    loss = None
    if return_loss:
        if lpt.shape[0] != lpt.shape[1]:
            raise ValueError("the contrastive loss needs as many images as captions")
        t = torch.arange(lpt.shape[0])
        loss = (F.cross_entropy(lpt, t) + F.cross_entropy(lpi, t)) / 2
    return dict(text_embeds=te, image_embeds=ie, logits_per_text=lpt, logits_per_image=lpi, loss=loss,
                last_hidden_state=lhs, text_features=tf, image_features=imf)
