"""Text-tower half of the CLIPModel contrastive training step (host side of pg_text_forward_train / pg_text_backward).

What autograd runs through HF `CLIPTextTransformer` (transformers 4.23.1 modeling_clip.py) for the `loss.backward()` of the HF
`Trainer` that reference training/train_modes.py:30-64 drives: the training forward keeps its activations in one arena (the
vision tower's per-layer layout, rows = n * S), the backward runs as hand-written kernels and leaves fp32 gradients under the
HF parameter names.  Every text parameter trains, as in the reference (nothing is frozen in `pretrain`).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib
from ._lib import PigeonB200Error, check, current_stream_ptr, load, ptr
from .clip_text import admissible_keys
from .vit_train import (LAYER_GRADS, _aligned_empty, _align, layer_grad_shapes, put_grad, put_layer_grads,
                        transpose_layers)


class TextTrainer:
    """Owns the activation arena, the transposed bf16 weights and the fused gradient buffer of one CLIPTextTower."""

    def __init__(self, tower):
        self.tower = tower
        self.dims = tower.dims
        self._lib = load()
        self._arena: Optional[torch.Tensor] = None
        self._ws: Optional[torch.Tensor] = None
        self._saved = None
        self._shape = None
        self._inputs = None
        self._wt = [None] * self.dims.layers
        self._wt_version: dict = {}
        self._pending: Optional[Dict[str, torch.Tensor]] = None

    def check_trainable(self) -> None:
        frozen = [n for n, p in self.tower.named_parameters() if not p.requires_grad]
        if frozen:
            raise NotImplementedError(f"the CLIPModel training step trains every text-tower parameter (as the reference's "
                                      f"pretraining does); frozen: {frozen[:3]}{' ...' if len(frozen) > 3 else ''}")

    def _build_saved(self, n: int, S: int):
        d = self.dims
        rows = n * S
        H, I = d.hidden, d.intermediate
        per_layer = [("x0", rows * H * 4), ("xn1", rows * H * 2), ("qkv", rows * 3 * H * 2), ("lse2", n * d.heads * S * 4),
                     ("ao", rows * H * 2), ("x1", rows * H * 4), ("xn2", rows * H * 2), ("u", rows * I * 2),
                     ("h", rows * I * 2)]
        total = _align(rows * H * 4) + d.layers * sum(_align(b) for _, b in per_layer)
        dev = next(self.tower.parameters()).device
        if self._arena is None or self._arena.numel() < total:
            self._arena = None
            self._arena = _aligned_empty(total, dev)
        base, off = self._arena.data_ptr(), 0
        saved = _lib.TextSaved()
        saved.x_final = base
        off += _align(rows * H * 4)
        layers = (_lib.VitSavedLayer * d.layers)()
        for l in range(d.layers):
            for name, b in per_layer:
                setattr(layers[l], name, base + off)
                off += _align(b)
        saved.layers_host = layers
        self._saved, self._saved_layers, self._shape = saved, layers, (n, S)

    def _pending_grads(self) -> Dict[str, torch.Tensor]:
        if self._pending is not None:
            return self._pending
        d = self.dims
        dev = next(self.tower.parameters()).device
        shapes = [("token_emb", (d.vocab, d.hidden)), ("pos_emb", (d.max_positions, d.hidden)),
                  ("final_ln_g", (d.hidden,)), ("final_ln_b", (d.hidden,))]
        for l in range(d.layers):
            shapes += layer_grad_shapes(l, d.hidden, d.intermediate)
        offs, total = [], 0
        for _, shp in shapes:
            offs.append(total)
            total += (int(torch.Size(shp).numel()) + 3) // 4 * 4
        flat = torch.zeros(total, dtype=torch.float32, device=dev)
        self._pending = {name: flat[o:o + int(torch.Size(shp).numel())].view(shp) for (name, shp), o in zip(shapes, offs)}
        return self._pending

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor]) -> torch.Tensor:
        """input_ids [n, S] and attention_mask [n, S] or None (CUDA) -> pooled output f32 [n, hidden]; the activations stay
        in the arena until the next forward."""
        self.check_trainable()
        d = self.dims
        n, S = input_ids.shape
        ids = input_ids.to(dtype=torch.int64).contiguous()
        mask = None if attention_mask is None else admissible_keys(attention_mask)
        self._build_saved(n, S)
        self._inputs = (ids, mask)
        eng = self.tower.engine()
        pooled = torch.empty((n, d.hidden), dtype=torch.float32, device=ids.device)
        check(self._lib.pg_text_forward_train(eng._handle, ptr(ids), ptr(mask), n, S, C.byref(self._saved), ptr(pooled),
                                              current_stream_ptr()), "pg_text_forward_train")
        return pooled

    @torch.no_grad()
    def backward(self, d_pooled: torch.Tensor) -> None:
        """d_pooled f32 [n, hidden] for the captions of the last forward; gradients accumulate in the pending buffer."""
        d = self.dims
        if self._saved is None or tuple(d_pooled.shape) != (self._shape[0], d.hidden):
            raise PigeonB200Error("backward() must follow forward() with one gradient row per caption")
        n, S = self._shape
        ids, mask = self._inputs
        d_pooled = d_pooled.to(torch.float32).contiguous()
        eng = self.tower.engine()
        transpose_layers(self.tower.text_model.encoder.layers, self.tower._group_versions(), self._wt, self._wt_version)
        g = self._pending_grads()
        lb = (_lib.VitLayerBwd * d.layers)()
        for l in range(d.layers):
            for k, t in self._wt[l].items():
                setattr(lb[l], k, t.data_ptr())
            for k in LAYER_GRADS:
                setattr(lb[l], "d_" + k, g[f"{l}.{k}"].data_ptr())
        grads = _lib.TextGrads(ptr(g["token_emb"]), ptr(g["pos_emb"]), ptr(g["final_ln_g"]), ptr(g["final_ln_b"]), lb)
        need = int(self._lib.pg_text_backward_workspace_bytes(eng._handle, n, S))
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = _aligned_empty(need, d_pooled.device)
        check(self._lib.pg_text_backward(eng._handle, C.byref(self._saved), ptr(ids), ptr(mask), ptr(d_pooled), n, S,
                                         C.byref(grads), ptr(self._ws), self._ws.numel(), current_stream_ptr()),
              "pg_text_backward")

    @torch.no_grad()
    def finalize(self) -> None:
        """Pending fused gradients -> `param.grad` (accumulating) under the HF names."""
        if self._pending is None:
            return
        g, tm = self._pending, self.tower.text_model
        put_grad(tm.embeddings.token_embedding.weight, g["token_emb"])
        put_grad(tm.embeddings.position_embedding.weight, g["pos_emb"])
        put_grad(tm.final_layer_norm.weight, g["final_ln_g"])
        put_grad(tm.final_layer_norm.bias, g["final_ln_b"])
        for l, L in enumerate(tm.encoder.layers):
            put_layer_grads(L, g, l, self.dims.hidden)
        self._pending = None
