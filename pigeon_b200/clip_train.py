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
from .vit_train import (carve_saved, flat_grads, grow_aligned, layer_grad_shapes, layers_bwd, put_grad, put_layer_grads,
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
        saved = _lib.TextSaved()
        carve_saved(self, saved, n, S, [("x_final", n * S * self.dims.hidden * 4)])
        self._saved, self._shape = saved, (n, S)

    def _pending_grads(self) -> Dict[str, torch.Tensor]:
        if self._pending is None:
            d = self.dims
            shapes = [("token_emb", (d.vocab, d.hidden)), ("pos_emb", (d.max_positions, d.hidden)),
                      ("final_ln_g", (d.hidden,)), ("final_ln_b", (d.hidden,))]
            for l in range(d.layers):
                shapes += layer_grad_shapes(l, d.hidden, d.intermediate)
            _, self._pending = flat_grads(shapes, next(self.tower.parameters()).device)
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
        grads = _lib.TextGrads(ptr(g["token_emb"]), ptr(g["pos_emb"]), ptr(g["final_ln_g"]), ptr(g["final_ln_b"]),
                               layers_bwd(self._wt, g, [True] * d.layers))
        ws = grow_aligned(self, "_ws", int(self._lib.pg_text_backward_workspace_bytes(eng._handle, n, S)), d_pooled.device)
        check(self._lib.pg_text_backward(eng._handle, C.byref(self._saved), ptr(ids), ptr(mask), ptr(d_pooled), n, S,
                                         C.byref(grads), ptr(ws), ws.numel(), current_stream_ptr()), "pg_text_backward")

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
