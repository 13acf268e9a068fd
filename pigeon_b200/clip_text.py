"""CLIP text tower on the GPU: HF `CLIPTextModel` / `CLIPTextTransformer` (transformers 4.23.1 modeling_clip.py), the text
half of the `CLIPModel` that reference training/train_modes.py:30-64 pretrains into StreetCLIP.

    TextDims        geometry (openai/clip-vit-large-patch14-336: 12 layers of 768, 12 heads, MLP 3072, 77 positions)
    TextEngine      packs HF-named weights into the kernel layouts, holds the C handle and runs `pg_text_forward`
    CLIPTextTower   nn.Module with HF `CLIPTextModel` parameter names; `tower(input_ids, attention_mask)` ->
                    `.last_hidden_state` (after final_layer_norm), `.pooler_output` (row of the largest input id)

Pinned semantics (4.23.1): embeddings = token_embedding[ids] + position_embedding[0..S-1], no pre-LayerNorm; causal
attention plus the padding mask; final_layer_norm; pooled row = first position of the row's largest input id
(`input_ids.argmax(-1)`, the EOS token 49407 for CLIP's tokenizer).  1 <= S <= max_position_embeddings.
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace
from typing import Dict, Optional

import torch
from torch import Tensor, nn
from torch.nn.parameter import Parameter

from . import _lib
from ._lib import PigeonB200Error, check, current_stream_ptr, ptr
from .encoder import EncoderEngine, EncoderTower, Holder, Pack, encoder_holder, norm


@dataclass
class TextDims:
    vocab: int = 49408
    max_positions: int = 77
    hidden: int = 768
    heads: int = 12
    intermediate: int = 3072
    layers: int = 12
    ln_eps: float = 1e-5

    @classmethod
    def from_hf_config(cls, cfg) -> "TextDims":
        return cls(vocab=cfg.vocab_size, max_positions=cfg.max_position_embeddings, hidden=cfg.hidden_size,
                   heads=cfg.num_attention_heads, intermediate=cfg.intermediate_size, layers=cfg.num_hidden_layers,
                   ln_eps=float(cfg.layer_norm_eps))


def admissible_keys(attention_mask: Tensor) -> Tensor:
    """attention_mask [n, S] of any dtype -> the kernels' 0/1 int64 mask.  HF 4.23.1's `_expand_mask` adds finfo.min
    wherever `1 - mask` is nonzero, so a key is attended only where its mask is exactly 1 (2, -1 or 1.5 exclude it)."""
    return (attention_mask == 1).to(torch.int64).contiguous()


def check_sequence_length(S: int, max_positions: int) -> None:
    """HF CLIPTextEmbeddings rejects sequences longer than the position table (the message of transformers 4.23.1+)."""
    if S > max_positions:
        raise ValueError(f"Sequence length must be less than max_position_embeddings (got `sequence length`: {S} and "
                         f"max_position_embeddings: {max_positions})")
    if S < 1:
        raise ValueError("input_ids must hold at least one token per caption")


class TextEngine(EncoderEngine):
    """H100 execution engine of HF CLIPTextTransformer.forward (pooled output, optionally last_hidden_state)."""
    PREFIXES = ("text_model.",)   # keys start at 'embeddings.' / 'encoder.' / 'final_layer_norm.'
    CREATE, DESTROY, WORKSPACE = "pg_text_create", "pg_text_destroy", "pg_text_workspace_bytes"

    def __init__(self, state_dict: Dict[str, Tensor], dims: TextDims, device: torch.device | str = "cuda",
                 max_texts_per_pass: int = 256):
        self.max_texts_per_pass = int(max_texts_per_pass)
        super().__init__(state_dict, dims, device)

    def _pack_embeddings(self, sd: Dict[str, Tensor], pack: Pack) -> tuple:
        """The "embeddings" group: token / position tables and final_layer_norm."""
        d = self.dims
        tok = pack.f32(sd["embeddings.token_embedding.weight"])
        pos = pack.f32(sd["embeddings.position_embedding.weight"])
        if tok.shape != (d.vocab, d.hidden) or pos.shape != (d.max_positions, d.hidden):
            raise PigeonB200Error(f"token_embedding {tuple(tok.shape)} / position_embedding {tuple(pos.shape)} do not "
                                  f"match ({d.vocab}, {d.hidden}) / ({d.max_positions}, {d.hidden})")
        return ptr(tok), ptr(pos), ptr(pack.f32(sd["final_layer_norm.weight"])), ptr(pack.f32(sd["final_layer_norm.bias"]))

    def _structs(self):
        d = self.dims
        cfg = _lib.TextConfig(d.vocab, d.max_positions, d.hidden, d.heads, d.intermediate, d.layers, d.ln_eps)
        return cfg, _lib.TextWeights(self._top[0], self._top[1], self._layers, self._top[2], self._top[3])

    @torch.no_grad()
    def forward(self, input_ids: Tensor, attention_mask: Optional[Tensor] = None, return_hidden: bool = False):
        """input_ids [n, S] (integer), attention_mask [n, S] or None (all ones) -> pooled [n, hidden] fp32
        (and last_hidden_state [n, S, hidden] fp32 when `return_hidden`)."""
        d = self.dims
        if input_ids.dim() != 2:
            raise ValueError(f"input_ids must be [batch, sequence], got {tuple(input_ids.shape)}")
        n, S = input_ids.shape
        check_sequence_length(S, d.max_positions)
        ids = input_ids.to(device=self.device, dtype=torch.int64).contiguous()
        mask = None
        if attention_mask is not None:
            if tuple(attention_mask.shape) != (n, S):
                raise ValueError(f"attention_mask {tuple(attention_mask.shape)} does not match input_ids {(n, S)}")
            mask = admissible_keys(attention_mask.to(self.device))
        pooled = torch.empty((n, d.hidden), dtype=torch.float32, device=self.device)
        hidden = torch.empty((n, S, d.hidden), dtype=torch.float32, device=self.device) if return_hidden else None
        if n == 0:
            return (pooled, hidden) if return_hidden else pooled
        step = max(1, min(self.max_texts_per_pass, n))
        ws = self._workspace(step, S)
        stream = current_stream_ptr()
        for s in range(0, n, step):
            e = min(n, s + step)
            check(self._lib.pg_text_forward(self._handle, ptr(ids[s:e]), ptr(mask[s:e]) if mask is not None else None,
                                            e - s, S, ptr(ws), ws.numel(), ptr(pooled[s:e]),
                                            ptr(hidden[s:e]) if hidden is not None else None, stream), "pg_text_forward")
        return (pooled, hidden) if return_hidden else pooled

    __call__ = forward


class CLIPTextTower(EncoderTower, nn.Module):
    """Drop-in for HF `CLIPTextModel`'s forward: parameters `text_model.embeddings.{token,position}_embedding.weight`,
    `text_model.encoder.layers.N....`, `text_model.final_layer_norm.*`; fp32 masters here, fp16 kernel layouts (re)packed
    lazily by `TextEngine` when parameters change."""
    ENGINE, PASS_LIMIT = TextEngine, "max_texts_per_pass"

    def __init__(self, dims: TextDims = TextDims()):
        super().__init__()
        self.dims = dims
        self.config = SimpleNamespace(vocab_size=dims.vocab, max_position_embeddings=dims.max_positions,
                                      hidden_size=dims.hidden, intermediate_size=dims.intermediate,
                                      num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                                      layer_norm_eps=dims.ln_eps)
        tm = Holder()
        emb = Holder()
        tok = Holder()
        tok.weight = Parameter(torch.zeros(dims.vocab, dims.hidden))
        emb.token_embedding = tok
        pos = Holder()
        pos.weight = Parameter(torch.zeros(dims.max_positions, dims.hidden))
        emb.position_embedding = pos
        tm.embeddings = emb
        tm.encoder = encoder_holder(dims.hidden, dims.intermediate, dims.layers)
        tm.final_layer_norm = norm(dims.hidden)
        self.text_model = tm
        self.max_texts_per_pass = 256

    @classmethod
    def from_hf(cls, hf_model) -> "CLIPTextTower":
        """Build from a HuggingFace CLIPTextModel / CLIPTextTransformer instance (weights copied by name)."""
        tower = cls(TextDims.from_hf_config(hf_model.config))
        sd = {k if k.startswith("text_model.") else "text_model." + k: v for k, v in hf_model.state_dict().items()
              if "position_ids" not in k}
        missing, unexpected = tower.load_state_dict(sd, strict=False)
        if missing or unexpected:
            raise PigeonB200Error(f"cannot map HF weights: missing={missing} unexpected={unexpected}")
        return tower

    def _repack_groups(self):
        tm = self.text_model
        return list(tm.embeddings.parameters()) + list(tm.final_layer_norm.parameters()), tm.encoder.layers

    @torch.no_grad()
    def pooled(self, input_ids: Tensor, attention_mask: Optional[Tensor] = None) -> Tensor:
        """pooler_output only (last_hidden_state is not written)."""
        return self.engine().forward(input_ids, attention_mask)

    @torch.no_grad()
    def forward(self, input_ids: Tensor = None, attention_mask: Optional[Tensor] = None, **kwargs):
        if input_ids is None:
            raise ValueError("You have to specify input_ids")
        pooled, hidden = self.engine().forward(input_ids, attention_mask, return_hidden=True)
        return SimpleNamespace(last_hidden_state=hidden, pooler_output=pooled)
