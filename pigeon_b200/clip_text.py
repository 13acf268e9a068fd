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

import ctypes as C
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Dict, Optional

import torch
from torch import Tensor, nn
from torch.nn.parameter import Parameter

from . import _lib, _versions
from ._lib import PigeonB200Error, check, current_stream_ptr, load, ptr


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


def _strip_prefix(sd: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """Normalise HF key names to start at 'embeddings.' / 'encoder.' / 'final_layer_norm.'."""
    out = {}
    for k, v in sd.items():
        while k.startswith("text_model."):
            k = k[len("text_model."):]
        out[k] = v
    return out


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


class TextEngine:
    """H100 execution engine of HF CLIPTextTransformer.forward (pooled output, optionally last_hidden_state)."""

    def __init__(self, state_dict: Dict[str, Tensor], dims: TextDims, device: torch.device | str = "cuda",
                 max_texts_per_pass: int = 256):
        self.dims = dims
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise PigeonB200Error("TextEngine runs on a CUDA device only (no CPU path)")
        self.max_texts_per_pass = int(max_texts_per_pass)
        self._lib = load()
        self._handle = C.c_void_p()
        self._ws: Optional[Tensor] = None
        self._packs = None
        self.load_state_dict(state_dict)

    def load_state_dict(self, state_dict: Dict[str, Tensor], changed=None) -> None:
        """(Re)pack weights; `changed` limits the work to groups ("embeddings" = token / position tables and
        final_layer_norm, or encoder layer indices) whose parameters moved (None = everything)."""
        d, dev = self.dims, self.device
        sd = _strip_prefix(state_dict)
        if changed is None or self._packs is None:
            changed = {"embeddings", *range(d.layers)}
            self._packs = {}
            self._layers = (_lib.VitLayer * d.layers)()

        def group(key):
            keep = []
            self._packs[key] = keep

            def f32(t):
                t = t.detach().to(device=dev, dtype=torch.float32).contiguous()
                keep.append(t)
                return t

            def f16(t):
                t = t.detach().to(device=dev, dtype=torch.float32).to(torch.float16).contiguous()
                keep.append(t)
                return t
            return f32, f16

        if "embeddings" in changed:
            f32, _ = group("embeddings")
            tok = f32(sd["embeddings.token_embedding.weight"])
            pos = f32(sd["embeddings.position_embedding.weight"])
            if tok.shape != (d.vocab, d.hidden) or pos.shape != (d.max_positions, d.hidden):
                raise PigeonB200Error(f"token_embedding {tuple(tok.shape)} / position_embedding {tuple(pos.shape)} do not "
                                      f"match ({d.vocab}, {d.hidden}) / ({d.max_positions}, {d.hidden})")
            self._top = (ptr(tok), ptr(pos), ptr(f32(sd["final_layer_norm.weight"])), ptr(f32(sd["final_layer_norm.bias"])))

        for i in sorted(k for k in changed if k != "embeddings"):
            f32, f16 = group(i)
            p = f"encoder.layers.{i}."
            L = self._layers[i]
            L.ln1_g, L.ln1_b = ptr(f32(sd[p + "layer_norm1.weight"])), ptr(f32(sd[p + "layer_norm1.bias"]))
            L.w_qkv = ptr(f16(torch.cat([sd[p + f"self_attn.{n}_proj.weight"] for n in "qkv"], dim=0)))
            L.b_qkv = ptr(f32(torch.cat([sd[p + f"self_attn.{n}_proj.bias"] for n in "qkv"], dim=0)))
            L.w_o, L.b_o = ptr(f16(sd[p + "self_attn.out_proj.weight"])), ptr(f32(sd[p + "self_attn.out_proj.bias"]))
            L.ln2_g, L.ln2_b = ptr(f32(sd[p + "layer_norm2.weight"])), ptr(f32(sd[p + "layer_norm2.bias"]))
            L.w_fc1, L.b_fc1 = ptr(f16(sd[p + "mlp.fc1.weight"])), ptr(f32(sd[p + "mlp.fc1.bias"]))
            L.w_fc2, L.b_fc2 = ptr(f16(sd[p + "mlp.fc2.weight"])), ptr(f32(sd[p + "mlp.fc2.bias"]))
            # the LayerNorm-fold fields stay NULL: the text tower runs the LayerNorm kernels

        cfg = _lib.TextConfig(d.vocab, d.max_positions, d.hidden, d.heads, d.intermediate, d.layers, d.ln_eps)
        w = _lib.TextWeights(self._top[0], self._top[1], self._layers, self._top[2], self._top[3])
        if self._handle:
            self._lib.pg_text_destroy(self._handle)
            self._handle = C.c_void_p()
        check(self._lib.pg_text_create(C.byref(cfg), C.byref(w), C.byref(self._handle)), "pg_text_create")

    def __del__(self):
        try:
            if self._handle:
                self._lib.pg_text_destroy(self._handle)
        except Exception:
            pass

    def workspace_bytes(self, n: int, S: int) -> int:
        return int(self._lib.pg_text_workspace_bytes(self._handle, n, S))

    def _workspace(self, n: int, S: int) -> Tensor:
        need = self.workspace_bytes(n, S)
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

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


class _Holder(nn.Module):
    """Parameter container (no forward): keeps the HF module tree so state_dict() key names match."""


def _linear(out_f: int, in_f: int, bias: bool = True) -> nn.Module:
    h = _Holder()
    h.weight = Parameter(torch.zeros(out_f, in_f))
    if bias:
        h.bias = Parameter(torch.zeros(out_f))
    return h


def _norm(n: int) -> nn.Module:
    h = _Holder()
    h.weight = Parameter(torch.ones(n))
    h.bias = Parameter(torch.zeros(n))
    return h


def encoder_holder(hidden: int, intermediate: int, layers: int) -> nn.Module:
    """`encoder.layers.N.{self_attn.{q,k,v,out}_proj, layer_norm1, mlp.fc1, mlp.fc2, layer_norm2}` (HF CLIPEncoder)."""
    enc = _Holder()
    out = []
    for _ in range(layers):
        L = _Holder()
        sa = _Holder()
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            setattr(sa, n, _linear(hidden, hidden))
        L.self_attn = sa
        L.layer_norm1 = _norm(hidden)
        mlp = _Holder()
        mlp.fc1 = _linear(intermediate, hidden)
        mlp.fc2 = _linear(hidden, intermediate)
        L.mlp = mlp
        L.layer_norm2 = _norm(hidden)
        out.append(L)
    enc.layers = nn.ModuleList(out)
    return enc


class CLIPTextTower(nn.Module):
    """Drop-in for HF `CLIPTextModel`'s forward: parameters `text_model.embeddings.{token,position}_embedding.weight`,
    `text_model.encoder.layers.N....`, `text_model.final_layer_norm.*`; fp32 masters here, fp16 kernel layouts (re)packed
    lazily by `TextEngine` when parameters change."""

    def __init__(self, dims: TextDims = TextDims()):
        super().__init__()
        self.dims = dims
        self.config = SimpleNamespace(vocab_size=dims.vocab, max_position_embeddings=dims.max_positions,
                                      hidden_size=dims.hidden, intermediate_size=dims.intermediate,
                                      num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                                      layer_norm_eps=dims.ln_eps)
        tm = _Holder()
        emb = _Holder()
        tok = _Holder()
        tok.weight = Parameter(torch.zeros(dims.vocab, dims.hidden))
        emb.token_embedding = tok
        pos = _Holder()
        pos.weight = Parameter(torch.zeros(dims.max_positions, dims.hidden))
        emb.position_embedding = pos
        tm.embeddings = emb
        tm.encoder = encoder_holder(dims.hidden, dims.intermediate, dims.layers)
        tm.final_layer_norm = _norm(dims.hidden)
        self.text_model = tm
        self._engine: Optional[TextEngine] = None
        self._packed_version = None
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

    def _group_versions(self):
        def key(params):
            return tuple((p.data_ptr(), p._version, _versions.get(p)) for p in params)
        tm = self.text_model
        groups = {"embeddings": key(list(tm.embeddings.parameters()) + list(tm.final_layer_norm.parameters()))}
        for i, layer in enumerate(tm.encoder.layers):
            groups[i] = key(layer.parameters())
        return groups

    def engine(self) -> TextEngine:
        p0 = next(self.parameters())
        if not p0.is_cuda:
            raise PigeonB200Error("CLIPTextTower is on the CPU: move the model with .to('cuda') — the H100 path has no CPU "
                                  "implementation")
        v = self._group_versions()
        if self._engine is None or self._packed_version != v:
            sd = {k: t.detach() for k, t in self.state_dict().items()}
            if self._engine is None or self._engine.device != p0.device:
                self._engine = TextEngine(sd, self.dims, device=p0.device, max_texts_per_pass=self.max_texts_per_pass)
            else:
                old = self._packed_version
                changed = None if old is None else {g for g, k in v.items() if old.get(g) != k}
                self._engine.load_state_dict(sd, changed=changed)
            self._packed_version = v
        self._engine.max_texts_per_pass = self.max_texts_per_pass
        return self._engine

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
