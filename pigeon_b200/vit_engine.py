"""Host-side owner of the CLIP vision tower on the GPU: packs HF-named weights into the kernel layouts,
holds the C handle and the scratch buffer, and runs `pg_vit_forward` in view chunks.

Accepts the state-dict key names of HF `CLIPVisionModel` (the module the reference builds at
models/clip_embedder.py:26 and evaluation/evaluate.py:36), so checkpoints written by the reference load by name.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict

import torch

from . import _lib
from ._lib import PigeonB200Error, check, current_stream_ptr, ptr
from .encoder import EncoderEngine, Pack


@dataclass
class VitDims:
    image_size: int = 336
    patch_size: int = 14
    hidden: int = 1024
    heads: int = 16
    intermediate: int = 4096
    layers: int = 24
    ln_eps: float = 1e-5

    @property
    def tokens(self) -> int:
        return (self.image_size // self.patch_size) ** 2 + 1

    @property
    def patch_k(self) -> int:
        return 3 * self.patch_size * self.patch_size

    @property
    def patch_k_pad(self) -> int:
        return (self.patch_k + 63) // 64 * 64

    @classmethod
    def from_hf_config(cls, cfg) -> "VitDims":
        return cls(image_size=cfg.image_size, patch_size=cfg.patch_size, hidden=cfg.hidden_size,
                   heads=cfg.num_attention_heads, intermediate=cfg.intermediate_size, layers=cfg.num_hidden_layers,
                   ln_eps=float(cfg.layer_norm_eps))


class VitEngine(EncoderEngine):
    """H100 execution engine of HF CLIPVisionTransformer.forward(...).last_hidden_state (+ token mean)."""
    PREFIXES = ("base_model.", "clip_model.", "vision_model.")   # keys start at 'embeddings.' / 'encoder.' / 'pre_layrnorm.'
    CREATE, DESTROY, WORKSPACE = "pg_vit_create", "pg_vit_destroy", "pg_vit_workspace_bytes"

    def __init__(self, state_dict: Dict[str, torch.Tensor], dims: VitDims, device: torch.device | str = "cuda",
                 max_views_per_pass: int = 256, fold_layernorm: bool = True):
        """fold_layernorm: feed the GEMMs the raw fp16 residual row and apply LayerNorm in their epilogues (no LayerNorm
        kernel, no normalised copy in HBM; see csrc/gemm.h EPI_F16_LN_*).  False keeps the LayerNorm kernels (A/B switch)."""
        self.fold_layernorm = bool(fold_layernorm)
        self.max_views_per_pass = int(max_views_per_pass)
        super().__init__(state_dict, dims, device)

    # ------------------------------------------------------------------------------------------ weights
    def _pack_embeddings(self, sd: Dict[str, torch.Tensor], pack: Pack) -> tuple:
        d, dev = self.dims, self.device
        pw = sd["embeddings.patch_embedding.weight"].detach().to(dev, torch.float32).reshape(d.hidden, d.patch_k)
        pw_pad = torch.zeros((d.hidden, d.patch_k_pad), dtype=torch.float32, device=dev)
        pw_pad[:, : d.patch_k] = pw
        pos = pack.f32(sd["embeddings.position_embedding.weight"])
        if pos.shape != (d.tokens, d.hidden):
            raise PigeonB200Error(f"position_embedding {tuple(pos.shape)} != ({d.tokens}, {d.hidden})")
        return (ptr(pack.f16(pw_pad)), ptr(pack.f32(sd["embeddings.class_embedding"])), ptr(pos),
                ptr(pack.f32(sd["pre_layrnorm.weight"])), ptr(pack.f32(sd["pre_layrnorm.bias"])))

    def _structs(self):
        d = self.dims
        cfg = _lib.VitConfig(d.image_size, d.patch_size, d.hidden, d.heads, d.intermediate, d.layers, d.ln_eps,
                             d.patch_k_pad)
        return cfg, _lib.VitWeights(*self._top, self._layers)

    # ------------------------------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, pixel_values: torch.Tensor, return_hidden: bool = False):
        """pixel_values [N, 3, H, W] (fp32 or fp16, CUDA) -> token-mean embedding [N, hidden] fp32
        (and last_hidden_state [N, tokens, hidden] fp32 when `return_hidden`)."""
        d = self.dims
        if not pixel_values.is_cuda:
            return self._forward_from_host(pixel_values, return_hidden)
        if pixel_values.dim() != 4 or tuple(pixel_values.shape[1:]) != (3, d.image_size, d.image_size):
            raise ValueError(f"Input image size ({tuple(pixel_values.shape[1:])}) doesn't match model "
                             f"(3, {d.image_size}, {d.image_size}).")
        if pixel_values.dtype not in (torch.float32, torch.float16):
            pixel_values = pixel_values.float()
        pixel_values = pixel_values.contiguous()
        n = pixel_values.shape[0]
        emb = torch.empty((n, d.hidden), dtype=torch.float32, device=self.device)
        hidden = torch.empty((n, d.tokens, d.hidden), dtype=torch.float32, device=self.device) if return_hidden else None
        step = max(1, min(self.max_views_per_pass, n))
        ws = self._workspace(step)
        stream = current_stream_ptr()
        for s in range(0, n, step):
            e = min(n, s + step)
            check(self._lib.pg_vit_forward(self._handle, ptr(pixel_values[s:e]), int(pixel_values.dtype == torch.float16),
                                           e - s, ptr(ws), ws.numel(), ptr(emb[s:e]),
                                           ptr(hidden[s:e]) if hidden is not None else None, stream), "pg_vit_forward")
        return (emb, hidden) if return_hidden else emb

    @torch.no_grad()
    def forward_cls(self, pixel_values: torch.Tensor):
        """pixel_values [N, 3, H, W] (fp32 or fp16; host tensors are copied over first) -> (token-mean embedding [N, hidden],
        CLS rows of last_hidden_state [N, hidden]) fp32, through pg_vit_forward_cls: the CLS rows that CLIPModel's image
        features start from, without the [N, tokens, hidden] last_hidden_state."""
        d = self.dims
        if pixel_values.dim() != 4 or tuple(pixel_values.shape[1:]) != (3, d.image_size, d.image_size):
            raise ValueError(f"Input image size ({tuple(pixel_values.shape[1:])}) doesn't match model "
                             f"(3, {d.image_size}, {d.image_size}).")
        if pixel_values.dtype not in (torch.float32, torch.float16):
            pixel_values = pixel_values.float()
        pixel_values = pixel_values.to(self.device).contiguous()
        n = pixel_values.shape[0]
        emb = torch.empty((n, d.hidden), dtype=torch.float32, device=self.device)
        cls = torch.empty((n, d.hidden), dtype=torch.float32, device=self.device)
        step = max(1, min(self.max_views_per_pass, n))
        ws = self._workspace(step)
        stream = current_stream_ptr()
        for s in range(0, n, step):
            e = min(n, s + step)
            check(self._lib.pg_vit_forward_cls(self._handle, ptr(pixel_values[s:e]), int(pixel_values.dtype == torch.float16),
                                               e - s, ptr(ws), ws.numel(), ptr(emb[s:e]), None, ptr(cls[s:e]), stream),
                  "pg_vit_forward_cls")
        return emb, cls

    @torch.no_grad()
    def _forward_from_host(self, pixel_values: torch.Tensor, return_hidden: bool, host_chunk: int = 256):
        """Host (ideally pinned) pixels: the H2D copy of chunk i+1 runs on a side stream while chunk i computes,
        through two device staging buffers (the reference copies the whole batch up front, super_guessr.py:193-217)."""
        d = self.dims
        if pixel_values.dim() != 4 or tuple(pixel_values.shape[1:]) != (3, d.image_size, d.image_size):
            raise ValueError(f"Input image size ({tuple(pixel_values.shape[1:])}) doesn't match model "
                             f"(3, {d.image_size}, {d.image_size}).")
        if pixel_values.dtype not in (torch.float32, torch.float16):
            pixel_values = pixel_values.float()
        pixel_values = pixel_values.contiguous()
        n = pixel_values.shape[0]
        step = max(1, min(host_chunk, self.max_views_per_pass, n))
        emb = torch.empty((n, d.hidden), dtype=torch.float32, device=self.device)
        hidden = torch.empty((n, d.tokens, d.hidden), dtype=torch.float32, device=self.device) if return_hidden else None
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        key = (step, pixel_values.dtype)
        if getattr(self, "_stage_key", None) != key:
            self._stage = [torch.empty((step,) + tuple(pixel_values.shape[1:]), dtype=pixel_values.dtype, device=self.device)
                           for _ in range(2)]
            self._stage_key = key
        ws = self._workspace(step)
        main = torch.cuda.current_stream(self.device)
        copied = [torch.cuda.Event(), torch.cuda.Event()]
        consumed = [torch.cuda.Event(), torch.cuda.Event()]
        chunks = list(range(0, n, step))

        def start_copy(i):
            s0, b = chunks[i], i & 1
            e0 = min(n, s0 + step)
            with torch.cuda.stream(self._copy_stream):
                if i >= 2:
                    self._copy_stream.wait_event(consumed[b])      # staging buffer b free again
                else:
                    self._copy_stream.wait_stream(main)            # order after earlier users of the staging buffers
                self._stage[b][: e0 - s0].copy_(pixel_values[s0:e0], non_blocking=True)
                copied[b].record(self._copy_stream)

        start_copy(0)
        for i, s0 in enumerate(chunks):
            e0, b = min(n, s0 + step), i & 1
            if i + 1 < len(chunks):
                start_copy(i + 1)
            main.wait_event(copied[b])
            check(self._lib.pg_vit_forward(self._handle, ptr(self._stage[b]), int(pixel_values.dtype == torch.float16),
                                           e0 - s0, ptr(ws), ws.numel(), ptr(emb[s0:e0]),
                                           ptr(hidden[s0:e0]) if hidden is not None else None, main.cuda_stream),
                  "pg_vit_forward")
            consumed[b].record(main)
        return (emb, hidden) if return_hidden else emb

    __call__ = forward
