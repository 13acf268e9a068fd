"""Host side of the pre-LN encoder stack that the CLIP vision and text towers share (`encoder_layers` in csrc/capi.cu):

    Holder, linear, norm, encoder_holder   the HF module tree, so state_dict() key names match HF checkpoints
    pack_layer                             encoder layer i of a state dict -> the kernel layouts of one `_lib.VitLayer`
    EncoderEngine                          owns the C handle and the packed weights, repacked group by group
    EncoderTower                           nn.Module mixin: repacks only the groups whose parameters moved
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Iterable, Optional

import torch
from torch import Tensor, nn
from torch.nn.parameter import Parameter

from . import _lib, _versions
from ._lib import PigeonB200Error, check, load, ptr


# ---------------------------------------------------------------------------------------------- parameter tree
class Holder(nn.Module):
    """Parameter container (no forward): keeps the HF module tree so state_dict() key names match."""


def linear(out_f: int, in_f: int, bias: bool = True) -> nn.Module:
    h = Holder()
    h.weight = Parameter(torch.zeros(out_f, in_f))
    if bias:
        h.bias = Parameter(torch.zeros(out_f))
    return h


def norm(n: int) -> nn.Module:
    h = Holder()
    h.weight = Parameter(torch.ones(n))
    h.bias = Parameter(torch.zeros(n))
    return h


def encoder_holder(hidden: int, intermediate: int, layers: int) -> nn.Module:
    """`encoder.layers.N.{self_attn.{q,k,v,out}_proj, layer_norm1, mlp.fc1, mlp.fc2, layer_norm2}` (HF CLIPEncoder)."""
    enc = Holder()
    out = []
    for _ in range(layers):
        L = Holder()
        sa = Holder()
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            setattr(sa, n, linear(hidden, hidden))
        L.self_attn = sa
        L.layer_norm1 = norm(hidden)
        mlp = Holder()
        mlp.fc1 = linear(intermediate, hidden)
        mlp.fc2 = linear(hidden, intermediate)
        L.mlp = mlp
        L.layer_norm2 = norm(hidden)
        out.append(L)
    enc.layers = nn.ModuleList(out)
    return enc


# ---------------------------------------------------------------------------------------------- weight packing
def strip_prefix(sd: Dict[str, Tensor], prefixes: Iterable[str]) -> Dict[str, Tensor]:
    """Normalise HF key names: every leading repeat of each of `prefixes` is dropped, in order."""
    out = {}
    for k, v in sd.items():
        for pre in prefixes:
            while k.startswith(pre):
                k = k[len(pre):]
        out[k] = v
    return out


class Pack(list):
    """The device tensors of one repack group.  The C side references them by raw pointer, so they live as long as the
    group does."""

    def __init__(self, device: torch.device):
        super().__init__()
        self.device = device

    def f32(self, t: Tensor) -> Tensor:
        t = t.detach().to(device=self.device, dtype=torch.float32).contiguous()
        self.append(t)
        return t

    def f16(self, t: Tensor) -> Tensor:
        t = t.detach().to(device=self.device, dtype=torch.float32).to(torch.float16).contiguous()
        self.append(t)
        return t


def pack_layer(L: _lib.VitLayer, sd: Dict[str, Tensor], i: int, pack: Pack, fold: bool) -> None:
    """Point `L` at the kernel layouts of encoder layer i of the prefix-stripped state dict `sd`, kept in `pack`.  `fold`
    also fills the LayerNorm-folded fields (w_*_ln, b_*_ln, cs_*); without it they stay NULL and the layer runs the
    LayerNorm kernels."""
    f32, f16, dev = pack.f32, pack.f16, pack.device
    p = f"encoder.layers.{i}."
    w_qkv = torch.cat([sd[p + f"self_attn.{n}_proj.weight"] for n in "qkv"], dim=0)
    b_qkv = torch.cat([sd[p + f"self_attn.{n}_proj.bias"] for n in "qkv"], dim=0)
    L.ln1_g, L.ln1_b = ptr(f32(sd[p + "layer_norm1.weight"])), ptr(f32(sd[p + "layer_norm1.bias"]))
    L.w_qkv, L.b_qkv = ptr(f16(w_qkv)), ptr(f32(b_qkv))
    L.w_o, L.b_o = ptr(f16(sd[p + "self_attn.out_proj.weight"])), ptr(f32(sd[p + "self_attn.out_proj.bias"]))
    L.ln2_g, L.ln2_b = ptr(f32(sd[p + "layer_norm2.weight"])), ptr(f32(sd[p + "layer_norm2.bias"]))
    L.w_fc1, L.b_fc1 = ptr(f16(sd[p + "mlp.fc1.weight"])), ptr(f32(sd[p + "mlp.fc1.bias"]))
    L.w_fc2, L.b_fc2 = ptr(f16(sd[p + "mlp.fc2.weight"])), ptr(f32(sd[p + "mlp.fc2.bias"]))
    if fold:
        # LN(x) W^T + b = rstd * (x (gamma*W)^T - mu * rowsum(gamma*W)) + (b + W beta): the tensor cores see the raw
        # row x and W' = gamma * W; rowsum is taken over the fp16 values of W' so that acc - mu * rowsum is exact.
        def fold_ln(w, b, g, beta):
            w32 = w.detach().to(dev, torch.float32)
            wf = f16(w32 * g.detach().to(dev, torch.float32)[None, :])
            cs = f32(wf.float().sum(dim=1))
            bf = f32(b.detach().to(dev, torch.float32) + w32 @ beta.detach().to(dev, torch.float32))
            return ptr(wf), ptr(bf), ptr(cs)
        L.w_qkv_ln, L.b_qkv_ln, L.cs_qkv = fold_ln(w_qkv, b_qkv, sd[p + "layer_norm1.weight"], sd[p + "layer_norm1.bias"])
        L.w_fc1_ln, L.b_fc1_ln, L.cs_fc1 = fold_ln(sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"],
                                                   sd[p + "layer_norm2.weight"], sd[p + "layer_norm2.bias"])


class EncoderEngine:
    """Packed weights and the C handle of one tower.  A subclass names its key prefixes and C entry points, packs its
    embeddings group (`_pack_embeddings`) and builds the create-call structs (`_structs`)."""
    PREFIXES: tuple = ()
    CREATE = DESTROY = WORKSPACE = ""
    fold_layernorm = False   # LayerNorm folded into the GEMM epilogues (the vision tower's default)

    def __init__(self, state_dict: Dict[str, Tensor], dims, device: torch.device | str = "cuda"):
        self.dims = dims
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise PigeonB200Error(f"{type(self).__name__} runs on a CUDA device only (no CPU path)")
        self._lib = load()
        self._handle = C.c_void_p()
        self._ws: Optional[Tensor] = None
        self._packs = None   # group ("embeddings" | layer index) -> its Pack
        self.load_state_dict(state_dict)

    def load_state_dict(self, state_dict: Dict[str, Tensor], changed=None) -> None:
        """(Re)pack weights for the kernels.  `changed` limits the work to the groups whose parameters moved: a set holding
        "embeddings" and / or encoder layer indices (None = everything).  Under the reference's fine-tune policy only the last
        layer changes between optimizer steps, so one layer is repacked per step instead of 24."""
        d = self.dims
        sd = strip_prefix(state_dict, self.PREFIXES)
        if changed is None or self._packs is None:
            changed = {"embeddings", *range(d.layers)}
            self._packs = {}
            self._layers = (_lib.VitLayer * d.layers)()
        if "embeddings" in changed:
            self._top = self._pack_embeddings(sd, self._group("embeddings"))
        for i in sorted(k for k in changed if k != "embeddings"):
            pack_layer(self._layers[i], sd, i, self._group(i), self.fold_layernorm)
        cfg, w = self._structs()
        if self._handle:
            getattr(self._lib, self.DESTROY)(self._handle)
            self._handle = C.c_void_p()
        check(getattr(self._lib, self.CREATE)(C.byref(cfg), C.byref(w), C.byref(self._handle)), self.CREATE)  # copies the structs

    def _group(self, key) -> Pack:
        self._packs[key] = Pack(self.device)
        return self._packs[key]

    def __del__(self):
        try:
            if self._handle:
                getattr(self._lib, self.DESTROY)(self._handle)
        except Exception:
            pass

    def workspace_bytes(self, *shape: int) -> int:
        return int(getattr(self._lib, self.WORKSPACE)(self._handle, *shape))

    def _workspace(self, *shape: int) -> Tensor:
        need = self.workspace_bytes(*shape)
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws


# ---------------------------------------------------------------------------------------------- repack policy
def _version_key(params) -> tuple:
    return tuple((p.data_ptr(), p._version, _versions.get(p)) for p in params)


class EncoderTower:
    """Mixin of the tower nn.Modules: fp32 master parameters live in the module, and `engine()` hands out an engine whose
    packed copies match them, repacking only the groups ("embeddings", encoder layer indices) whose parameters moved.  A
    tower supplies `ENGINE`, `PASS_LIMIT` (the attribute name of its per-pass limit, the same on tower and engine),
    `_repack_groups()` and `_engine_kwargs()`."""
    ENGINE = EncoderEngine
    PASS_LIMIT = ""
    _engine = None
    _packed_version = None

    def _repack_groups(self):
        """(parameters of the "embeddings" group, the encoder layers)."""
        raise NotImplementedError

    def _engine_kwargs(self) -> dict:
        """Engine constructor arguments besides the limit; an existing engine that differs in one of them is replaced."""
        return {}

    def _weights_changed(self):
        self._packed_version = None

    def _weights_version(self):
        return _version_key(self.parameters())

    def _group_versions(self):
        """Version key per repack group: "embeddings" and one per encoder layer — under the reference's fine-tune policy only
        the last layer moves between optimizer steps."""
        emb, layers = self._repack_groups()
        groups = {"embeddings": _version_key(emb)}
        for i, layer in enumerate(layers):
            groups[i] = _version_key(layer.parameters())
        return groups

    def engine(self):
        p0 = next(self.parameters())
        if not p0.is_cuda:
            raise PigeonB200Error(f"{type(self).__name__} is on the CPU: move the model with .to('cuda') — the H100 path "
                                  "has no CPU implementation")
        v = self._group_versions()
        if self._engine is None or self._packed_version != v:
            sd = {k: t.detach() for k, t in self.state_dict().items()}
            kw, eng = self._engine_kwargs(), self._engine
            if eng is None or eng.device != p0.device or any(getattr(eng, k) != x for k, x in kw.items()):
                self._engine = self.ENGINE(sd, self.dims, device=p0.device, **kw)
            else:
                old = self._packed_version
                changed = None if old is None else {g for g, key in v.items() if old.get(g) != key}
                eng.load_state_dict(sd, changed=changed)
            self._packed_version = v
        setattr(self._engine, self.PASS_LIMIT, int(getattr(self, self.PASS_LIMIT)))
        return self._engine
