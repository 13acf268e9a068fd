"""Fine-tune step of the vision tower (host side of pg_vit_forward_train / pg_vit_backward).

What the reference gets from autograd + DDP for `accelerator.backward(output.loss)` (training/train_eval_loop.py:216)
with the freeze policy of models/super_guessr.py:159-160 (embeddings, pre_layrnorm and the LAST encoder layer
trainable; `requires_grad` decides here too): the training-mode forward keeps its activations in one arena, the
backward runs as hand-written kernels (bf16 operands, fp32 accumulation) and leaves fp32 gradients in `param.grad`
under the HuggingFace parameter names, ready for `pigeon_b200.training.AdamW`.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import torch

from . import _lib
from ._lib import PigeonB200Error, check, current_stream_ptr, load, ptr


def _align(n: int, a: int = 1024) -> int:
    return (n + a - 1) // a * a


def _aligned_empty(nbytes: int, device) -> torch.Tensor:
    """uint8 buffer whose data pointer is 1024-byte aligned (the caching allocator only guarantees 512)."""
    raw = torch.empty(nbytes + 1024, dtype=torch.uint8, device=device)
    off = (-raw.data_ptr()) % 1024
    return raw[off:off + nbytes]


def grow_aligned(owner, name: str, nbytes: int, device) -> torch.Tensor:
    """owner.<name>, replaced by a 1024-byte aligned buffer of nbytes when it holds fewer (the old one is freed first)."""
    buf = getattr(owner, name)
    if buf is None or buf.numel() < nbytes:
        setattr(owner, name, None)
        buf = _aligned_empty(nbytes, device)
        setattr(owner, name, buf)
    return buf


def put_grad(p, t) -> None:
    """p.grad += t (p.grad = a copy of t when there is none yet): gradient accumulation across backward calls."""
    t = t.contiguous()
    p.grad = t.clone() if p.grad is None else p.grad.add_(t)


LAYER_GRADS = ("ln1_g", "ln1_b", "w_qkv", "b_qkv", "w_o", "b_o", "ln2_g", "ln2_b", "w_fc1", "b_fc1", "w_fc2", "b_fc2")


def layer_grad_shapes(l: int, H: int, I: int):
    return [(f"{l}.ln1_g", (H,)), (f"{l}.ln1_b", (H,)), (f"{l}.w_qkv", (3 * H, H)), (f"{l}.b_qkv", (3 * H,)),
            (f"{l}.w_o", (H, H)), (f"{l}.b_o", (H,)), (f"{l}.ln2_g", (H,)), (f"{l}.ln2_b", (H,)),
            (f"{l}.w_fc1", (I, H)), (f"{l}.b_fc1", (I,)), (f"{l}.w_fc2", (H, I)), (f"{l}.b_fc2", (H,))]


def put_layer_grads(L, g: Dict[str, torch.Tensor], l: int, H: int) -> None:
    """Publish the fused gradients of encoder layer l (HF CLIPEncoderLayer L) into its parameters' .grad."""
    sa, mlp = L.self_attn, L.mlp
    for i, proj in enumerate((sa.q_proj, sa.k_proj, sa.v_proj)):
        put_grad(proj.weight, g[f"{l}.w_qkv"][i * H:(i + 1) * H])
        put_grad(proj.bias, g[f"{l}.b_qkv"][i * H:(i + 1) * H])
    put_grad(sa.out_proj.weight, g[f"{l}.w_o"]); put_grad(sa.out_proj.bias, g[f"{l}.b_o"])
    put_grad(L.layer_norm1.weight, g[f"{l}.ln1_g"]); put_grad(L.layer_norm1.bias, g[f"{l}.ln1_b"])
    put_grad(L.layer_norm2.weight, g[f"{l}.ln2_g"]); put_grad(L.layer_norm2.bias, g[f"{l}.ln2_b"])
    put_grad(mlp.fc1.weight, g[f"{l}.w_fc1"]); put_grad(mlp.fc1.bias, g[f"{l}.b_fc1"])
    put_grad(mlp.fc2.weight, g[f"{l}.w_fc2"]); put_grad(mlp.fc2.bias, g[f"{l}.b_fc2"])


@torch.no_grad()
def transpose_layers(layers, versions, wt: list, wt_version: dict) -> None:
    """wt[l] = bf16 transposes of encoder layer l's four weight matrices, redone only where versions[l] moved."""
    bf = torch.bfloat16
    for l, L in enumerate(layers):
        if wt[l] is not None and wt_version.get(l) == versions[l]:
            continue
        sa, mlp = L.self_attn, L.mlp
        wqkv = torch.cat([sa.q_proj.weight, sa.k_proj.weight, sa.v_proj.weight], dim=0)      # [3H, H]
        wt[l] = dict(w_qkv_t=wqkv.t().contiguous().to(bf), w_o_t=sa.out_proj.weight.t().contiguous().to(bf),
                     w_fc1_t=mlp.fc1.weight.t().contiguous().to(bf), w_fc2_t=mlp.fc2.weight.t().contiguous().to(bf))
        wt_version[l] = versions[l]


def carve_saved(owner, saved, n: int, seq: int, top) -> Dict[str, int]:
    """Lay the activations a training forward keeps out in owner._arena (grown when too small) for n sequences of seq rows
    (tokens or S): the tower's `top` entries [(field of `saved`, bytes)] first, then x0 ... h of every encoder layer.  Points
    `saved` and owner._saved_layers at them and returns the arena offset of each top entry."""
    d = owner.dims
    rows, H, I = n * seq, d.hidden, d.intermediate
    per_layer = [("x0", rows * H * 4), ("xn1", rows * H * 2), ("qkv", rows * 3 * H * 2), ("lse2", n * d.heads * seq * 4),
                 ("ao", rows * H * 2), ("x1", rows * H * 4), ("xn2", rows * H * 2), ("u", rows * I * 2), ("h", rows * I * 2)]
    total = sum(_align(b) for _, b in top) + d.layers * sum(_align(b) for _, b in per_layer)
    base, off, offs = grow_aligned(owner, "_arena", total, next(owner.tower.parameters()).device).data_ptr(), 0, {}
    if base % 1024:
        raise PigeonB200Error("activation arena is not 1024-byte aligned")
    for name, b in top:
        setattr(saved, name, base + off)
        offs[name] = off
        off += _align(b)
    layers = (_lib.VitSavedLayer * d.layers)()
    for l in range(d.layers):
        for name, b in per_layer:
            setattr(layers[l], name, base + off)
            off += _align(b)
    saved.layers_host = owner._saved_layers = layers
    return offs


def flat_grads(shapes, device):
    """ONE zeroed flat fp32 buffer holding a tensor per (name, shape) of `shapes`, each 16-byte aligned inside it, so a single
    all-reduce averages them all -> (buffer, {name: view})."""
    offs, total = [], 0
    for _, shp in shapes:
        offs.append(total)
        total += (int(torch.Size(shp).numel()) + 3) // 4 * 4
    flat = torch.zeros(total, dtype=torch.float32, device=device)
    return flat, {name: flat[o:o + int(torch.Size(shp).numel())].view(shp) for (name, shp), o in zip(shapes, offs)}


def layers_bwd(wt: list, g: Dict[str, torch.Tensor], trainable) -> C.Array:
    """The VitLayerBwd array of a backward: every layer's transposed weights, and the gradient buffers of the layers whose
    `trainable` flag is set."""
    lb = (_lib.VitLayerBwd * len(wt))()
    for l, w in enumerate(wt):
        for k, t in w.items():
            setattr(lb[l], k, t.data_ptr())
        if trainable[l]:
            for k in LAYER_GRADS:
                setattr(lb[l], "d_" + k, g[f"{l}.{k}"].data_ptr())
    return lb


class TowerTrainer:
    """Owns the activation arena, the transposed bf16 weights and the fused gradient buffers of one CLIPVisionTower."""

    def __init__(self, tower, max_views: int = 64):
        self.tower = tower
        self.dims = tower.dims
        self.max_views = int(max_views)
        self._lib = load()
        self._arena: Optional[torch.Tensor] = None
        self._arena_views = 0
        self._ws: Optional[torch.Tensor] = None
        self._saved = None
        self._saved_layers = None
        self._saved_views = 0
        self._wt: Optional[List[Dict[str, torch.Tensor]]] = None
        self._wt_version = None
        self._pending: Optional[Dict[str, torch.Tensor]] = None
        self._keep = []

    # ---------------------------------------------------------------------------------- which parameters train
    def layout(self):
        vm = self.tower.vision_model
        emb_params = [vm.embeddings.class_embedding, vm.embeddings.patch_embedding.weight,
                      vm.embeddings.position_embedding.weight, vm.pre_layrnorm.weight, vm.pre_layrnorm.bias]
        flags = [p.requires_grad for p in emb_params]
        if any(flags) and not all(flags):
            raise PigeonB200Error("embeddings and pre_layrnorm must be trainable or frozen together")
        layers = []
        for i, L in enumerate(vm.encoder.layers):
            f = [p.requires_grad for p in L.parameters()]
            if any(f) and not all(f):
                raise PigeonB200Error(f"encoder layer {i}: parameters must be trainable or frozen together")
            layers.append(all(f))
        return all(flags), layers

    def any_trainable(self) -> bool:
        e, layers = self.layout()
        return e or any(layers)

    # ---------------------------------------------------------------------------------- buffers
    def _build_saved(self, n_views: int):
        d = self.dims
        rows = n_views * d.tokens
        top = [("im2col", n_views * (d.tokens - 1) * d.patch_k_pad * 2), ("e", rows * d.hidden * 4),
               ("x_out", rows * d.hidden * 4)]
        saved = _lib.VitSaved()
        self._x_out_off = carve_saved(self, saved, n_views, d.tokens, top)["x_out"]
        self._saved, self._saved_views = saved, n_views

    def _transposed_weights(self):
        """bf16 transposes of the four weight matrices of every layer (B operands of the backward GEMMs); only the layers whose
        parameters moved since the last call are redone (the last one, under the reference's fine-tune policy)."""
        if self._wt is None:
            self._wt, self._wt_version = [None] * self.dims.layers, {}
        transpose_layers(self.tower.vision_model.encoder.layers, self.tower._group_versions(), self._wt, self._wt_version)
        return self._wt

    def _pending_grads(self):
        if self._pending is not None:
            return self._pending
        d = self.dims
        dev = next(self.tower.parameters()).device
        emb_train, layers = self.layout()
        shapes = []
        if emb_train:
            shapes += [("patch_w", (d.hidden, d.patch_k_pad)), ("class_emb", (d.hidden,)), ("pos_emb", (d.tokens, d.hidden)),
                       ("pre_ln_g", (d.hidden,)), ("pre_ln_b", (d.hidden,))]
        for l, t in enumerate(layers):
            if t:
                shapes += layer_grad_shapes(l, d.hidden, d.intermediate)
        self._pending_flat, self._pending = flat_grads(shapes, dev)
        return self._pending

    # ---------------------------------------------------------------------------------- forward / backward
    @torch.no_grad()
    def forward(self, pixel_values: torch.Tensor) -> torch.Tensor:
        """pixel_values CUDA [n, 3, S, S] (fp16 or fp32), n <= max_views -> token-mean embedding [n, hidden] f32;
        the activations stay in the arena until the next forward."""
        d = self.dims
        n = pixel_values.shape[0]
        if n > self.max_views:
            raise PigeonB200Error(f"{n} views exceed max_views={self.max_views} of the training arena")
        if not pixel_values.is_cuda or tuple(pixel_values.shape[1:]) != (3, d.image_size, d.image_size):
            raise ValueError(f"pixel_values must be CUDA [n, 3, {d.image_size}, {d.image_size}]")
        if pixel_values.dtype not in (torch.float16, torch.float32):
            pixel_values = pixel_values.float()
        pixel_values = pixel_values.contiguous()
        self._build_saved(n)
        eng = self.tower.engine()
        emb = torch.empty((n, d.hidden), dtype=torch.float32, device=pixel_values.device)
        check(self._lib.pg_vit_forward_train(eng._handle, ptr(pixel_values), int(pixel_values.dtype == torch.float16), n,
                                             C.byref(self._saved), ptr(emb), current_stream_ptr()), "pg_vit_forward_train")
        return emb

    def _buckets(self):
        """Gradient buckets of the flat pending buffer in the order the backward completes them: encoder layers from the
        top down, then the embeddings.  (event slot, first element, one past the last element)"""
        g, d = self._pending_grads(), self.dims
        base = self._pending_flat.data_ptr()
        off = lambda t: (t.data_ptr() - base) // 4
        out = []
        emb_train, layers = self.layout()
        for l in reversed(range(d.layers)):
            if layers[l]:
                out.append((l, off(g[f"{l}.ln1_g"]), off(g[f"{l}.b_fc2"]) + g[f"{l}.b_fc2"].numel()))
        if emb_train:
            out.append((d.layers, off(g["patch_w"]), off(g["pre_ln_b"]) + g["pre_ln_b"].numel()))
        return out

    def cls_rows(self) -> torch.Tensor:
        """last_hidden_state[:, 0] of the views of the last forward, f32 [n, hidden] (a copy out of the arena): the CLS rows
        that CLIPModel feeds to post_layernorm and visual_projection."""
        if self._saved is None:
            raise PigeonB200Error("cls_rows() needs a preceding forward()")
        d, n = self.dims, self._saved_views
        nbytes = n * d.tokens * d.hidden * 4
        x = self._arena[self._x_out_off:self._x_out_off + nbytes].view(torch.float32).view(n, d.tokens, d.hidden)
        return x[:, 0].contiguous()

    @torch.no_grad()
    def backward(self, d_emb: torch.Tensor, overlap_world: int = 1) -> None:
        """d_emb f32 [n, hidden] for the views of the last forward; gradients accumulate in the pending buffers.

        overlap_world > 1 (the LAST chunk of a micro-batch under torch.distributed): each layer's gradient bucket is summed
        over the ranks by an NCCL all-reduce on a side stream as soon as pg_vit_backward reports the layer done, while the
        layers below are still in their backward; `finalize` then only waits for the outstanding buckets."""
        self._backward(d_emb, "pg_vit_backward", overlap_world)

    @torch.no_grad()
    def backward_cls(self, d_cls: torch.Tensor) -> None:
        """d_cls f32 [n, hidden]: gradient of the CLS rows (`cls_rows()`) of the views of the last forward (pg_vit_backward_cls);
        gradients accumulate in the pending buffers."""
        self._backward(d_cls, "pg_vit_backward_cls", 1)

    def _backward(self, d_emb: torch.Tensor, entry: str, overlap_world: int) -> None:
        d = self.dims
        n = self._saved_views
        if self._saved is None or d_emb.shape != (n, d.hidden):
            raise PigeonB200Error("backward() must follow forward() with one gradient row per view")
        d_emb = d_emb.to(torch.float32).contiguous()
        eng = self.tower.engine()
        wt = self._transposed_weights()
        g = self._pending_grads()
        emb_train, layers = self.layout()
        grads = _lib.VitGrads()
        if emb_train:
            grads.d_patch_w, grads.d_class_emb, grads.d_pos_emb = g["patch_w"].data_ptr(), g["class_emb"].data_ptr(), g["pos_emb"].data_ptr()
            grads.d_pre_ln_g, grads.d_pre_ln_b = g["pre_ln_g"].data_ptr(), g["pre_ln_b"].data_ptr()
        grads.layers_host = layers_bwd(wt, g, layers)
        events, ev_arr = None, None
        if overlap_world > 1:
            if getattr(self, "_bucket_events", None) is None:
                self._bucket_events = [torch.cuda.Event() for _ in range(d.layers + 1)]
                for e in self._bucket_events:
                    e.record()                                    # materialises the cudaEvent_t handle
                self._side = torch.cuda.Stream(device=d_emb.device)
            events = self._bucket_events
            ev_arr = (C.c_void_p * (d.layers + 1))(*[e.cuda_event for e in events])
            grads.layer_done_events = ev_arr
        ws = grow_aligned(self, "_ws", int(self._lib.pg_vit_backward_workspace_bytes(eng._handle, n)), d_emb.device)
        check(getattr(self._lib, entry)(eng._handle, C.byref(self._saved), ptr(d_emb), n, C.byref(grads), ptr(ws), ws.numel(),
                                        current_stream_ptr()), entry)
        if overlap_world > 1:
            self._works = []
            with torch.cuda.stream(self._side):
                for slot, lo, hi in self._buckets():
                    self._side.wait_event(events[slot])
                    self._works.append(torch.distributed.all_reduce(self._pending_flat[lo:hi], async_op=True))

    @torch.no_grad()
    def finalize(self, world: int = 1) -> None:
        """Pending fused gradients -> `param.grad` (accumulating), averaged over `world` ranks after a summing all-reduce."""
        if self._pending is None:
            return
        g, d = self._pending, self.dims
        if world > 1:                                  # DDP: average of the per-rank gradients (train_eval_loop.py:192)
            works, self._works = getattr(self, "_works", None), None
            if works:                                  # buckets already in flight behind the last chunk's backward
                for wk in works:
                    wk.wait()                          # the current stream waits for the NCCL stream
            else:
                torch.distributed.all_reduce(self._pending_flat)
            self._pending_flat.mul_(1.0 / world)
        vm = self.tower.vision_model
        put = put_grad
        if "patch_w" in g:
            e = vm.embeddings
            put(e.patch_embedding.weight, g["patch_w"][:, : d.patch_k].reshape(e.patch_embedding.weight.shape))
            put(e.class_embedding, g["class_emb"])
            put(e.position_embedding.weight, g["pos_emb"])
            put(vm.pre_layrnorm.weight, g["pre_ln_g"])
            put(vm.pre_layrnorm.bias, g["pre_ln_b"])
        for l, L in enumerate(vm.encoder.layers):
            if f"{l}.w_qkv" in g:
                put_layer_grads(L, g, l, d.hidden)
        self._pending = None
