"""torch.Tensor-level wrappers over the C ABI building blocks (tests, and callers that fuse differently).

Every function requires CUDA tensors and raises `PigeonB200Error` otherwise — there is no eager fallback.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import PigeonB200Error, check, current_stream_ptr, load, ptr


def _need_cuda(*ts: torch.Tensor) -> None:
    for t in ts:
        if t is not None and not t.is_cuda:
            raise PigeonB200Error("pigeon_b200 kernels need CUDA tensors (there is no CPU path)")
        if t is not None and not t.is_contiguous():
            raise PigeonB200Error("pigeon_b200 kernels need contiguous tensors")


def gemm_f16(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None, epilogue: int,
             out: torch.Tensor | None = None) -> torch.Tensor:
    """out = epilogue(a @ w.T + bias); a [M,K] fp16, w [N,K] fp16 (nn.Linear layout), fp32 accumulate."""
    _need_cuda(a, w, bias, out)
    assert a.dtype == torch.float16 and w.dtype == torch.float16 and a.shape[1] == w.shape[1]
    M, K = a.shape
    N = w.shape[0]
    if out is None:
        assert epilogue != _lib.EPI_F32_BIAS_RESID, "residual epilogue accumulates into `out`"
        dt = torch.float16 if epilogue in (_lib.EPI_F16_BIAS, _lib.EPI_F16_BIAS_QGELU) else torch.float32
        out = torch.empty((M, N), dtype=dt, device=a.device)
    check(load().pg_gemm_f16(ptr(a), a.stride(0), ptr(w), w.stride(0), ptr(out), out.stride(0), ptr(bias), M, N, K,
                             epilogue, current_stream_ptr()), "pg_gemm_f16")
    return out


def gemm_set_schedule(mode: int) -> None:
    """Kernel of every K-major GEMM, process-wide: 0 = automatic (128 x 256 for the fp16-output projections, else
    ping-pong), 1 = the single-warpgroup kernel, 2 = the ping-pong kernel (all the same bits)."""
    check(load().pg_gemm_set_schedule(int(mode)), "pg_gemm_set_schedule")


def layernorm_f16(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float) -> torch.Tensor:
    _need_cuda(x, gamma, beta)
    assert x.dtype == torch.float32
    rows, hidden = x.reshape(-1, x.shape[-1]).shape
    y = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    check(load().pg_layernorm_f16(ptr(x), ptr(y), ptr(gamma), ptr(beta), rows, hidden, eps, current_stream_ptr()),
          "pg_layernorm_f16")
    return y


def attention_f16(qkv: torch.Tensor, n_views: int, seq: int, heads: int, variant: int | None = None,
                  poly: int = -1, return_lse2: bool = False):
    """qkv fp16 [n_views*seq, 3*heads*64] -> fp16 [n_views*seq, heads*64].

    `variant` (0..3) and `poly` are kept from earlier ABI versions that had several forward kernels; the sm_90a library
    has one, and every value runs it.  None = pg_attention_f16.  `return_lse2` (with an explicit variant): also the log2-domain log-sum-exp of the scaled
    logits, f32 [n_views*heads, seq], the side output the training forward keeps for the backward pass."""
    _need_cuda(qkv)
    assert qkv.dtype == torch.float16 and qkv.shape == (n_views * seq, 3 * heads * 64)
    out = torch.empty((n_views * seq, heads * 64), dtype=torch.float16, device=qkv.device)
    lse2 = torch.empty((n_views * heads, seq), dtype=torch.float32, device=qkv.device) if return_lse2 else None
    if variant is None:
        if return_lse2:
            raise ValueError("return_lse2 needs an explicit variant (pg_attention_f16 has no lse2 argument)")
        check(load().pg_attention_f16(ptr(qkv), ptr(out), n_views, seq, heads, current_stream_ptr()), "pg_attention_f16")
    else:
        check(load().pg_attention_f16_variant(ptr(qkv), ptr(out), ptr(lse2) if return_lse2 else None, n_views, seq, heads,
                                              variant, poly, current_stream_ptr()), "pg_attention_f16_variant")
    return (out, lse2) if return_lse2 else out


def attention_f16_masked(qkv: torch.Tensor, n_views: int, seq: int, heads: int, mask: torch.Tensor | None = None,
                         causal: bool = False) -> torch.Tensor:
    """The text tower's attention: qkv fp16 [n_views*seq, 3*heads*64] -> fp16 [n_views*seq, heads*64] with key j admissible
    for query i only if (not causal or j <= i) and mask[view, j] != 0; mask i64 [n_views, seq] or None (mask[:, 0] must be
    1).  No mask and causal=False is `attention_f16`."""
    if mask is not None:
        mask = mask.to(torch.int64).contiguous()
    _need_cuda(qkv, mask)
    assert qkv.dtype == torch.float16 and qkv.shape == (n_views * seq, 3 * heads * 64)
    assert mask is None or mask.shape == (n_views, seq)
    out = torch.empty((n_views * seq, heads * 64), dtype=torch.float16, device=qkv.device)
    check(load().pg_attention_f16_masked(ptr(qkv), ptr(out), ptr(mask), int(bool(causal)), n_views, seq, heads,
                                         current_stream_ptr()), "pg_attention_f16_masked")
    return out


def attention_f16_masked_lse(qkv: torch.Tensor, n_views: int, seq: int, heads: int, mask: torch.Tensor | None = None,
                             causal: bool = False):
    """`attention_f16_masked` plus lse2 f32 [n_views*heads, seq] (log2-sum-exp over the admissible keys), the side output the
    text tower's training forward keeps for the backward pass -> (out, lse2)."""
    if mask is not None:
        mask = mask.to(torch.int64).contiguous()
    _need_cuda(qkv, mask)
    assert qkv.dtype == torch.float16 and qkv.shape == (n_views * seq, 3 * heads * 64)
    assert mask is None or mask.shape == (n_views, seq)
    out = torch.empty((n_views * seq, heads * 64), dtype=torch.float16, device=qkv.device)
    lse2 = torch.empty((n_views * heads, seq), dtype=torch.float32, device=qkv.device)
    check(load().pg_attention_f16_masked_lse(ptr(qkv), ptr(out), ptr(lse2), ptr(mask), int(bool(causal)), n_views, seq, heads,
                                             current_stream_ptr()), "pg_attention_f16_masked_lse")
    return out, lse2


def attention_backward_masked(qkv: torch.Tensor, out: torch.Tensor, d_out: torch.Tensor, lse2: torch.Tensor, n_views: int,
                              seq: int, heads: int, mask: torch.Tensor | None = None, causal: bool = False) -> torch.Tensor:
    """Backward of `attention_f16_masked_lse`: qkv / out fp16, d_out f32 [n_views*seq, heads*64] -> dqkv bf16
    [n_views*seq, 3*heads*64].  No mask and causal=False runs pg_attention_backward's kernels."""
    if mask is not None:
        mask = mask.to(torch.int64).contiguous()
    d_out = d_out.to(torch.float32).contiguous()
    _need_cuda(qkv, out, d_out, lse2, mask)
    lib = load()
    dqkv = torch.empty((n_views * seq, 3 * heads * 64), dtype=torch.bfloat16, device=qkv.device)
    ws = torch.empty(int(lib.pg_attention_backward_workspace_bytes(n_views, seq, heads)) + 256, dtype=torch.uint8,
                     device=qkv.device)
    ws = ws[(-ws.data_ptr()) % 256:]
    check(lib.pg_attention_backward_masked(ptr(qkv), ptr(out), ptr(d_out), ptr(lse2), ptr(mask), int(bool(causal)), ptr(dqkv),
                                           n_views, seq, heads, ptr(ws), ws.numel(), current_stream_ptr()),
          "pg_attention_backward_masked")
    return dqkv


def layernorm_f32(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float) -> torch.Tensor:
    """fp32 LayerNorm over the last dim: x f32 [rows, hidden] -> f32 [rows, hidden]."""
    _need_cuda(x, gamma, beta)
    assert x.dtype == torch.float32
    rows, hidden = x.reshape(-1, x.shape[-1]).shape
    y = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    check(load().pg_layernorm_f32(ptr(x), ptr(y), ptr(gamma), ptr(beta), rows, hidden, eps, current_stream_ptr()),
          "pg_layernorm_f32")
    return y


def clip_loss_grad(image_embeds: torch.Tensor, text_embeds: torch.Tensor, logit_scale: torch.Tensor,
                   grad_scale: float = 1.0) -> dict:
    """HF `clip_loss(logits_per_text)` and its gradient for n images and n captions: image_embeds, text_embeds f32 [n, P]
    (not normalised), logit_scale f32 scalar CUDA tensor -> dict(loss [], d_image_embeds [n, P], d_text_embeds [n, P],
    d_logit_scale [], logits_per_image [n, n], logits_per_text [n, n]); gradients times grad_scale."""
    img = image_embeds.to(torch.float32).contiguous()
    txt = text_embeds.to(torch.float32).contiguous()
    ls = logit_scale.detach().to(torch.float32).reshape(()).contiguous()
    _need_cuda(img, txt, ls)
    n, P = img.shape
    if tuple(txt.shape) != (n, P):
        raise ValueError(f"the contrastive loss needs as many images as captions of one width (got {tuple(img.shape)} images, "
                         f"{tuple(txt.shape)} captions)")
    lib = load()
    dev = img.device
    out = dict(loss=torch.empty((), dtype=torch.float32, device=dev), d_image_embeds=torch.empty_like(img),
               d_text_embeds=torch.empty_like(txt), d_logit_scale=torch.empty((), dtype=torch.float32, device=dev),
               logits_per_image=torch.empty((n, n), dtype=torch.float32, device=dev),
               logits_per_text=torch.empty((n, n), dtype=torch.float32, device=dev))
    if n == 0:
        return out
    ws = torch.empty(int(lib.pg_clip_loss_grad_workspace_bytes(n, P)), dtype=torch.uint8, device=dev)
    check(lib.pg_clip_loss_grad(ptr(img), ptr(txt), n, P, ptr(ls), float(grad_scale), ptr(ws), ws.numel(), ptr(out["loss"]),
                                ptr(out["d_image_embeds"]), ptr(out["d_text_embeds"]), ptr(out["d_logit_scale"]),
                                ptr(out["logits_per_image"]), ptr(out["logits_per_text"]), current_stream_ptr()),
          "pg_clip_loss_grad")
    return out


def grad_norm_clip(grad: torch.Tensor, max_norm: float, grad_scale: float = 1.0,
                   workspace: torch.Tensor | None = None):
    """`torch.nn.utils.clip_grad_norm_` over one flat fp32 CUDA gradient read as grad * grad_scale, without modifying it:
    -> (total_norm, clip_coef), two f32 CUDA scalars (clip_coef = min(max_norm / (total_norm + 1e-6), 1)); no host sync.
    Deterministic.  A non-finite norm passes through (inf -> clip_coef 0, NaN -> NaN), as torch does."""
    _need_cuda(grad, workspace)
    if grad.dtype != torch.float32:
        raise PigeonB200Error("grad_norm_clip needs an fp32 gradient")
    lib = load()
    n = grad.numel()
    need = int(lib.pg_grad_norm_clip_workspace_bytes(n))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=grad.device)
    out = torch.empty(2, dtype=torch.float32, device=grad.device)
    check(lib.pg_grad_norm_clip(ptr(grad), n, float(grad_scale), float(max_norm), ptr(out[0]), ptr(out[1]), ptr(workspace),
                                workspace.numel(), current_stream_ptr()), "pg_grad_norm_clip")
    return out[0], out[1]


def adamw_hf_step(param: torch.Tensor, grad: torch.Tensor, exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, step: int,
                  lr: float, betas=(0.9, 0.999), eps: float = 1e-6, weight_decay: float = 0.0, grad_scale: float = 1.0,
                  clip_coef: torch.Tensor | None = None) -> None:
    """transformers.optimization.AdamW.step (4.23.1, correct_bias=True) in place on one contiguous fp32 CUDA tensor;
    `clip_coef` is an f32 CUDA scalar (None = 1), `step` counts from 1."""
    _need_cuda(param, grad, exp_avg, exp_avg_sq, clip_coef)
    if any(t.dtype != torch.float32 for t in (param, grad, exp_avg, exp_avg_sq)):
        raise PigeonB200Error("adamw_hf_step needs fp32 parameter, gradient and state")
    if not (param.numel() == grad.numel() == exp_avg.numel() == exp_avg_sq.numel()):
        raise PigeonB200Error("adamw_hf_step: parameter, gradient and state sizes differ")
    check(load().pg_adamw_hf_step(ptr(param), ptr(grad), ptr(exp_avg), ptr(exp_avg_sq), param.numel(), float(lr),
                                  float(betas[0]), float(betas[1]), float(eps), float(weight_decay), int(step),
                                  float(grad_scale), ptr(clip_coef), current_stream_ptr()), "pg_adamw_hf_step")


def clip_project(x: torch.Tensor, w3: torch.Tensor, ln_weight: torch.Tensor | None = None,
                 ln_bias: torch.Tensor | None = None, eps: float = 1e-5) -> torch.Tensor:
    """x f32 [n, D] -> f32 [n, P] = LN(x) W^T (LN only when ln_weight / ln_bias are given), W packed by `head_pack_weight`
    into w3 fp16 [P, 3*D]: the error-compensated split GEMM of the geocell head (visual_projection / text_projection)."""
    _need_cuda(x, w3, ln_weight, ln_bias)
    if (ln_weight is None) != (ln_bias is None):
        raise ValueError("ln_weight and ln_bias go together")
    assert x.dtype == torch.float32 and x.dim() == 2 and w3.dtype == torch.float16
    n, D = x.shape
    P = w3.shape[0]
    if w3.shape[1] != 3 * D:
        raise PigeonB200Error(f"packed weight {tuple(w3.shape)} does not match input dim {D}")
    lib = load()
    out = torch.empty((n, P), dtype=torch.float32, device=x.device)
    if n == 0:
        return out
    ws = torch.empty(lib.pg_clip_project_workspace_bytes(n, D), dtype=torch.uint8, device=x.device)
    check(lib.pg_clip_project(ptr(x), n, D, ptr(ln_weight), ptr(ln_bias), float(eps), ptr(w3), P, ptr(ws), ws.numel(),
                              ptr(out), current_stream_ptr()), "pg_clip_project")
    return out


def clip_logits(image_embeds: torch.Tensor, text_embeds: torch.Tensor, logit_scale: float, per_text: bool = True,
                probs: bool = False, pred: bool = False, loss: bool = False) -> dict:
    """CLIPModel's logits from UNnormalised embeds (normalised inside): image_embeds f32 [Ni, P], text_embeds f32 [Nt, P]
    -> dict(logits_per_image [Ni, Nt] and, on request, logits_per_text [Nt, Ni], probs [Ni, Nt] (softmax over captions),
    pred i64 [Ni] (first argmax), loss f32 [] (symmetric cross-entropy against arange; needs Ni == Nt))."""
    img = image_embeds.to(torch.float32).contiguous()
    txt = text_embeds.to(torch.float32).contiguous()
    _need_cuda(img, txt)
    Ni, P = img.shape
    Nt = txt.shape[0]
    if txt.shape[1] != P:
        raise ValueError(f"image embeds have dim {P}, text embeds {txt.shape[1]}")
    if loss and Ni != Nt:
        raise ValueError(f"the contrastive loss needs as many images as captions (got {Ni} images, {Nt} captions)")
    dev = img.device
    out = dict(logits_per_image=torch.empty((Ni, Nt), dtype=torch.float32, device=dev))
    if per_text:
        out["logits_per_text"] = torch.empty((Nt, Ni), dtype=torch.float32, device=dev)
    if probs:
        out["probs"] = torch.empty((Ni, Nt), dtype=torch.float32, device=dev)
    if pred:
        out["pred"] = torch.empty((Ni,), dtype=torch.int64, device=dev)
    if loss:
        out["loss"] = torch.empty((), dtype=torch.float32, device=dev)
    check(load().pg_clip_logits(ptr(img), Ni, ptr(txt), Nt, P, float(logit_scale), ptr(out["logits_per_image"]),
                                ptr(out.get("logits_per_text")), ptr(out.get("probs")), ptr(out.get("pred")),
                                ptr(out.get("loss")), current_stream_ptr()), "pg_clip_logits")
    return out


def refiner_scan(bank: "DeviceBank", emb: torch.Tensor, cand_idx: torch.Tensor, topk: int):
    """Scan stage only (cell-sharded banks): per (query, candidate) partials (best_logit [B, topk], best_lnglat
    [B, topk, 2], best_proto [B, topk]); pairs whose geocell this bank does not hold come back as -100000 / (0, 0) / -1."""
    import ctypes as C
    if emb.dim() == 2:
        emb = emb.unsqueeze(1)
    emb = emb.to(torch.float32).contiguous()
    cand_idx = cand_idx.to(torch.int64).contiguous()
    _need_cuda(emb, cand_idx)
    B, V, D = emb.shape
    if D != bank.dim:
        raise PigeonB200Error(f"embedding dim {D} != bank dim {bank.dim}")
    dev = emb.device
    lib = load()
    ws = torch.empty(lib.pg_refiner_workspace_bytes(B, topk, D, bank.num_cells), dtype=torch.uint8, device=dev)
    bl = torch.empty((B, topk), dtype=torch.float32, device=dev)
    bll = torch.empty((B, topk, 2), dtype=torch.float32, device=dev)
    bp = torch.empty((B, topk), dtype=torch.int32, device=dev)
    check(lib.pg_refiner_scan(C.byref(bank.c_struct), ptr(emb), B, V, ptr(cand_idx), cand_idx.shape[1], topk, ptr(ws),
                              ws.numel(), ptr(bl), ptr(bll), ptr(bp), current_stream_ptr()), "pg_refiner_scan")
    return bl, bll, bp


def refiner_finalize(best_logit: torch.Tensor, best_lnglat: torch.Tensor, init_lnglat: torch.Tensor,
                     cand_idx: torch.Tensor, cand_prob: torch.Tensor, topk: int, temperature: float,
                     max_refinement_km: float):
    """Final stage on merged partials -> (preds_LLH f32 [B, 2], preds_geocell i64 [B], choice i32 [B])."""
    best_logit = best_logit.to(torch.float32).contiguous()
    best_lnglat = best_lnglat.to(torch.float32).contiguous()
    init_lnglat = init_lnglat.to(torch.float64).contiguous()
    cand_idx = cand_idx.to(torch.int64).contiguous()
    cand_prob = cand_prob.to(torch.float32).contiguous()
    _need_cuda(best_logit, best_lnglat, init_lnglat, cand_idx, cand_prob)
    B = best_logit.shape[0]
    dev = best_logit.device
    out_ll = torch.empty((B, 2), dtype=torch.float32, device=dev)
    out_cell = torch.empty((B,), dtype=torch.int64, device=dev)
    choice = torch.empty((B,), dtype=torch.int32, device=dev)
    check(load().pg_refiner_finalize(ptr(best_logit), ptr(best_lnglat), ptr(init_lnglat), ptr(cand_idx), ptr(cand_prob),
                                     cand_idx.shape[1], B, topk, float(temperature), float(max_refinement_km),
                                     ptr(out_ll), ptr(out_cell), ptr(choice), current_stream_ptr()),
          "pg_refiner_finalize")
    return out_ll, out_cell, choice


def head_set_fused(on: bool) -> None:
    """A/B switch of the geocell head: False (default) three kernels, True the single fused kernel (same results)."""
    check(load().pg_head_set_fused(1 if on else 0), "pg_head_set_fused")


def refiner_set_schedule(mode: int) -> None:
    """A/B switch of the refiner scan: 0 automatic, 1 query-major, 2 cell-major, 3 tile scan, 4 slab scan (same selections)."""
    check(load().pg_refiner_set_schedule(int(mode)), "pg_refiner_set_schedule")


def head_pack_weight(weight: torch.Tensor) -> torch.Tensor:
    """cell_layer.weight f32 [C, D] -> fp16 [C, 3*D] error-compensated split consumed by `head_forward`."""
    _need_cuda(weight)
    w = weight.detach().to(torch.float32).contiguous()
    C_, D = w.shape
    w3 = torch.empty((C_, 3 * D), dtype=torch.float16, device=w.device)
    check(load().pg_head_pack_weight(ptr(w), ptr(w3), C_, D, current_stream_ptr()), "pg_head_pack_weight")
    return w3


def head_forward(emb: torch.Tensor, w3: torch.Tensor, bias: torch.Tensor, centroids: torch.Tensor, k: int):
    """emb f32 [B, V, D] -> dict(pooled, logits, probs, pred_cell, pred_lnglat, topk_val, topk_idx)."""
    _need_cuda(emb, w3, bias, centroids)
    assert emb.dtype == torch.float32 and emb.dim() == 3
    assert centroids.dtype == torch.float64 and bias.dtype == torch.float32
    B, V, D = emb.shape
    C_ = w3.shape[0]
    dev = emb.device
    lib = load()
    ws = torch.empty(lib.pg_head_workspace_bytes(B, D), dtype=torch.uint8, device=dev)
    out = dict(
        pooled=torch.empty((B, D), dtype=torch.float32, device=dev),
        logits=torch.empty((B, C_), dtype=torch.float32, device=dev),
        probs=torch.empty((B, C_), dtype=torch.float32, device=dev),
        pred_cell=torch.empty((B,), dtype=torch.int64, device=dev),
        pred_lnglat=torch.empty((B, 2), dtype=torch.float64, device=dev),
        topk_val=torch.empty((B, k), dtype=torch.float32, device=dev),
        topk_idx=torch.empty((B, k), dtype=torch.int64, device=dev),
    )
    check(lib.pg_head_forward(ptr(emb), B, V, D, ptr(w3), ptr(bias), ptr(centroids), C_, k, ptr(ws), ws.numel(),
                              ptr(out["pooled"]), ptr(out["logits"]), ptr(out["probs"]), ptr(out["pred_cell"]),
                              ptr(out["pred_lnglat"]), ptr(out["topk_val"]), ptr(out["topk_idx"]),
                              current_stream_ptr()), "pg_head_forward")
    return out


def view_attention_forward(emb: torch.Tensor, pe: torch.Tensor, w_in3: torch.Tensor, b_in: torch.Tensor,
                           w_out3: torch.Tensor, b_out: torch.Tensor, heads: int = 16, n0: int = 0, p_x: float = 0.0,
                           p_attn: float = 0.0, seed: int = 0, offset: int = 0, return_masks: bool = False) -> dict:
    """The hierarchical head's view self-attention (pg_view_attn_forward): emb f32 [N, 4, E], pe = pos_encoder.pos_encoding
    f32 [rows, 1, E] (sample n uses row n0 + n), in_proj / out_proj packed by `head_pack_weight` -> dict(cls f32 [N, E],
    saved f32 (what `view_attention_backward` reads; `view_attention_saved` names its parts)) and, with `return_masks`,
    mask_x bool [N, 4, E] and mask_p bool [N, heads, 4]: where the two dropouts kept the element."""
    _need_cuda(emb, pe, w_in3, b_in, w_out3, b_out)
    if emb.dtype != torch.float32 or emb.dim() != 3 or emb.shape[1] != 4:
        raise PigeonB200Error(f"view attention needs f32 embeddings [N, 4, E], got {emb.dtype} {tuple(emb.shape)}")
    N, _, E = emb.shape
    if pe.shape[-1] != E or w_in3.shape != (3 * E, 3 * E) or w_out3.shape != (E, 3 * E):
        raise PigeonB200Error(f"view attention weights {tuple(w_in3.shape)}, {tuple(w_out3.shape)} or positional encoding "
                              f"{tuple(pe.shape)} do not match E = {E}")
    lib = load()
    dev = emb.device
    saved = torch.empty(max(1, lib.pg_view_attn_saved_floats(N, E, heads)), dtype=torch.float32, device=dev)
    ws = torch.empty(max(1, lib.pg_view_attn_workspace_bytes(N, E)), dtype=torch.uint8, device=dev)
    cls = torch.empty((N, E), dtype=torch.float32, device=dev)
    mask_x = torch.empty((N, 4, E), dtype=torch.uint8, device=dev) if return_masks else None
    mask_p = torch.empty((N, heads, 4), dtype=torch.uint8, device=dev) if return_masks else None
    check(lib.pg_view_attn_forward(ptr(emb), N, E, heads, ptr(pe), pe.shape[0], n0, ptr(w_in3), ptr(b_in), ptr(w_out3),
                                   ptr(b_out), float(p_x), float(p_attn), int(seed), int(offset), ptr(ws), ws.numel(),
                                   ptr(saved), ptr(mask_x), ptr(mask_p), ptr(cls), current_stream_ptr()),
          "pg_view_attn_forward")
    out = dict(cls=cls, saved=saved)
    if return_masks:
        out.update(mask_x=mask_x.bool(), mask_p=mask_p.bool())
    return out


def view_attention_saved(saved: torch.Tensor, N: int, E: int, heads: int = 16) -> dict:
    """Named views of `view_attention_forward`'s saved activations: x [N, 4, E] (after the positional encoding and its
    dropout), q0 [N, E], k [N, 4, E], v [N, 4, E], o [N, E] (attention output before out_proj), probs [N, heads, 4]."""
    ne = N * E
    kv = saved[5 * ne:13 * ne].view(N, 4, 2 * E)
    return dict(x=saved[:4 * ne].view(N, 4, E), q0=saved[4 * ne:5 * ne].view(N, E), k=kv[..., :E], v=kv[..., E:],
                o=saved[13 * ne:14 * ne].view(N, E), probs=saved[14 * ne:14 * ne + 4 * N * heads].view(N, heads, 4))


def view_attention_backward(dcls: torch.Tensor, saved: torch.Tensor, w_in: torch.Tensor, w_out: torch.Tensor,
                            heads: int = 16, n0: int = 0, p_x: float = 0.0, p_attn: float = 0.0, seed: int = 0,
                            offset: int = 0, grads=None, accumulate: bool = False) -> torch.Tensor:
    """Backward of `view_attention_forward` (same n0, dropout probabilities, seed and offset): dcls f32 [N, E] -> d emb
    f32 [N, 4, E].  `grads` = (d in_proj_weight [3E, E], d in_proj_bias [3E], d out_proj.weight [E, E], d out_proj.bias [E])
    f32 tensors written, or added into with `accumulate` (entries may be None)."""
    dcls = dcls.to(torch.float32).contiguous()
    w_in, w_out = w_in.detach().contiguous(), w_out.detach().contiguous()
    grads = tuple(grads) if grads is not None else (None,) * 4
    _need_cuda(dcls, saved, w_in, w_out, *grads)
    N, E = dcls.shape
    lib = load()
    dev = dcls.device
    ws = torch.empty(max(1, lib.pg_view_attn_workspace_bytes(N, E)), dtype=torch.uint8, device=dev)
    demb = torch.empty((N, 4, E), dtype=torch.float32, device=dev)
    check(lib.pg_view_attn_backward(ptr(dcls), N, E, heads, n0, ptr(w_in), ptr(w_out), ptr(saved), float(p_x),
                                    float(p_attn), int(seed), int(offset), int(bool(accumulate)), *(ptr(g) for g in grads),
                                    ptr(demb), ptr(ws), ws.numel(), current_stream_ptr()), "pg_view_attn_backward")
    return demb


class DeviceBank:
    """CSR prototype bank resident in HBM (layout of `pg_refiner_bank`, include/pigeon_b200.h)."""

    FIELDS = ("cell_off", "proto_emb", "proto_lnglat", "proto_count", "member_off", "member_idx", "data_emb",
              "data_lnglat")
    DTYPES = dict(cell_off=torch.int64, proto_emb=torch.float32, proto_lnglat=torch.float32, proto_count=torch.int32,
                  member_off=torch.int64, member_idx=torch.int64, data_emb=torch.float32, data_lnglat=torch.float32)

    def __init__(self, device, **arrays):
        self.device = torch.device(device)
        for f in self.FIELDS:
            t = torch.as_tensor(arrays[f]).to(device=self.device, dtype=self.DTYPES[f]).contiguous()
            if t.numel() == 0:  # keep a valid (never dereferenced) pointer for empty arrays
                t = torch.zeros((1,) + tuple(t.shape[1:]), dtype=t.dtype, device=self.device)
            setattr(self, f, t)
        self.num_cells = int(arrays["cell_off"].shape[0]) - 1
        self.dim = int(self.proto_emb.shape[1])
        # |p|^2 per prototype, once per bank: the tile scan (schedule 3) scores in the |p|^2 + |q|^2 - 2 p.q form
        self.proto_sqnorm = None
        P = int(arrays["proto_emb"].shape[0])
        if self.device.type == "cuda" and P > 0:
            self.proto_sqnorm = torch.empty(P, dtype=torch.float32, device=self.device)
            with torch.cuda.device(self.device):
                check(load().pg_refiner_bank_sqnorm(ptr(self.proto_emb), P, self.dim, ptr(self.proto_sqnorm),
                                                    current_stream_ptr()), "pg_refiner_bank_sqnorm")
        self.c_struct = _lib.RefinerBank(self.num_cells, self.dim, *(ptr(getattr(self, f)) for f in self.FIELDS),
                                         ptr(self.proto_sqnorm) if self.proto_sqnorm is not None else None, P,
                                         int((self.cell_off[1:] > self.cell_off[:-1]).sum().item()))


def refiner_forward(bank: DeviceBank, emb: torch.Tensor, init_lnglat: torch.Tensor, cand_idx: torch.Tensor,
                    cand_prob: torch.Tensor, topk: int, temperature: float, max_refinement_km: float,
                    debug: bool = False):
    """ProtoRefiner.forward on the GPU. emb f32 [B, D] or [B, V, D]; returns (preds_LLH f32 [B,2], preds_geocell i64 [B])
    and, with `debug`, a dict of the per-candidate intermediates."""
    import ctypes as C
    if emb.dim() == 2:
        emb = emb.unsqueeze(1)
    emb = emb.to(torch.float32).contiguous()
    init_lnglat = init_lnglat.to(torch.float64).contiguous()
    cand_idx = cand_idx.to(torch.int64).contiguous()
    cand_prob = cand_prob.to(torch.float32).contiguous()
    _need_cuda(emb, init_lnglat, cand_idx, cand_prob)
    B, V, D = emb.shape
    if D != bank.dim:
        raise PigeonB200Error(f"embedding dim {D} != bank dim {bank.dim}")
    stride = cand_idx.shape[1]
    dev = emb.device
    lib = load()
    ws = torch.empty(lib.pg_refiner_workspace_bytes(B, topk, D, bank.num_cells), dtype=torch.uint8, device=dev)
    out_ll = torch.empty((B, 2), dtype=torch.float32, device=dev)
    out_cell = torch.empty((B,), dtype=torch.int64, device=dev)
    dbg = None
    if debug:
        dbg = dict(best_logit=torch.empty((B, topk), dtype=torch.float32, device=dev),
                   best_lnglat=torch.empty((B, topk, 2), dtype=torch.float32, device=dev),
                   best_proto=torch.empty((B, topk), dtype=torch.int32, device=dev),
                   choice=torch.empty((B,), dtype=torch.int32, device=dev))
    check(lib.pg_refiner_forward(C.byref(bank.c_struct), ptr(emb), B, V, ptr(init_lnglat), ptr(cand_idx),
                                 ptr(cand_prob), stride, topk, float(temperature), float(max_refinement_km), ptr(ws),
                                 ws.numel(), ptr(out_ll), ptr(out_cell),
                                 ptr(dbg["best_logit"]) if dbg else None, ptr(dbg["best_lnglat"]) if dbg else None,
                                 ptr(dbg["best_proto"]) if dbg else None, ptr(dbg["choice"]) if dbg else None,
                                 current_stream_ptr()), "pg_refiner_forward")
    return (out_ll, out_cell, dbg) if debug else (out_ll, out_cell)
