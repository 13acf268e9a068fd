"""fp64 references and per-element error bounds for the geocell head (csrc/head.cu, csrc/head_fused_wgmma.cu) and the
fp32 backward of its Linear (csrc/train.cu).

Every function takes the operands the kernels read, computes the operation in float64 on whatever device they live on, and
returns the result together with a bound B such that |kernel - reference| <= B element by element.

Notation: u = 2^-24 (fp32 unit roundoff), gamma_n = n u / (1 - n u) (a chain of n roundings, Higham).

View mean (view_mean_split_kernel, and the A-operand producer of head_fused_kernel): both add the V views in order from 0.f
and divide by V, as `view_mean_f32` does in fp32.  The kernels' pooled output is therefore checked bit for bit against it;
against the fp64 mean it is within gamma_V sum_v |emb_v| / V.

Logits.  Both paths evaluate x.W^T + b, x the fp32 pooled row and W the fp32 weight, as one fp16 GEMM with K = 3D:
    hi = rn16(x), lo = rn16(x - hi), Whi = rn16(W), Wlo = rn16(W - Whi),   S = hi.Whi + lo.Whi + hi.Wlo.
  * Split error, per term.  x - hi is exact in fp32.  If hi is normal, |x - hi| <= 2^-11 |x| and lo adds a relative 2^-11
    of that, or 2^-25 absolute once lo falls below 2^-14 (fp16 subnormal spacing 2^-24); if hi itself is subnormal,
    |x - hi| <= 2^-25 and lo is 0 or 2^-24.  So x = hi + lo + e_x with |e_x| <= 1.001 * 2^-22 |x| + 2^-25 (and |e_x| <= |x|),
    |lo| <= 1.001 * 2^-11 |x| + 2^-25, and likewise for W.  Then
        x W - (hi Whi + lo Whi + hi Wlo) = lo Wlo + e_x W + e_W (x - e_x),
    whose size is at most 3.01 * 2^-22 |x W| + 1.01 * 2^-25 (|x| + |W|): the first part from lo Wlo, e_x W and e_W x, the
    floor from the 2^-25 parts of e_x and e_W (the cross terms are 2^-11 of these).  Below 2^-3 the lo parts are fp16
    subnormals, and from there on this floor, not 2^-22 relative, is what a term keeps.
  * Accumulation.  The 3D fp16 products are exact in fp32.  The tensor cores add them into the fp32 accumulator 16 at a
    time (one wgmma k-step) and round toward zero, so each step can lose up to one fp32 ulp of the accumulator, 2^-23 |acc|,
    and |acc| <= sum_d |x_d W_cd| (1 + 2^-10) over the whole chain (the lo terms add at most 2^-10 of it).  With
    n = 3D / 16 steps:  n 2^-23 (1 + 2^-10) sum_d |x_d W_cd|.  The truncation does not average out when the partial sums
    keep their sign, so this is a worst case, not a random walk.
  * The bias is added once in fp32: u (|ref| + the bound above).
    Together: |logit' - logit| <= alpha sum_d |x_d W_cd| + 1.01 * 2^-25 (sum_d |x_d| + sum_d |W_cd|) + u (|logit| + ...),
    alpha = 3.01 * 2^-22 + (3D / 16) 2^-23 (1 + 2^-10).   Plain fp16 operands (no lo terms) miss by 2^-12 |x W| per term
    on average, and dropping any one of the three products by 2^-13: far above alpha at every D up to 256 and still above it
    at D = 1024 in the largest elements.

Probabilities (softmax_topk_kernel, and the last-CTA rows of head_fused_kernel): p_c = expf(x_c - m) / s, s = sum_c expf(..)
in fp32, m the row maximum.  With L_c the logit bound above, the reference row is shifted by at most
sum_c p_c L_c in its log-sum-exp; x_c - m rounds once (u |x_c - m|), expf is within 2 ulp (4u relative), the sum of the
exponentials adds gamma_n relative (n = ceil(C / 32) + 13 covers both kernels' per-lane chains, shuffle trees and the
8-warp tail) and the division one more u:
    |p' - p| <= p expm1(1.01 (L_c + sum_c' p_c' (L_c' + u |x_c' - m| + 4u) + gamma_n + u |x_c - m| + 6u)) + 2^-126.
The top-k ranks the probabilities the kernel writes, so it is checked EXACTLY against `stable_topk` of the kernel's own
probs (descending, first index on ties, NaN first); against the fp64 probabilities it is exact at every rank whose margin
exceeds the bounds (`safe_ranks`).

Loss (ce_loss_kernel) is evaluated in fp64 from the fp32 logits, so the reference matches it to a few fp64 ulps of the
terms: 1e-13 sum_c t_c (|lse| + |x_c|), plus for the haversine targets the relative error of t_c = exp(-(d_c - d_min) / s)
from fp64 distances that are within 1e-13 (d + 1) km: 4e-13 (20038 + 1) / s.  The gradient is that fp64 value rounded to
fp32: u |g| + the fp64 part + 2^-149; for the haversine targets the kernel keeps t in the fp32 gradient row until sum t is
known, which adds u (p sum t + t) scaled like the gradient.

Backward (sgemm_kernel: one fmaf per k in order, then fmaf(beta, c, acc) when accumulating; column_sum_kernel: rows in
order, then one fmaf): gamma_{K+1} (sum_k |a_k b_k| + |c0|), K the reduction length.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24
FLOOR16 = 2.0 ** -25          # half the fp16 subnormal spacing


def gamma(n) -> float:
    n = float(n)
    return n * U / (1.0 - n * U)


def view_mean_f32(emb: torch.Tensor) -> torch.Tensor:
    """[B, V, D] fp32 -> [B, D] fp32: views added in order from 0, then divided by V (the kernels' arithmetic)."""
    s = torch.zeros(emb.shape[0], emb.shape[2], dtype=torch.float32, device=emb.device)
    for v in range(emb.shape[1]):
        s = s + emb[:, v]
    # a true division: torch turns a division by a Python scalar into a multiply by its reciprocal on CUDA, which differs
    # from the kernels' s / V for V = 7
    return s / torch.full_like(s, emb.shape[1])


def view_mean(emb: torch.Tensor):
    """fp64 mean over the views and its bound for any fp32 evaluation that adds the views in order and divides once."""
    e = emb.double()
    V = emb.shape[1]
    return e.mean(1), gamma(V) * e.abs().sum(1) / V


def split_f16(x: torch.Tensor):
    """fp32 -> (hi, lo) fp16 with hi = rn(x), lo = rn(x - hi) (torch's fp16 cast rounds to nearest even, like
    __float2half_rn)."""
    x = x.float()
    hi = x.half()
    lo = (x - hi.float()).half()
    return hi, lo


def split_operands(x: torch.Tensor, W: torch.Tensor):
    """The GEMM's operands: a3 = [hi | lo | hi] [B, 3D] and w3 = [Whi | Whi | Wlo] [C, 3D], fp16."""
    hi, lo = split_f16(x)
    whi, wlo = split_f16(W)
    return torch.cat([hi, lo, hi], 1), torch.cat([whi, whi, wlo], 1)


def alpha(D: int) -> float:
    """Relative part of the logit bound (module docstring): split error plus truncating accumulation over 3D / 16 steps."""
    return 3.01 * 2.0 ** -22 + (3 * D / 16) * 2.0 ** -23 * (1 + 2.0 ** -10)


def logits(x: torch.Tensor, W: torch.Tensor, b: torch.Tensor | None):
    """x [B, D] fp32 pooled, W [C, D], b [C] -> (fp64 logits, per-element bound)."""
    xd, Wd = x.double(), W.double()
    ref = xd @ Wd.t()
    if b is not None:
        ref = ref + b.double()
    D = x.shape[1]
    # NaN in x must not poison the bound of the other rows (a NaN row is checked by other means)
    xa = torch.nan_to_num(xd.abs(), nan=0.0)
    absprod = xa @ Wd.abs().t()
    floor = 1.01 * FLOOR16 * (xa.sum(1, keepdim=True) + Wd.abs().sum(1)[None, :])
    bound = alpha(D) * absprod + floor
    bound = bound + U * (torch.nan_to_num(ref.abs(), nan=0.0) + bound)
    return ref, bound


def probs(ref_logits: torch.Tensor, L: torch.Tensor):
    """fp64 softmax of the reference logits and its per-element bound, L the logit bound."""
    p = torch.softmax(ref_logits, -1)
    C = ref_logits.shape[1]
    m = ref_logits.max(-1, keepdim=True).values
    dx = U * (ref_logits - m).abs()
    shift = (p * (L + dx + 4 * U)).sum(-1, keepdim=True)
    r = 1.01 * (L + shift + gamma(-(-C // 32) + 13) + dx + 6 * U)
    return p, p * torch.expm1(r) + 2.0 ** -126


def stable_topk(p: torch.Tensor, k: int):
    """Top-k of every row: descending, the first index first among equal values, NaN above everything (torch.argmax's
    order, which torch.topk does not promise among ties)."""
    n = p.shape[1]
    idx = torch.arange(n, device=p.device).expand_as(p)
    key = torch.where(torch.isnan(p), torch.full_like(p, math.inf), p)
    nan_first = torch.isnan(p).to(torch.int64)
    # lexicographic: NaN, then value descending, then index ascending; sort is stable, so sort by the later keys first
    order = torch.argsort(idx, dim=1, stable=True)
    order = torch.gather(order, 1, torch.argsort(-torch.gather(key, 1, order), dim=1, stable=True))
    order = torch.gather(order, 1, torch.argsort(-torch.gather(nan_first, 1, order), dim=1, stable=True))
    top = order[:, :k]
    return torch.gather(p, 1, top), top


def safe_ranks(p_ref: torch.Tensor, P: torch.Tensor, k: int) -> torch.Tensor:
    """[B, k] bool: rank j of the fp64 top-k is safe when every rank up to j beats all lower-ranked cells by more than the
    two probability bounds, so that any values within the bounds rank the same."""
    order = torch.argsort(-p_ref, dim=1, stable=True)
    lo = torch.gather(p_ref - P, 1, order)
    hi = torch.gather(p_ref + P, 1, order)
    # best upper value among the cells ranked below position j
    below = torch.flip(torch.cummax(torch.flip(hi, [1]), 1).values, [1])
    below = torch.cat([below[:, 1:], torch.full_like(below[:, :1], -math.inf)], 1)
    ok = (lo > below)[:, :k]
    return ok.to(torch.int64).cumprod(1).bool()


def targets(mode: int, C: int, labels_idx=None, soft=None, labels_lnglat=None, centroids=None, smoothing: float = 65.0):
    """[B, C] fp64 targets of the three loss modes (mode 2: the reference's haversine smoothing with constant `smoothing`)."""
    if mode == 0:
        t = torch.zeros(labels_idx.shape[0], C, dtype=torch.float64, device=labels_idx.device)
        t[torch.arange(labels_idx.shape[0], device=t.device), labels_idx] = 1.0
        return t
    if mode == 1:
        return soft.double()
    x = torch.deg2rad(labels_lnglat.double())
    y = torch.deg2rad(centroids.double())
    dlat = x[:, None, 1] - y[None, :, 1]
    dlng = x[:, None, 0] - y[None, :, 0]
    a = torch.sin(dlat / 2) ** 2 + torch.cos(x[:, None, 1]) * torch.cos(y[None, :, 1]) * torch.sin(dlng / 2) ** 2
    d = 6378137.0 * (2 * torch.arcsin(torch.sqrt(a))) / 1000
    t = torch.exp(-(d - d.min(-1, keepdim=True).values) / smoothing)
    return torch.nan_to_num(t, nan=0.0, posinf=0.0, neginf=0.0)


def loss(x: torch.Tensor, t: torch.Tensor, mode: int, smoothing: float = 65.0, grad_scale: float = 1.0):
    """Soft-target cross entropy of fp32 logits x [B, C] with fp64 targets t: (per-sample loss, its bound, the gradient of
    grad_scale * mean loss with respect to x, its bound)."""
    xd = x.double()
    B = x.shape[0]
    lse = torch.logsumexp(xd, -1, keepdim=True)
    per = (t * (lse - xd)).sum(-1)
    et = 4e-13 * (20038.0 + 1.0) / smoothing if mode == 2 else 0.0
    per_bound = 1e-13 * (t * (lse.abs() + xd.abs())).sum(-1) + et * (t * (lse - xd).abs()).sum(-1)
    p = torch.exp(xd - lse)
    tsum = t.sum(-1, keepdim=True)
    g = grad_scale / B * (p * tsum - t)
    # mode 2 parks t in the fp32 gradient row before forming the gradient: t and sum t are rounded to fp32 first
    eg = 1e-13 * (1 + lse.abs() + xd.abs()) + 2 * et + (1.01 * U if mode == 2 else 0.0)
    g_bound = U * g.abs() + abs(grad_scale) / B * (p * tsum + t) * eg + 2.0 ** -149
    return per, per_bound, g, g_bound


def gemm(a: torch.Tensor, b: torch.Tensor, c0: torch.Tensor | None = None):
    """a [M, K] . b [K, N] (+ c0) in fp64 and the bound of an in-order fp32 FMA chain (plus one FMA for c0)."""
    ref = a.double() @ b.double()
    absum = a.double().abs() @ b.double().abs()
    if c0 is not None:
        ref = ref + c0.double()
        absum = absum + c0.double().abs()
    return ref, gamma(a.shape[1] + 1) * absum


def ratio(err: torch.Tensor, bound: torch.Tensor) -> float:
    """Largest |error| / bound; an error where the bound is zero counts as infinite."""
    err, bound = err.double().abs(), bound.double()
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0
