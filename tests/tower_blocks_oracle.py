"""fp64 references and per-element error bounds for the memory-bound building blocks of the two towers (csrc/vit_misc.cu,
csrc/train_vit.cu and the text-tower kernels of csrc/clip_train.cu).

Every function takes the same fp32 / fp16 / bf16 operands the kernel reads, computes the operation in float64 on whatever
device they live on, and returns the exact-ish result together with a bound B such that |kernel - reference| <= B element by
element.  A bound is c * u * sum|terms| for the terms each output element is built from, never a global rel-L2.

Notation: u = 2^-24 (fp32 unit roundoff), gamma_n = n u / (1 - n u) (Higham's bound for a length-n chain of roundings: a
recursive sum of n + 1 terms in any order, or a product of n factors (1 + delta_i)).  Derivations, term by term:

LayerNorm row statistics (ln_row in vit_misc.cu, ln_backward_kernel in train_vit.cu, text_pool_ln_backward_kernel in
clip_train.cu; all three share the layout).  One warp owns a row; lane l holds the float4 slots l + 32 i, i < NV4 = hidden / 128.
  * sum of x: each lane adds (x + y) + (z + w) of a slot (2 levels) onto its running sum (NV4 levels), then a 5-level xor
    shuffle tree: depth D = NV4 + 7, so |S' - S| <= gamma_D sum|x|, and the division by hidden rounds once:
        dmu = gamma_{D+1} sum|x| / hidden.
  * sum of squares: each centred value x - mu' rounds once and its square once more, the float4 adds twice more, then NV4
    + 5 levels as above: depth D + 3, plus the division: var' = (var + dmu^2)(1 + theta_{D+4}) (the centring error enters
    as + dmu^2 because the exact deviations sum to zero).  var' + eps rounds once, rsqrtf is within 2 ulp (4 u relative):
        tau = (gamma_{D+4} (var + dmu^2) + dmu^2) / (var + eps) + u,   rho = 0.51 tau + 4.01 u   (relative error of rstd).
  * forward output y = ((x - mu') rstd') g + b: the subtraction, two products and the add round once each:
        |y' - y| <= 1.01 (|g| rstd dmu + |g xhat| (rho + gamma_3)) + u (|g xhat| + |b|).
    An fp16 output rounds that fp32 value to nearest: plus half an fp16 ulp of |y| + bound (the rounded value may sit in the
    next binade), or 2^-25 below the normal range.
  * backward: xhat' = (x - mu') rstd' is within dxh = 1.01 (rstd dmu + |xhat| (rho + gamma_2)); gd = g dy rounds once; the
    row means s1 = mean(gd) and s2 = mean(gd xhat) add one product rounding and the division to the tree depth:
        ds1 = gamma_{D+2} sum|gd| / hidden,   ds2 = 1.01 (gamma_{D+3} sum|gd xhat| + sum |gd| dxh) / hidden,
    and dx = rstd' ((gd - s1) - xhat s2) rounds four more times:
        |dx' - dx| <= 1.01 rstd (gamma_4 (|gd| + |s1| + |xhat s2|) + ds1 + |xhat| ds2 + |s2| dxh) + 1.01 |dx| (rho + u);
    accumulating onto a previous dx adds u (|dx| + |dx0|).
  * dgamma / dbeta of ln_backward_kernel: a warp adds its rows (rpw of them) into shared memory in order, the block adds its 8
    warps in order, and every block adds its partial with one atomicAdd in any order (B blocks, plus the initial value):
        |dgamma' - dgamma| <= gamma_{rpw + 8 + B + 1} (sum|dy xhat| + |dgamma0|) + sum |dy| dxh,
        |dbeta' - dbeta|   <= gamma_{rpw + 8 + B} (sum|dy| + |dbeta0|).
    text_pool_ln_backward orders its n per-caption partials instead: depth n + 1 (+ 1 for the product of dgamma).

Column sums (column_sum_kernel): a thread adds 128 rows in order, and ceil(rows / 128) partials meet in atomics:
        (128 + ceil(rows / 128)) u (sum|x| + |out0|)   (as gamma_n).
Token mean (token_mean_kernel): ny = min(8, 1024 / (hidden / 4)) threads per column each add every ny-th token in order, the
first adds the other ny - 1 partials, and the sum is multiplied by fp32(1 / tokens) (one rounding for the reciprocal, one
for the product):  gamma_{ceil(tokens / ny) + ny + 1} sum|x| / tokens.
Token-embedding gradient (token_embedding_grad_kernel): per id the rows holding it are added in ascending order, then once
onto dtok: gamma_{count + 1} (sum|dx| + |dtok0|).
Patch embedding (the wgmma GEMM, bound as in test_gpu_gemm_epilogues.py): fp32 accumulation of K exact fp16 products is within
C_ACC u sqrt(K) (|A| |W|^T) (Higham & Mary's probabilistic lambda sqrt(K) u with C_ACC = 2), and adding the position
embedding rounds once: u |e|.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24
C_ACC = 2.0


def gamma(n) -> float:
    n = float(n)
    return n * U / (1.0 - n * U)


def ln_depth(hidden: int) -> int:
    """Depth D of the fp32 row sums of the LayerNorm kernels (see the module docstring)."""
    return hidden // 128 + 7


def half_ulp_f16(mag: torch.Tensor) -> torch.Tensor:
    """Half a unit in the last place of fp16 at magnitude `mag` (2^-25 in the subnormal range)."""
    e = torch.floor(torch.log2(mag.clamp_min(2.0 ** -14)))
    return torch.exp2(e - 11.0)


def _row_stats(x: torch.Tensor, eps: float):
    eps = float(torch.tensor(eps, dtype=torch.float32))   # the kernels take eps as a float
    x = x.double()
    n = x.shape[-1]
    D = ln_depth(n)
    mean = x.mean(-1, keepdim=True)
    a = x - mean
    var = (a * a).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    dmu = gamma(D + 1) * x.abs().mean(-1, keepdim=True)
    tau = (gamma(D + 4) * (var + dmu * dmu) + dmu * dmu) / (var + eps) + U
    rho = 0.51 * tau + 4.01 * U
    return a * rstd, rstd, dmu, rho


def layernorm_forward(x, g, b, eps: float, out_f16: bool = False):
    """y = LayerNorm(x) * g + b in fp64 and its per-element bound for the fp32 (or, out_f16, the fp16) output."""
    xhat, rstd, dmu, rho = _row_stats(x, eps)
    g, b = g.double(), b.double()
    y = xhat * g + b
    bound = 1.01 * (g.abs() * rstd * dmu + (g * xhat).abs() * (rho + gamma(3))) + U * ((g * xhat).abs() + b.abs())
    if out_f16:
        bound = bound + half_ulp_f16(y.abs() + bound)
    return y, bound


def layernorm_backward(dy, x, g, eps: float, dx0=None):
    """dx (+ dx0) of LayerNorm with respect to x and its per-element bound; also the per-column |term| sums and the
    xhat error that the dgamma / dbeta bounds need (`ln_param_bounds`)."""
    xhat, rstd, dmu, rho = _row_stats(x, eps)
    n = x.shape[-1]
    D = ln_depth(n)
    dy, g = dy.double(), g.double()
    gd = dy * g
    s1 = gd.mean(-1, keepdim=True)
    s2 = (gd * xhat).mean(-1, keepdim=True)
    dx = rstd * (gd - s1 - xhat * s2)
    dxh = 1.01 * (rstd * dmu + xhat.abs() * (rho + gamma(2)))
    ds1 = gamma(D + 2) * gd.abs().mean(-1, keepdim=True)
    ds2 = 1.01 * (gamma(D + 3) * (gd * xhat).abs().sum(-1, keepdim=True) + (gd.abs() * dxh).sum(-1, keepdim=True)) / n
    bound = 1.01 * rstd * (gamma(4) * (gd.abs() + s1.abs() + (xhat * s2).abs()) + ds1 + xhat.abs() * ds2 + s2.abs() * dxh) \
        + 1.01 * dx.abs() * (rho + U)
    if dx0 is not None:
        dx0 = dx0.double()
        dx = dx + dx0
        bound = bound * (1 + U) + U * (dx.abs() + dx0.abs())
    return dict(dx=dx, bound=bound, dgamma=(dy * xhat).sum(0), dbeta=dy.sum(0), abs_dg=(dy * xhat).abs().sum(0),
                abs_db=dy.abs().sum(0), dxh_term=(dy.abs() * dxh).sum(0))


def ln_backward_schedule(rows: int, sms: int):
    """(blocks, rows per warp) of layernorm_backward's launch: 8 warps per block, at most 8 blocks per SM."""
    blocks = min((rows + 7) // 8, 8 * sms)
    return blocks, -(-rows // (8 * blocks))


def ln_param_bounds(ref: dict, dgamma0, dbeta0, depth: int):
    """Bounds of dgamma0 + dgamma and dbeta0 + dbeta when every column is a sum of `depth` fp32 additions in some order."""
    bg = gamma(depth + 1) * (ref["abs_dg"] + dgamma0.double().abs()) + 1.01 * ref["dxh_term"]
    bb = gamma(depth) * (ref["abs_db"] + dbeta0.double().abs())
    return bg, bb


def column_sum(x, out0):
    """out0 + x.sum(0) in fp64 and the bound of column_sum_kernel (rows chunks of 128, atomics across chunks)."""
    rows = x.shape[0]
    ref = out0.double() + x.double().sum(0)
    bound = gamma(min(rows, 128) + -(-rows // 128)) * (x.double().abs().sum(0) + out0.double().abs())
    return ref, bound


def token_mean(x, hidden: int):
    """x [n, tokens, hidden] -> mean over tokens in fp64 and the bound of token_mean_kernel."""
    tokens = x.shape[1]
    ny = max(1, min(8, 1024 // (hidden // 4)))
    xd = x.double()
    return xd.mean(1), gamma(-(-tokens // ny) + ny + 1) * xd.abs().sum(1) / tokens


def first_argmax(ids: torch.Tensor) -> torch.Tensor:
    """First index of the largest id of every row (transformers' `input_ids.argmax(dim=-1)`)."""
    S = ids.shape[1]
    t = torch.arange(S, device=ids.device).expand_as(ids)
    return torch.where(ids == ids.max(1, keepdim=True).values, t, S).min(1).values


def token_embedding_grad(ids, dx, vocab: int, dtok0):
    """dtok0 + per-id sums of the rows of dx (ids outside [0, vocab) skipped) in fp64, the bound, and the ids that occur."""
    ok = (ids >= 0) & (ids < vocab)
    idv, dxv = ids[ok], dx[ok].double()
    ref = dtok0.double().index_add(0, idv, dxv)
    absum = torch.zeros_like(ref).index_add_(0, idv, dxv.abs())
    count = torch.bincount(idv, minlength=vocab).double()
    g = count * U / (1 - count * U) + gamma(1)
    bound = g[:, None] * (absum + dtok0.double().abs())
    return ref, bound, count > 0


def patch_embedding(a16, w16, pos):
    """e[:, 1:] of embed_preln: im2col [rows, K] fp16 . patch weight [hidden, K] fp16 ^T + pos, and the GEMM bound."""
    acc = a16.double() @ w16.double().t()
    absprod = a16.double().abs() @ w16.double().abs().t()
    e = acc + pos.double()
    return e, 1.01 * C_ACC * U * math.sqrt(a16.shape[1]) * absprod + 1.01 * U * e.abs()


def ratio(err: torch.Tensor, bound: torch.Tensor) -> float:
    """Largest |error| / bound; an error where the bound is zero counts as infinite."""
    err, bound = err.double().abs(), bound.double()
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0
