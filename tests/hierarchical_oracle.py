"""fp64 restatement of the hierarchical panorama head (reference models/super_guessr.py:94-103,414-433 with
models/layers/positional_encoder.py and nn.MultiheadAttention(E, 16, batch_first=True)), for the tests and for
tools/make_hierarchical_golden.py, which draws the same synthetic weights from `synthetic_params`.

Everything here is differentiable torch on whatever dtype it is given (the tests pass fp64): gradients come from autograd."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle.geo import haversine_matrix, smooth_labels

HEADS = 16
FULL, STRIDE = 4096, 37   # the golden keeps tensors of up to FULL elements whole, larger ones every STRIDE-th element
ATTN_KEYS = ("self_attn.in_proj_weight", "self_attn.in_proj_bias", "self_attn.out_proj.weight", "self_attn.out_proj.bias")


def synthetic_params(E: int, C: int, seed: int) -> dict:
    """fp32 self_attn and cell_layer entries of a hierarchical SuperGuessr's state_dict, drawn from a CPU generator (the
    biases are non-zero so that every bias path is exercised; nn.MultiheadAttention initialises them to zero)."""
    g = torch.Generator().manual_seed(seed)
    s = 1.0 / math.sqrt(E)
    return {"self_attn.in_proj_weight": torch.randn(3 * E, E, generator=g) * s,
            "self_attn.in_proj_bias": torch.randn(3 * E, generator=g) * 0.05,
            "self_attn.out_proj.weight": torch.randn(E, E, generator=g) * s,
            "self_attn.out_proj.bias": torch.randn(E, generator=g) * 0.05,
            "cell_layer.weight": torch.randn(C, E, generator=g) * (1.4 * s),  # logits ~ 1 sd: top-1 / top-2 margins
            "cell_layer.bias": torch.randn(C, generator=g) * 0.01}


def embeddings(N: int, E: int, seed: int) -> torch.Tensor:
    """Panorama embeddings f32 [N, 4, E] of a case."""
    return torch.randn(N, 4, E, generator=torch.Generator().manual_seed(seed)) * 0.3


def sample(t) -> torch.Tensor:
    """What tests/golden/hierarchical.npz keeps of a tensor: all of it flattened if it has at most FULL elements, else every
    STRIDE-th element (37 is prime, so the sample crosses rows, heads and the q / k / v blocks)."""
    flat = torch.as_tensor(t).reshape(-1)
    return flat if flat.numel() <= FULL else flat[::STRIDE]


def labels(N: int, seed: int, C: int = 1000):
    """(labels (lng, lat) f64 [N, 2], labels_clf i64 [N], labels_multi_task [N, 6], labels_climate one-hot [N, 28],
    labels_month i64 [N]) of a case."""
    from pigeon_b200 import synthetic
    g = torch.Generator().manual_seed(seed + 500)
    return (torch.tensor(synthetic.synthetic_geocells(N, seed + 7)), torch.randint(0, C, (N,), generator=g),
            torch.randn(N, 6, generator=g), F.one_hot(torch.randint(0, 28, (N,), generator=g), 28).float(),
            torch.randint(0, 12, (N,), generator=g))


def attention(emb, pe, in_w, in_b, out_w, out_b, heads: int = HEADS, mask_x=None, mask_p=None, p_x: float = 0.0,
              p_attn: float = 0.0, n0: int = 0) -> dict:
    """emb [N, 4, E], pe = pos_encoding [rows, 1, E] -> dict(x, q0, k, v, probs, o, cls).  Sample n gets PE row n0 + n on
    all four views (positional_encoder.py:44 with batch_first inputs); mask_x [N, 4, E] and mask_p [N, heads, 4] are the
    dropout keep-masks (None = no dropout)."""
    N, V, E = emb.shape
    hd = E // heads
    x = emb + pe[n0:n0 + N]
    if mask_x is not None:
        x = x * mask_x.to(x.dtype) / (1.0 - p_x)
    wq, wk, wv = in_w.split(E)
    bq, bk, bv = in_b.split(E)
    q0 = F.linear(x[:, 0], wq, bq)
    k = F.linear(x, wk, bk)
    v = F.linear(x, wv, bv)
    scores = torch.einsum("nhd,njhd->nhj", q0.view(N, heads, hd), k.view(N, V, heads, hd)) / math.sqrt(hd)
    probs = torch.softmax(scores, dim=-1)
    pd = probs if mask_p is None else probs * mask_p.to(probs.dtype) / (1.0 - p_attn)
    o = torch.einsum("nhj,njhd->nhd", pd, v.view(N, V, heads, hd)).reshape(N, E)
    return dict(x=x, q0=q0, k=k, v=v, probs=probs, o=o, cls=F.linear(o, out_w, out_b))


def head(cls, W, b, centroids, k: int):
    """cell_layer, softmax, arg-max, centroid and top-k (super_guessr.py:447-459) -> (logits, probs, pred, pred_LLH, topk)."""
    logits = F.linear(cls, W, b)
    probs = torch.softmax(logits, dim=-1)
    pred = torch.argmax(probs, dim=-1)
    return logits, probs, pred, centroids[pred], torch.topk(probs, k, dim=-1)


def classification_loss(logits, centroids, labels=None, labels_clf=None, smooth: bool = False):
    """super_guessr.py:468-474: CE against geocell indices, or against haversine-smoothed targets."""
    if smooth:
        return F.cross_entropy(logits, smooth_labels(haversine_matrix(labels.double(), centroids.t())).to(logits.dtype))
    return F.cross_entropy(logits, labels_clf)


def multi_task_loss(cls, heads: dict, labels_mt, labels_climate, labels_month):
    """super_guessr.py:315-348 with the loss scalings 8, 2, 1; `heads` maps multi_task_head / climate_layer / month_layer to
    (weight, bias)."""
    mt = F.linear(cls, *heads["multi_task_head"])
    climate = F.linear(cls, *heads["climate_layer"])
    month = F.linear(cls, *heads["month_layer"])
    return (F.mse_loss(mt, labels_mt.to(cls.dtype)) * 8 + F.cross_entropy(climate, labels_climate.to(cls.dtype)) * 2
            + F.cross_entropy(month, labels_month))
