"""Deterministic synthetic weights / geocells / prototype banks (no network: the reference's checkpoints,
geocell CSV and datasets are not shipped — README.md:11, data/README.md:3).  Used by tests and bench.py."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from .vit_engine import VitDims


def random_vit_state_dict(dims: VitDims, seed: int = 0, std: float = 0.02) -> Dict[str, torch.Tensor]:
    """HF-named CLIPVisionModel state dict with N(0, std) matrices, unit-ish LayerNorms, small biases."""
    g = torch.Generator().manual_seed(seed)

    def n(*shape, s=std):
        return torch.randn(*shape, generator=g) * s

    sd = {
        "vision_model.embeddings.class_embedding": n(dims.hidden),
        "vision_model.embeddings.patch_embedding.weight": n(dims.hidden, 3, dims.patch_size, dims.patch_size),
        "vision_model.embeddings.position_embedding.weight": n(dims.tokens, dims.hidden),
        "vision_model.pre_layrnorm.weight": 1 + n(dims.hidden),
        "vision_model.pre_layrnorm.bias": n(dims.hidden),
        "vision_model.post_layernorm.weight": 1 + n(dims.hidden),
        "vision_model.post_layernorm.bias": n(dims.hidden),
    }
    for i in range(dims.layers):
        p = f"vision_model.encoder.layers.{i}."
        for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + f"self_attn.{nm}.weight"] = n(dims.hidden, dims.hidden)
            sd[p + f"self_attn.{nm}.bias"] = n(dims.hidden)
        sd[p + "layer_norm1.weight"] = 1 + n(dims.hidden)
        sd[p + "layer_norm1.bias"] = n(dims.hidden)
        sd[p + "layer_norm2.weight"] = 1 + n(dims.hidden)
        sd[p + "layer_norm2.bias"] = n(dims.hidden)
        sd[p + "mlp.fc1.weight"] = n(dims.intermediate, dims.hidden)
        sd[p + "mlp.fc1.bias"] = n(dims.intermediate)
        sd[p + "mlp.fc2.weight"] = n(dims.hidden, dims.intermediate)
        sd[p + "mlp.fc2.bias"] = n(dims.hidden)
    return sd


def random_clip_state_dict(text_dims, vision_dims: VitDims, seed: int = 0, std: float = 0.02,
                           projection_dim: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """HF-named CLIPModel state dict: `random_vit_state_dict(vision_dims, seed)` for `vision_model.*`, N(0, std) text tower
    (`text_model.*`, unit-ish LayerNorms, small biases), bias-free projections to `projection_dim` (default: the text
    width, as in CLIP-L/14) and logit_scale = log(1 / 0.07)."""
    sd = random_vit_state_dict(vision_dims, seed=seed, std=std)
    g = torch.Generator().manual_seed(seed + 7919)
    P = text_dims.hidden if projection_dim is None else projection_dim
    H = text_dims.hidden

    def n(*shape, s=std):
        return torch.randn(*shape, generator=g) * s

    sd["text_model.embeddings.token_embedding.weight"] = n(text_dims.vocab, H)
    sd["text_model.embeddings.position_embedding.weight"] = n(text_dims.max_positions, H)
    for i in range(text_dims.layers):
        p = f"text_model.encoder.layers.{i}."
        for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + f"self_attn.{nm}.weight"] = n(H, H)
            sd[p + f"self_attn.{nm}.bias"] = n(H)
        sd[p + "layer_norm1.weight"] = 1 + n(H)
        sd[p + "layer_norm1.bias"] = n(H)
        sd[p + "layer_norm2.weight"] = 1 + n(H)
        sd[p + "layer_norm2.bias"] = n(H)
        sd[p + "mlp.fc1.weight"] = n(text_dims.intermediate, H)
        sd[p + "mlp.fc1.bias"] = n(text_dims.intermediate)
        sd[p + "mlp.fc2.weight"] = n(H, text_dims.intermediate)
        sd[p + "mlp.fc2.bias"] = n(H)
    sd["text_model.final_layer_norm.weight"] = 1 + n(H)
    sd["text_model.final_layer_norm.bias"] = n(H)
    sd["visual_projection.weight"] = n(P, vision_dims.hidden)
    sd["text_projection.weight"] = n(P, H)
    sd["logit_scale"] = torch.tensor(float(np.log(1 / 0.07)), dtype=torch.float32)
    return sd


def synthetic_geocells(num_cells: int, seed: int = 0) -> np.ndarray:
    """(C, 2) float64 (lng, lat): lng ~ U(-180, 180), lat ~ U(-90, 90)   (SURVEY.md §8d cfg1)."""
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(-180, 180, num_cells), rng.uniform(-90, 90, num_cells)], axis=1)


def synthetic_bank(num_cells: int, num_protos: int, dim: int, seed: int = 2, members_mean: float = 0.0,
                   empty_cells: int = 0, emb_std: float = 0.3, max_members: int = 64) -> Dict[str, np.ndarray]:
    """CSR prototype bank (layout of `pg_refiner_bank`).

    Cell sizes ~ multinomial; `empty_cells` cells get no prototypes (reference quirk: protos[cell] is None).
    members_mean == 0 -> every cluster has count == 1 (prototype == its single member);
    otherwise cluster sizes ~ 1 + Poisson(members_mean - 1) and the prototype is the member mean
    (reference models/proto_refiner.py:359-378)."""
    rng = np.random.default_rng(seed)
    live = np.ones(num_cells, bool)
    if empty_cells:
        live[rng.choice(num_cells, size=empty_cells, replace=False)] = False
    pvals = live / live.sum()
    sizes = rng.multinomial(num_protos, pvals)
    cell_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    P = int(cell_off[-1])
    if members_mean and members_mean > 1:
        count = np.minimum(1 + rng.poisson(members_mean - 1, size=P), max_members).astype(np.int32)
    else:
        count = np.ones(P, np.int32)
    member_off = np.concatenate([[0], np.cumsum(count)]).astype(np.int64)
    n_train = int(member_off[-1])
    member_idx = rng.permutation(n_train).astype(np.int64)
    data_emb = (rng.standard_normal((n_train, dim), dtype=np.float32) * emb_std).astype(np.float32)
    data_lnglat = np.stack([rng.uniform(-180, 180, n_train), rng.uniform(-90, 90, n_train)], axis=1).astype(np.float32)
    proto_emb = np.empty((P, dim), np.float32)
    proto_lnglat = np.empty((P, 2), np.float32)
    # prototype embedding = mean of member embeddings; cluster (lng, lat) = mean member location
    seg = np.repeat(np.arange(P), count)
    order_emb = data_emb[member_idx]
    sums = np.zeros((P, dim), np.float64)
    np.add.at(sums, seg, order_emb)
    proto_emb[:] = (sums / count[:, None]).astype(np.float32)
    ll = np.zeros((P, 2), np.float64)
    np.add.at(ll, seg, data_lnglat[member_idx])
    proto_lnglat[:] = (ll / count[:, None]).astype(np.float32)
    return dict(cell_off=cell_off, proto_emb=proto_emb, proto_lnglat=proto_lnglat, proto_count=count,
                member_off=member_off, member_idx=member_idx, data_emb=data_emb, data_lnglat=data_lnglat)


def synthetic_candidates(batch: int, k: int, num_cells: int, seed: int = 3):
    """k distinct candidate cells per query, sorted-descending Dirichlet probabilities (SURVEY.md §8d cfg5)."""
    rng = np.random.default_rng(seed)
    cand = np.stack([rng.choice(num_cells, size=k, replace=False) for _ in range(batch)]).astype(np.int64)
    probs = -np.sort(-rng.dirichlet(np.ones(k), size=batch), axis=1)
    return cand, probs.astype(np.float32)


def synthetic_queries(bank: Dict[str, np.ndarray], cand: np.ndarray, views: int = 4, near_frac: float = 0.6,
                      noise: float = 0.05, emb_std: float = 0.3, seed: int = 4) -> np.ndarray:
    """(B, views, D) float32 queries.  A fraction sits next to a prototype of one of its candidate cells so that
    the refinement actually moves guesses (random embeddings are all ~equidistant and never change the arg-max)."""
    rng = np.random.default_rng(seed)
    B, k = cand.shape
    D = bank["proto_emb"].shape[1]
    q = (rng.standard_normal((B, D), dtype=np.float32) * emb_std).astype(np.float32)
    for b in range(B):
        if rng.random() < near_frac:
            cell = cand[b, rng.integers(0, k)]
            lo, hi = bank["cell_off"][cell], bank["cell_off"][cell + 1]
            if hi > lo:
                q[b] = bank["proto_emb"][rng.integers(lo, hi)] + rng.standard_normal(D, dtype=np.float32) * noise
    v = q[:, None, :] + rng.standard_normal((B, views, D), dtype=np.float32) * (noise * 0.1)
    return v.astype(np.float32)


def synthetic_photo(height: int, width: int, seed: int = 0) -> np.ndarray:
    """Deterministic uint8 RGB test image [H, W, 3] from integer arithmetic only (triangle-wave gradients, PCG64 integer
    noise, two saturated blocks so that bicubic overshoot has to clip): identical on every machine."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:height, 0:width].astype(np.int64)
    img = np.empty((height, width, 3), dtype=np.int64)
    for c in range(3):
        t = (xx * (3 + c) + yy * (5 - c)) % 510
        tri = np.where(t > 255, 510 - t, t)
        u = (xx * yy // (17 + 4 * c)) % 256
        img[..., c] = (tri * 3 + u) // 4
    img += rng.integers(-40, 41, size=img.shape)
    img = np.clip(img, 0, 255)
    h4, w4 = height // 4, width // 4
    img[h4:h4 + height // 10, w4:w4 + width // 8] = 255
    img[h4 + height // 10:h4 + height // 5, w4:w4 + width // 8] = 0
    return img.astype(np.uint8)
