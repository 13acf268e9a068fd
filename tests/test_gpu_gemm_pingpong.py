"""The ping-pong GEMM kernel (gemm_pingpong.cu) against the single-warpgroup kernel (pg_gemm_set_schedule(1)): same
tiles, same MMA sequence, same epilogue arithmetic, so every output must be the same bits — the building blocks at ragged
shapes, the vision tower with LayerNorm folded into the epilogues, and a fine-tune step."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _both(fn):
    """fn() under the automatic schedule (ping-pong) and under the single-warpgroup kernel."""
    from pigeon_b200 import ops
    try:
        ops.gemm_set_schedule(0)
        new = fn()
        ops.gemm_set_schedule(1)
        old = fn()
    finally:
        ops.gemm_set_schedule(0)
    torch.cuda.synchronize()
    return new, old


# M: one row, one tile plus two rows, ragged, 9 x 128 + 2, the real row count of 64 views; tiles from 3 to 13 848
@pytest.mark.parametrize("M", [1, 130, 300, 1154, 577 * 64])
@pytest.mark.parametrize("N,K", [(384, 64), (1000, 96), (3072, 1024), (1024, 4096)])
@pytest.mark.parametrize("bf16", [0, 1])
def test_building_block_epilogues_bit_identical(cuda, M, N, K, bf16):
    from pigeon_b200._lib import check, current_stream_ptr, load, ptr
    lib = load()
    g = torch.Generator().manual_seed(M * 7 + N + K)
    dt = torch.bfloat16 if bf16 else torch.float16
    a = (torch.randn(M, K, generator=g) * 0.5).to(cuda, dt)
    w = (torch.randn(N, K, generator=g) * 0.05).to(cuda, dt)
    bias = torch.randn(N, generator=g).to(cuda)
    resid = torch.randn(M, N, generator=g).to(cuda)

    def run(epi, variant):
        """variant: epilogue 2 updates `out` in place (True) or reads the residual from a separate buffer (False);
        epilogue 3 with a bias (False) or without one (True)."""
        if epi == 2 and variant:
            out = resid.clone()
        else:
            out = torch.full((M, N), float("nan"), device=cuda, dtype=torch.float16 if epi in (0, 1) else torch.float32)
        src = resid if epi == 2 and not variant else None
        b = None if epi == 3 and variant else bias
        check(lib.pg_gemm_ex(ptr(a), K, ptr(w), K, ptr(out), N, ptr(b), ptr(src), M, N, K, epi, bf16,
                             current_stream_ptr()), "pg_gemm_ex")
        return out

    for epi in (0, 1, 2, 3):
        for variant in ((True, False) if epi in (2, 3) else (False,)):
            new, old = _both(lambda: run(epi, variant))
            assert torch.equal(new.view(torch.int16 if new.dtype == torch.float16 else torch.int32),
                               old.view(torch.int16 if old.dtype == torch.float16 else torch.int32)), (epi, variant)


def test_gemm_f16_wrapper_bit_identical(cuda):
    from pigeon_b200 import ops
    g = torch.Generator().manual_seed(5)
    a = torch.randn(577 * 3, 1024, generator=g).half().to(cuda)
    w = (torch.randn(4096, 1024, generator=g) * 0.03).half().to(cuda)
    b = torch.randn(4096, generator=g).to(cuda)
    for epi in (0, 1, 3):
        new, old = _both(lambda: ops.gemm_f16(a, w, b, epi))
        assert torch.equal(new, old), epi


def _tower_embeddings(cuda, dims, n_views, seed):
    from pigeon_b200 import synthetic
    from pigeon_b200.vit_engine import VitEngine
    sd = synthetic.random_vit_state_dict(dims, seed=seed)
    px = torch.randn(n_views, 3, dims.image_size, dims.image_size, generator=torch.Generator().manual_seed(seed)).to(cuda)
    eng = VitEngine(sd, dims, device=cuda, max_views_per_pass=n_views, fold_layernorm=True)
    return _both(lambda: eng.forward(px, return_hidden=True))


def test_tower_with_folded_layernorm_small_geometry(cuda):
    """Epilogues 4 (patch embedding), 7 (out_proj / fc2 with LayerNorm moments), 8 (qkv) and 9 (fc1)."""
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims(image_size=238, patch_size=14, hidden=256, heads=4, intermediate=768, layers=2)
    (e_new, h_new), (e_old, h_old) = _tower_embeddings(cuda, dims, 5, 11)
    assert torch.equal(e_new, e_old) and torch.equal(h_new, h_old)


def test_tower_with_folded_layernorm_real_geometry(cuda):
    """16 views of ViT-L/14-336: 9 232 GEMM rows, 73 row blocks."""
    from pigeon_b200.vit_engine import VitDims
    (e_new, h_new), (e_old, h_old) = _tower_embeddings(cuda, VitDims(), 16, 12)
    assert torch.equal(e_new, e_old) and torch.equal(h_new, h_old)


def _reduced_with_atomics(name):
    """LayerNorm and bias gradients come from the fine-tune's float-atomic column reductions; every other gradient is
    reduced in a fixed order."""
    return name.endswith(".bias") or "layer_norm" in name or "layrnorm" in name


def test_fine_tune_step_gradients(cuda):
    """Epilogues 5 (backward through fc1's activation) and 6 (training forward of fc1) and the bf16 backward GEMMs."""
    from pigeon_b200 import CLIPVisionTower, SuperGuessr, VitDims, synthetic
    z = np.load(os.path.join(GOLD, "train_tower_small.npz"))
    meta = json.loads(str(z["meta"]))
    dims = VitDims(**meta["dims"])
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=meta["sd_seed"], std=meta["std"]), strict=True)
    sg = SuperGuessr(tower, panorama=False, should_smooth_labels=True, num_candidates=5, geocells=z["centroids"]).to(cuda)
    px = torch.randn(meta["n_views"], 3, dims.image_size, dims.image_size,
                     generator=torch.Generator().manual_seed(meta["px_seed"])).to(cuda)
    sg.train()

    def step():
        sg.zero_grad(set_to_none=True)
        out = sg(pixel_values=px, labels=torch.tensor(z["labels"]), labels_clf=torch.tensor(z["labels_clf"]))
        sg.backward(out.loss)
        return out.loss.detach().clone(), {n: p.grad.detach().clone() for n, p in sg.named_parameters() if p.grad is not None}

    (loss_new, g_new), (loss_old, g_old) = _both(step)
    assert torch.equal(loss_new, loss_old)
    assert g_new.keys() == g_old.keys() and len(g_new) > 0
    for n in g_new:
        if _reduced_with_atomics(n):
            rel = ((g_new[n].double() - g_old[n].double()).norm() / g_old[n].double().norm().clamp_min(1e-30)).item()
            assert rel <= 1e-6, (n, rel)
        else:
            assert torch.equal(g_new[n], g_old[n]), n
