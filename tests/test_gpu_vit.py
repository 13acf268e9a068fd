"""Vision-tower parity on the H100: pg_vit_forward (fp16 tensor-core operands, fp32 accumulate / residual /
statistics) against the fp32 CPU oracle of HF CLIPVisionTransformer (oracle/vit.py).

Tolerance (BASELINE.json north_star): <= 1e-3 relative on fp32 embeddings."""
import pytest
import torch

pytestmark = pytest.mark.gpu

REL_TOL = 1e-3


def _record(line):
    """Measured parity numbers are appended to a parity log when its directory exists; never fails a test."""
    import os
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    if os.path.isdir(d):
        with open(os.path.join(d, "parity.log"), "a") as f:
            f.write(line + "\n")


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _run(cuda, dims, n_views, seed, std=0.02, fold=True, mutate=None, pass_size=3):
    from oracle import vit as ovit
    from pigeon_b200 import synthetic
    from pigeon_b200.vit_engine import VitEngine
    sd = synthetic.random_vit_state_dict(dims, seed=seed, std=std)
    if mutate is not None:
        mutate(sd)
    g = torch.Generator().manual_seed(seed + 100)
    px = torch.randn(n_views, 3, dims.image_size, dims.image_size, generator=g)
    ref_h, ref_layers = ovit.vit_last_hidden_state(sd, px, patch=dims.patch_size, heads=dims.heads, layers=dims.layers,
                                                   eps=dims.ln_eps, return_layers=True)
    eng = VitEngine(sd, dims, device=cuda, max_views_per_pass=pass_size, fold_layernorm=fold)
    emb, hid = eng.forward(px.to(cuda), return_hidden=True)
    torch.cuda.synchronize()
    return emb, hid, ref_h


@pytest.mark.parametrize("fold", [True, False])
def test_vit_tiny(cuda, fold):
    """fold=True: LayerNorm applied in the GEMM epilogues (the default); fold=False: LayerNorm kernels."""
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=2)
    emb, hid, ref_h = _run(cuda, dims, n_views=5, seed=1, std=0.05, fold=fold)
    assert torch.isfinite(hid).all()
    assert _rel(hid, ref_h) < REL_TOL, _rel(hid, ref_h)
    assert _rel(emb, ref_h.mean(1)) < REL_TOL


@pytest.mark.parametrize("fold", [True, False])
def test_vit_336_one_pass_past_the_layernorm_grid_cap(cuda, fold):
    """30 views of 577 tokens in one pass: 17,310 rows, more than the 16 blocks x 8 warps per SM of the LayerNorm kernels on
    132 SMs, so their warps loop over several rows; with fold=True this covers the LayerNorm-fold statistics that embed_preln
    writes for the first GEMM."""
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims(image_size=336, patch_size=14, hidden=256, heads=4, intermediate=1024, layers=1)
    emb, hid, ref_h = _run(cuda, dims, n_views=30, seed=4, std=0.05, fold=fold, pass_size=30)
    assert torch.isfinite(hid).all()
    assert _rel(hid, ref_h) < REL_TOL, _rel(hid, ref_h)
    assert _rel(emb, ref_h.mean(1)) < REL_TOL


def test_vit_tiny_wide_tokens(cuda):
    """more than one 128-row q tile and a ragged last KV block (tokens = 10*10+1 = 101 ... 17*17+1 = 290)."""
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims(image_size=238, patch_size=14, hidden=256, heads=4, intermediate=768, layers=2)
    emb, hid, ref_h = _run(cuda, dims, n_views=2, seed=2, std=0.05)
    assert _rel(hid, ref_h) < REL_TOL, _rel(hid, ref_h)
    assert _rel(emb, ref_h.mean(1)) < REL_TOL


def test_vit_large_336(cuda):
    """The real geometry: ViT-L/14 at 336 px (577 tokens, 24 layers), random-init weights, 2 views."""
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims()
    emb, hid, ref_h = _run(cuda, dims, n_views=2, seed=3)
    e_h, e_e = _rel(hid, ref_h), _rel(emb, ref_h.mean(1))
    print(f"ViT-L/14-336 rel-L2: last_hidden_state {e_h:.3e}  embedding {e_e:.3e}")
    _record(f"vit_large_336 (24 layers, 577 tokens, 2 views) vs fp32 CPU oracle: rel-L2 last_hidden_state {e_h:.3e}, embedding {e_e:.3e}")
    assert e_h < REL_TOL and e_e < REL_TOL, (e_h, e_e)


@pytest.mark.parametrize("fold", [True, False])
def test_vit_large_336_outlier_channels(cuda, fold):
    """Real CLIP-L carries a few residual-stream channels two orders of magnitude above the rest ("massive activations").
    HF default-init weights have none, so they are injected: pre_layrnorm.bias puts 150 into one channel and 30 into three
    more of EVERY token, layer_norm gammas of those channels are damped as trained models do.  The fp16 operand of the
    LayerNorm-folded GEMMs is then the raw row (|x| up to 150) and the epilogue subtracts mu * colsum: this is the regime
    the folded scheme has to survive inside the 1e-3 budget."""
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims()
    chans = {7: 150.0, 100: 30.0, 500: -30.0, 901: 30.0}

    def mutate(sd):
        for ch, v in chans.items():
            sd["vision_model.pre_layrnorm.bias"][ch] = v
            for i in range(dims.layers):
                for ln in ("layer_norm1", "layer_norm2"):
                    sd[f"vision_model.encoder.layers.{i}.{ln}.weight"][ch] *= 0.05

    emb, hid, ref_h = _run(cuda, dims, n_views=2, seed=5, fold=fold, mutate=mutate)
    assert float(ref_h.abs().max()) > 100, "the injected outlier channel must survive to last_hidden_state"
    e_h, e_e = _rel(hid, ref_h), _rel(emb, ref_h.mean(1))
    # the outlier channels dominate the L2 norm: also compare with them removed
    keep = torch.ones(dims.hidden, dtype=torch.bool)
    keep[list(chans)] = False
    e_rest = _rel(hid[..., keep.to(hid.device)], ref_h[..., keep])
    _record(f"vit_large_336 with outlier channels {chans} (fold_layernorm={fold}): rel-L2 last_hidden_state {e_h:.3e}, "
            f"without the outlier channels {e_rest:.3e}, embedding {e_e:.3e}")
    assert e_h < REL_TOL and e_e < REL_TOL and e_rest < REL_TOL, (e_h, e_rest, e_e)


def test_vit_fp16_pixels_and_chunking(cuda):
    """fp16 pixel input path and chunked execution give the same answer as one pass on fp32 pixels of the same values."""
    from pigeon_b200 import synthetic
    from pigeon_b200.vit_engine import VitDims, VitEngine
    dims = VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    sd = synthetic.random_vit_state_dict(dims, seed=7, std=0.05)
    px = torch.randn(7, 3, 56, 56, generator=torch.Generator().manual_seed(1)).half()
    a = VitEngine(sd, dims, device=cuda, max_views_per_pass=2).forward(px.to(cuda))
    b = VitEngine(sd, dims, device=cuda, max_views_per_pass=64).forward(px.float().to(cuda))
    assert torch.equal(a, b)
