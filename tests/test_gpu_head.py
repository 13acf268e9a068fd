"""The geocell head per element against fp64 (tests/head_oracle.py): both forward paths (the fused kernel and the three
kernels view mean + split / wgmma GEMM / softmax + top-k) at every tile edge, size limit, tie and magnitude, the loss in all
three modes and the fp32 backward of the Linear with each operand form its callers use.

Every forward case asserts which kernel ran (torch.profiler kernel names), checks pooled bit for bit against the in-order
fp32 view mean, logits and probabilities against their bounds, the top-k exactly against the stable reference of the
kernel's own probabilities, and the ranking against fp64 wherever the fp64 margins exceed the bounds."""
import pytest
import torch

import head_oracle as O

pytestmark = pytest.mark.gpu

FUSED, THREE = "head_fused_kernel", "softmax_topk_kernel"


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    return res, {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


def _forward(emb, W, b, cent, k, fused):
    """ops.head_forward with the fused kernel switched on or off -> (outputs, names of the CUDA kernels that ran)."""
    from pigeon_b200 import ops
    w3 = ops.head_pack_weight(W)
    torch.cuda.synchronize()
    ops.head_set_fused(fused)
    try:
        return _kernels(lambda: ops.head_forward(emb, w3, b, cent, k))
    finally:
        ops.head_set_fused(False)


def _expect_kernel(names, fused_ran):
    want, other = (FUSED, THREE) if fused_ran else (THREE, FUSED)
    assert any(want in n for n in names) and not any(other in n for n in names), names


def _same(a, b):
    """bitwise equality with NaN == NaN"""
    return bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def _check(emb, W, b, cent, k, out, min_safe=0.0):
    """Every output of one forward against the references; returns (logit ratio, prob ratio)."""
    B, C = emb.shape[0], W.shape[0]
    x = O.view_mean_f32(emb)
    assert _same(out["pooled"], x), "pooled differs from the in-order fp32 view mean"
    ref, L = O.logits(x, W, b)
    p, P = O.probs(ref, L)
    nan_row = torch.isnan(x).any(1)
    ok = ~nan_row
    rl = O.ratio(out["logits"][ok] - ref[ok], L[ok])
    rp = O.ratio(out["probs"][ok] - p[ok], P[ok])
    assert rl <= 1, f"logit error {rl:.3g} x its bound"
    assert rp <= 1, f"probability error {rp:.3g} x its bound"
    # NaN rows: torch semantics (all-NaN logits and probs, NaN first in index order)
    if nan_row.any():
        assert torch.isnan(out["logits"][nan_row]).all() and torch.isnan(out["probs"][nan_row]).all()
    # the top-k ranks exactly the probabilities the kernel wrote
    sv, si = O.stable_topk(out["probs"], k)
    assert torch.equal(out["topk_idx"], si), "top-k differs from the stable order of the kernel's own probabilities"
    assert _same(out["topk_val"], sv)
    assert torch.equal(out["pred_cell"], si[:, 0])
    assert torch.equal(out["pred_lnglat"], cent[si[:, 0]])
    # and the fp64 ranking wherever its margins exceed the bounds
    safe = O.safe_ranks(p, P, k) & ok[:, None]
    _, ri = O.stable_topk(p, k)
    assert torch.equal(out["topk_idx"][safe], ri[safe])
    assert safe[ok, 0].float().mean().item() >= min_safe if ok.any() else True
    print(f"  B={B} C={C} D={W.shape[1]} k={k}: logits {rl:.3g}, probs {rp:.3g} of the bound; top-1 safe "
          f"{safe[:, 0].float().mean().item():.2f}")
    return rl, rp


def _operands(B, V, D, C, kind, seed, cuda):
    g = torch.Generator().manual_seed(seed)
    emb = torch.randn(B, V, D, generator=g) * 0.3
    W = torch.randn(C, D, generator=g) * D ** -0.5
    if kind == "small":                      # |x| ~ 1e-3, |W| ~ 1e-4: the lo halves are fp16 subnormals
        emb, W = emb * 3e-3, W * (3e-4 * D ** 0.5)
    elif kind == "large":                    # |x| ~ 1e2, |W| ~ 1: logits of thousands, most probabilities exactly 0
        emb, W = emb * 300, W * D ** 0.5
    elif kind == "outlier":                  # a few channels two orders above the rest
        emb[:, :, :3] = 50.0
        W[:, :3] *= 10
    elif kind == "positive":                 # every partial sum of the accumulator keeps its sign
        emb, W = emb.abs(), W.abs()
    b = torch.randn(C, generator=g) * 0.1
    cent = torch.rand(C, 2, generator=g, dtype=torch.float64) * 100
    return emb.to(cuda), W.to(cuda), b.to(cuda), cent.to(cuda)


# (B, V, D, C, k): tile edges of both paths; the fused kernel takes D % 64 == 0 and C <= 6144
SHAPES = [(1, 4, 64, 1, 1), (127, 4, 64, 127, 5), (128, 1, 1024, 128, 50), (129, 7, 64, 129, 129), (257, 4, 1024, 130, 5),
          (1000, 4, 1024, 2203, 50), (129, 4, 64, 6144, 50), (129, 4, 64, 6145, 5), (5, 4, 72, 130, 5), (3, 1, 8, 2, 2),
          (3, 4, 1024, 12289, 50), (2, 4, 64, 51200, 5)]


def _fused_supported(B, V, D, C, k):
    return D % 64 == 0 and C <= 6144


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("B,V,D,C,k", SHAPES)
def test_head_forward_shapes(cuda, B, V, D, C, k, fused):
    emb, W, b, cent = _operands(B, V, D, C, "plain", B * 7 + C, cuda)
    out, names = _forward(emb, W, b, cent, k, fused)
    _expect_kernel(names, fused and _fused_supported(B, V, D, C, k))
    _check(emb, W, b, cent, k, out, min_safe=0.5)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("kind", ["small", "large", "outlier", "positive"])
@pytest.mark.parametrize("D", [64, 1024])
def test_head_forward_magnitudes(cuda, D, kind, fused):
    B, V, C, k = 257, 4, 2203, 50
    emb, W, b, cent = _operands(B, V, D, C, kind, D, cuda)
    out, names = _forward(emb, W, b, cent, k, fused)
    _expect_kernel(names, fused)
    _check(emb, W, b, cent, k, out)
    if kind == "large":      # k above the count of non-zero probabilities: the tail is a tie at 0, in index order
        nz = (out["probs"] > 0).sum(1)
        assert (nz < k).float().mean().item() > 0.5, nz
        assert (out["topk_val"][:, -1] == 0).any()


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("B,D,C,k", [(129, 64, 130, 50), (3, 1024, 2203, 2203), (2, 72, 129, 129)])
def test_head_zero_layer_ties_in_index_order(cuda, B, D, C, k, fused):
    """A cell layer of zeros gives every logit the same value: the top-k is 0, 1, ..., k - 1."""
    emb = torch.randn(B, 4, D, generator=torch.Generator().manual_seed(C)).to(cuda)
    W, b = torch.zeros(C, D, device=cuda), torch.zeros(C, device=cuda)
    cent = torch.rand(C, 2, dtype=torch.float64, generator=torch.Generator().manual_seed(1)).to(cuda)
    out, names = _forward(emb, W, b, cent, k, fused)
    _expect_kernel(names, fused and D % 64 == 0)
    assert (out["logits"] == 0).all() and (out["probs"] == out["probs"][0, 0]).all()
    assert torch.equal(out["topk_idx"], torch.arange(k, device=cuda).expand(B, k))
    assert (out["pred_cell"] == 0).all()
    _check(emb, W, b, cent, k, out)


@pytest.mark.parametrize("fused", [False, True])
def test_head_duplicate_rows_tie_in_index_order(cuda, fused):
    """Cells 2j and 2j + 1 share weights and bias: equal probabilities, the even cell ranked first."""
    B, D, C, k = 257, 1024, 2204, 50
    emb, W, b, cent = _operands(B, 4, D, C, "plain", 11, cuda)
    W[1::2], b[1::2] = W[0::2], b[0::2]
    out, names = _forward(emb, W, b, cent, k, fused)
    _expect_kernel(names, fused)
    assert torch.equal(out["probs"][:, 0::2], out["probs"][:, 1::2])
    _check(emb, W, b, cent, k, out)
    both = torch.isin(out["topk_idx"] ^ 1, out["topk_idx"])
    assert both.any()
    idx = out["topk_idx"]
    for r in range(B):
        rank = {c: j for j, c in enumerate(idx[r].tolist())}
        for c, j in rank.items():
            if c % 2 == 0 and c + 1 in rank:
                assert j + 1 == rank[c + 1], (r, c)


@pytest.mark.parametrize("fused", [False, True])
def test_head_nan_sample_leaves_its_block_exact(cuda, fused):
    B, D, C, k = 257, 64, 130, 5
    emb, W, b, cent = _operands(B, 4, D, C, "plain", 12, cuda)
    emb[130, 2, 17] = float("nan")
    out, names = _forward(emb, W, b, cent, k, fused)
    _expect_kernel(names, fused)
    assert torch.equal(out["topk_idx"][130], torch.arange(k, device=cuda)) and out["pred_cell"][130].item() == 0
    ref = torch.softmax(out["logits"][130], -1)
    assert torch.isnan(ref).all() and torch.isnan(out["probs"][130]).all()
    _check(emb, W, b, cent, k, out)


def test_head_fused_back_to_back_batches(cuda):
    """The sample-block tickets are reused by the next launch: B = 300 then B = 129 on the same weights."""
    from pigeon_b200 import ops
    D, C, k = 1024, 2203, 50
    e1, W, b, cent = _operands(300, 4, D, C, "plain", 13, cuda)
    e2 = _operands(129, 4, D, C, "plain", 14, cuda)[0]
    w3 = ops.head_pack_weight(W)
    ops.head_set_fused(True)
    try:
        (o1, o2), names = _kernels(lambda: (ops.head_forward(e1, w3, b, cent, k), ops.head_forward(e2, w3, b, cent, k)))
    finally:
        ops.head_set_fused(False)
    _expect_kernel(names, True)
    _check(e1, W, b, cent, k, o1)
    _check(e2, W, b, cent, k, o2)


def test_head_unaligned_embedding_falls_back(cuda):
    B, V, D, C, k = 129, 4, 1024, 2203, 50
    emb, W, b, cent = _operands(B, V, D, C, "plain", 15, cuda)
    buf = torch.empty(B * V * D + 1, device=cuda)
    shifted = buf[1:].view(B, V, D)
    shifted.copy_(emb)
    assert shifted.data_ptr() % 16 == 4
    out, names = _forward(shifted, W, b, cent, k, True)
    _expect_kernel(names, False)
    _check(emb, W, b, cent, k, out)


def test_head_refuses_rows_beyond_shared_memory(cuda):
    from pigeon_b200 import PigeonB200Error
    emb, W, b, cent = _operands(2, 1, 8, 51201, "plain", 16, cuda)
    with pytest.raises(PigeonB200Error, match="too large"):
        _forward(emb, W, b, cent, 5, False)


@pytest.mark.parametrize("fused", [False, True])
def test_head_empty_batch(cuda, fused):
    """B = 0 returns empty outputs of the right shapes, like the reference's Linear, softmax and topk, and launches nothing."""
    emb, W, b, cent = _operands(1, 4, 64, 130, "plain", 17, cuda)
    out, names = _forward(emb[:0].contiguous(), W, b, cent, 5, fused)
    assert not names, names
    shapes = dict(pooled=(0, 64), logits=(0, 130), probs=(0, 130), pred_cell=(0,), pred_lnglat=(0, 2), topk_val=(0, 5),
                  topk_idx=(0, 5))
    assert {n: tuple(t.shape) for n, t in out.items()} == shapes


# ------------------------------------------------------------------------------------------------ loss
def _loss_call(logits, mode, idx, soft, lab, cent, smoothing, grad_scale):
    from pigeon_b200._lib import check, current_stream_ptr, load, ptr
    lib = load()
    B, C = logits.shape
    dev = logits.device
    per = torch.empty(B, dtype=torch.float64, device=dev)
    out = torch.empty(1, dtype=torch.float64, device=dev)
    dl = torch.empty(B, C, dtype=torch.float32, device=dev)
    args = (ptr(idx) if mode == 0 else None, ptr(soft) if mode == 1 else None, ptr(lab) if mode == 2 else None,
            ptr(cent) if mode == 2 else None, smoothing)
    check(lib.pg_head_loss_grad(ptr(logits), B, C, mode, *args, grad_scale, ptr(per), ptr(out), ptr(dl),
                                current_stream_ptr()), "pg_head_loss_grad")
    per2 = torch.empty_like(per)
    out2 = torch.empty_like(out)
    check(lib.pg_head_loss(ptr(logits), B, C, mode, *args, ptr(per2), ptr(out2), current_stream_ptr()), "pg_head_loss")
    torch.cuda.synchronize()
    assert torch.equal(per, per2) and torch.equal(out, out2), "pg_head_loss and pg_head_loss_grad disagree"
    return per, out, dl


LOSS_CASES = [  # (B, C, logit scale, smoothing km, grad_scale)
    (1, 1, 3.0, 65.0, 1.0), (3, 255, 3.0, 65.0, 1.0), (3, 256, 3.0, 65.0, 0.37), (4, 257, 1e3, 65.0, 1.0),
    (2, 12289, 3.0, 65.0, 2.5), (5, 2203, 1e3, 1e-3, 1.0), (3, 130, 3.0, 1e-3, 1.0)]


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("B,C,scale,smoothing,grad_scale", LOSS_CASES)
def test_loss_and_gradient_per_element(cuda, B, C, scale, smoothing, grad_scale, mode):
    g = torch.Generator().manual_seed(B * C + mode)
    logits = (torch.randn(B, C, generator=g) * scale).to(cuda)
    idx = torch.randint(0, C, (B,), generator=g).to(cuda)
    soft = torch.rand(B, C, generator=g) * (torch.rand(B, C, generator=g) < 0.3)
    soft[0] = 0                                    # a row that sums to 0
    if B > 1:
        soft[1] *= 3.7 / max(soft[1].sum().item(), 1e-30)   # and one that sums to more than 1
    soft = soft.to(cuda)
    cent = torch.stack([torch.rand(C, generator=g, dtype=torch.float64) * 360 - 180,
                        torch.rand(C, generator=g, dtype=torch.float64) * 180 - 90], 1)
    cent[0] = torch.tensor([179.95, 10.0], dtype=torch.float64)
    lab = torch.stack([torch.rand(B, generator=g, dtype=torch.float64) * 360 - 180,
                       torch.rand(B, generator=g, dtype=torch.float64) * 180 - 90], 1)
    lab[0] = cent[C // 2]                          # on a centroid
    if B > 1:
        lab[1] = torch.tensor([-179.97, 10.01], dtype=torch.float64)   # across the antimeridian from centroid 0
    if B > 2:
        lab[2] = torch.tensor([30.0, 90.0], dtype=torch.float64)       # at the pole
    cent, lab = cent.to(cuda), lab.to(cuda)
    per, out, dl = _loss_call(logits, mode, idx, soft, lab, cent, smoothing, grad_scale)
    t = O.targets(mode, C, idx, soft, lab, cent, smoothing)
    rper, pbound, rg, gbound = O.loss(logits, t, mode, smoothing, grad_scale)
    assert O.ratio(per - rper, pbound) <= 1, O.ratio(per - rper, pbound)
    assert abs(out.item() - rper.mean().item()) <= pbound.sum().item() / B + 1e-15 * rper.abs().mean().item()
    assert O.ratio(dl - rg, gbound) <= 1, O.ratio(dl - rg, gbound)
    if mode == 2 and B > 1 and C > 1:
        assert t[1, 0] > 0.5 or smoothing < 1          # 5 km across the antimeridian, not 40000


# ------------------------------------------------------------------------------------------------ backward
BWD_FORMS = {"all": (1, 1, 1), "no_bias": (1, 0, 1), "dpooled": (0, 0, 1), "weights": (1, 1, 0)}


@pytest.mark.parametrize("acc", [0, 1])
@pytest.mark.parametrize("B,C,D", [(1, 1, 8), (15, 63, 72), (17, 65, 1024), (65, 2203, 72), (65, 2203, 1024),
                                   (17, 1, 72), (1, 65, 8)])
def test_head_backward_per_element(cuda, B, C, D, acc):
    from pigeon_b200._lib import check, current_stream_ptr, load, ptr
    lib = load()
    g = torch.Generator().manual_seed(B * 31 + C + D)
    dl = (torch.randn(B, C, generator=g) * 0.01).to(cuda)
    x = (torch.randn(B, D, generator=g) * 0.5).to(cuda)
    w = (torch.randn(C, D, generator=g) * 0.03).to(cuda)
    dw0 = (torch.randn(C, D, generator=g) * 0.01).to(cuda)
    db0 = (torch.randn(C, generator=g) * 0.01).to(cuda)
    for form, (want_w, want_b, want_x) in BWD_FORMS.items():
        dw, db = dw0.clone(), db0.clone()
        dx = torch.full((B, D), float("nan"), device=cuda)
        check(lib.pg_head_backward(ptr(dl), ptr(x) if want_w else None, ptr(w) if want_x else None, B, C, D, acc,
                                   ptr(dw) if want_w else None, ptr(db) if want_b else None, ptr(dx) if want_x else None,
                                   current_stream_ptr()), "pg_head_backward")
        torch.cuda.synchronize()
        if want_w:
            ref, bound = O.gemm(dl.t(), x, dw0 if acc else None)
            assert O.ratio(dw - ref, bound) <= 1, (form, "dw")
        else:
            assert torch.equal(dw, dw0)
        if want_b:
            ref, bound = O.gemm(dl.t(), torch.ones(B, 1, device=cuda), db0[:, None] if acc else None)
            assert O.ratio(db - ref[:, 0], bound[:, 0]) <= 1, (form, "db")
        else:
            assert torch.equal(db, db0)
        if want_x:
            ref, bound = O.gemm(dl, w)
            assert O.ratio(dx - ref, bound) <= 1, (form, "dpooled")
        else:
            assert torch.isnan(dx).all()
