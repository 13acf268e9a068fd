"""The bounds of tests/head_oracle.py are neither loose enough to pass a broken head nor too tight for the kernels' own
arithmetic.  The split GEMM is restated in torch with fp32 accumulation and must stay within the logit bound; plain fp16
operands and a split missing any one of its three products must not.  The top-k reference breaks ties by the first index,
so a last-index tie-break must not match it."""
import pytest
import torch

import head_oracle as O


def _operands(kind, B, C, D, gen):
    x = torch.randn(B, D, generator=gen) * 0.3
    W = torch.randn(C, D, generator=gen) * D ** -0.5
    if kind == "small":                 # lo and Wlo deep in the fp16 subnormals
        x, W = x * 3e-3, W * 3e-3
    elif kind == "large":
        x = x * 300
    elif kind == "outlier":             # a few channels far above the rest
        x[:, :3] = 80.0
        W[:, :3] *= 20
    elif kind == "positive":            # every partial sum keeps its sign
        x, W = x.abs(), W.abs()
    b = torch.randn(C, generator=gen) * 0.1
    return x.float(), W.float(), b.float()


def _split_logits(x, W, b, drop=None):
    """The kernel's GEMM with fp32 accumulation; drop = 0, 1 or 2 leaves out hi.Whi, lo.Whi or hi.Wlo."""
    a3, w3 = O.split_operands(x, W)
    D = x.shape[1]
    if drop is not None:
        a3 = a3.clone()
        a3[:, drop * D:(drop + 1) * D] = 0
    return a3.float() @ w3.float().t() + b


@pytest.mark.parametrize("D", [8, 64, 256, 1024])
@pytest.mark.parametrize("kind", ["plain", "small", "large", "outlier", "positive"])
def test_logit_bound_holds_for_the_split(kind, D):
    gen = torch.Generator().manual_seed(D)
    x, W, b = _operands(kind, 64, 257, D, gen)
    ref, bound = O.logits(x, W, b)
    assert O.ratio(_split_logits(x, W, b) - ref, bound) <= 1


@pytest.mark.parametrize("D", [64, 256, 1024])
def test_logit_bound_catches_plain_fp16_and_each_missing_product(D):
    gen = torch.Generator().manual_seed(D + 1)
    x, W, b = _operands("plain", 128, 1024, D, gen)
    ref, bound = O.logits(x, W, b)
    plain = x.half().float() @ W.half().float().t() + b
    assert O.ratio(plain - ref, bound) > 1
    for drop in range(3):
        r = O.ratio(_split_logits(x, W, b, drop) - ref, bound)
        assert r > 1, (drop, r)


def test_logit_bound_floor_is_what_keeps_small_magnitudes():
    """At |x|, |W| ~ 1e-3 the lo parts are fp16 subnormals: without the 2^-25 floor the exact split would fail."""
    gen = torch.Generator().manual_seed(3)
    x, W, b = _operands("small", 64, 257, 256, gen)
    b = torch.zeros_like(b)
    ref, bound = O.logits(x, W, b)
    got = _split_logits(x, W, b)
    assert O.ratio(got - ref, bound) <= 1
    rel = O.alpha(256) * (x.double().abs() @ W.double().abs().t())
    assert O.ratio(got - ref, rel * (1 + O.U)) > 1


def test_prob_bound_holds_and_catches_a_shifted_row():
    gen = torch.Generator().manual_seed(4)
    x, W, b = _operands("plain", 32, 2203, 1024, gen)
    W = W * 8
    ref, L = O.logits(x, W, b)
    p, P = O.probs(ref, L)
    got = torch.softmax(_split_logits(x, W, b), -1)
    assert O.ratio(got - p, P) <= 1
    bad = torch.softmax(_split_logits(x, W, b) + 1e-4 * torch.arange(2203.0), -1)   # a drift of 0.2 across the row
    assert O.ratio(bad - p, P) > 1


def test_stable_topk_orders_ties_and_nan():
    p = torch.tensor([[0.1, 0.3, 0.3, 0.0, 0.3],
                      [0.0, 0.0, 0.0, 0.0, 0.0],
                      [0.2, float("nan"), 0.5, float("nan"), 0.5]])
    v, i = O.stable_topk(p, 5)
    assert i.tolist() == [[1, 2, 4, 0, 3], [0, 1, 2, 3, 4], [1, 3, 2, 4, 0]]
    assert torch.equal(v[0], torch.tensor([0.3, 0.3, 0.3, 0.1, 0.0]))


def test_last_index_tie_break_fails_the_stable_reference():
    gen = torch.Generator().manual_seed(5)
    p = torch.randint(0, 4, (16, 40), generator=gen).float() / 4        # many exact ties
    _, first = O.stable_topk(p, 10)
    # last index among ties: the stable reference of the reversed row, mapped back
    _, rev = O.stable_topk(p.flip(1), 10)
    last = 39 - rev
    assert not torch.equal(first, last)
    assert torch.equal(torch.gather(p, 1, first), torch.gather(p, 1, last))   # the same values, in another order


def test_safe_ranks():
    p = torch.tensor([[0.5, 0.3, 0.1, 0.1], [0.4, 0.4, 0.1, 0.1]], dtype=torch.float64)
    P = torch.full_like(p, 1e-3)
    assert O.safe_ranks(p, P, 3).tolist() == [[True, True, False], [False, False, False]]


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_loss_reference_matches_torch_cross_entropy(mode):
    gen = torch.Generator().manual_seed(mode)
    B, C = 6, 300
    x = (torch.randn(B, C, generator=gen) * 4).float()
    idx = torch.randint(0, C, (B,), generator=gen)
    soft = torch.rand(B, C, generator=gen)
    lab = torch.stack([torch.rand(B, generator=gen, dtype=torch.float64) * 360 - 180,
                       torch.rand(B, generator=gen, dtype=torch.float64) * 180 - 90], 1)
    cent = torch.stack([torch.rand(C, generator=gen, dtype=torch.float64) * 360 - 180,
                        torch.rand(C, generator=gen, dtype=torch.float64) * 180 - 90], 1)
    t = O.targets(mode, C, idx, soft, lab, cent)
    if mode == 2:
        from oracle.geo import haversine_matrix, smooth_labels
        assert torch.allclose(t, smooth_labels(haversine_matrix(lab, cent.t())), rtol=1e-12, atol=0)
    xl = x.double().requires_grad_(True)
    ce = torch.nn.functional.cross_entropy(xl, t if mode else idx)
    ce.backward()
    per, pb, g, gb = O.loss(x, t, mode)
    assert abs(per.mean().item() - ce.item()) <= 1e-12 * abs(ce.item())
    assert O.ratio(g - xl.grad, gb) <= 1


def test_gemm_bound_catches_a_dropped_accumulator():
    gen = torch.Generator().manual_seed(6)
    a, b, c0 = torch.randn(17, 65, generator=gen), torch.randn(65, 72, generator=gen), torch.randn(17, 72, generator=gen)
    ref, bound = O.gemm(a, b, c0)
    got = (a.double() @ b.double()).float() + c0
    assert O.ratio(got - ref, bound) <= 1
    assert O.ratio((a.double() @ b.double()).float() - ref, bound) > 1
