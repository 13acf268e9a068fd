"""The bounds of tests/tower_blocks_oracle.py are neither loose enough to pass anything nor too tight for the kernels' own
arithmetic.  Each kernel's fp32 arithmetic is restated here in torch, in the kernel's order (warp layout, shuffle tree,
per-warp / per-block / atomic partial sums), and must stay within the bound; two plausible slips must not."""
import numpy as np
import pytest
import torch

import tower_blocks_oracle as O

EPS = 1e-5


def _warp_sum(v):
    """xor-shuffle tree over the last dim (32 lanes): every lane ends with the same total."""
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lane ^ o]
    return v


def _slots(x):
    """[rows, hidden] -> [rows, NV4, 32, 4]: lane l holds columns 4 (l + 32 i) .. + 3 of slot i."""
    return x.reshape(x.shape[0], -1, 32, 4)


def _lane_sum(v):
    """sum of a [rows, NV4, 32, 4] tensor as the kernels add it: (x + y) + (z + w) per slot, slots in order, then the tree."""
    s = torch.zeros(v.shape[0], 32, dtype=torch.float32)
    for i in range(v.shape[1]):
        s = s + ((v[:, i, :, 0] + v[:, i, :, 1]) + (v[:, i, :, 2] + v[:, i, :, 3]))
    return _warp_sum(s)[:, 0].reshape(-1, 1, 1, 1)


def _stats(x, hidden, var_div=None):
    v = _slots(x)
    mean = _lane_sum(v) / hidden
    a = v - mean
    var = _lane_sum(a * a) / (hidden if var_div is None else var_div)
    rstd = torch.rsqrt(var + torch.tensor(EPS, dtype=torch.float32))
    return a, rstd


def sim_layernorm(x, g, b, var_div=None):
    hidden = x.shape[1]
    a, rstd = _stats(x, hidden, var_div)
    y = (a * rstd) * _slots(g[None]) + _slots(b[None])
    return y.reshape(x.shape)


def sim_layernorm_backward(dy, x, g, drop_slot=False):
    hidden = x.shape[1]
    a, rstd = _stats(x, hidden)
    xh = a * rstd
    dv = _slots(dy)
    gd = dv * _slots(g[None])
    s1 = _lane_sum(gd) / hidden
    s2 = _lane_sum(gd * xh) / hidden
    corr = xh * s2
    if drop_slot:                                   # one float4 slot (the last lane's last slot) forgets xhat * s2
        corr[:, -1, 31, :] = 0
    dx = rstd * ((gd - s1) - corr)
    return dx.reshape(x.shape), (dv * xh).reshape(x.shape), dy


def sim_param_sums(prod, init, sms, gen, reset=False):
    """ln_backward_kernel's dgamma / dbeta: per-warp row sums, 8 warps per block in order, blocks by atomics in any order.
    reset: a warp that restarts its sums at every row (keeps only its last row)."""
    rows, n = prod.shape
    blocks, rpw = O.ln_backward_schedule(rows, sms)
    warps = 8 * blocks
    pad = torch.zeros(rpw * warps, n, dtype=torch.float32)
    pad[:rows] = prod
    acc = torch.zeros(warps, n, dtype=torch.float32)
    for k in range(rpw):
        acc = (0 if reset else acc) + pad[k * warps:(k + 1) * warps]
    t = torch.zeros(blocks, n, dtype=torch.float32)
    for w in range(8):
        t = t + acc.view(blocks, 8, n)[:, w]
    out = init.clone()
    for blk in torch.randperm(blocks, generator=gen).tolist():
        out = out + t[blk]
    return out


def _inputs(kind, rows, hidden, gen):
    x = torch.randn(rows, hidden, generator=gen) * 2 + 0.3
    if kind == "offset":
        x = 1000 + torch.randn(rows, hidden, generator=gen)
    elif kind == "constant":
        x = torch.full((rows, hidden), 0.7) + torch.arange(rows)[:, None] * 0.01
    elif kind == "outlier":
        x[:, 7] = 150.0
    g = 1 + 0.2 * torch.randn(hidden, generator=gen)
    b = 0.1 * torch.randn(hidden, generator=gen)
    return x.float(), g.float(), b.float()


@pytest.mark.parametrize("hidden", [128, 256, 512, 768, 1024])
@pytest.mark.parametrize("kind", ["plain", "offset", "constant", "outlier"])
def test_layernorm_forward_bound_holds_and_catches_bessel(hidden, kind):
    gen = torch.Generator().manual_seed(hidden)
    x, g, b = _inputs(kind, 64, hidden, gen)
    ref, bound = O.layernorm_forward(x, g, b, EPS)
    y = sim_layernorm(x, g, b)
    assert O.ratio(y - ref, bound) <= 1
    ref16, bound16 = O.layernorm_forward(x, g, b, EPS, out_f16=True)
    assert O.ratio(y.half().double() - ref16, bound16) <= 1
    if kind == "plain":
        bad = sim_layernorm(x, g, b, var_div=hidden - 1)
        assert O.ratio(bad - ref, bound) > 1
        if hidden <= 256:                          # 1 / (2 hidden) above half an fp16 ulp
            assert O.ratio(bad.half().double() - ref16, bound16) > 1


@pytest.mark.parametrize("hidden", [128, 256, 512, 768, 1024])
@pytest.mark.parametrize("kind", ["plain", "offset", "constant", "outlier"])
def test_layernorm_backward_bound_holds_and_catches_dropped_slot(hidden, kind):
    gen = torch.Generator().manual_seed(hidden + 1)
    rows, sms = 300, 4                              # 32 blocks of 8 warps: 2 rows per warp
    x, g, _ = _inputs(kind, rows, hidden, gen)
    dy = (torch.randn(rows, hidden, generator=gen) * 1e-3).float()
    dx0 = (torch.randn(rows, hidden, generator=gen) * 1e-3).float()
    ref = O.layernorm_backward(dy, x, g, EPS, dx0=dx0)
    dx, pg, pb = sim_layernorm_backward(dy, x, g)
    assert O.ratio(dx + dx0 - ref["dx"], ref["bound"]) <= 1
    dg0, db0 = torch.full((hidden,), 0.5), torch.full((hidden,), -0.25)
    blocks, rpw = O.ln_backward_schedule(rows, sms)
    bg, bb = O.ln_param_bounds(ref, dg0, db0, rpw + 8 + blocks)
    dg = sim_param_sums(pg, dg0, sms, gen)
    db = sim_param_sums(pb, db0, sms, gen)
    assert O.ratio(dg - (dg0.double() + ref["dgamma"]), bg) <= 1
    assert O.ratio(db - (db0.double() + ref["dbeta"]), bb) <= 1
    if kind == "plain":
        bad, _, _ = sim_layernorm_backward(dy, x, g, drop_slot=True)
        assert O.ratio(bad + dx0 - ref["dx"], ref["bound"]) > 1
        reset = sim_param_sums(pg, dg0, sms, gen, reset=True)
        assert O.ratio(reset - (dg0.double() + ref["dgamma"]), bg) > 1


@pytest.mark.parametrize("rows,cols", [(1, 1), (129, 257), (1000, 300)])
def test_column_sum_bound(rows, cols):
    gen = torch.Generator().manual_seed(rows)
    x = torch.randn(rows, cols, generator=gen).float()
    out0 = torch.randn(cols, generator=gen).float()
    ref, bound = O.column_sum(x, out0)
    parts = []
    for r0 in range(0, rows, 128):
        s = torch.zeros(cols, dtype=torch.float32)
        for r in range(r0, min(rows, r0 + 128)):
            s = s + x[r]
        parts.append(s)
    out = out0.clone()
    for i in torch.randperm(len(parts), generator=gen).tolist():
        out = out + parts[i]
    assert O.ratio(out - ref, bound) <= 1
    short = out - x[min(rows, 128) - 1]             # a chunk that stops one row early
    assert O.ratio(short - ref, bound) > 1


@pytest.mark.parametrize("tokens,hidden", [(577, 1024), (50, 128), (257, 768)])
def test_token_mean_bound(tokens, hidden):
    gen = torch.Generator().manual_seed(tokens)
    x = (torch.randn(3, tokens, hidden, generator=gen) + 0.5).float()
    ref, bound = O.token_mean(x, hidden)
    ny = max(1, min(8, 1024 // (hidden // 4)))
    parts = []
    for y in range(ny):
        s = torch.zeros(3, hidden, dtype=torch.float32)
        for t in range(y, tokens, ny):
            s = s + x[:, t]
        parts.append(s)
    acc = parts[0]
    for p in parts[1:]:
        acc = acc + p
    inv = torch.tensor(1.0, dtype=torch.float32) / tokens
    assert O.ratio(acc * inv - ref, bound) <= 1
    assert O.ratio((acc - parts[-1]) * inv - ref, bound) > 1


def test_token_embedding_grad_bound():
    gen = torch.Generator().manual_seed(3)
    vocab, rows, hidden = 50, 600, 128
    ids = torch.randint(0, vocab, (rows,), generator=gen)
    ids[::3] = 7                                    # one id repeated 200 times
    dx = torch.randn(rows, hidden, generator=gen).float()
    dtok0 = torch.randn(vocab, hidden, generator=gen).float()
    ref, bound, seen = O.token_embedding_grad(ids, dx, vocab, dtok0)
    out = dtok0.clone()
    for i in ids.unique().tolist():
        s = torch.zeros(hidden, dtype=torch.float32)
        for r in (ids == i).nonzero().flatten().tolist():
            s = s + dx[r]
        out[i] = out[i] + s
    assert O.ratio(out - ref, bound) <= 1
    skip_first = out.clone()
    skip_first[7] -= dx[0]
    assert O.ratio(skip_first - ref, bound) > 1


def test_first_argmax_takes_the_first_of_ties():
    ids = torch.tensor([[5, 9, 9, 1], [9, 0, 0, 9], [0, 0, 0, 0], [1, 2, 3, 4]])
    assert O.first_argmax(ids).tolist() == [1, 0, 0, 3]


def test_half_ulp_f16():
    v = torch.tensor([1.0, 1.5, 2.0, 65504.0, 2.0 ** -14, 1e-6], dtype=torch.float64)
    expect = np.array([2.0 ** -11, 2.0 ** -11, 2.0 ** -10, 16.0, 2.0 ** -25, 2.0 ** -25])
    assert np.array_equal(O.half_ulp_f16(v).numpy(), expect)
