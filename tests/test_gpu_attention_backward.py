"""Both attention backward kernels (pg_attention_backward and pg_attention_backward_masked, with their attention_delta
prologue) against plain float64 arithmetic, per element, at the head counts, masks and tile edges where they go wrong: one
token, one partial 64-row tile, a last tile with one valid row (S = 577), odd head counts, causal and padding masks, a
non-causal mask with interior zeros and a whole masked key block, and logits from near-uniform to peaked.

The inputs are built directly, so the backward is tested on its own: random fp16 qkv, `out` = fp64 attention rounded to
fp16, `lse2` = fp64 log2-sum-exp over the admissible keys rounded to fp32, fp32 d_out.  The reference is torch float64 on the
device applied to what the kernel reads, rounding where the kernel rounds (attention_bwd_wgmma.cu):
  delta = rowsum(d_out * out),  dO = bf16(d_out),  q, k, v = bf16(qkv),  S = q16 k16^T (fp16 operands),
  P = 2^(S c - lse2) with the kernel's fp32 c = 0.125f * 1.4426950408889634f (0 where inadmissible or below 2^-126),
  dP = dO v^T,  dS = P (dP - delta) / 8,  dQ = bf16(dS) k,  dK = bf16(dS)^T q,  dV = bf16(P)^T dO,  output bf16.
So the reference differs from the kernel by accumulation order, the fp32 arithmetic that forms P and dS, and the output
rounding.  Per-element bound, with u = 2^-24:
  * accumulation: C_ACC * u * sqrt(K) * A, A = sum_k |a_k||b_k| over the contraction, K its length padded to the 64-row
    tile (the probabilistic bound of the GEMM epilogue test, C_ACC = 2);
  * rounding flips of P and dS: the kernel's fp32 P is within e_P = P (ln2 (c e_S + u |S c - lse2|) + EX2_REL) of the fp64
    value, e_S = C_ACC u sqrt(64) |q16||k16|^T being the logits' accumulation error and EX2_REL ex2.approx's relative
    error; its dS is within e_dS = P/8 (|dP - delta| (e_P/P + 2u) + e_dP + e_delta) + 2^-149, e_dP the accumulation error of
    dP and e_delta = 8 u rowsum|d_out * out| that of delta (a product and seven adds).  Both are doubled for the
    second-order terms.  The kernel's bf16 operand then lies between bf16(x - e) and bf16(x + e) (0 when x - e < 2^-126 for
    P: ex2.approx.ftz flushes), so that span (zero away from a rounding boundary, one ulp near one) times |partner operand|,
    one more matmul, bounds what the flips can change;
  * output rounding: one bf16 ulp of |reference| + the two terms above.
The largest error / bound per case is printed at the end of the module.

Exact properties: two runs give the same bits (no atomics); each view's rows do not change when every other view's qkv,
out, d_out and lse2 are NaN, and equal a one-view call; keys with mask == 0 get dK = dV = 0; scaling d_out by 2^-17 scales
dqkv by exactly 2^-17; the masked instantiation with an all-ones mask and causal = 0 gives the unmasked kernel's bits; NaN
guard rows around dqkv survive.  A plain fp32-autograd comparison (rel-L2 1.5e-2 per q / k / v; 3e-2 with at most two
keys, and for dQ at near-uniform attention a bar widened by the worst case of the rounding that `_autograd` explains) keeps
the rounding emulation from hiding a misreading of the maths shared by kernel and reference.

The forward's lse2, which the backward uses to rebuild P, is checked per element against fp64 logsumexp * log2(e) within
the fp32 bound derived at `_lse2_bound`."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_ACC = 2.0
EX2_REL = 2.0 ** -21            # ex2.approx.ftz.f32: a relative error of a few fp32 ulp
FTZ = 2.0 ** -126
LOG2E = 1.4426950408889634
C_LOG2 = (torch.tensor(0.125, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)).item()   # the kernel's c
GUARD = 2                       # NaN guard rows before and after dqkv
SENT = 0x7FD5                   # bf16 NaN with a payload the kernel never writes
AUTOGRAD_REL = 1.5e-2
RATIOS = {}                     # case -> largest observed error / bound, printed at the end of the module
AUTOGRAD = {}                   # case -> rel-L2 of dq, dk, dv against fp32 autograd

# id: (n_views, S, heads, mask, logits, d_out scale).  Masks: none = pg_attention_backward; causal; pad = causal + padding
# with lengths 1, S // 2, S, ...; interior = causal 0 with interior zeros (and, from S = 128, one whole masked key block);
# ones = causal 0 with an all-ones mask (the masked kernel).  Logits: typical q, k x 0.8; uniform q, k x 0.05 plus a key
# component shared by all tokens of a head, as the text tower's keys have (the softmax ignores it, bf16(dS) does not);
# peaked q, k x 3; ramp = keys growing along the sequence (the forward test's online-softmax ramp).
CASES = {
    "S1-h1": (1, 1, 1, "none", "typical", 1.0),
    "S2-h2-causal": (3, 2, 2, "causal", "typical", 1e-5),
    "S2-h5-interior": (1, 2, 5, "interior", "peaked", 1.0),
    "S17-h3": (3, 17, 3, "none", "peaked", 1.0),
    "S17-h1-pad": (3, 17, 1, "pad", "typical", 1e-5),
    "S63-h5-causal": (1, 63, 5, "causal", "ramp", 1e-5),
    "S64-h16-interior": (3, 64, 16, "interior", "typical", 1.0),
    "S65-h2-pad": (3, 65, 2, "pad", "peaked", 1e-5),
    "S65-h3": (1, 65, 3, "none", "uniform", 1.0),
    "S77-h12-pad-uniform": (3, 77, 12, "pad", "uniform", 1.0),
    "S77-h12-text-batch": (64, 77, 12, "pad", "uniform", 1e-5),
    "S77-h5-ones": (1, 77, 5, "ones", "typical", 1e-5),
    "S128-h1-interior": (3, 128, 1, "interior", "ramp", 1.0),
    "S129-h3-ones": (1, 129, 3, "ones", "peaked", 1.0),
    "S129-h12-causal": (3, 129, 12, "causal", "uniform", 1e-5),
    "S577-h16": (3, 577, 16, "none", "typical", 1e-5),
    "S577-h5-pad": (3, 577, 5, "pad", "ramp", 1.0),
    "S577-h1-interior": (1, 577, 1, "interior", "uniform", 1e-5),
}


@pytest.fixture(scope="module")
def lib(cuda):
    from pigeon_b200 import _lib
    lib = _lib.load()
    yield lib
    if RATIOS:
        print("\nmax |error| / bound per case:", {k: round(v, 4) for k, v in RATIOS.items()})
    if AUTOGRAD:
        print("rel-L2 (dq, dk, dv) against fp32 autograd:", {k: tuple(round(x, 5) for x in v) for k, v in AUTOGRAD.items()})


def _note(key, ratio):
    RATIOS[key] = max(RATIOS.get(key, 0.0), ratio)


# ------------------------------------------------------------------------------------------------ inputs
def _mask(kind, n, S, seed):
    """(mask i64 [n, S] or None, causal) of a mask kind; mask[:, 0] = 1 as the forward requires."""
    if kind == "none":
        return None, False
    if kind == "causal":
        return None, True
    g = torch.Generator().manual_seed(seed + 1)
    if kind == "pad":
        lengths = [1, max(1, S // 2), S] + torch.randint(1, S + 1, (max(0, n - 3),), generator=g).tolist()
        m = torch.zeros(n, S, dtype=torch.int64)
        for b in range(n):
            m[b, :lengths[b % len(lengths)]] = 1
        return m, True
    if kind == "interior":
        m = (torch.rand(n, S, generator=g) > 0.3).to(torch.int64)
        if S >= 128:
            m[n // 2, 64:128] = 0            # a key block with no admissible key
        m[:, 0] = 1
        return m, False
    assert kind == "ones"
    return torch.ones(n, S, dtype=torch.int64), False


def _admissible(n, S, mask, causal, dev):
    ok = torch.ones(n, 1, S, S, dtype=torch.bool, device=dev)
    if causal:
        ok &= torch.ones(S, S, dtype=torch.bool, device=dev).tril()
    if mask is not None:
        ok &= mask.bool()[:, None, None, :]
    return ok


def _qkv(n, S, heads, logits, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, S, 3, heads, 64, generator=g)
    if logits == "typical":
        x[:, :, :2] *= 0.8
    elif logits == "uniform":
        x[:, :, :2] *= 0.05
        x[:, :, 1] += torch.randn(1, heads, 64, generator=g)
    elif logits == "peaked":
        x[:, :, :2] *= 3.0
    else:
        assert logits == "ramp"
        x[:, :, 1] *= (0.25 + 6.0 * torch.arange(S) / S).view(1, S, 1, 1)
    return x.reshape(n * S, 3 * heads * 64).half()


def _split(t, n, S, heads):
    """[n*S, 3*heads*64] -> q, k, v [n, heads, S, 64]."""
    return t.reshape(n, S, 3, heads, 64).permute(2, 0, 3, 1, 4)


def _heads(t, n, S, heads):
    """[n*S, heads*64] -> [n, heads, S, 64]."""
    return t.reshape(n, S, heads, 64).permute(0, 2, 1, 3)


def _case(name, cuda, spec=None):
    n, S, heads, kind, logits, dscale = spec or CASES[name]
    seed = sum(map(ord, name))
    qkv = _qkv(n, S, heads, logits, seed).to(cuda)
    mask, causal = _mask(kind, n, S, seed)
    mask = None if mask is None else mask.to(cuda)
    ok = _admissible(n, S, mask, causal, cuda)
    q, k, v = _split(qkv.double(), n, S, heads)
    logit = (q @ k.transpose(-1, -2)).masked_fill(~ok, -math.inf)
    lse = torch.logsumexp(logit * 0.125, -1)
    out = (torch.exp(logit * 0.125 - lse[..., None]) @ v).permute(0, 2, 1, 3).reshape(n * S, heads * 64).half()
    lse2 = (lse * LOG2E).reshape(n * heads, S).float()
    g = torch.Generator().manual_seed(seed + 2)
    d_out = (torch.randn(n * S, heads * 64, generator=g) * dscale).to(cuda)
    return dict(name=name, n=n, S=S, heads=heads, kind=kind, logits=logits, qkv=qkv, out=out, lse2=lse2, d_out=d_out,
                mask=mask, causal=causal, ok=ok)


# ------------------------------------------------------------------------------------------------ the kernel
def _run(lib, c, masked_abi=None, **over):
    """dqkv of one call with NaN-payload guard rows before and after it, which must survive."""
    from pigeon_b200._lib import check, current_stream_ptr, ptr
    from pigeon_b200.vit_train import _aligned_empty
    c = dict(c, **over)
    n, S, heads = c["n"], c["S"], c["heads"]
    rows, hidden = n * S, heads * 64
    big = torch.empty(rows + 2 * GUARD, 3 * hidden, dtype=torch.bfloat16, device=c["qkv"].device)
    big.view(torch.int16).fill_(SENT)
    dqkv = big[GUARD:GUARD + rows]
    need = lib.pg_attention_backward_workspace_bytes(n, S, heads)
    ws = _aligned_empty(need, c["qkv"].device)
    if masked_abi is None:
        masked_abi = c["kind"] != "none"
    args = (ptr(c["qkv"]), ptr(c["out"]), ptr(c["d_out"]), ptr(c["lse2"]))
    if masked_abi:
        check(lib.pg_attention_backward_masked(*args, ptr(c["mask"]), int(c["causal"]), ptr(dqkv), n, S, heads, ptr(ws), need,
                                               current_stream_ptr()), "pg_attention_backward_masked")
    else:
        check(lib.pg_attention_backward(*args, ptr(dqkv), n, S, heads, ptr(ws), need, current_stream_ptr()),
              "pg_attention_backward")
    torch.cuda.synchronize()
    guards = torch.cat([big[:GUARD], big[GUARD + rows:]]).view(torch.int16)
    assert (guards == SENT).all(), "attention backward wrote outside dqkv"
    return dqkv.clone()


def _bits(t):
    return t.view(torch.int16)


# ------------------------------------------------------------------------------------------------ the fp64 reference
def _bf(x):
    return x.to(torch.bfloat16).double()


def _ulp_bf16(x):
    """One bf16 unit in the last place of x >= 0 (subnormal spacing 2^-133 below the normal range and at 0)."""
    _, e = torch.frexp(x)
    e = (e - 1).clamp_min(-126)
    return torch.where(x > 0, torch.ldexp(torch.ones_like(x), e - 7), torch.full_like(x, 2.0 ** -133))


def _reference(c):
    """([dq, dk, dv] fp64 [n, heads, S, 64], their per-element bounds, the fp64 P, dS and bf16 operands)."""
    n, S, heads, ok = c["n"], c["S"], c["heads"], c["ok"]
    q16, k16, _ = _split(c["qkv"].double(), n, S, heads)
    qb, kb, vb = _split(_bf(c["qkv"]), n, S, heads)
    d_out = _heads(c["d_out"].double(), n, S, heads)
    out = _heads(c["out"].double(), n, S, heads)
    dob = _bf(d_out)
    lse2 = c["lse2"].double().reshape(n, heads, S, 1)
    delta = (d_out * out).sum(-1, keepdim=True)
    e_delta = 8 * U * (d_out * out).abs().sum(-1, keepdim=True)

    s = q16 @ k16.transpose(-1, -2)
    e_s = C_ACC * U * 8 * (q16.abs() @ k16.abs().transpose(-1, -2))
    x = s * C_LOG2 - lse2
    p = torch.where(ok, torch.exp2(x), torch.zeros_like(x))
    e_p = 2 * p * (math.log(2) * (C_LOG2 * e_s + U * x.abs()) + EX2_REL)
    p_ref = torch.where(p < FTZ, torch.zeros_like(p), p)
    p_lo = torch.where(p - e_p < FTZ, torch.zeros_like(p), _bf(p - e_p))
    p_hi = torch.where(p + e_p < FTZ, torch.zeros_like(p), _bf(p + e_p))
    p_flip = p_hi - p_lo

    dp = dob @ vb.transpose(-1, -2)
    e_dp = C_ACC * U * 8 * (dob.abs() @ vb.abs().transpose(-1, -2))
    diff = dp - delta
    ds = p_ref * diff * 0.125
    rel_p = torch.where(p > 0, e_p / p.clamp_min(1e-300), torch.zeros_like(p))
    e_ds = 2 * (p * 0.125 * (diff.abs() * (rel_p + 2 * U) + e_dp + e_delta) + 2.0 ** -149)
    ds_lo, ds_hi = _bf(ds - e_ds), _bf(ds + e_ds)
    flush = p - e_p < FTZ                    # the kernel's P may be 0 here, and then so is its dS
    ds_lo = torch.where(flush, ds_lo.clamp_max(0), ds_lo)
    ds_hi = torch.where(flush, ds_hi.clamp_min(0), ds_hi)
    ds_flip = torch.where(ok, ds_hi - ds_lo, torch.zeros_like(ds))

    pb, dsb = _bf(p_ref), _bf(ds)
    kpad = math.sqrt((S + 63) // 64 * 64)
    refs, bounds = [], []
    for a, flip, b in ((dsb, ds_flip, kb), (dsb.transpose(-1, -2), ds_flip.transpose(-1, -2), qb),
                       (pb.transpose(-1, -2), p_flip.transpose(-1, -2), dob)):
        ref = a @ b
        f = flip @ b.abs()
        e = C_ACC * U * kpad * (a.abs() @ b.abs() + f) + f
        refs.append(ref)
        bounds.append(_ulp_bf16(ref.abs() + e) + e)
    return refs, bounds, dict(p=p_ref, ds=ds, kb=kb, dob=dob, vb=vb)


def _check(c, got, refs, bounds):
    name, n, S, heads = c["name"], c["n"], c["S"], c["heads"]
    for part, g, ref, bound in zip("qkv", _split(got.double(), n, S, heads), refs, bounds):
        err = (g - ref).abs()
        err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
        r = err / bound
        r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
        ratio = r.max().item()
        _note(name, ratio)
        if ratio > 1.0:
            i = tuple(int(j) for j in torch.unravel_index(r.argmax(), r.shape))
            raise AssertionError(f"{name}: d{part} |error| / bound = {ratio:.3g} at [view, head, row, col] = {list(i)}: "
                                 f"got {g[i].item()!r}, reference {ref[i].item()!r}, bound {bound[i].item():.3g}")


def _autograd(c, got, parts):
    """rel-L2 per q / k / v against fp32 autograd of the plain maths on the same inputs; `parts` are the fp64 reference's
    P, dS and bf16 operands."""
    name, n, S, heads, ok = c["name"], c["n"], c["S"], c["heads"], c["ok"]
    x = c["qkv"].float().clone().requires_grad_(True)
    q, k, v = _split(x, n, S, heads)
    w = ((q @ k.transpose(-1, -2)) * 0.125).masked_fill(~ok, -math.inf)
    o = (torch.softmax(w, -1) @ v).permute(0, 2, 1, 3).reshape(n * S, heads * 64)
    o.backward(c["d_out"])
    ref = _split(x.grad.double(), n, S, heads)
    gd = _split(got.double(), n, S, heads)
    scale = max(r.norm().item() for r in ref)
    rels = []
    for i, part in enumerate("qkv"):
        if ref[i].norm().item() < 1e-4 * scale:      # one admissible key per row: dS = 0, so dQ = dK = 0
            assert gd[i].norm().item() < AUTOGRAD_REL * scale, (name, part)
            rels.append(0.0)
            continue
        rel = ((gd[i] - ref[i]).norm() / ref[i].norm()).item()
        # with at most two keys per row, dS is the difference of two terms, and the bf16 dO inside dP (delta uses the fp32
        # d_out) is not averaged out over the keys
        bar = AUTOGRAD_REL if S > 2 else 2 * AUTOGRAD_REL
        if part == "q" and c["logits"] == "uniform":
            # sum_j dS_ij = 0, so a key component shared by every token drops out of dQ.  The kernel's dS does not sum to 0:
            # bf16(dS) rounds each element (2^-9 relative) and dP = bf16(dO) bf16(v)^T is not the dP of the fp32 delta
            # (2^-8 + 2^-18 relative to |dO||v|^T); the shared component enters through both, at most by this much
            p, ds, dob, vb = parts["p"], parts["ds"], parts["dob"], parts["vb"]
            e_ds = 2.0 ** -9 * ds.abs() + (2.0 ** -8 + 2.0 ** -18) * p / 8 * (dob.abs() @ vb.abs().transpose(-1, -2))
            bar += ((e_ds @ parts["kb"].abs()).norm() / ref[i].norm()).item()
        rels.append(rel)
        assert rel < bar, (name, part, rel, bar)
    AUTOGRAD[name] = tuple(rels)


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("name", list(CASES))
def test_backward_matches_fp64_reference(lib, cuda, name):
    c = _case(name, cuda)
    got = _run(lib, c)
    again = _run(lib, c)
    assert torch.equal(_bits(got), _bits(again)), f"{name}: dqkv differs run to run"
    refs, bounds, parts = _reference(c)
    _check(c, got, refs, bounds)
    if c["mask"] is not None:
        # keys excluded by the mask get exactly zero dK and dV
        n, S, heads = c["n"], c["S"], c["heads"]
        _, dk, dv = _split(got, n, S, heads)
        off = (c["mask"] == 0)[:, None, :, None].expand(n, heads, S, 64)
        assert (dk[off] == 0).all() and (dv[off] == 0).all(), f"{name}: masked keys got a gradient"
    if c["kind"] == "ones":
        # the masked kernel with every key admissible and causal = 0 is the unmasked kernel, bit for bit
        assert torch.equal(_bits(got), _bits(_run(lib, c, masked_abi=False))), name
    _autograd(c, got, parts)


@pytest.mark.parametrize("name", ["S2-h2-causal", "S17-h3", "S64-h16-interior", "S65-h2-pad", "S577-h5-pad"])
def test_views_are_independent(lib, cuda, name):
    """With NaN in every other view's qkv, out, d_out and lse2, a view's rows are the bits of a one-view call on its data."""
    c = _case(name, cuda)
    n, S, heads = c["n"], c["S"], c["heads"]
    full = _run(lib, c)
    for view in range(n):
        rows = slice(view * S, (view + 1) * S)
        stats = slice(view * heads, (view + 1) * heads)
        one = _run(lib, c, n=1, qkv=c["qkv"][rows].contiguous(), out=c["out"][rows].contiguous(),
                   d_out=c["d_out"][rows].contiguous(), lse2=c["lse2"][stats].contiguous(),
                   mask=None if c["mask"] is None else c["mask"][view:view + 1].contiguous())
        poisoned = {k: torch.full_like(c[k], math.nan) for k in ("qkv", "out", "d_out", "lse2")}
        for k in ("qkv", "out", "d_out"):
            poisoned[k][rows] = c[k][rows]
        poisoned["lse2"][stats] = c["lse2"][stats]
        got = _run(lib, c, **poisoned)
        assert torch.equal(_bits(got[rows]), _bits(one)), f"{name}: view {view} depends on the other views"
        assert torch.equal(_bits(full[rows]), _bits(one)), f"{name}: view {view} differs from a one-view call"


@pytest.mark.parametrize("name", ["S2-h2-causal", "S17-h1-pad", "S64-h16-interior", "S77-h5-ones", "S577-h16"])
def test_scaling_d_out_by_a_power_of_two_is_exact(lib, cuda, name):
    c = _case(name, cuda)
    got = _run(lib, c)
    scaled = _run(lib, c, d_out=c["d_out"] * 2.0 ** -17)
    nz = got.float().abs()
    assert (nz[nz > 0] * 2.0 ** -17).min().item() >= FTZ, "the scaled gradients must stay in bf16's normal range"
    assert torch.equal(_bits(scaled), _bits((got.float() * 2.0 ** -17).to(torch.bfloat16))), name


@pytest.mark.parametrize("heads", [1, 3, 5, 6, 7, 9, 10, 13, 17])
def test_delta_prologue_takes_any_head_count(lib, cuda, heads):
    """attention_delta used to dispatch on hidden / 128 alone: odd counts ran with the wrong row stride (3, 5, 9, 13, 17)
    or were refused (1, 7, 10).  One view of 65 tokens against the fp64 reference at every such count."""
    c = _case(f"delta-h{heads}", cuda, spec=(1, 65, heads, "none", "typical", 1.0))
    refs, bounds, _ = _reference(c)
    _check(c, _run(lib, c), refs, bounds)


# ------------------------------------------------------------------------------------------------ forward lse2
def _lse2_bound(c):
    """Per-row bound on the forward's fp32 lse2 = m c + log2 l (attention_wgmma.cu), in log2 units:
      * logits: c e_S with e_S the accumulation bound of q16 k16^T, and |c_f32 - log2(e)/8| |S| for the constant;
      * exponents: u |m c| for m c, u |S c - m c| <= 2 u M for each fmaf (M = max |S c|), and per KV block 4 u M for the
        rescale's argument plus one ex2 error -- (3 + 4 nb) u M in all;
      * the sum l: EX2_REL per term and u per add, (nb + 1) EX2_REL + (S + 2 nb + 4) u relative, over ln 2, plus the terms
        ex2.approx.ftz flushes (S 2^-126 relative, as l >= 1);
      * log2f (1 ulp of a value below log2(S) + 1) and the final add (u |lse2|)."""
    n, S, heads, ok = c["n"], c["S"], c["heads"], c["ok"]
    q16, k16, _ = _split(c["qkv"].double(), n, S, heads)
    s = q16 @ k16.transpose(-1, -2)
    zero = torch.zeros_like(s)
    e_s = torch.where(ok, C_ACC * U * 8 * (q16.abs() @ k16.abs().transpose(-1, -2)), zero).amax(-1)
    big = torch.where(ok, s.abs(), zero).amax(-1)
    nb = (S + 63) // 64
    dc = abs(C_LOG2 - LOG2E / 8)
    b = (C_LOG2 * e_s + dc * big + (3 + 4 * nb) * U * C_LOG2 * big
         + ((nb + 1) * EX2_REL + (S + 2 * nb + 4) * U + S * FTZ) / math.log(2) + 2 * U * (math.log2(S) + 1))
    ref = torch.logsumexp(s.masked_fill(~ok, -math.inf) * 0.125, -1) * LOG2E
    return ref, b + U * ref.abs()


@pytest.mark.parametrize("name", list(CASES))
def test_forward_lse2_matches_fp64(lib, cuda, name):
    from pigeon_b200 import ops
    c = _case(name, cuda)
    n, S, heads = c["n"], c["S"], c["heads"]
    if c["kind"] == "none":
        _, lse2 = ops.attention_f16(c["qkv"], n, S, heads, variant=0, return_lse2=True)
    else:
        _, lse2 = ops.attention_f16_masked_lse(c["qkv"], n, S, heads, c["mask"], causal=c["causal"])
    ref, bound = _lse2_bound(c)
    err = (lse2.double().reshape(n, heads, S) - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    ratio = (err / bound).max().item()
    _note("lse2 " + name, ratio)
    assert ratio <= 1.0, f"{name}: lse2 |error| / bound = {ratio:.3g}"
