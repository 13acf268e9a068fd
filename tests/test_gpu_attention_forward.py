"""Both attention forward kernels (attention_kernel<false> behind pg_attention_f16, _lse and _variant, attention_kernel<true>
behind pg_attention_f16_masked and _masked_lse) against plain float64 arithmetic, per element, at the head counts, masks and
tile edges where they go wrong: one token, one partial 64-row tile, exact tile multiples, a last q-tile with one valid row
(S = 577), odd head counts, causal and padding masks, a non-causal mask with interior zeros and a whole masked key block,
logits from near-uniform to peaked, a key-norm ramp that makes the running maximum rise from block to block, and a v small
enough that `out` lands among fp16's subnormals.

The reference is torch float64 (on the device, or on the CPU for the test that checks the bound itself) applied to what the
kernel reads, rounding where the kernel rounds (attention_wgmma.cu).  Per row i with admissible keys A_i and 64-key blocks b:
  s = q16 k16^T (exact in fp64);  M_b = the largest admissible s in blocks <= b (the kernel's running maximum after block b;
  a block without admissible keys leaves it unchanged, and a causal q-tile that stops at its diagonal block only skips such
  blocks);  P'_ij = 2^(c (s_ij - M_b(j))) with the kernel's fp32 c = 0.125f * 1.4426950408889634f;
  alpha_b = 2^(c (M_b - M_last));  ref_i = sum_j alpha_b fp16(P'_ij) v16_j / sum_j alpha_b P'_ij
(the PV product takes P packed to fp16, the row sum l adds the fp32 P).  Per-element bound, with u = 2^-24, w_j = alpha P'_ij
and l = sum_j w_j:
  * the exponent: the kernel's argument fmaf(s, c, -fl(m c)) differs from c (s - M_b) by c e_S (the logits' accumulation
    error, e_S = C_ACC u sqrt(64) |q16||k16|^T, C_ACC = 2 as in the GEMM epilogue test), c E (E = the row's largest e_S, the
    error of the running maximum m), u |c M_b| (rounding m c) and u |x| (the fmaf), so P' is within
    e_P = 2 P' (ln2 (c (e_S + E) + u |c M_b| + u |x|) + EX2_REL), EX2_REL being ex2.approx's relative error, doubled for the
    second-order terms;
  * the rescale: each block's alpha = ex2((m - n) c) adds EX2_REL, ln2 4 u c max|s| (the subtraction and the product) and
    the two multiplies of O and l (2 u): eps_j = e_P / P' + nb (EX2_REL + 4 ln2 u c max|s| + 2 u) is the relative error of
    the weight w_j, common to the numerator and l, which enters as sum_j w_j eps_j (|v_j| + |ref_i|) / l;
  * the fp16 packing of P': the kernel's fp16(P') lies between fp16(P' - e_P) and fp16(P' + e_P) (0 below 2^-25), so that
    span times alpha |v|, summed, over l, bounds what a rounding flip changes;
  * the fp32 accumulation of O: C_ACC u sqrt(K) sum_j alpha fp16(P') |v_j| / l, K the key count padded to 64, plus one
    rounding per block for the rescale multiply (nb u on the same sum);
  * l's summation: each thread adds 16 terms per block and the quad adds four partial sums, (17 nb + 2) u |ref|, plus the
    terms ex2.approx.ftz flushes (S 2^-126 |ref|, as l >= 1);
  * 1/l and o * inv: 2 u |ref|;
  * output rounding: one fp16 ulp of |ref| + E (spacing 2^-24 among the subnormals) + E, E the sum of the terms above.
The largest error / bound per case is printed at the end of the module.  A CPU test checks that the bound is not vacuous: a
reference that rounds P to bf16 (peaked logits) and one that skips the rescale of rows +8 of each 16-row group (the ramp,
whose maximum rises after block 0) both break it, and the emulated reference does not.

A plain fp64 softmax comparison (rel-L2 below 1e-3 plus the rel-L2 of one fp16 ulp of the result, which matters only for
the subnormal outputs) keeps the emulation from hiding a misreading of the maths shared by kernel and reference.

Exact properties: two runs give the same bits; every unmasked entry point (pg_attention_f16, _lse, _variant 0..3 with and
without lse2, _masked and _masked_lse with no mask and causal 0) returns the same `out`; the all-ones mask gives the
unmasked kernel's bits; a view's rows equal a one-view call on its data with NaN in every other view's qkv; the k and v of
keys a row does not admit do not change its bits; a row with one admissible key returns v16 of key 0; scaling v by 2^+-3
scales `out` exactly; NaN guard rows around `out` and guard entries around lse2 survive; n_views = 0 is a no-op and
n_views > 65535 an error before any launch."""
import math

import pytest
import torch

U = 2.0 ** -24
C_ACC = 2.0
EX2_REL = 2.0 ** -21            # ex2.approx.ftz.f32: a relative error of a few fp32 ulp
FTZ = 2.0 ** -126
LN2 = math.log(2)
LOG2E = 1.4426950408889634
C_LOG2 = (torch.tensor(0.125, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)).item()   # the kernel's c
GUARD = 2                       # NaN guard rows before and after out, guard entries before and after lse2
SENT16 = 0x7E55                 # fp16 NaN with a payload the kernel never writes
SENT32 = 0x7FC0_1234            # fp32 NaN with a payload
PLAIN_REL = 1e-3
RATIOS = {}                     # case -> largest observed error / bound, printed at the end of the module
PLAIN = {}                      # case -> rel-L2 against the unemulated fp64 softmax

# id: (n_views, S, heads, mask, logits, v scale).  Masks: none = attention_kernel<false>; causal; pad = causal + padding
# with lengths 1, S // 2, S, ...; interior = causal 0 with interior zeros (and, from S = 128, one whole masked key block);
# ones = causal 0 with an all-ones mask (the masked kernel).  Logits: typical q, k x 0.8; uniform q, k x 0.05 plus a key
# component shared by all tokens of a head, as the text tower's keys have; peaked q, k x 3 (many P' among fp16's
# subnormals or flushed); ramp = key norms growing along the sequence, so the running maximum rises across blocks.
CASES = {
    "S1-h1": (1, 1, 1, "none", "typical", 1.0),
    "S1-h3-causal": (2, 1, 3, "causal", "peaked", 1.0),
    "S2-h2-causal": (3, 2, 2, "causal", "typical", 1.0),
    "S2-h5-interior": (1, 2, 5, "interior", "peaked", 1.0),
    "S17-h3": (3, 17, 3, "none", "peaked", 1.0),
    "S17-h1-pad": (3, 17, 1, "pad", "typical", 1.0),
    "S63-h5-causal-ramp": (1, 63, 5, "causal", "ramp", 1.0),
    "S64-h16-interior": (3, 64, 16, "interior", "typical", 1.0),
    "S64-h2-causal-peaked": (2, 64, 2, "causal", "peaked", 1.0),
    "S65-h2-pad": (3, 65, 2, "pad", "peaked", 1.0),
    "S65-h3-uniform": (1, 65, 3, "none", "uniform", 1.0),
    "S65-h17-tiny-v": (2, 65, 17, "none", "typical", 2.0 ** -16),
    "S77-h12-pad-uniform": (3, 77, 12, "pad", "uniform", 1.0),
    "S77-h12-text-batch": (64, 77, 12, "pad", "uniform", 1.0),
    "S77-h5-ones": (1, 77, 5, "ones", "typical", 1.0),
    "S77-h1-pad-tiny-v": (3, 77, 1, "pad", "peaked", 2.0 ** -18),
    "S128-h1-interior-ramp": (3, 128, 1, "interior", "ramp", 1.0),
    "S128-h3-causal-ramp": (2, 128, 3, "causal", "ramp", 1.0),
    "S129-h3-ones": (1, 129, 3, "ones", "peaked", 1.0),
    "S129-h12-causal": (3, 129, 12, "causal", "uniform", 1.0),
    "S129-h17-ramp": (2, 129, 17, "none", "ramp", 1.0),
    "S577-h16-vision": (4, 577, 16, "none", "typical", 1.0),
    "S577-h2-peaked": (2, 577, 2, "none", "peaked", 1.0),
    "S577-h3-causal": (2, 577, 3, "causal", "typical", 1.0),
    "S577-h5-pad-ramp": (3, 577, 5, "pad", "ramp", 1.0),
    "S577-h1-interior-uniform": (1, 577, 1, "interior", "uniform", 1.0),
}


@pytest.fixture(scope="module")
def lib(cuda):
    from pigeon_b200 import _lib
    lib = _lib.load()
    yield lib
    if RATIOS:
        print("\nmax |error| / bound per case:", {k: round(v, 4) for k, v in RATIOS.items()})
    if PLAIN:
        print("rel-L2 against the fp64 softmax:", {k: float(f"{v:.3g}") for k, v in PLAIN.items()})


def _note(key, ratio):
    RATIOS[key] = max(RATIOS.get(key, 0.0), ratio)


# ------------------------------------------------------------------------------------------------ inputs
def _mask(kind, n, S, seed):
    """(mask i64 [n, S] or None, causal) of a mask kind; mask[:, 0] = 1 as the kernel requires."""
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
            m[n // 2, 64:128] = 0            # a key block with no admissible key: b = -inf there
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


def _qkv(n, S, heads, logits, vscale, seed):
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
    x[:, :, 2] *= vscale
    return x.reshape(n * S, 3 * heads * 64).half()


def _split(t, n, S, heads):
    """[n*S, 3*heads*64] -> q, k, v [n, heads, S, 64]."""
    return t.reshape(n, S, 3, heads, 64).permute(2, 0, 3, 1, 4)


def _heads(t, n, S, heads):
    """[n*S, heads*64] -> [n, heads, S, 64]."""
    return t.reshape(n, S, heads, 64).permute(0, 2, 1, 3)


def _case(name, dev, spec=None):
    n, S, heads, kind, logits, vscale = spec or CASES[name]
    seed = sum(map(ord, name))
    qkv = _qkv(n, S, heads, logits, vscale, seed).to(dev)
    mask, causal = _mask(kind, n, S, seed)
    mask = None if mask is None else mask.to(dev)
    return dict(name=name, n=n, S=S, heads=heads, kind=kind, logits=logits, qkv=qkv, mask=mask, causal=causal)


# ------------------------------------------------------------------------------------------------ the kernels
def _run(lib, c, entry=None, lse=True, **over):
    """(out, lse2 or None) of one call, with NaN-payload guard rows around out and guard entries around lse2, which must
    survive.  entry: "f16", "lse", "variant<k>", "masked", "masked_lse"; None = _lse or _masked_lse by the mask kind."""
    from pigeon_b200._lib import check, current_stream_ptr, ptr
    c = dict(c, **over)
    n, S, heads = c["n"], c["S"], c["heads"]
    if entry is None:
        entry = "masked_lse" if c["kind"] != "none" else "lse"
    dev = c["qkv"].device
    rows, hidden = n * S, heads * 64
    big = torch.empty(rows + 2 * GUARD, hidden, dtype=torch.float16, device=dev)
    big.view(torch.int16).fill_(SENT16)
    out = big[GUARD:GUARD + rows]
    want_lse = entry in ("lse", "masked_lse") or (entry.startswith("variant") and lse)
    lbig = torch.empty(n * heads * S + 2 * GUARD, dtype=torch.float32, device=dev)
    lbig.view(torch.int32).fill_(SENT32)
    lse2 = lbig[GUARD:GUARD + n * heads * S] if want_lse else None
    st, q, mask, causal = current_stream_ptr(), ptr(c["qkv"]), ptr(c["mask"]), int(c["causal"])
    o = big.data_ptr() + GUARD * hidden * 2                     # valid even when n = 0 leaves `out` empty
    ls = lbig.data_ptr() + GUARD * 4 if want_lse else None
    if entry == "f16":
        check(lib.pg_attention_f16(q, o, n, S, heads, st), entry)
    elif entry == "lse":
        check(lib.pg_attention_f16_lse(q, o, ls, n, S, heads, st), entry)
    elif entry.startswith("variant"):
        check(lib.pg_attention_f16_variant(q, o, ls, n, S, heads, int(entry[7:]), -1, st), entry)
    elif entry == "masked":
        check(lib.pg_attention_f16_masked(q, o, mask, causal, n, S, heads, st), entry)
    else:
        assert entry == "masked_lse"
        check(lib.pg_attention_f16_masked_lse(q, o, ls, mask, causal, n, S, heads, st), entry)
    torch.cuda.synchronize()
    guards = torch.cat([big[:GUARD], big[GUARD + rows:]]).view(torch.int16)
    assert (guards == SENT16).all(), f"{entry}: attention wrote outside out"
    lguards = torch.cat([lbig[:GUARD], lbig[lbig.numel() - GUARD:]]).view(torch.int32)
    assert (lguards == SENT32).all(), f"{entry}: attention wrote outside lse2"
    if lse2 is None:
        assert (lbig.view(torch.int32) == SENT32).all(), f"{entry}: lse2 written though not requested"
    return out.clone(), None if lse2 is None else lse2.clone()


def _bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------ the fp64 reference
def _f16(x):
    return x.to(torch.float16).double()


def _bf16(x):
    return x.to(torch.bfloat16).double()


def _ulp_f16(x):
    """One fp16 unit in the last place of x >= 0 (spacing 2^-24 among the subnormals and at 0)."""
    _, e = torch.frexp(x)
    e = (e - 1).clamp_min(-14)
    return torch.where(x > 0, torch.ldexp(torch.ones_like(x), e - 10), torch.full_like(x, U))


def _reference(c, round_p=_f16, skip_rescale_hi=False):
    """(ref fp64 [n, heads, S, 64], its per-element bound, the unemulated fp64 softmax) on the device of c["qkv"].
    round_p and skip_rescale_hi build the perturbed references of the bound's self-test."""
    n, S, heads = c["n"], c["S"], c["heads"]
    dev = c["qkv"].device
    ok = _admissible(n, S, c["mask"], c["causal"], dev)
    q16, k16, v16 = _split(c["qkv"].double(), n, S, heads)
    s = q16 @ k16.transpose(-1, -2)
    sm = s.masked_fill(~ok, -math.inf)
    nb = (S + 63) // 64
    blocks = torch.nn.functional.pad(sm, (0, nb * 64 - S), value=-math.inf).unflatten(-1, (nb, 64)).amax(-1)
    M = torch.cummax(blocks, -1).values                           # running maximum after each block [n, heads, S, nb]
    Mb = M.repeat_interleave(64, -1)[..., :S]                     # M_b(j) per key
    Mlast = M[..., -1:]
    zero = torch.zeros_like(s)
    x = torch.where(ok, (s - Mb) * C_LOG2, zero)
    p = torch.where(ok, torch.exp2(x), zero)
    alpha = torch.where(ok, torch.exp2((Mb - Mlast) * C_LOG2), zero)
    if skip_rescale_hi:                                           # rows r_loc + 8 of each 16-row group keep their old O, l
        hi = (torch.arange(S, device=dev) % 16 >= 8).view(1, 1, S, 1)
        alpha = torch.where(hi & ok, torch.ones_like(alpha), alpha)
    h = round_p(p)
    w = alpha * p
    l = w.sum(-1, keepdim=True)
    ref = (alpha * h) @ v16 / l
    av = v16.abs()

    e_s = C_ACC * U * 8 * (q16.abs() @ k16.abs().transpose(-1, -2))
    e_row = torch.where(ok, e_s, zero).amax(-1, keepdim=True)
    s_abs = torch.where(ok, s.abs(), zero).amax(-1, keepdim=True)
    mc = torch.where(ok, (Mb * C_LOG2).abs(), zero)
    e_p = 2 * p * (LN2 * (C_LOG2 * (e_s + e_row) + U * mc + U * x.abs()) + EX2_REL)
    flip = torch.where(ok, _f16(p + e_p) - _f16(p - e_p), zero)
    eps = torch.where(ok, e_p / p.clamp_min(1e-300), zero) + nb * (EX2_REL + 4 * LN2 * U * C_LOG2 * s_abs + 2 * U)
    we = w * eps
    pv = (alpha * h) @ av
    aref = ref.abs()
    E = ((alpha * flip) @ av + we @ av + aref * we.sum(-1, keepdim=True)
         + (C_ACC * U * math.sqrt(nb * 64) + nb * U) * pv) / l \
        + aref * ((17 * nb + 2) * U + S * FTZ + 2 * U)
    bound = _ulp_f16(aref + E) + E
    plain = torch.softmax(sm * 0.125, -1) @ v16
    return ref, bound, plain


def _ratio(got, ref, bound):
    """max |got - ref| / bound (inf where got is not finite) and its index."""
    err = (got.double() - ref).abs()
    r = err / bound
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    return r.max().item(), torch.unravel_index(r.argmax(), r.shape)


def _check(c, out, ref, bound, plain):
    name, n, S, heads = c["name"], c["n"], c["S"], c["heads"]
    got = _heads(out.double(), n, S, heads)
    ratio, at = _ratio(got, ref, bound)
    _note(name, ratio)
    if ratio > 1.0:
        i = tuple(int(j) for j in at)
        raise AssertionError(f"{name}: out |error| / bound = {ratio:.3g} at [view, head, row, col] = {list(i)}: got "
                             f"{got[i].item()!r}, reference {ref[i].item()!r}, bound {bound[i].item():.3g}")
    rel = ((got - plain).norm() / plain.norm()).item()
    bar = PLAIN_REL + (_ulp_f16(plain.abs()).norm() / plain.norm()).item()
    PLAIN[name] = rel
    assert rel < bar, (name, rel, bar)


# ------------------------------------------------------------------------------------------------ the bound, without a GPU
def test_bound_rejects_perturbed_references():
    """The bound is tight enough to catch P rounded to bf16 (peaked logits) and a skipped rescale of rows +8 of each 16-row
    group (the ramp: the running maximum rises after block 0); the emulated reference itself stays inside it."""
    cpu = torch.device("cpu")
    checks = [("peaked", (2, 129, 2, "none", "peaked", 1.0), dict(round_p=_bf16)),
              ("peaked-pad", (3, 77, 2, "pad", "peaked", 1.0), dict(round_p=_bf16)),
              ("ramp", (2, 129, 2, "none", "ramp", 1.0), dict(skip_rescale_hi=True)),
              ("ramp-causal", (1, 192, 1, "causal", "ramp", 1.0), dict(skip_rescale_hi=True))]
    for name, spec, perturb in checks:
        c = _case("cpu-" + name, cpu, spec=spec)
        ref, bound, _ = _reference(c)
        ratio, _ = _ratio(_f16(ref), ref, bound)
        assert ratio <= 0.5, (name, ratio)
        bad, _, _ = _reference(c, **perturb)
        ratio, _ = _ratio(_f16(bad), ref, bound)
        assert ratio > 1.0, (name, perturb, ratio)


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_forward_matches_fp64_reference(lib, cuda, name):
    c = _case(name, cuda)
    out, lse2 = _run(lib, c)
    again, lse2_again = _run(lib, c)
    assert torch.equal(_bits(out), _bits(again)), f"{name}: out differs run to run"
    assert torch.equal(lse2.view(torch.int32), lse2_again.view(torch.int32)), f"{name}: lse2 differs run to run"
    ref, bound, plain = _reference(c)
    _check(c, out, ref, bound, plain)
    n, S, heads = c["n"], c["S"], c["heads"]
    got = _heads(out, n, S, heads)
    v0 = _heads(c["qkv"][:, 2 * heads * 64:], n, S, heads)[:, :, 0]     # v16 of key 0 [n, heads, 64]
    if c["causal"]:
        # row 0 admits key 0 alone: l = 1, O = v16, out = v16 exactly
        assert torch.equal(_bits(got[:, :, 0]), _bits(v0)), f"{name}: causal row 0 is not v of key 0"
    if c["kind"] == "pad":
        # the length-1 caption (view 0): every row admits key 0 alone
        assert torch.equal(_bits(got[0]), _bits(v0[0, :, None].expand(heads, S, 64))), f"{name}: a length-1 caption"
    if c["kind"] == "ones":
        # the masked kernel with every key admissible and causal = 0 is the unmasked kernel, bit for bit
        plain_out, _ = _run(lib, c, entry="lse")
        assert torch.equal(_bits(out), _bits(plain_out)), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["S1-h1", "S17-h3", "S65-h3-uniform", "S65-h17-tiny-v", "S129-h17-ramp", "S577-h16-vision"])
def test_unmasked_entry_points_agree(lib, cuda, name):
    """pg_attention_f16, _lse, every _variant with and without lse2, and the masked entry points with no mask and causal 0
    return the same out; requesting lse2 does not change it, and every lse2 is the same."""
    c = _case(name, cuda)
    out, lse2 = _run(lib, c, entry="lse")
    entries = [("f16", True), ("masked", True), ("masked_lse", True)]
    entries += [(f"variant{k}", lse) for k in range(4) for lse in (False, True)]
    for entry, lse in entries:
        o, l2 = _run(lib, c, entry=entry, lse=lse, mask=None, causal=False)
        assert torch.equal(_bits(o), _bits(out)), f"{name}: {entry} (lse2 {l2 is not None}) changes out"
        if l2 is not None:
            assert torch.equal(l2.view(torch.int32), lse2.view(torch.int32)), f"{name}: {entry} changes lse2"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["S2-h2-causal", "S17-h3", "S17-h1-pad", "S64-h16-interior", "S77-h5-ones",
                                  "S128-h1-interior-ramp", "S129-h12-causal", "S577-h5-pad-ramp", "S577-h2-peaked"])
def test_views_are_independent(lib, cuda, name):
    """With NaN in every other view's qkv (the mask left as it is), a view's rows are the bits of a one-view call."""
    c = _case(name, cuda)
    n, S = c["n"], c["S"]
    full, _ = _run(lib, c)
    for view in range(n):
        rows = slice(view * S, (view + 1) * S)
        one, _ = _run(lib, c, n=1, qkv=c["qkv"][rows].contiguous(),
                      mask=None if c["mask"] is None else c["mask"][view:view + 1].contiguous())
        poisoned = torch.full_like(c["qkv"], math.nan)
        poisoned[rows] = c["qkv"][rows]
        got, _ = _run(lib, c, qkv=poisoned)
        assert torch.equal(_bits(got[rows]), _bits(one)), f"{name}: view {view} depends on the other views"
        assert torch.equal(_bits(full[rows]), _bits(one)), f"{name}: view {view} differs from a one-view call"


def _replace_keys(c, keys, seed):
    """qkv with the k and v of `keys` (bool [n, S]) replaced by other finite values."""
    n, S, heads = c["n"], c["S"], c["heads"]
    g = torch.Generator().manual_seed(seed)
    x = c["qkv"].clone().view(n, S, 3, heads, 64)
    other = (torch.randn(n, S, 2, heads, 64, generator=g) * 4).half().to(x.device)
    sel = keys.to(x.device)[:, :, None, None, None]
    x[:, :, 1:] = torch.where(sel, other, x[:, :, 1:])
    return x.view(n * S, 3 * heads * 64)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["S2-h2-causal", "S17-h1-pad", "S63-h5-causal-ramp", "S64-h16-interior",
                                  "S64-h2-causal-peaked", "S128-h3-causal-ramp", "S129-h12-causal",
                                  "S577-h1-interior-uniform", "S577-h3-causal"])
def test_inadmissible_keys_do_not_matter(lib, cuda, name):
    """Other k and v for keys with mask 0 leave every row's bits; for causal rows, other k and v for every key >= t leave
    the bits of rows < t (t at and around the tile edges: a diagonal off by one changes them)."""
    c = _case(name, cuda)
    n, S = c["n"], c["S"]
    out, _ = _run(lib, c)
    if c["mask"] is not None:
        off = c["mask"].cpu() == 0
        if off.any():
            got, _ = _run(lib, c, qkv=_replace_keys(c, off, 7))
            assert torch.equal(_bits(got), _bits(out)), f"{name}: keys with mask 0 change the output"
    if c["causal"]:
        for t in sorted({1, S // 2, S - 1, 63, 64, 65, 127, 128, 129} & set(range(1, S))):
            keys = (torch.arange(S) >= t).expand(n, S)
            got, _ = _run(lib, c, qkv=_replace_keys(c, keys, t))
            rows = torch.arange(n * S, device=cuda) % S < t
            assert torch.equal(_bits(got[rows]), _bits(out[rows])), f"{name}: keys >= {t} change rows < {t}"
            assert not torch.equal(_bits(got[~rows]), _bits(out[~rows])), f"{name}: the replaced keys were never read"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["S2-h2-causal", "S17-h3", "S65-h2-pad", "S77-h5-ones", "S128-h1-interior-ramp",
                                  "S577-h16-vision"])
def test_scaling_v_by_a_power_of_two_is_exact(lib, cuda, name):
    """v in [1, 4) keeps out (a convex combination) and out x 2^+-3 in fp16's normal range, where rounding commutes with
    the scaling; P does not depend on v."""
    c = _case(name, cuda)
    heads = c["heads"]
    g = torch.Generator().manual_seed(5)
    c["qkv"][:, 2 * heads * 64:] = (1 + torch.rand(c["qkv"].shape[0], heads * 64, generator=g) * 3).half().to(cuda)
    out, _ = _run(lib, c)
    a = out.float().abs()
    for e in (3, -3):
        f = 2.0 ** e
        qkv = c["qkv"].clone()
        v = qkv[:, 2 * heads * 64:]
        assert torch.equal((v.float() * f).half().float(), v.float() * f), "the scaled v must stay exact in fp16"
        assert (a * f).min().item() >= 2.0 ** -14 and (a * f).max().item() <= 65504, "out must stay in fp16's normal range"
        qkv[:, 2 * heads * 64:] = (v.float() * f).half()
        scaled, _ = _run(lib, c, qkv=qkv)
        assert torch.equal(_bits(scaled), _bits((out.float() * f).half())), f"{name}: v x 2^{e}"


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["f16", "lse", "variant2", "masked", "masked_lse"])
def test_view_count_edges(lib, cuda, entry):
    """n_views = 0 with valid pointers leaves out and lse2 untouched; n_views > 65535 (the grid's z limit) is refused before
    any launch, naming the limit."""
    from pigeon_b200._lib import PigeonB200Error
    c = _case("views0", cuda, spec=(1, 65, 2, "pad" if entry.startswith("masked") else "none", "typical", 1.0))
    out, _ = _run(lib, c, entry=entry, n=0)
    assert out.numel() == 0
    with pytest.raises(PigeonB200Error, match="65535"):
        _run(lib, c, entry=entry, n=65536, S=1)
