"""Every epilogue of both wgmma GEMM kernels against plain float64 arithmetic, per element, at the shapes and strides where a
GEMM goes wrong: one row, ragged M and N, a partial K block, CTAs with an odd number of tiles (the ping-pong hand-off), row
strides that rule out vector stores, the row map of the patch embedding, and the activation's overflow / underflow ranges.

Each case runs under pg_gemm_set_schedule(0) (ping-pong kernel) twice and under pg_gemm_set_schedule(1) (single-warpgroup
kernel) once.  Every run must match the fp64 reference within the bound derived below, leave every sentinel around its
outputs intact, and be bit-identical to the other two runs.

The reference is torch in float64 on the device, applied to the same fp16 / bf16 operands the kernel reads.  Error bounds,
with u = 2^-24 (fp32 unit roundoff):
  * accumulation: the fp32 sum of K exact fp16 x fp16 (or bf16 x bf16) products is within C_ACC * u * sqrt(K) * (|A| |W|^T)
    of the exact sum (the probabilistic bound lambda * sqrt(K) * u of Higham & Mary, 2019, with C_ACC = 2 leaving room for the
    tensor core's truncating alignment of addends);
  * each fp32 add / fma of the epilogue rounds once: u * |its result|;
  * an activation scales what comes in by its slope: |quick_gelu'| <= 1.0998 (at x = 1.41), QGELU_SLOPE = 1.1;
  * quick_gelu / quick_gelu' run on ex2.approx + __fdividef (a few fp32 ulps relative, plus the rounding of the
    exponent's argument, relative 1.7 u |x|): 2^-20 (1 + |x|) relative;
  * a 2-byte output rounds to nearest: half a unit in the last place; one full ulp of |reference| is allowed because the
    fp32 value being rounded may sit across a binade boundary from the reference.
For fp32 outputs the bound is the accumulation and rounding terms alone."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_ACC = 2.0
QGELU_SLOPE = 1.1
APPROX = 2.0 ** -20
POISON = 1.0e4                  # operand padding columns [K, ld): finite, and large enough that reading it shows at once
LN_EPS = 1e-5
SENT = {torch.float16: 0x7E5A, torch.bfloat16: 0x7FD5, torch.float32: 0x7FD5A5A5}   # NaNs with a payload the kernels never write
IVIEW = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32}
ACT_EDGES = [20.0, -20.0, 60.0, -60.0, 65504.0, -65504.0]   # ex2 underflow / overflow, __fdividef's huge-divisor branch
RATIOS = {}                     # epilogue -> largest observed error / bound, printed at the end of the module


@pytest.fixture(scope="module")
def lib(cuda):
    from pigeon_b200 import _lib
    lib = _lib.load()
    yield lib
    if RATIOS:
        print("\nmax |error| / bound per epilogue:", {k: round(v, 4) for k, v in sorted(RATIOS.items(), key=str)})


def _note(key, ratio):
    RATIOS[key] = max(RATIOS.get(key, 0.0), ratio)


def _run(lib, **kw):
    from pigeon_b200 import _lib
    p = _lib.GemmProblem(**kw)
    return lib.pg_gemm_problem_run(C.byref(p), _lib.current_stream_ptr())


def _set_schedule(lib, mode):
    assert lib.pg_gemm_set_schedule(mode) == 0


def _sentinel(rows, cols, dt, dev):
    t = torch.empty(rows, cols, dtype=dt, device=dev)
    t.view(IVIEW[dt]).fill_(SENT[dt])
    return t


def _bits(t):
    return t.view(IVIEW[t.dtype]) if t.dtype in IVIEW else t


def _assert_sentinels(buf, valid, what):
    bad = (_bits(buf) != SENT[buf.dtype]) & ~valid
    assert not bad.any(), f"{what}: {int(bad.sum())} writes outside the output, first at {bad.nonzero()[0].tolist()}"


def _operand(rows, k, scale, dt, g, dev, shift=None):
    """[rows, ld] with ld a multiple of 8 and at least 8 poisoned columns past k."""
    ld = (k + 7) // 8 * 8 + 8
    t = torch.full((rows, ld), POISON, dtype=dt, device=dev)
    v = torch.randn(rows, k, generator=g, device=dev) * scale
    if shift is not None:
        v += shift
    t[:, :k] = v.to(dt)
    return t, ld


def _ulp(x, dt):
    """One unit in the last place of |x| in the 2-byte output type (subnormal spacing below the normal range)."""
    bits, emin = (10, -14) if dt == torch.float16 else (7, -126)
    _, e = torch.frexp(x.abs())
    e = (e - 1).clamp_min(emin)
    return torch.ldexp(torch.ones_like(x), e - bits)


def _qg(x):
    return x * torch.sigmoid(1.702 * x)


def _dqg(x):
    s = torch.sigmoid(1.702 * x)
    return s * (1 + 1.702 * x * (1 - s))


def _check(got, ref, bound, key, what):
    err = (got.double() - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    ratio = (err / bound).max().item()
    _note(key, ratio)
    if ratio > 1.0:
        i = int((err / bound).argmax())
        r, c = divmod(i, ref.shape[1])
        raise AssertionError(f"{what}: |error| / bound = {ratio:.3g} at [{r}, {c}]: got {got[r, c].item()!r}, "
                             f"reference {ref[r, c].item()!r}, bound {bound[r, c].item():.3g}")


def _three_runs(lib, call, what):
    """call() under the ping-pong kernel twice and the single-warpgroup kernel once; all three must be the same bits."""
    try:
        _set_schedule(lib, 0)
        r0 = call()
        r0b = call()
        _set_schedule(lib, 1)
        r1 = call()
    finally:
        _set_schedule(lib, 0)
    torch.cuda.synchronize()
    for name in r0:
        assert torch.equal(_bits(r0[name]), _bits(r0b[name])), f"{what}: {name} differs run to run"
        assert torch.equal(_bits(r0[name]), _bits(r1[name])), f"{what}: {name} differs between the two kernels"
    return r0


def _sm_count(lib):
    n = lib.pg_device_sm_count()
    assert n > 0
    return n


# ------------------------------------------------------------------------------------------------ epilogues 0 - 6
# (M, N, K, extra ldo columns): one row with N below one chunk and K below one K block; every ragged M edge of a 128-row
# tile; N ragged for the 32- and 64-column chunks; K of 8 / 72 / 1024 / 4096; ldo = N, N + 8 (vector stores) and N + 1 /
# N + 3 (the scalar path); "T1" / "T2" rows give sm_count + 1 / 2 sm_count + 1 tiles at N = 128 (a CTA with an odd number of
# tiles: the last goes to consumer 0 with no partner).
SHAPES = [(1, 40, 8, 0), (127, 64, 72, 3), (129, 200, 1024, 8), (300, 384, 4096, 1), (1731, 1000, 72, 0),
          ("T1", 128, 1024, 0), ("T2", 128, 72, 8), (1731, 3072, 1024, 8), (300, 200, 8, 3), (129, 64, 4096, 1)]
BIG = (577 * 64, 1024, 1024, 0)


def _rows(lib, M):
    return {"T1": 128 * _sm_count(lib) + 1, "T2": 256 * _sm_count(lib) + 1}.get(M, M)


def _epilogue_case(lib, dev, epi, M, N, K, pad, bf16, variant=0, rowmap=(7, 10, 3)):
    """One problem with epilogue `epi`; variant: epilogue 2 in place (0) / out of place (1); epilogue 3 with (0) / without
    (1) a bias."""
    from pigeon_b200 import _lib
    dt = torch.bfloat16 if bf16 else torch.float16
    g = torch.Generator(device=dev).manual_seed(1000 * epi + 7 * M + 3 * N + K + pad + 17 * bf16 + 5 * variant)
    a, lda = _operand(M, K, 0.5, dt, g, dev)
    w, ldw = _operand(N, K, 0.05, dt, g, dev)
    ldo = N + pad
    f16_out = epi in (_lib.EPI_F16_BIAS, _lib.EPI_F16_BIAS_QGELU, _lib.EPI_F16_BIAS_QGELU_SAVE)
    out_dt = torch.float16 if f16_out else torch.bfloat16 if epi == _lib.EPI_BF16_DGELU else torch.float32
    bias = torch.randn(N, generator=g, device=dev)
    gelu = epi in (_lib.EPI_F16_BIAS_QGELU, _lib.EPI_F16_BIAS_QGELU_SAVE)
    if gelu:
        bias[:len(ACT_EDGES)] = torch.tensor(ACT_EDGES[:N], device=dev)
    if epi == _lib.EPI_BF16_DGELU:
        bias = None
    if epi == _lib.EPI_F32_BIAS and variant == 1:
        bias = None
    if epi == _lib.EPI_F32_ROWMAP:
        div, mul, add = rowmap
        out_rows = mul * ((M - 1) // div) + (M - 1) % div + add + 1
        r = torch.arange(M, device=dev)
        orow = mul * (r // div) + r % div + add
    else:
        div = mul = add = 0
        out_rows, orow = M, torch.arange(M, device=dev)
    resid = None
    R = torch.randn(M, N, generator=g, device=dev) * 2
    aux_in = None
    if epi == _lib.EPI_BF16_DGELU:   # the fc1 pre-activation the backward reads; [N, ldo) never read
        aux_in = _sentinel(M, ldo, torch.float16, dev)
        u = torch.randn(M, N, generator=g, device=dev) * 3
        u[:, :len(ACT_EDGES)] = torch.tensor(ACT_EDGES[:N], device=dev)
        aux_in[:, :N] = u.half()
    if epi == _lib.EPI_F32_BIAS_RESID and variant == 1:
        resid = _sentinel(M, ldo, torch.float32, dev)
        resid[:, :N] = R

    def call():
        out = _sentinel(out_rows + 2, ldo, out_dt, dev)
        if epi == _lib.EPI_F32_BIAS_RESID and variant == 0:
            out[:M, :N] = R
        aux = aux_in
        if epi == _lib.EPI_F16_BIAS_QGELU_SAVE:
            aux = _sentinel(M + 2, ldo, torch.float16, dev)
        st = _run(lib, M=M, N=N, K=K, a=a.data_ptr(), lda=lda, w=w.data_ptr(), ldw=ldw, out=out.data_ptr(), ldo=ldo,
                  bias=None if bias is None else bias.data_ptr(), epilogue=epi, rowmap_div=div, rowmap_mul=mul,
                  rowmap_add=add, operand_bf16=bf16, resid=None if resid is None else resid.data_ptr(),
                  aux=None if aux is None else aux.data_ptr())
        assert st == 0, lib.pg_last_error().decode()
        res = {"out": out}
        if epi == _lib.EPI_F16_BIAS_QGELU_SAVE:
            res["aux"] = aux
        return res

    what = f"epilogue {epi} M={M} N={N} K={K} ldo={ldo} bf16={bf16} variant={variant}"
    res = _three_runs(lib, call, what)
    out = res["out"]
    valid = torch.zeros(out.shape, dtype=torch.bool, device=dev)
    valid[orow, :N] = True
    _assert_sentinels(out, valid, what)
    got = out[orow, :N]

    a64, w64 = a[:, :K].double(), w[:, :K].double()
    z = a64 @ w64.t()
    acc_err = C_ACC * U * math.sqrt(K) * (a64.abs() @ w64.abs().t())
    b64 = torch.zeros(N, dtype=torch.float64, device=dev) if bias is None else bias.double()
    v = z + b64
    rnd = 2 * U * (z.abs() + b64.abs())                     # the bias add, and the conversion rounding of an fp32 output
    key = f"{epi}" + ("" if variant == 0 else f".{variant}")
    if epi in (_lib.EPI_F32_BIAS, _lib.EPI_F32_ROWMAP):
        _check(got, v, acc_err + rnd, key, what)
    elif epi == _lib.EPI_F32_BIAS_RESID:
        r64 = R.double()
        _check(got, r64 + v, acc_err + 2 * U * (r64.abs() + z.abs() + b64.abs()), key, what)
    elif epi == _lib.EPI_F16_BIAS:
        _check(got, v, _ulp(v, torch.float16) + acc_err + rnd, key, what)
    elif gelu:
        ref = _qg(v)
        assert torch.isfinite(got.float()).all(), what
        _check(got, ref, _ulp(ref, torch.float16) + QGELU_SLOPE * (acc_err + rnd) + APPROX * (1 + v.abs()) * ref.abs(),
               key, what)
        if epi == _lib.EPI_F16_BIAS_QGELU_SAVE:
            aux = res["aux"]
            valid = torch.zeros(aux.shape, dtype=torch.bool, device=dev)
            valid[:M, :N] = True
            _assert_sentinels(aux, valid, what + " (aux)")
            _check(aux[:M, :N], v, _ulp(v, torch.float16) + acc_err + rnd, key + ".aux", what + " (aux)")
    elif epi == _lib.EPI_BF16_DGELU:
        u64 = aux_in[:, :N].double()
        ref = z * _dqg(u64)
        assert torch.isfinite(got.float()).all(), what
        _check(got, ref, _ulp(ref, torch.bfloat16) + QGELU_SLOPE * acc_err + APPROX * (1 + 2 * u64.abs()) * z.abs(),
               key, what)
    else:
        raise AssertionError(epi)


@pytest.mark.parametrize("bf16", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("epi", [0, 1, 2, 3, 4, 5, 6])
def test_epilogue_against_fp64(cuda, lib, epi, bf16):
    variants = (0, 1) if epi in (2, 3) else (0,)
    for M, N, K, pad in SHAPES:
        for variant in variants:
            _epilogue_case(lib, cuda, epi, _rows(lib, M), N, K, pad, bf16, variant)
    if epi == 2:
        for variant in variants:
            _epilogue_case(lib, cuda, epi, *BIG, bf16, variant)


@pytest.mark.parametrize("bf16", [0, 1], ids=["fp16", "bf16"])
def test_rowmap_patch_embedding_geometry(cuda, lib, bf16):
    """The patch embedding's scatter: row (view, patch) -> token row view * 577 + 1 + patch; the CLS rows (token 0 of every
    view) and the rows past the last view must keep their sentinels.  K = 640 is patch_k_pad of 14 x 14 x 3 pixels."""
    for views, ldo_pad in ((3, 0), (5, 3)):
        _epilogue_case(lib, cuda, 4, views * 576, 1024 - 24 * ldo_pad, 640, ldo_pad, bf16, rowmap=(576, 577, 1))


# ------------------------------------------------------------------------------------------------ LayerNorm producer (7)
STATS_SHAPES = [(1, 128, 8, 0), (127, 384, 72, 8), (129, 1024, 1024, 0), (300, 3072, 1024, 8), (1731, 128, 4096, 0),
                ("T1", 128, 72, 0), ("T2", 128, 1024, 8), BIG]


def _producer(lib, dev, M, N, K, ldo, bf16, a, lda, w, ldw, bias, R, inplace):
    """Epilogue 7 on fresh sentinel buffers; returns out, aux, stats (each with two sentinel rows past M)."""
    out = _sentinel(M + 2, ldo, torch.float32, dev)
    resid = None
    if inplace:
        out[:M, :N] = R
    else:
        resid = _sentinel(M, ldo, torch.float32, dev)
        resid[:, :N] = R
    aux = _sentinel(M + 2, ldo, torch.float16, dev)
    stats = _sentinel(M + 2, N // 128 * 2, torch.float32, dev)
    st = _run(lib, M=M, N=N, K=K, a=a.data_ptr(), lda=lda, w=w.data_ptr(), ldw=ldw, out=out.data_ptr(), ldo=ldo,
              bias=None if bias is None else bias.data_ptr(), epilogue=7, operand_bf16=bf16,
              resid=None if resid is None else resid.data_ptr(), aux=aux.data_ptr(), stats=stats.data_ptr())
    assert st == 0, lib.pg_last_error().decode()
    return {"out": out, "aux": aux, "stats": stats}


def _check_producer(res, M, N, K, a, w, bias, R, key, what):
    dev = R.device
    out, aux, stats = res["out"], res["aux"], res["stats"]
    for name, buf, cols in (("out", out, N), ("aux", aux, N), ("stats", stats, N // 128 * 2)):
        valid = torch.zeros(buf.shape, dtype=torch.bool, device=dev)
        valid[:M, :cols] = True
        _assert_sentinels(buf, valid, f"{what} ({name})")
    a64, w64 = a[:, :K].double(), w[:, :K].double()
    z = a64 @ w64.t()
    acc_err = C_ACC * U * math.sqrt(K) * (a64.abs() @ w64.abs().t())
    b64 = torch.zeros(N, dtype=torch.float64, device=dev) if bias is None else bias.double()
    r64 = R.double()
    _check(out[:M, :N], r64 + z + b64, acc_err + 2 * U * (r64.abs() + z.abs() + b64.abs()), key, what)
    # aux is exactly the fp32 result rounded to fp16
    assert torch.equal(aux[:M, :N], out[:M, :N].half()), what + ": aux != fp16(out)"
    # stats: per 128 columns, the fp32 (sum, sum of squares) of the fp16 values; each is a sum of 128 terms of depth <= 12
    # (16 per lane in 4 chunks, pairwise in twos, then a 3-level shuffle tree), so within 16 u * sum |term|
    x = aux[:M, :N].double().reshape(M, N // 128, 128)
    s = stats[:M].view(M, N // 128, 2).double()
    for j, (ref, mag) in enumerate(((x.sum(-1), x.abs().sum(-1)), ((x * x).sum(-1), (x * x).sum(-1)))):
        err = (s[..., j] - ref).abs()
        ratio = (err / (16 * U * mag).clamp_min(1e-30)).max().item()
        _note(key + ".stats", ratio)
        assert ratio <= 1.0, f"{what}: stats[{j}] |error| / bound = {ratio}"


@pytest.mark.parametrize("bf16", [0, 1], ids=["fp16", "bf16"])
def test_layernorm_producer_epilogue_against_fp64(cuda, lib, bf16):
    dt = torch.bfloat16 if bf16 else torch.float16
    for i, (M, N, K, pad) in enumerate(STATS_SHAPES):
        M = _rows(lib, M)
        g = torch.Generator(device=cuda).manual_seed(7000 + 13 * i + bf16)
        a, lda = _operand(M, K, 0.5, dt, g, cuda)
        w, ldw = _operand(N, K, 0.05, dt, g, cuda)
        bias = torch.randn(N, generator=g, device=cuda) if i % 3 else None
        R = torch.randn(M, N, generator=g, device=cuda) * 2
        for inplace in ((True, False) if i % 2 else (True,)):
            what = f"epilogue 7 M={M} N={N} K={K} ldo={N + pad} bf16={bf16} inplace={inplace}"
            res = _three_runs(lib, lambda: _producer(lib, cuda, M, N, K, N + pad, bf16, a, lda, w, ldw, bias, R, inplace), what)
            _check_producer(res, M, N, K, a, w, bias, R, "7", what)


# ------------------------------------------------------------------------------------------------ LayerNorm consumers (8, 9)
def _fold(wraw, b, gamma, beta, dt):
    """W' = fp16/bf16(gamma * W), colsum = row sums of W' (fp32), b' = b + W beta: as VitEngine builds them."""
    wf = (wraw * gamma[None, :]).to(dt)
    return wf, wf.float().sum(dim=1), b + wraw @ beta


def _consumer(lib, dev, epi, M, N, K, ldo, bf16, x, ldx, wf, ldw, cs, bf, stats):
    out = _sentinel(M + 2, ldo, torch.float16, dev)
    st = _run(lib, M=M, N=N, K=K, a=x.data_ptr(), lda=ldx, w=wf.data_ptr(), ldw=ldw, out=out.data_ptr(), ldo=ldo,
              bias=bf.data_ptr(), epilogue=epi, operand_bf16=bf16, stats=stats.data_ptr(), colsum=cs.data_ptr(),
              ln_eps=LN_EPS)
    assert st == 0, lib.pg_last_error().decode()
    return {"out": out}


def _ln_reference(epi, x16, wf, cs, bf):
    """fp64 rstd * (x W'^T - mu colsum) + b' with (mu, rstd) of the fp16 row, and its per-element bound (no allowance for
    the error of the kernel's one-pass fp32 variance: that has to fit inside the fp16 output budget)."""
    K = x16.shape[1]
    x = x16.double()
    w64 = wf.double()
    mu = x.mean(dim=1, keepdim=True)
    rstd = torch.rsqrt(x.var(dim=1, unbiased=False, keepdim=True) + LN_EPS)
    z = x @ w64.t()
    cs64, b64 = cs.double()[None, :], bf.double()[None, :]
    lin = rstd * (z - mu * cs64) + b64
    acc_err = C_ACC * U * math.sqrt(K) * (x.abs() @ w64.abs().t())
    # fmaf(rstd, acc, fmaf(-rstd * mu, colsum, b')): two fma roundings, the rounding of -rstd * mu and of mu, and rsqrtf's
    # approximation (2 ulp relative) on rstd * (acc - mu colsum)
    fma = 4 * U * (rstd * z.abs() + rstd * mu.abs() * cs64.abs() + b64.abs()) + 2 ** -21 * (lin - b64).abs()
    inner = rstd * acc_err + fma
    if epi == 8:
        return lin, _ulp(lin, torch.float16) + inner, (mu, rstd)
    ref = _qg(lin)
    return ref, _ulp(ref, torch.float16) + QGELU_SLOPE * inner + APPROX * (1 + lin.abs()) * ref.abs(), (mu, rstd)


def _stats_of(x16, slots):
    """(sum, sum of squares) per 128 columns of the fp16 row, rounded once to fp32 (what a perfect producer would store)."""
    x = x16.double().reshape(x16.shape[0], slots, 128)
    return torch.stack((x.sum(-1), (x * x).sum(-1)), dim=-1).float().reshape(x16.shape[0], slots * 2).contiguous()


LN_SHAPES = [(1, 64, 1024, 0), (127, 384, 1024, 3), (129, 3072, 4096, 8), (1731, 64, 1024, 1), ("T1", 128, 1024, 0),
             ("T2", 128, 4096, 8), (300, 1024, 128, 0)]


@pytest.mark.parametrize("bf16", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("epi", [8, 9])
def test_layernorm_consumer_epilogue_against_fp64(cuda, lib, epi, bf16):
    dt = torch.bfloat16 if bf16 else torch.float16
    shapes = LN_SHAPES + ([(577 * 64, 3072, 1024, 0)] if epi == 8 else [])
    for i, (M, N, K, pad) in enumerate(shapes):
        M = _rows(lib, M)
        g = torch.Generator(device=cuda).manual_seed(9000 + 31 * i + 2 * epi + bf16)
        x, ldx = _operand(M, K, 1.0, dt, g, cuda, shift=0.3)
        wraw = torch.randn(N, K, generator=g, device=cuda) * 0.03
        gamma = 1 + 0.1 * torch.randn(K, generator=g, device=cuda)
        beta = 0.1 * torch.randn(K, generator=g, device=cuda)
        b = torch.randn(N, generator=g, device=cuda)
        wf16, cs, bf = _fold(wraw, b, gamma, beta, dt)
        if epi == 9:
            bf[:len(ACT_EDGES)] = torch.tensor(ACT_EDGES, device=cuda)
        wf = torch.full((N, ldx), POISON, dtype=dt, device=cuda)
        wf[:, :K] = wf16
        stats = _stats_of(x[:, :K], K // 128)
        what = f"epilogue {epi} M={M} N={N} K={K} ldo={N + pad} bf16={bf16}"
        res = _three_runs(lib, lambda: _consumer(lib, cuda, epi, M, N, K, N + pad, bf16, x, ldx, wf, ldx, cs, bf, stats), what)
        out = res["out"]
        valid = torch.zeros(out.shape, dtype=torch.bool, device=cuda)
        valid[:M, :N] = True
        _assert_sentinels(out, valid, what)
        ref, bound, _ = _ln_reference(epi, x[:, :K], wf16, cs, bf)
        if epi == 9:
            assert torch.isfinite(out[:M, :N].float()).all(), what
        _check(out[:M, :N], ref, bound, str(epi), what)


def _ln_rows(M, N, g, dev):
    """Residual rows of the LayerNorm chain: |mean| / std of 0, 4 and 30, one channel at 150, and constant rows."""
    R = torch.randn(M, N, generator=g, device=dev)
    kind = torch.arange(M, device=dev) % 8
    shift = torch.tensor([0.0, 4.0, -4.0, 30.0, -30.0, 0.0, 0.0, 0.0], device=dev)[kind]
    R += shift[:, None]
    R[kind == 5, 7] = 150.0
    const = torch.tensor([-4.0, -1.5, 0.3701171875, 3.990234375], device=dev)
    rows = (kind == 6) | (kind == 7)
    R[rows] = const[torch.arange(int(rows.sum()), device=dev) % 4][:, None].expand(-1, N)
    return R, rows


@pytest.mark.parametrize("M,N", [(300, 1024), (577 * 64, 1024)])
def test_layernorm_chain_producer_then_consumers(cuda, lib, M, N):
    """Epilogue 7 writes the new residual, its fp16 copy and the per-128-column moments; epilogues 8 and 9 normalise that fp16
    row on the fly.  Compared with the fp64 fold of the same fp16 row (the kernel's contract, strict bound) and with fp64
    LayerNorm(new fp32 residual) W^T + b (the module the fold stands for; the bound adds the first-order effect of rounding
    the row and gamma * W to fp16, computed from the actual rounding errors)."""
    g = torch.Generator(device=cuda).manual_seed(M + 1)
    K0 = 1024
    a, lda = _operand(M, K0, 0.5, torch.float16, g, cuda)
    w, ldw = _operand(N, K0, 0.002, torch.float16, g, cuda)     # small update: the rows keep their designed mean / std
    R, const_rows = _ln_rows(M, N, g, cuda)
    a[const_rows, :K0] = 0                                        # constant rows stay constant (no bias in the producer)
    what = f"chain M={M} N={N}"
    prod = _three_runs(lib, lambda: _producer(lib, cuda, M, N, K0, N, 0, a, lda, w, ldw, None, R, True), what + " (7)")
    _check_producer(prod, M, N, K0, a, w, None, R, "7", what + " (7)")
    x16, stats, x32 = prod["aux"][:M], prod["stats"][:M], prod["out"][:M, :N]
    assert torch.equal(x16[const_rows, :N].float(), R[const_rows]), "constant rows must stay constant"
    for epi, N2 in ((8, 3072), (9, 4096)):
        wraw = torch.randn(N2, N, generator=g, device=cuda) * 0.03
        gamma = 1 + 0.1 * torch.randn(N, generator=g, device=cuda)
        beta = 0.1 * torch.randn(N, generator=g, device=cuda)
        b = torch.randn(N2, generator=g, device=cuda)
        wf, cs, bf = _fold(wraw, b, gamma, beta, torch.float16)
        wh = f"{what} (epilogue {epi})"
        res = _three_runs(lib, lambda: _consumer(lib, cuda, epi, M, N2, N, N2, 0, x16, N, wf, N, cs, bf, stats), wh)
        out = res["out"]
        valid = torch.zeros(out.shape, dtype=torch.bool, device=cuda)
        valid[:M, :N2] = True
        _assert_sentinels(out, valid, wh)
        got = out[:M, :N2]
        ref, bound, (mu, rstd) = _ln_reference(epi, x16[:, :N], wf, cs, bf)
        _check(got, ref, bound, f"{epi}.chain", wh)
        # against the module: LayerNorm of the fp32 residual, unrounded gamma * W
        x = x32.double()
        ln = torch.nn.functional.layer_norm(x, (N,), gamma.double(), beta.double(), LN_EPS)
        lin32 = ln @ wraw.double().t() + b.double()
        ref32 = lin32 if epi == 8 else _qg(lin32)
        mu32 = x.mean(1, keepdim=True)
        rstd32 = torch.rsqrt(x.var(1, unbiased=False, keepdim=True) + LN_EPS)
        dx = (x - x16[:, :N].double()).abs()
        dw = (wraw.double() * gamma.double()[None, :] - wf.double()).abs()
        quant = (rstd * (dx @ wf.double().abs().t() + (x - mu32).abs() @ dw.t()) + (rstd32 - rstd).abs() *
                 ((x - mu32) @ wf.double().t()).abs() + rstd * (mu32 - mu).abs() * cs.double().abs()[None, :])
        _check(got, ref32, bound + (QGELU_SLOPE if epi == 9 else 1.0) * quant, f"{epi}.module", wh + " vs LayerNorm")


# ------------------------------------------------------------------------------------------------ MN-major (pg_gemm_tn)
@pytest.mark.parametrize("bf16", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("M", [129, 300, 577])
def test_mn_major_weight_gradient_form(cuda, lib, M, bf16):
    """D (+)= a^T w with a [K, lda] and w [K, ldw] (contraction index outermost): poison in the padding columns of both,
    sentinels around the output; overwrite (epilogue 3) and accumulate (epilogue 2)."""
    dt = torch.bfloat16 if bf16 else torch.float16
    for N in (256, 768):
        for K in (1, 70, 577):
            g = torch.Generator(device=cuda).manual_seed(M * 31 + N + K + bf16)
            a, lda = _operand(K, M, 1e-2, dt, g, cuda)
            w, ldw = _operand(K, N, 0.3, dt, g, cuda)
            acc0 = torch.randn(M, N, generator=g, device=cuda) * 1e-2
            ldo = N + 8
            for accumulate in (0, 1):
                def call():
                    out = _sentinel(M + 2, ldo, torch.float32, dev=cuda)
                    if accumulate:
                        out[:M, :N] = acc0
                    st = _run(lib, M=M, N=N, K=K, a=a.data_ptr(), lda=lda, w=w.data_ptr(), ldw=ldw, out=out.data_ptr(),
                              ldo=ldo, epilogue=2 if accumulate else 3, operand_bf16=bf16, mn_major=1)
                    assert st == 0, lib.pg_last_error().decode()
                    return {"out": out}
                what = f"mn-major M={M} N={N} K={K} bf16={bf16} accumulate={accumulate}"
                out = _three_runs(lib, call, what)["out"]
                valid = torch.zeros(out.shape, dtype=torch.bool, device=cuda)
                valid[:M, :N] = True
                _assert_sentinels(out, valid, what)
                a64, w64 = a[:, :M].double(), w[:, :N].double()
                z = a64.t() @ w64
                bound = C_ACC * U * math.sqrt(K) * (a64.abs().t() @ w64.abs()) + 2 * U * z.abs()
                ref = z
                if accumulate:
                    ref = z + acc0.double()
                    bound = bound + 2 * U * acc0.double().abs()
                _check(out[:M, :N], ref, bound, "tn", what)


# ------------------------------------------------------------------------------------------------ rejections
def test_rejected_problems_enqueue_nothing(cuda, lib):
    """Each problem a kernel cannot run returns an error before anything is enqueued, and the output keeps its sentinels."""
    M, N, K = 256, 256, 256
    g = torch.Generator(device=cuda).manual_seed(3)
    a, lda = _operand(M, K, 0.5, torch.float16, g, cuda)
    w, ldw = _operand(N, K, 0.05, torch.float16, g, cuda)
    bias = torch.randn(N + 8, generator=g, device=cuda)
    raw = torch.zeros((M + 1) * (N + 8) + 16, device=cuda)            # room for misaligned views
    aux = torch.zeros(M, N + 8, dtype=torch.float16, device=cuda)
    stats = torch.zeros(M * 8 + 8, device=cuda)
    cs = torch.zeros(N + 8, device=cuda)
    base = dict(M=M, N=N, K=K, a=a.data_ptr(), lda=lda, w=w.data_ptr(), ldw=ldw, ldo=N + 8, bias=bias.data_ptr())
    f32, f16p = 4, 2
    cases = {
        "ldo < N": dict(epilogue=3, ldo=N - 8),
        "lda < K": dict(epilogue=3, lda=K - 8),
        "ldw < K": dict(epilogue=3, ldw=K - 8),
        "lda not a multiple of 8": dict(epilogue=3, lda=lda + 1),
        "unknown epilogue": dict(epilogue=10),
        "residual 4 bytes off 16-byte alignment": dict(epilogue=2, resid=raw.data_ptr() + f32),
        "producer: stats 4 bytes off 8-byte alignment": dict(epilogue=7, aux=aux.data_ptr(), stats=stats.data_ptr() + f32),
        "consumer 8: stats 4 bytes off 8-byte alignment": dict(epilogue=8, stats=stats.data_ptr() + f32, colsum=cs.data_ptr()),
        "consumer 9: stats 4 bytes off 8-byte alignment": dict(epilogue=9, stats=stats.data_ptr() + f32, colsum=cs.data_ptr()),
        "producer: N % 128": dict(epilogue=7, N=192, aux=aux.data_ptr(), stats=stats.data_ptr()),
        "producer: ldo % 8": dict(epilogue=7, ldo=N + 4, aux=aux.data_ptr(), stats=stats.data_ptr()),
        "producer: no stats": dict(epilogue=7, aux=aux.data_ptr()),
        "producer: no aux": dict(epilogue=7, stats=stats.data_ptr()),
        "save: no aux": dict(epilogue=6),
        "save: aux off 16-byte alignment": dict(epilogue=6, aux=aux.data_ptr() + 4 * f16p),
        "dgelu: no aux": dict(epilogue=5),
        "consumer: K % 128": dict(epilogue=8, K=192, stats=stats.data_ptr(), colsum=cs.data_ptr()),
        "consumer: N % 64": dict(epilogue=9, N=200, stats=stats.data_ptr(), colsum=cs.data_ptr()),
        "consumer: no colsum": dict(epilogue=8, stats=stats.data_ptr()),
        "consumer: colsum off 16-byte alignment": dict(epilogue=8, stats=stats.data_ptr(), colsum=cs.data_ptr() + f32),
        "consumer: no bias": dict(epilogue=9, bias=None, stats=stats.data_ptr(), colsum=cs.data_ptr()),
        "consumer: no stats": dict(epilogue=8, colsum=cs.data_ptr()),
        "mn-major: N % 256": dict(epilogue=3, mn_major=1, N=200, lda=M, ldw=200),
        "mn-major: M <= 128": dict(epilogue=3, mn_major=1, M=128, lda=128, ldw=N),
        "mn-major: lda < M": dict(epilogue=3, mn_major=1, lda=M - 8, ldw=N),
        "mn-major: ldw < N": dict(epilogue=3, mn_major=1, lda=M, ldw=N - 8),
    }
    for name, over in cases.items():
        out_dt = torch.float16 if over.get("epilogue") in (0, 1, 6, 8, 9) else torch.float32
        out = _sentinel(M + 1, N + 8, out_dt, cuda)
        kw = dict(base, out=out.data_ptr(), **over)
        for mode in (0, 1):
            _set_schedule(lib, mode)
            try:
                st = _run(lib, **kw)
            finally:
                _set_schedule(lib, 0)
            assert st != 0, f"{name}: accepted"
            assert lib.pg_last_error().decode(), name
        torch.cuda.synchronize()
        _assert_sentinels(out, torch.zeros(out.shape, dtype=torch.bool, device=cuda), name)
