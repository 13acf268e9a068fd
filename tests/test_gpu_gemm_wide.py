"""The 128 x 256 GEMM kernel (gemm_wide.cu, schedule 0 for the fp16-output epilogues) against the ping-pong kernel
(schedule 2) and the single-warpgroup kernel (schedule 1): the same products summed in the same order and the same
epilogue arithmetic, so every output must be the same bits.  Rows past M, 256-column tiles partly or wholly past N, partial
K blocks, an output row pitch wider than N with NaN guard columns and guard rows that must stay NaN, and a row pitch the
TMA store cannot take (it falls back to the ping-pong kernel and must give the same bits)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

SENT = 0x7E5A                   # fp16 NaN with a payload no kernel writes
POISON = 1.0e4                  # operand columns [K, ld): reading them would show at once
LN_EPS = 1e-5
MS = [1, 64, 65, 130, 577 * 16]
NS = [128, 320, 1000, 3072, 4096]
KS = [64, 96, 1024]


@pytest.fixture(scope="module")
def lib(cuda):
    from pigeon_b200 import _lib
    return _lib.load()


def _operand(rows, k, dt, g, dev, shift=0.0):
    """[rows, ld] with ld a multiple of 8 and at least 8 poisoned columns past k."""
    ld = (k + 7) // 8 * 8 + 8
    t = torch.full((rows, ld), POISON, dtype=dt, device=dev)
    t[:, :k] = (torch.randn(rows, k, generator=g, device=dev) + shift).to(dt)
    return t, ld


def _case(lib, dev, epi, bf16, M, N, K, ldo, seed, bias=True):
    """out = [M + 2, ldo] fp16 filled with the sentinel, under schedules 0, 2 and 1; returns the three buffers."""
    from pigeon_b200 import _lib
    dt = torch.bfloat16 if bf16 else torch.float16
    g = torch.Generator(device=dev).manual_seed(seed)
    ln = epi in (_lib.EPI_F16_LN_BIAS, _lib.EPI_F16_LN_BIAS_QGELU)
    x, ldx = _operand(M, K, dt, g, dev, shift=0.3 if ln else 0.0)
    w = torch.full((N, ldx), POISON, dtype=dt, device=dev)
    if ln:   # as VitEngine folds a LayerNorm: W' = gamma * W, colsum = row sums of W', b' = b + W beta
        wraw = torch.randn(N, K, generator=g, device=dev) * 0.03
        gamma = 1 + 0.1 * torch.randn(K, generator=g, device=dev)
        beta = 0.1 * torch.randn(K, generator=g, device=dev)
        wf = (wraw * gamma[None, :]).to(dt)
        w[:, :K] = wf
        colsum = wf.float().sum(dim=1)
        b = torch.randn(N, generator=g, device=dev) + wraw @ beta
        xs = x[:, :K].double().reshape(M, K // 128, 128)   # per-128-column (sum, sum of squares) of the A row
        stats = torch.stack((xs.sum(-1), (xs * xs).sum(-1)), dim=-1).float().reshape(M, K // 64).contiguous()
    else:
        w[:, :K] = (torch.randn(N, K, generator=g, device=dev) * 0.05).to(dt)
        b = torch.randn(N, generator=g, device=dev)
        colsum = stats = None
    outs = {}
    try:
        for sched in (0, 2, 1):
            assert lib.pg_gemm_set_schedule(sched) == 0
            out = torch.empty(M + 2, ldo, dtype=torch.float16, device=dev)
            out.view(torch.int16).fill_(SENT)
            p = _lib.GemmProblem(M=M, N=N, K=K, a=x.data_ptr(), lda=ldx, w=w.data_ptr(), ldw=ldx, out=out.data_ptr(), ldo=ldo,
                                 bias=b.data_ptr() if bias else None, epilogue=epi, operand_bf16=bf16,
                                 stats=None if stats is None else stats.data_ptr(),
                                 colsum=None if colsum is None else colsum.data_ptr(), ln_eps=LN_EPS)
            st = lib.pg_gemm_problem_run(C.byref(p), _lib.current_stream_ptr())
            assert st == 0, lib.pg_last_error().decode()
            outs[sched] = out
    finally:
        assert lib.pg_gemm_set_schedule(0) == 0
    torch.cuda.synchronize()
    return outs


def _check(outs, M, N, what):
    bits = {s: o.view(torch.int16) for s, o in outs.items()}
    assert torch.equal(bits[0], bits[2]), f"{what}: schedule 0 differs from the ping-pong kernel"
    assert torch.equal(bits[0], bits[1]), f"{what}: schedule 0 differs from the single-warpgroup kernel"
    guard = torch.ones_like(bits[0], dtype=torch.bool)
    guard[:M, :N] = False
    assert (bits[0][guard] == SENT).all(), f"{what}: write outside the output"
    assert not (bits[0][:M, :N] == SENT).any(), f"{what}: output element left unwritten"


@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("bf16", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("epi", [0, 1, 8, 9])
def test_wide_kernel_bit_identical(cuda, lib, epi, bf16, M):
    ln = epi in (8, 9)
    for i, N in enumerate(NS):
        for j, K in enumerate(KS):
            if ln and (K % 128 or N % 64):   # the LayerNorm-consumer epilogues' own requirements
                continue
            ldo = (N + 7) // 8 * 8 + 8   # TMA-storable pitch, 8+ NaN guard columns
            what = f"epilogue {epi} bf16={bf16} M={M} N={N} K={K} ldo={ldo}"
            bias = not (epi == 0 and i == 1)   # EPI_F16_BIAS without a bias too
            _check(_case(lib, cuda, epi, bf16, M, N, K, ldo, 100 * i + 10 * j + epi + bf16, bias), M, N, what)


@pytest.mark.parametrize("bf16", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("epi", [0, 1, 8, 9])
def test_unaligned_pitch_falls_back_with_the_same_bits(cuda, lib, epi, bf16):
    M, N, K = 577 * 16, 3072, 1024
    ldo = N + 4   # rows 8 bytes apart from a 16-byte multiple: no TMA store, the ping-pong kernel runs under schedule 0
    _check(_case(lib, cuda, epi, bf16, M, N, K, ldo, 7 + epi + bf16), M, N, f"epilogue {epi} bf16={bf16} ldo={ldo}")
