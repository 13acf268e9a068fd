"""The fp32 residual epilogues (out_proj and fc2) of the 128 x 256 GEMM kernel (gemm_wide_resid.cu, schedule 0) against the
ping-pong kernel (schedule 2) and the single-warpgroup kernel (schedule 1).  out fp32 = (acc + bias) + resid, in place or
from a separate source; EPI_F32_BIAS_RESID_STATS also writes the fp16 copy (aux) and the per-128-column moments (stats).
All three must be the same bits under every schedule.  Rows past M, 256-column tiles partly or wholly past N, partial K
blocks, NaN guard columns and rows around out, aux and stats that must stay NaN, and a row pitch the TMA boxes cannot take
(it falls back to the ping-pong kernel and must give the same bits)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

SENT = 0x7E5A                   # fp16 NaN with a payload no kernel writes
SENT32 = 0x7FC0DEAD             # fp32 NaN with a payload no kernel writes
POISON = 1.0e4                  # operand columns [K, ld): reading them would show at once
RESID_NS = {2: [128, 384, 1000, 1024], 7: [128, 384, 1024]}   # 1000: a ragged last tile (epilogue 7 needs N % 128 == 0)
RESID_KS = [64, 96, 1024, 4096]


@pytest.fixture(scope="module")
def lib(cuda):
    from pigeon_b200 import _lib
    return _lib.load()


def _operand(rows, k, dt, g, dev):
    """[rows, ld] with ld a multiple of 8 and at least 8 poisoned columns past k."""
    ld = (k + 7) // 8 * 8 + 8
    t = torch.full((rows, ld), POISON, dtype=dt, device=dev)
    t[:, :k] = torch.randn(rows, k, generator=g, device=dev).to(dt)
    return t, ld


def _resid_case(lib, dev, epi, bf16, M, N, K, ldo, inplace, seed):
    """Runs the problem under schedules 0, 2 and 1 on fresh buffers; returns {schedule: (out, aux, stats)} with guard rows
    and columns (aux and stats None for epilogue 2)."""
    from pigeon_b200 import _lib
    dt = torch.bfloat16 if bf16 else torch.float16
    g = torch.Generator(device=dev).manual_seed(seed)
    x, ldx = _operand(M, K, dt, g, dev)
    w = torch.full((N, ldx), POISON, dtype=dt, device=dev)
    w[:, :K] = (torch.randn(N, K, generator=g, device=dev) * 0.05).to(dt)
    b = torch.randn(N, generator=g, device=dev)
    resid = torch.full((M + 2, ldo), float("nan"), device=dev)
    resid[:M, :N] = torch.randn(M, N, generator=g, device=dev) * 2
    stats_ok = epi == _lib.EPI_F32_BIAS_RESID_STATS
    slots = N // 128
    outs = {}
    try:
        for sched in (0, 2, 1):
            assert lib.pg_gemm_set_schedule(sched) == 0
            out = torch.empty(M + 2, ldo, device=dev)
            out.view(torch.int32).fill_(SENT32)
            if inplace:
                out[:M, :N] = resid[:M, :N]
            aux = stats = None
            if stats_ok:
                aux = torch.empty(M + 2, ldo, dtype=torch.float16, device=dev)
                aux.view(torch.int16).fill_(SENT)
                stats = torch.empty(M + 2, slots, 2, device=dev)
                stats.view(torch.int32).fill_(SENT32)
            p = _lib.GemmProblem(M=M, N=N, K=K, a=x.data_ptr(), lda=ldx, w=w.data_ptr(), ldw=ldx, out=out.data_ptr(), ldo=ldo,
                                 bias=b.data_ptr(), epilogue=epi, operand_bf16=bf16,
                                 resid=None if inplace else resid.data_ptr(),
                                 aux=None if aux is None else aux.data_ptr(), stats=None if stats is None else stats.data_ptr())
            st = lib.pg_gemm_problem_run(C.byref(p), _lib.current_stream_ptr())
            assert st == 0, lib.pg_last_error().decode()
            outs[sched] = (out, aux, stats)
    finally:
        assert lib.pg_gemm_set_schedule(0) == 0
    torch.cuda.synchronize()
    return outs


def _check_resid(outs, M, N, what):
    for i, name in enumerate(("out", "aux", "stats")):
        if outs[0][i] is None:
            continue
        bits = {s: o[i].view(torch.int16 if name == "aux" else torch.int32) for s, o in outs.items()}
        assert torch.equal(bits[0], bits[2]), f"{what}: {name} of schedule 0 differs from the ping-pong kernel"
        assert torch.equal(bits[0], bits[1]), f"{what}: {name} of schedule 0 differs from the single-warpgroup kernel"
        sent = SENT if name == "aux" else SENT32
        b0 = bits[0]
        if name == "stats":
            assert (b0[M:] == sent).all(), f"{what}: stats written past row M"
            assert not (b0[:M] == sent).any(), f"{what}: stats left unwritten"
            continue
        guard = torch.ones_like(b0, dtype=torch.bool)
        guard[:M, :N] = False
        assert (b0[guard] == sent).all(), f"{what}: {name} written outside [M, N]"
        assert not (b0[:M, :N] == sent).any(), f"{what}: {name} element left unwritten"
        assert torch.isfinite(outs[0][i][:M, :N].float()).all(), f"{what}: {name} not finite"


@pytest.mark.parametrize("M", [1, 65, 577 * 16])
@pytest.mark.parametrize("inplace", [1, 0], ids=["inplace", "separate"])
@pytest.mark.parametrize("bf16", [0, 1], ids=["fp16", "bf16"])
@pytest.mark.parametrize("epi", [2, 7])
def test_wide_residual_epilogues_bit_identical(cuda, lib, epi, bf16, inplace, M):
    for i, N in enumerate(RESID_NS[epi]):
        for j, K in enumerate(RESID_KS):
            ldo = (N + 7) // 8 * 8 + 8   # TMA-storable pitch, 8+ NaN guard columns
            what = f"epilogue {epi} bf16={bf16} inplace={inplace} M={M} N={N} K={K} ldo={ldo}"
            outs = _resid_case(lib, cuda, epi, bf16, M, N, K, ldo, inplace, 1000 + 100 * i + 10 * j + epi + bf16)
            _check_resid(outs, M, N, what)


@pytest.mark.parametrize("inplace", [1, 0], ids=["inplace", "separate"])
@pytest.mark.parametrize("bf16", [0, 1], ids=["fp16", "bf16"])
def test_residual_unaligned_pitch_falls_back_with_the_same_bits(cuda, lib, bf16, inplace):
    M, N, K = 577 * 16, 1024, 1024
    ldo = N + 4   # fp32 rows 16-byte aligned but not an fp16-box pitch: the ping-pong kernel runs under schedule 0
    outs = _resid_case(lib, cuda, 2, bf16, M, N, K, ldo, inplace, 11 + bf16)
    _check_resid(outs, M, N, f"epilogue 2 bf16={bf16} inplace={inplace} ldo={ldo}")
