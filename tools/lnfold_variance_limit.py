"""How far from zero-mean can a residual row be before the folded LayerNorm's one-pass variance spoils the fp16 output?

The LayerNorm-producer epilogue (7) stores per-128-column (sum, sum of squares) of the fp16 row; the consumer epilogues (8, 9)
form mu = sum / K and var = sum_sq / K - mu^2 in fp32 and scale by rstd = rsqrt(var + eps).  Every output then carries the
relative error of rstd times |out - b'| (the normalised product before the bias), so the variance stays inside the fp16
output budget while rstd's relative error is at most half an fp16 ulp, 2^-12.  The error of var grows like u (mu / sigma)^2.

For rows x = +-r + N(0, 1) this runs the producer on the GPU, forms rstd from its statistics with the consumer's fp32 operations,
and reports per r = |mean| / std the largest relative error of rstd against fp64 statistics of the same fp16 row, and the
largest |error| / bound of the consumer epilogue (8) against the per-element bound of tests/test_gpu_gemm_epilogues.py.
Prints one JSON line per r, the first r whose rstd error exceeds 2^-12, and the GPU it ran on.
python tools/lnfold_variance_limit.py"""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pigeon_b200 import _lib  # noqa: E402

U = 2.0 ** -24
EPS = 1e-5


def run(lib, **kw):
    p = _lib.GemmProblem(**kw)
    _lib.check(lib.pg_gemm_problem_run(C.byref(p), _lib.current_stream_ptr()), "pg_gemm_problem_run")


def ulp16(x):
    _, e = torch.frexp(x.abs())
    return torch.ldexp(torch.ones_like(x), (e - 1).clamp_min(-14) - 10)


def main():
    dev = torch.device("cuda:0")
    lib = _lib.load()
    M, K, N = 4096, 1024, 3072
    g = torch.Generator(device=dev).manual_seed(0)
    wraw = torch.randn(N, K, generator=g, device=dev) * 0.03
    gamma = 1 + 0.1 * torch.randn(K, generator=g, device=dev)
    beta = 0.1 * torch.randn(K, generator=g, device=dev)
    b = torch.randn(N, generator=g, device=dev)
    wf = (wraw * gamma[None, :]).half()
    cs = wf.float().sum(dim=1)
    bf = b + wraw @ beta
    zero_a = torch.zeros(M, K, dtype=torch.float16, device=dev)
    w_any = torch.zeros(K, K, dtype=torch.float16, device=dev)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip()
    except OSError:
        q = "unknown"
    print(json.dumps({"gpu": q, "M": M, "K": K, "N": N}))
    limit = None
    for r in (0, 1, 2, 4, 8, 16, 30, 45, 64, 90, 128, 181, 256, 362, 512):
        R = torch.randn(M, K, generator=g, device=dev) + r * torch.where(torch.arange(M, device=dev) % 2 == 0, 1.0, -1.0)[:, None]
        x32 = R.clone()
        aux = torch.empty(M, K, dtype=torch.float16, device=dev)
        stats = torch.empty(M, K // 128, 2, device=dev)
        # producer: A = 0, no bias, so the new residual is R itself
        run(lib, M=M, N=K, K=K, a=zero_a.data_ptr(), lda=K, w=w_any.data_ptr(), ldw=K, out=x32.data_ptr(), ldo=K,
            epilogue=7, aux=aux.data_ptr(), stats=stats.data_ptr())
        out = torch.empty(M, N, dtype=torch.float16, device=dev)
        run(lib, M=M, N=N, K=K, a=aux.data_ptr(), lda=K, w=wf.data_ptr(), ldw=K, out=out.data_ptr(), ldo=N,
            bias=bf.data_ptr(), epilogue=8, stats=stats.data_ptr(), colsum=cs.data_ptr(), ln_eps=EPS)
        torch.cuda.synchronize()
        x = aux.double()
        mu = x.mean(1, keepdim=True)
        rstd = torch.rsqrt(x.var(1, unbiased=False, keepdim=True) + EPS)
        # the consumer's arithmetic on the producer's statistics: fp32 slot sums in order, one-pass variance
        s1 = torch.zeros(M, device=dev)
        s2 = torch.zeros(M, device=dev)
        for k in range(K // 128):
            s1 += stats[:, k, 0]
            s2 += stats[:, k, 1]
        mu_k = s1 * (1.0 / K)
        var_k = (s2 * (1.0 / K) - mu_k * mu_k).clamp_min(0.0)
        rstd_k = torch.rsqrt(var_k + EPS).double()
        rstd_err = ((rstd_k - rstd.squeeze(1)).abs() / rstd.squeeze(1)).max().item()
        cs64, b64 = cs.double()[None, :], bf.double()[None, :]
        z = x @ wf.double().t()
        ref = rstd * (z - mu * cs64) + b64
        bound = (ulp16(ref) + rstd * 2 * U * math.sqrt(K) * (x.abs() @ wf.double().abs().t()) +
                 4 * U * (rstd * z.abs() + rstd * mu.abs() * cs64.abs() + b64.abs()) + 2 ** -21 * (ref - b64).abs())
        o = out.double()
        ratio = ((o - ref).abs() / bound).max().item()
        sd = x.std(1, unbiased=False)
        print(json.dumps({"mean_over_std": round((mu.abs().squeeze(1) / sd).median().item(), 2),
                          "rstd_rel_err": float(f"{rstd_err:.3g}"), "rstd_err_over_half_fp16_ulp": round(rstd_err / 2 ** -12, 4),
                          "error_over_test_bound": round(ratio, 4)}), flush=True)
        if limit is None and rstd_err > 2 ** -12:
            limit = r
    print(json.dumps({"first_r_outside_fp16_budget": limit}))


if __name__ == "__main__":
    main()
