"""GEMM schedules on one GPU: the automatic choice (schedule 0, the default: the 128 x 256 kernel for the fp16-output
projections and the fp32 residual updates, ping-pong for the rest) against the ping-pong kernel for every K-major GEMM
(schedule 2, pg_gemm_set_schedule).  Writes one JSON file, <out>/gemm_bench.json, with the card's name, power limit and SM clocks
(read-only nvidia-smi queries) beside the numbers.

  1. per GEMM family at the real shapes: VitEngine.forward on --views views of ViT-L/14-336 (LayerNorm folded), device
     time per family from the library's launch events, both schedules alternating, --rounds rounds each;
  2. K-sweep: M = 590 848 (1024 views x 577 tokens), N in {1024, 3072}, K in {256 .. 4096}, EPI_F16_BIAS and
     EPI_F16_BIAS_QGELU, and at N = 1024 EPI_F32_BIAS_RESID_STATS in place (K = 1024 is out_proj, K = 4096 fc2, which
     the per-family profile cannot tell apart), both schedules, fitted to t = a + b K: b gives the mainloop rate, a the
     per-tile fixed cost (epilogue, fill, drain); torch.matmul (cuBLAS) at the same shapes as a reference point on the same card;
  3. --bench-ab: bench.py --steps 10 --warmup 3 --no-cpu-baseline --dump-outputs as a subprocess, 3 times with
     PG_GEMM_SCHEDULE=2 and 3 times without, alternating; every dumped array of the two schedules compared bit for bit.

usage: python tools/gemm_bench.py [--out DIR] [--bench-ab] [--skip-families] [--skip-sweep]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TOKENS = 577
SCHEDULES = (0, 2)   # the automatic choice, and its reference: the ping-pong kernel for every K-major GEMM
SWEEP_K = (256, 512, 1024, 2048, 4096)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        v = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": v[0], "power_limit_w": float(v[1]), "sm_mhz": float(v[2]), "sm_max_mhz": float(v[3])}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(0), "nvidia_smi": f"unavailable ({e})"}


def read_profile(lib):
    n = lib.pg_profile_end()
    names, ms, counts = (C.c_char_p * n)(), (C.c_float * n)(), (C.c_int32 * n)()
    lib.pg_profile_read(names, ms, counts, n)
    return {names[i].decode(): (float(ms[i]), int(counts[i])) for i in range(n)}


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "runs": xs}


def families(views, rounds):
    """Per-family device ms and algorithmic TFLOP/s of one VitEngine.forward, schedules alternating."""
    from pigeon_b200 import _lib, ops, synthetic
    from pigeon_b200.vit_engine import VitDims, VitEngine
    dims = VitDims()
    lib = _lib.load()
    eng = VitEngine(synthetic.random_vit_state_dict(dims, seed=0), dims, device="cuda", max_views_per_pass=views,
                    fold_layernorm=True)
    px = torch.randn(views, 3, dims.image_size, dims.image_size, generator=torch.Generator().manual_seed(0)).half().cuda()
    M, H, I, L = views * TOKENS, dims.hidden, dims.intermediate, dims.layers
    patch_k = 3 * dims.patch_size ** 2
    flop = {"gemm_f16_ln_bias": 2 * M * 3 * H * H * L,                          # qkv
            "gemm_f16_ln_bias_qgelu": 2 * M * I * H * L,                        # fc1
            "out_proj+fc2": 2 * M * H * H * L + 2 * M * H * I * L,              # gemm_f32_bias_resid(_stats)
            "gemm_f32_rowmap": 2 * views * (TOKENS - 1) * H * patch_k}          # patch embedding
    res = {s: [] for s in SCHEDULES}
    for sched in SCHEDULES:                   # warm-up: module load, tensor maps, attributes
        ops.gemm_set_schedule(sched)
        eng.forward(px)
    torch.cuda.synchronize()
    for _ in range(rounds):
        for sched in SCHEDULES:
            ops.gemm_set_schedule(sched)
            lib.pg_profile_begin()
            eng.forward(px)
            torch.cuda.synchronize()
            fam = read_profile(lib)
            g = {k: v[0] for k, v in fam.items() if k.startswith("gemm")}
            g["out_proj+fc2"] = g.pop("gemm_f32_bias_resid_stats", 0.0) + g.pop("gemm_f32_bias_resid", 0.0)
            g["gemm_total"] = sum(v for k, v in g.items())
            res[sched].append(g)
    ops.gemm_set_schedule(0)
    total_flop = sum(flop.values())
    out = {}
    for sched, runs in res.items():
        d = {}
        for k in runs[0]:
            ms = [r[k] for r in runs]
            f = total_flop if k == "gemm_total" else flop.get(k)
            d[k] = {"ms": spread(ms), "tflops_median": (f / (statistics.median(ms) / 1e3) / 1e12) if f else None}
        out[f"schedule_{sched}"] = d
    out["views"], out["rounds"], out["gemm_rows"] = views, rounds, M
    return out


def sweep(reps=5):
    """K-sweep of the two schedules and cuBLAS at M = 590 848."""
    from pigeon_b200 import _lib, ops
    from pigeon_b200._lib import check, current_stream_ptr, ptr
    lib = _lib.load()
    M, Kmax = 1024 * TOKENS, max(SWEEP_K)
    g = torch.Generator(device="cuda").manual_seed(0)
    a = (torch.randn(M, Kmax, device="cuda", generator=g) * 0.5).half()
    out = {"M": M, "K": list(SWEEP_K), "configs": {}}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        fn()
        ev[0].record()
        for _ in range(reps):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / reps

    for N in (1024, 3072):
        w = (torch.randn(N, Kmax, device="cuda", generator=g) * 0.03).half()
        bias = torch.randn(N, device="cuda", generator=g)
        epis = ((0, "EPI_F16_BIAS"), (1, "EPI_F16_BIAS_QGELU")) + (((7, "EPI_F32_BIAS_RESID_STATS"),) if N == 1024 else ())
        for epi, name in epis:
            if epi == 7:   # the residual stream updated in place, its fp16 copy and per-128-column moments (out_proj, fc2)
                o = torch.randn(M, N, device="cuda", generator=g)
                aux = torch.empty(M, N, device="cuda", dtype=torch.float16)
                stats = torch.empty(M, N // 128, 2, device="cuda")

                def run(K):
                    p = _lib.GemmProblem(M=M, N=N, K=K, a=ptr(a), lda=Kmax, w=ptr(w), ldw=Kmax, out=ptr(o), ldo=N, bias=ptr(bias),
                                         epilogue=epi, aux=ptr(aux), stats=ptr(stats))
                    check(lib.pg_gemm_problem_run(C.byref(p), current_stream_ptr()), "pg_gemm_problem_run")
            else:
                o = torch.empty(M, N, device="cuda", dtype=torch.float16)

                def run(K):
                    check(lib.pg_gemm_f16(ptr(a), Kmax, ptr(w), Kmax, ptr(o), N, ptr(bias), M, N, K, epi, current_stream_ptr()),
                          "pg_gemm_f16")
            for sched in SCHEDULES:
                ops.gemm_set_schedule(sched)
                ts = [timed(lambda: run(K)) for K in SWEEP_K]
                b, a0 = np.polyfit(np.array(SWEEP_K, dtype=float), np.array(ts), 1)
                tiles = (M // 128) * (N // (256 if sched == 0 else 128))
                out["configs"][f"N{N}_{name}_schedule{sched}"] = {
                    "ms": ts, "tflops": [2 * M * N * K / (t / 1e3) / 1e12 for K, t in zip(SWEEP_K, ts)],
                    "fit_ms_intercept": a0, "fit_ms_per_k": b,
                    "mainloop_tflops_from_slope": 2 * M * N / (b / 1e3) / 1e12,
                    "fixed_us_per_tile_per_sm": a0 * 1e3 / (tiles / torch.cuda.get_device_properties(0).multi_processor_count)}
            del o
            if epi == 7:
                del aux, stats
        ops.gemm_set_schedule(0)
        ts = []
        for K in SWEEP_K:
            x, y = a[:, :K], w[:, :K].t()
            ts.append(timed(lambda: torch.matmul(x, y)))
        b, a0 = np.polyfit(np.array(SWEEP_K, dtype=float), np.array(ts), 1)
        out["configs"][f"N{N}_cublas_matmul_f16"] = {"ms": ts, "tflops": [2 * M * N * K / (t / 1e3) / 1e12 for K, t in zip(SWEEP_K, ts)],
                                                     "fit_ms_intercept": a0, "fit_ms_per_k": b,
                                                     "mainloop_tflops_from_slope": 2 * M * N / (b / 1e3) / 1e12}
        del w
    return out


def bench_ab(runs=3):
    """bench.py under both schedules, alternating; outputs compared bit for bit."""
    res = {f"schedule_{s}": [] for s in SCHEDULES}
    dirs = {s: [] for s in SCHEDULES}
    tmp = tempfile.mkdtemp(prefix="gemm_bench_ab_")
    for r in range(runs):
        for sched in SCHEDULES[::-1]:
            d = os.path.join(tmp, f"s{sched}_r{r}")
            env = dict(os.environ)
            env.pop("PG_GEMM_SCHEDULE", None)
            if sched != 0:
                env["PG_GEMM_SCHEDULE"] = str(sched)
            p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "10", "--warmup", "3",
                                "--no-cpu-baseline", "--dump-outputs", d], capture_output=True, text=True, env=env, cwd=ROOT)
            line = [l for l in p.stdout.splitlines() if l.startswith("{")]
            if p.returncode != 0 or not line:
                raise RuntimeError(f"bench.py failed (schedule {sched}):\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            j = json.loads(line[-1])
            res[f"schedule_{sched}"].append(j)
            dirs[sched].append(d)
    same = {}
    ref_dirs = dirs[SCHEDULES[1]]
    for name in sorted(os.listdir(ref_dirs[0])):
        ref = np.load(os.path.join(ref_dirs[0], name))
        same[name] = all(np.array_equal(np.load(os.path.join(d, name)), ref) for d in dirs[0] + ref_dirs)
    v = {s: [j["value"] for j in res[f"schedule_{s}"]] for s in SCHEDULES}
    summary = {"images_per_s": {f"schedule_{s}": spread(v[s]) for s in SCHEDULES},
               "speedup_median": statistics.median(v[0]) / statistics.median(v[SCHEDULES[1]]),
               "every_new_run_faster": min(v[0]) > max(v[SCHEDULES[1]]),
               "outputs_bit_identical": same, "all_outputs_bit_identical": all(same.values()),
               "parity_ok_all_runs": all(j["parity_check"]["ok"] for s in SCHEDULES for j in res[f"schedule_{s}"]),
               "runs": res}
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gemm_bench_out")
    ap.add_argument("--views", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-families", action="store_true")
    ap.add_argument("--skip-sweep", action="store_true")
    ap.add_argument("--bench-ab", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_bench needs a CUDA GPU")
    result = {"gpu": gpu_info()}
    if not args.skip_families:
        result["families"] = families(args.views, args.rounds)
        torch.cuda.empty_cache()
    if not args.skip_sweep:
        result["k_sweep"] = sweep()
        torch.cuda.empty_cache()
    if args.bench_ab:
        result["bench_ab"] = bench_ab()
    result["gpu_after"] = gpu_info()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gemm_bench.json"), "w") as f:
        json.dump(result, f, indent=1)
    brief = {k: v for k, v in result.get("bench_ab", {}).items() if k != "runs"}
    print(json.dumps({"gpu": result["gpu"], "bench_ab": brief,
                      "families": {f"schedule_{s}": {k: (round(v["ms"]["median"], 2), v["tflops_median"] and round(v["tflops_median"]))
                                                     for k, v in result["families"][f"schedule_{s}"].items()}
                                   for s in SCHEDULES}
                      if "families" in result else None}))


if __name__ == "__main__":
    main()
