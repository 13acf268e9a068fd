"""Kernel-level parity on the H100: each hand-written kernel against the same op in plain PyTorch fp32
(a floating-point kernel's torch reference, evaluated on the SAME fp16-rounded operands so that the
tolerance measures the kernel, not the quantisation)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 256, 128), (300, 384, 192), (577 * 2, 3072, 1024),
                                   (1154, 1024, 4096), (64, 1000, 3072), (1, 1000, 3072), (1000, 2076, 96)])
def test_gemm_f32_bias(cuda, M, N, K):
    from pigeon_b200 import _lib, ops
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(cuda)
    w = (torch.randn(N, K, generator=g) * 0.05).half().to(cuda)
    b = torch.randn(N, generator=g).to(cuda)
    ref = a.double() @ w.double().t() + b.double()
    out = ops.gemm_f16(a, w, b, _lib.EPI_F32_BIAS)
    torch.cuda.synchronize()
    # fp32 tensor-core accumulation over K up to 4096: ~sqrt(K) * 2^-24 relative
    assert _rel(out, ref) < 1e-5, _rel(out, ref)
    out2 = ops.gemm_f16(a, w, None, _lib.EPI_F32_BIAS)
    assert _rel(out2, ref - b.double()) < 1e-5


@pytest.mark.parametrize("M,N,K", [(256, 512, 256), (1154, 4096, 1024), (130, 384, 64)])
def test_gemm_epilogues(cuda, M, N, K):
    from pigeon_b200 import _lib, ops
    g = torch.Generator(device="cpu").manual_seed(11)
    a = (torch.randn(M, K, generator=g)).half().to(cuda)
    w = (torch.randn(N, K, generator=g) * 0.05).half().to(cuda)
    b = torch.randn(N, generator=g).to(cuda)
    acc = a.float() @ w.float().t() + b
    out = ops.gemm_f16(a, w, b, _lib.EPI_F16_BIAS)
    assert out.dtype == torch.float16 and _rel(out.float(), acc) < 6e-4
    out = ops.gemm_f16(a, w, b, _lib.EPI_F16_BIAS_QGELU)
    ref = acc * torch.sigmoid(1.702 * acc)
    assert _rel(out.float(), ref) < 8e-4
    resid = torch.randn(M, N, generator=g).to(cuda)
    out = resid.clone()
    ops.gemm_f16(a, w, b, _lib.EPI_F32_BIAS_RESID, out=out)
    assert _rel(out, resid + acc) < 1e-5


def test_gemm_many_tiles_persistent(cuda):
    """more tiles than SMs: exercises the persistent loop, the reuse of the accumulator tile and the ring wrap."""
    from pigeon_b200 import _lib, ops
    g = torch.Generator(device="cpu").manual_seed(5)
    M, N, K = 577 * 64, 1024, 1024
    a = (torch.randn(M, K, generator=g)).half().to(cuda)
    w = (torch.randn(N, K, generator=g) * 0.03).half().to(cuda)
    out = ops.gemm_f16(a, w, None, _lib.EPI_F32_BIAS)
    ref = a.float() @ w.float().t()
    assert _rel(out, ref) < 1e-5
    assert torch.equal(ops.gemm_f16(a, w, None, _lib.EPI_F32_BIAS), out), "GEMM must be run-to-run deterministic"


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("n_views,seq,heads", [(1, 128, 1), (1, 64, 2), (2, 577, 2), (3, 200, 1), (1, 577, 16),
                                               (2, 65, 1), (1, 129, 1), (1, 17, 4)])
def test_attention(cuda, n_views, seq, heads):
    from pigeon_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(seq * 3 + heads)
    hidden = heads * 64
    qkv = (torch.randn(n_views * seq, 3 * hidden, generator=g) * 1.5).half().to(cuda)
    out = ops.attention_f16(qkv, n_views, seq, heads)
    torch.cuda.synchronize()
    x = qkv.float().view(n_views, seq, 3, heads, 64)
    q, k, v = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    att = torch.softmax(q @ k.transpose(-1, -2) * 0.125, dim=-1)
    ref = (att @ v).permute(0, 2, 1, 3).reshape(n_views * seq, hidden)
    err = _rel(out.float(), ref)
    assert err < 2e-3, err  # P and the output are rounded to fp16
    assert torch.isfinite(out.float()).all()


ATTN_KERNELS = [(None, -1), (3, 2), (3, 12), (0, 2), (2, 2), (1, 0)]   # default entry point, then every (variant, poly) the ABI accepts


def _attention_reference(qkv, n_views, seq, heads):
    xf = qkv.float().view(n_views, seq, 3, heads, 64)
    q, k, v = (xf[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    logits = q @ k.transpose(-1, -2) * 0.125
    out = (torch.softmax(logits, dim=-1) @ v).permute(0, 2, 1, 3).reshape(n_views * seq, heads * 64)
    return out, logits


def test_attention_views_are_independent(cuda):
    """A view's last KV block ends inside the next view's rows: non-finite values there must not reach this view."""
    from pigeon_b200 import ops
    n_views, seq, heads = 2, 65, 2
    g = torch.Generator(device="cpu").manual_seed(5)
    qkv = (torch.randn(n_views * seq, 3 * heads * 64, generator=g) * 1.5).half()
    ref, _ = _attention_reference(qkv[:seq].to(cuda), 1, seq, heads)
    qkv[seq:] = float("nan")
    out = ops.attention_f16(qkv.to(cuda), n_views, seq, heads)
    assert torch.isfinite(out[:seq].float()).all()
    assert _rel(out[:seq].float(), ref) < 2e-3


@pytest.mark.parametrize("variant,poly", ATTN_KERNELS[1:])
@pytest.mark.parametrize("n_views,seq,heads", [(2, 577, 3), (1, 17, 4), (3, 200, 1), (2, 64, 2), (1, 129, 5)])
def test_attention_every_kernel_and_its_lse2(cuda, n_views, seq, heads, variant, poly):
    """Every (variant, poly) of the ABI against torch fp32, output and the log2-domain log-sum-exp side output (what the
    training forward keeps for the backward)."""
    from pigeon_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(seq * 5 + heads)
    qkv = (torch.randn(n_views * seq, 3 * heads * 64, generator=g) * 1.5).half().to(cuda)
    out, lse2 = ops.attention_f16(qkv, n_views, seq, heads, variant=variant, poly=poly, return_lse2=True)
    ref, logits = _attention_reference(qkv, n_views, seq, heads)
    assert torch.isfinite(out.float()).all() and _rel(out.float(), ref) < 2e-3
    lse_ref = torch.logsumexp(logits, dim=-1) * 1.4426950408889634
    assert (lse2.view(n_views, heads, seq) - lse_ref).abs().max().item() < 1e-2


@pytest.mark.parametrize("variant,poly", ATTN_KERNELS)
def test_attention_growing_logits_exercise_rescale(cuda, variant, poly):
    """Key norms grow along the sequence so that later KV blocks raise the row maximum far beyond what fp16 P can hold
    relative to the first block: the kernel must rescale O and l when the maximum rises and agree with an exact softmax."""
    from pigeon_b200 import ops
    n_views, seq, heads = 2, 577, 2
    g = torch.Generator(device="cpu").manual_seed(77)
    hidden = heads * 64
    x = torch.randn(n_views, seq, 3, heads, 64, generator=g)
    ramp = (0.25 + 6.0 * torch.arange(seq) / seq).view(1, seq, 1, 1)
    x[:, :, 1] *= ramp                                   # k
    qkv = x.reshape(n_views * seq, 3 * hidden).half().to(cuda)
    out = ops.attention_f16(qkv, n_views, seq, heads, variant=variant, poly=poly)
    ref, logits = _attention_reference(qkv, n_views, seq, heads)
    spread = (logits.max(-1).values - logits[..., :64].max(-1).values) * 1.4427
    assert (spread > 20).float().mean() > 0.05, "test must push a share of the rows out of the fp16 window"
    assert (spread < 18).float().mean() > 0.2, "and leave others inside it"
    err = _rel(out.float(), ref)
    assert torch.isfinite(out.float()).all() and err < 2e-3, err
    # row by row: the rescaled rows and the others are both right
    row_err = (out.float() - ref).norm(dim=1) / ref.norm(dim=1).clamp_min(1e-6)
    assert row_err.max().item() < 2e-2, row_err.max().item()


# ------------------------------------------------------------------------------------------------ head
@pytest.mark.parametrize("B,V,D,C,k", [(8, 4, 1024, 1000, 50), (3, 1, 1024, 2076, 5), (256, 4, 1024, 1000, 50),
                                       (5, 4, 256, 331, 7), (300, 4, 1024, 2076, 5)])
@pytest.mark.parametrize("fused", [False, True])
def test_head(cuda, B, V, D, C, k, fused):
    from pigeon_b200 import ops
    ops.head_set_fused(fused)
    try:
        _check_head(cuda, B, V, D, C, k)
    finally:
        ops.head_set_fused(False)


def _check_head(cuda, B, V, D, C, k):
    from pigeon_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(B + C)
    emb = (torch.randn(B, V, D, generator=g) * 0.3).to(cuda)
    lin = torch.nn.Linear(D, C)
    W, bias = lin.weight.detach().to(cuda), lin.bias.detach().to(cuda)
    cent = torch.rand(C, 2, generator=g, dtype=torch.float64).to(cuda) * 100
    out = ops.head_forward(emb, ops.head_pack_weight(W), bias, cent, k)
    pooled = emb.mean(1)
    logits = pooled.double() @ W.double().t() + bias.double()
    probs = torch.softmax(logits, -1)
    assert _rel(out["pooled"], pooled) < 1e-6
    # error-compensated fp16 split: ~1e-5 relative, two orders below the plain-fp16 5e-4
    assert _rel(out["logits"], logits) < 2e-5, _rel(out["logits"], logits)
    assert _rel(out["probs"], probs) < 2e-5
    tk = torch.topk(probs, k, dim=-1)
    assert torch.equal(out["pred_cell"], out["probs"].argmax(-1))
    assert torch.equal(out["topk_idx"], torch.topk(out["probs"], k, dim=-1).indices)
    # against the fp64 reference: identical ranking wherever its own margins exceed the logit error
    gaps = (tk.values[:, :-1] - tk.values[:, 1:]) / tk.values[:, :-1]
    safe = torch.cat([gaps > 1e-4, torch.ones_like(gaps[:, :1], dtype=torch.bool)], 1).cumprod(1).bool()
    assert safe.float().mean() > 0.2
    assert torch.equal(out["topk_idx"][safe], tk.indices[safe])
    assert torch.allclose(out["topk_val"].double(), tk.values, rtol=1e-4, atol=0)
    assert torch.equal(out["pred_lnglat"], cent[out["pred_cell"]])


# ------------------------------------------------------------------------------------------------ refiner
@pytest.mark.parametrize("C,P,D,B,kc,topk,members,T,maxref", [
    (50, 600, 1024, 64, 10, 5, 0.0, 1.6, 1000.0),
    (50, 600, 768, 64, 10, 10, 6.0, 0.6, 100000.0),
    (40, 300, 256, 33, 5, 5, 3.0, 1.0, 2000.0),
    # BASELINE.json configs[2] scale: the 100k-prototype bank of the bench, one rank's batch, top-5 and top-40
    (1000, 100_000, 1024, 256, 40, 5, 0.0, 1.6, 1000.0),
    (1000, 100_000, 1024, 256, 40, 40, 0.0, 0.6, 100000.0),
])
def test_refiner_vs_oracle(cuda, C, P, D, B, kc, topk, members, T, maxref):
    import numpy as np
    from oracle import refiner as oref
    from pigeon_b200 import ops, synthetic
    bank = synthetic.synthetic_bank(C, P, D, seed=2, members_mean=members, empty_cells=3)
    cand, probs = synthetic.synthetic_candidates(B, kc, C, seed=3)
    emb = torch.from_numpy(synthetic.synthetic_queries(bank, cand, views=4, seed=4))
    init = torch.from_numpy(synthetic.synthetic_geocells(B, seed=9))
    candt, probst = torch.from_numpy(cand), torch.from_numpy(probs)
    # put every other initial guess next to its refined location so that both outcomes of the
    # max-refinement gate (proto_refiner.py:202-203) occur
    ll0, _, _ = oref.refiner_forward(bank, emb, init, candt, probst, topk, T, 1e12)
    init[::2] = ll0[::2].double() + 0.25
    ll, cell, info = oref.refiner_forward(bank, emb, init, candt, probst, topk, T, maxref)
    dbank = ops.DeviceBank(cuda, **bank)
    oll, ocell, dbg = ops.refiner_forward(dbank, emb.to(cuda), init.to(cuda), candt.to(cuda), probst.to(cuda), topk, T,
                                          maxref, debug=True)
    torch.cuda.synchronize()
    # fp32 summation order differs between torch.cdist and the kernel: compare selections only where the
    # oracle's own decision margins are above that noise (and require that this is nearly everywhere)
    pair_ok = info["proto_gap"] > 2e-4
    row_ok = pair_ok.all(axis=1) & (info["margin"] > 1e-4)
    assert pair_ok.mean() > 0.95 and row_ok.mean() > 0.8
    assert np.array_equal(dbg["best_proto"].cpu().numpy()[pair_ok], info["best_proto"][pair_ok])
    np.testing.assert_allclose(dbg["best_logit"].cpu().numpy(), info["best_logit"], rtol=5e-5)
    assert np.array_equal(dbg["best_lnglat"].cpu().numpy()[pair_ok], info["best_lnglat"][pair_ok])
    assert np.array_equal(dbg["choice"].cpu().numpy()[row_ok], info["choice"][row_ok])
    assert (info["choice"] != 0).any(), "test data must exercise a refinement that changes the geocell"
    assert torch.equal(ocell.cpu()[row_ok], cell[row_ok])
    assert torch.equal(oll.cpu()[row_ok], ll[row_ok])


@pytest.mark.parametrize("C,P,D,B,kc,topk,members", [(30, 900, 1024, 256, 8, 8, 4.0), (64, 4000, 768, 512, 10, 5, 0.0),
                                                     (20, 150, 128, 3, 4, 4, 3.0)])
def test_refiner_cell_major_equals_query_major(cuda, C, P, D, B, kc, topk, members, monkeypatch):
    """The cell-major scan (pairs counting-sorted by geocell, register-tiled 4 prototypes x 8 queries) and the
    query-major scan (one warp per pair) are two schedules of the same arithmetic: same winners, same outputs."""
    import numpy as np
    from pigeon_b200 import ops, synthetic
    bank = synthetic.synthetic_bank(C, P, D, seed=12, members_mean=members, empty_cells=2)
    cand, probs = synthetic.synthetic_candidates(B, kc, C, seed=13)
    emb = torch.from_numpy(synthetic.synthetic_queries(bank, cand, views=1, seed=14)).to(cuda)
    init = torch.from_numpy(synthetic.synthetic_geocells(B, seed=15)).to(cuda)
    dbank = ops.DeviceBank(cuda, **bank)
    args = (dbank, emb, init, torch.from_numpy(cand).to(cuda), torch.from_numpy(probs).to(cuda), topk, 1.6, 1e6)
    try:
        ops.refiner_set_schedule(1)
        ll_q, cell_q, dq = ops.refiner_forward(*args, debug=True)
        ops.refiner_set_schedule(2)
        ll_c, cell_c, dc = ops.refiner_forward(*args, debug=True)
    finally:
        ops.refiner_set_schedule(0)
    torch.cuda.synchronize()
    # identical winners except where two prototypes tie to within fp32 summation-order noise
    same = (dq["best_proto"] == dc["best_proto"])
    assert same.float().mean() > 0.995
    assert torch.allclose(dq["best_logit"], dc["best_logit"], rtol=5e-5, atol=1e-5)   # direct differences vs |p|^2+|q|^2-2pq
    assert torch.equal(dq["best_lnglat"][same], dc["best_lnglat"][same])
    rows = same.all(dim=1)
    assert torch.equal(cell_q[rows], cell_c[rows]) and torch.equal(ll_q[rows], ll_c[rows])


@pytest.mark.parametrize("C,P,D,B,kc,topk,members", [
    (30, 900, 1024, 256, 8, 8, 4.0),       # D = 1024: 16 staged queries, 68 pairs per cell -> 5 query passes
    (64, 4000, 768, 512, 10, 5, 0.0),      # 40 pairs per cell -> two passes of 32 + 8, ragged last tiles
    (20, 150, 128, 3, 4, 4, 3.0),          # a handful of pairs, cells smaller than one tile
    (7, 3000, 512, 2000, 3, 3, 0.0),       # 857 pairs per cell (27 passes), 4-stage ring
    (200, 20000, 256, 1500, 6, 5, 2.0),    # more cells than SMs: ranges of several cells, straddling cells merged by atomicMin
    (3, 5000, 768, 40, 2, 2, 0.0),         # fewer cells than SMs: every cell cut across many CTAs
    (12, 9000, 768, 300, 4, 3, 0.0),       # geocells of ~900 prototypes: two 512-prototype CTA tiles each, three query passes
])
@pytest.mark.parametrize("sched", [3, 4])
def test_refiner_tile_scan_equals_cell_major(cuda, C, P, D, B, kc, topk, members, sched):
    """The tile scan (3: persistent CTAs, cp.async.bulk ring, 8-way split of D) and the slab scan (4: TMA-streamed embedding
    chunks, 8 x 8 register tiles), both merging through a packed atomicMin, against the cell-major and query-major schedules:
    same winners wherever two prototypes do not tie within fp32 summation-order noise."""
    from pigeon_b200 import ops, synthetic
    bank = synthetic.synthetic_bank(C, P, D, seed=31, members_mean=members, empty_cells=min(2, C - 1))
    cand, probs = synthetic.synthetic_candidates(B, kc, C, seed=32)
    emb = torch.from_numpy(synthetic.synthetic_queries(bank, cand, views=1, seed=33)).to(cuda)
    init = torch.from_numpy(synthetic.synthetic_geocells(B, seed=34)).to(cuda)
    dbank = ops.DeviceBank(cuda, **bank)
    assert dbank.proto_sqnorm is not None
    ref_norm = (dbank.proto_emb.double() ** 2).sum(1)
    assert torch.allclose(dbank.proto_sqnorm.double(), ref_norm, rtol=1e-6)
    args = (dbank, emb, init, torch.from_numpy(cand).to(cuda), torch.from_numpy(probs).to(cuda), topk, 1.6, 1e6)
    try:
        ops.refiner_set_schedule(1)
        _, _, dq = ops.refiner_forward(*args, debug=True)
        ops.refiner_set_schedule(2)
        ll_c, cell_c, dc = ops.refiner_forward(*args, debug=True)
        ops.refiner_set_schedule(sched)
        ll_t, cell_t, dt = ops.refiner_forward(*args, debug=True)
        ll_t2, cell_t2, dt2 = ops.refiner_forward(*args, debug=True)
    finally:
        ops.refiner_set_schedule(0)
    torch.cuda.synchronize()
    # run to run: the merge is an atomicMin on (d2, prototype), so the result does not depend on arrival order
    assert torch.equal(dt["best_proto"], dt2["best_proto"]) and torch.equal(dt["best_logit"], dt2["best_logit"])
    assert torch.equal(ll_t, ll_t2) and torch.equal(cell_t, cell_t2)
    for other in (dc, dq):
        same = dt["best_proto"] == other["best_proto"]
        assert same.float().mean() > 0.995, same.float().mean()
        assert torch.allclose(dt["best_logit"], other["best_logit"], rtol=5e-5, atol=1e-5)
        assert torch.equal(dt["best_lnglat"][same], other["best_lnglat"][same])
    rows = (dt["best_proto"] == dc["best_proto"]).all(dim=1)
    assert torch.equal(cell_t[rows], cell_c[rows]) and torch.equal(ll_t[rows], ll_c[rows])
    # the winner really is the nearest prototype of its cell (fp64 check on a sample of pairs)
    bp = dt["best_proto"].cpu()
    off = torch.as_tensor(bank["cell_off"])
    pe = dbank.proto_emb.double().cpu()
    q = emb[:, 0].double().cpu()
    for b in range(0, B, max(1, B // 16)):
        for j in range(topk):
            c = int(cand[b, j])
            lo, hi = int(off[c]), int(off[c + 1])
            if hi <= lo:
                assert int(bp[b, j]) == -1
                continue
            d = ((pe[lo:hi] - q[b]) ** 2).sum(1)
            win = int(bp[b, j]) - lo
            assert 0 <= win < hi - lo and d[win] <= d.min() * (1 + 1e-5) + 1e-6


@pytest.mark.parametrize("world,members", [(2, 0.0), (4, 3.0), (8, 0.0)])
def test_refiner_cell_sharded_equals_replicated(cuda, world, members):
    """SURVEY.md 8e-ii on one GPU: scan the same queries against each of `world` cell shards (bank.shard_bank), merge the
    partials by owner (dist.merge_partials_by_owner, what the ranks do after their all-gather), run the final stage:
    every output must equal the replicated bank's, bit for bit (the owner runs the same arithmetic on the same rows)."""
    from pigeon_b200 import bank as bank_mod, dist as pdist, ops, synthetic
    C, P, D, B, kc, topk = 300, 6000, 256, 700, 8, 5
    full = synthetic.synthetic_bank(C, P, D, seed=21, members_mean=members, empty_cells=4)
    cand, probs = synthetic.synthetic_candidates(B, kc, C, seed=22)
    emb = torch.from_numpy(synthetic.synthetic_queries(full, cand, views=1, seed=23)).to(cuda)
    init = torch.from_numpy(synthetic.synthetic_geocells(B, seed=24)).to(cuda)
    candt, probst = torch.from_numpy(cand).to(cuda), torch.from_numpy(probs).to(cuda)
    ll_ref, cell_ref, dbg = ops.refiner_forward(ops.DeviceBank(cuda, **full), emb, init, candt, probst, topk, 1.6, 1e6, debug=True)
    parts_l, parts_ll = [], []
    for r in range(world):
        bl, bll, _ = ops.refiner_scan(ops.DeviceBank(cuda, **bank_mod.shard_bank(full, r, world)), emb, candt, topk)
        parts_l.append(bl)
        parts_ll.append(bll)
    gathered = dict(best_logit=torch.cat(parts_l), best_lnglat=torch.cat(parts_ll))
    merged = pdist.merge_partials_by_owner(gathered, candt[:, :topk], world)
    assert torch.equal(merged["best_logit"], dbg["best_logit"]) and torch.equal(merged["best_lnglat"], dbg["best_lnglat"])
    ll, cell, choice = ops.refiner_finalize(merged["best_logit"], merged["best_lnglat"], init, candt, probst, topk, 1.6, 1e6)
    assert torch.equal(ll, ll_ref) and torch.equal(cell, cell_ref) and torch.equal(choice, dbg["choice"])
