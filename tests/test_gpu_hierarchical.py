"""Hierarchical panorama head on the GPU (pg_view_attn_forward / pg_view_attn_backward behind SuperGuessr(hierarchical=True))
against tests/golden/hierarchical.npz, outputs of the UNMODIFIED reference (tools/make_hierarchical_golden.py), and against the
fp64 oracle of tests/hierarchical_oracle.py.

Bounds.  The projections run the error-compensated split GEMM (fp16 hi/lo operands, fp32 accumulation): each product carries
a relative error of at most 3 * 2^-22 from the split, and the fp32 sum of K terms at most about sqrt(K) * 2^-24 of the sum of
their magnitudes in practice; the per-element bound below is 4x that, relative to sum |a| |w| + |b|.  The attention core is
fp32 arithmetic over 4 keys and a head dimension of hd terms.  The backward is fp32 throughout (CUDA-core GEMMs)."""
import json
import math
import os

import numpy as np
import pytest
import torch

import hierarchical_oracle as ho

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "hierarchical.npz")
U = 2.0 ** -24
GRAD_REL = 6e-3


@pytest.fixture(scope="module")
def gold():
    z = np.load(GOLD, allow_pickle=False)
    return z, json.loads(str(z["meta"]))


def _rel(a, b):
    a = torch.as_tensor(np.asarray(a.detach().cpu() if torch.is_tensor(a) else a), dtype=torch.float64)
    b = torch.as_tensor(np.asarray(b.detach().cpu() if torch.is_tensor(b) else b), dtype=torch.float64)
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _model(z, cuda, E, seed, base_model=None, **kw):
    """torch.manual_seed(seed); SuperGuessr(...) then the synthetic self_attn / cell_layer weights, as the generator did."""
    from pigeon_b200 import SuperGuessr
    torch.manual_seed(seed)
    sg = SuperGuessr(base_model, panorama=True, hierarchical=True, embed_dim=E, num_candidates=5, geocells=z["centroids"],
                     **kw)
    with torch.no_grad():
        for k, v in ho.synthetic_params(E, 1000, seed).items():
            sg.state_dict()[k].copy_(v)
    return sg.to(cuda)


def _no_dropout(sg):
    sg.pos_encoder.dropout.p = 0.0
    sg.self_attn.dropout = 0.0


def _gemm_bound(a_abs, w_abs, b_abs, K):
    return 4 * (3 * 4 * U + math.sqrt(K) * U) * (a_abs @ w_abs.t() + b_abs) + 1e-30


# ------------------------------------------------------------------------------------------------ evaluation vs reference
@pytest.mark.parametrize("name", ["eval_a", "eval_b", "eval_c", "serve"])
def test_eval_matches_reference_golden(cuda, gold, name):
    z, meta = gold
    case = meta["cases"][name]
    E, N, seed = case["E"], case["N"], int(z[f"{name}_seed"])
    sg = _model(z, cuda, E, seed, should_smooth_labels=case["smooth"], multi_task=case["mt"], serving=case["serving"]).eval()
    emb = ho.embeddings(N, E, seed)
    labels, labels_clf, lmt, lcl, lmo = ho.labels(N, seed)
    kw = dict(labels_multi_task=lmt, labels_climate=lcl, labels_month=lmo) if case["mt"] else {}
    o = sg(embedding=emb, labels=labels, labels_clf=labels_clf, **kw)
    assert (z[f"{name}_margin"] > meta["margin"]).all()            # every sample is decided by more than the fp32 budget
    topk, pred_llh, embedding = (o[1], o[0], o[-1]) if case["serving"] else (o.top5_geocells, o.preds_LLH, o.embedding)
    assert np.array_equal(topk.indices.cpu().numpy(), z[f"{name}_topk_idx"])
    assert np.array_equal(pred_llh.cpu().numpy(), z[f"{name}_preds_LLH"])
    np.testing.assert_allclose(topk.values.cpu().numpy(), z[f"{name}_topk_val"], rtol=2e-5)
    assert torch.equal(embedding.cpu(), emb)                          # the un-averaged [N, 4, E] input comes back
    if case["mt"]:
        np.testing.assert_allclose((o[2] if case["serving"] else o.preds_mt).cpu().numpy(), z[f"{name}_preds_mt"],
                                   rtol=1e-4, atol=1e-5)
    if case["serving"]:
        return
    assert np.array_equal(o.preds_geocell.cpu().numpy(), z[f"{name}_preds_geocell"])
    np.testing.assert_allclose(o.loss.item(), z[f"{name}_loss"], rtol=2e-5)
    np.testing.assert_allclose(o.loss_clf.item(), z[f"{name}_loss_clf"], rtol=2e-5)
    assert sg.last_pooled is None                                     # the refiner averages the raw views itself


def test_positional_encoding_limit_raises(cuda, gold):
    from pigeon_b200 import PigeonB200Error
    z, _ = gold
    sg = _model(z, cuda, 64, 1).eval()
    sg(embedding=torch.randn(1000, 4, 64), labels_clf=torch.zeros(1000, dtype=torch.long))
    with pytest.raises(PigeonB200Error, match="positional-encoding rows"):
        sg(embedding=torch.randn(1001, 4, 64), labels_clf=torch.zeros(1001, dtype=torch.long))


# ------------------------------------------------------------------------------------------------ kernels per element
def _core_sizes():
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    # the core kernels cap their grid at 4 blocks of 8 warps per SM, one warp per (sample, head): past 2 * SMs samples
    # every warp loops; the positional-encoding kernel caps at 8 blocks of 256 threads per SM, 4 elements per thread
    return [7, 2 * sms + 37]


@pytest.mark.parametrize("E", [128, 256, 1024])
@pytest.mark.parametrize("N", _core_sizes())
def test_view_attention_forward_per_element(cuda, N, E):
    """Every stage against fp64 recomputed from the kernel's own saved inputs to that stage, dropout on (masks read back)."""
    from pigeon_b200 import ops
    from pigeon_b200.super_guessr import PositionalEncoder
    p = {k: v.to(cuda) for k, v in ho.synthetic_params(E, 8, N + E).items()}
    pe = PositionalEncoder(E).pos_encoding.to(cuda)
    emb = ho.embeddings(N, E, N).to(cuda)
    n0 = 1000 - N if N < 1000 else 0
    a = ops.view_attention_forward(emb, pe, ops.head_pack_weight(p[ho.ATTN_KEYS[0]]), p[ho.ATTN_KEYS[1]],
                                   ops.head_pack_weight(p[ho.ATTN_KEYS[2]]), p[ho.ATTN_KEYS[3]], 16, n0, 0.1, 0.1, 1234, 99,
                                   return_masks=True)
    s = {k: v.double() for k, v in ops.view_attention_saved(a["saved"], N, E).items()}
    mx, mp = a["mask_x"], a["mask_p"]
    hd = E // 16
    # x = (emb + pe) * keep * fl(1 / 0.9): three fp32 roundings
    x_ref = (emb.double() + pe[n0:n0 + N].double()) * mx.double() / 0.9
    assert ((s["x"] - x_ref).abs() <= 4 * U * x_ref.abs() + 1e-30).all()
    # projections from the saved x
    W = {k: v.double() for k, v in p.items()}
    wq, wk, wv = W[ho.ATTN_KEYS[0]].split(E)
    bq, bk, bv = W[ho.ATTN_KEYS[1]].split(E)
    for got, xin, w, b in ((s["q0"], s["x"][:, 0], wq, bq), (s["k"], s["x"], wk, bk), (s["v"], s["x"], wv, bv)):
        ref = xin @ w.t() + b
        assert ((got - ref).abs() <= _gemm_bound(xin.abs(), w.abs(), b.abs(), 3 * E)).all()
    # scores, softmax and P.v from the saved q0, k, v
    q, k, v = s["q0"].view(N, 16, hd), s["k"].reshape(N, 4, 16, hd), s["v"].reshape(N, 4, 16, hd)
    sc = torch.einsum("nhd,njhd->nhj", q, k) / math.sqrt(hd)
    ds = (hd + 2) * U * torch.einsum("nhd,njhd->nhj", q.abs(), k.abs()).amax(-1, keepdim=True) / math.sqrt(hd)
    P = torch.softmax(sc, -1)
    assert ((s["probs"] - P).abs() <= 2 * ds * P + 8 * U).all()
    pd = s["probs"] * mp.double() / 0.9
    o_ref = torch.einsum("nhj,njhd->nhd", pd, v).reshape(N, E)
    o_bound = 8 * U * torch.einsum("nhj,njhd->nhd", pd.abs(), v.abs()).reshape(N, E) + 1e-30
    assert ((s["o"] - o_ref).abs() <= o_bound).all()
    cls_ref = s["o"] @ W[ho.ATTN_KEYS[2]].t() + W[ho.ATTN_KEYS[3]]
    assert ((a["cls"].double() - cls_ref).abs() <=
            _gemm_bound(s["o"].abs(), W[ho.ATTN_KEYS[2]].abs(), W[ho.ATTN_KEYS[3]].abs(), 3 * E)).all()
    # and end to end against the oracle with the same masks
    ref = ho.attention(emb.double(), pe.double(), *[W[k] for k in ho.ATTN_KEYS], mask_x=mx, mask_p=mp, p_x=0.1, p_attn=0.1,
                       n0=n0)
    assert _rel(a["cls"], ref["cls"]) < 1e-5


@pytest.mark.parametrize("E", [128, 256, 1024])
@pytest.mark.parametrize("N", _core_sizes())
def test_view_attention_backward_per_element(cuda, N, E):
    """dcls -> d weights, d biases, d emb against fp64 autograd through the oracle with the kernel's masks.  Each gradient
    element is a sum over samples and views of fp32 products: bounded by 16 (K + 8) 2^-24 times the same sum over |terms|,
    which autograd gives by running the backward on absolute values."""
    from pigeon_b200 import ops
    from pigeon_b200.super_guessr import PositionalEncoder
    p = {k: v.to(cuda) for k, v in ho.synthetic_params(E, 8, N + E + 1).items()}
    pe = PositionalEncoder(E).pos_encoding.to(cuda)
    emb = ho.embeddings(N, E, N + 1).to(cuda)
    a = ops.view_attention_forward(emb, pe, ops.head_pack_weight(p[ho.ATTN_KEYS[0]]), p[ho.ATTN_KEYS[1]],
                                   ops.head_pack_weight(p[ho.ATTN_KEYS[2]]), p[ho.ATTN_KEYS[3]], 16, 0, 0.1, 0.1, 77, 5,
                                   return_masks=True)
    dcls = torch.randn(N, E, generator=torch.Generator().manual_seed(N)).to(cuda) * 0.01
    grads = [torch.full_like(p[k], 0.5) for k in ho.ATTN_KEYS]                   # accumulate adds onto these
    demb = ops.view_attention_backward(dcls, a["saved"], p[ho.ATTN_KEYS[0]], p[ho.ATTN_KEYS[2]], 16, 0, 0.1, 0.1, 77, 5,
                                       grads=grads, accumulate=True)
    W = [p[k].double().requires_grad_(True) for k in ho.ATTN_KEYS]
    e64 = emb.double().requires_grad_(True)
    ref = ho.attention(e64, pe.double(), *W, mask_x=a["mask_x"], mask_p=a["mask_p"], p_x=0.1, p_attn=0.1)
    ref["cls"].backward(dcls.double())
    K = 4 * N + 3 * E
    for got, want in zip([demb] + [g - 0.5 for g in grads], [e64.grad] + [w.grad for w in W]):
        scale = want.abs().amax().item()
        err = (got.double() - want).abs()
        assert (err <= 16 * (K + 8) * U * scale + 1e-4 * want.abs()).all(), (err.max().item(), scale)
        assert _rel(got, want) < 1e-4


# ------------------------------------------------------------------------------------------------ training vs reference
def test_gradients_match_reference_golden(cuda, gold):
    z, meta = gold
    seed, E, N = int(z["grad_seed"]), 128, 24
    sg = _model(z, cuda, E, seed, should_smooth_labels=True, multi_task=True).train()
    _no_dropout(sg)
    labels, labels_clf, lmt, lcl, lmo = ho.labels(N, seed)
    emb = ho.embeddings(N, E, seed)
    o = sg(embedding=emb, labels=labels, labels_clf=labels_clf, labels_multi_task=lmt, labels_climate=lcl, labels_month=lmo)
    np.testing.assert_allclose(o.loss.item(), z["grad_loss"], rtol=1e-5)
    st = dict(sg._attn_state)
    sg.backward(o.loss)
    for k, prm in sg.named_parameters():
        if "grad/" + k in z.files:
            assert prm.grad is not None, k
            got = ho.sample(prm.grad.cpu())
            assert _rel(got, z["grad/" + k]) < GRAD_REL, (k, _rel(got, z["grad/" + k]))
    # d embedding: d loss / d cls from fp64 autograd, then the kernel backward
    heads = {n: (getattr(sg, n).weight.detach().double().cpu(), getattr(sg, n).bias.detach().double().cpu())
             for n in ("multi_task_head", "climate_layer", "month_layer")}
    pp = {k: v.double() for k, v in ho.synthetic_params(E, 1000, seed).items()}
    cls = ho.attention(emb.double(), sg.pos_encoder.pos_encoding.detach().double().cpu(),
                       *[pp[k] for k in ho.ATTN_KEYS])["cls"].detach().requires_grad_(True)
    logits = torch.nn.functional.linear(cls, pp["cell_layer.weight"], pp["cell_layer.bias"])
    loss = ho.classification_loss(logits, torch.tensor(z["centroids"]), labels, labels_clf, smooth=True) + \
        ho.multi_task_loss(cls, heads, lmt, lcl, lmo)
    loss.backward()
    from pigeon_b200 import ops
    demb = ops.view_attention_backward(cls.grad.float().to(cuda), st["saved"], sg.self_attn.in_proj_weight,
                                       sg.self_attn.out_proj.weight)
    assert _rel(ho.sample(demb.cpu()), z["grad/embedding"]) < GRAD_REL


def test_adamw_trajectory_matches_reference_golden(cuda, gold):
    """3 optimizer steps: the packed fp16 copies of in_proj / out_proj must follow every step (a stale copy would leave the
    second and third losses on the first step's weights)."""
    from pigeon_b200.training import AdamW
    z, meta = gold
    seed, E, N, steps, lr = int(z["adam_seed"]), 128, 24, int(z["adam_steps"]), float(z["adam_lr"])
    sg = _model(z, cuda, E, seed).train()
    _no_dropout(sg)
    opt = AdamW(sg.parameters(), lr=lr)
    for i in range(steps):
        _, labels_clf, *_ = ho.labels(N, seed + i)
        o = sg(embedding=ho.embeddings(N, E, seed + i), labels_clf=labels_clf)
        np.testing.assert_allclose(o.loss.item(), z["adam_losses"][i], rtol=1e-5)
        sg.backward(o.loss)
        opt.step()
        opt.zero_grad()
    sd = sg.state_dict()
    for k in ho.ATTN_KEYS + ("cell_layer.weight", "cell_layer.bias"):
        got, want = ho.sample(sd[k].double().cpu()), torch.from_numpy(z["adam/" + k]).double()
        if k == "self_attn.in_proj_bias":
            # the key bias has an exactly-zero gradient (the softmax cancels it): both runs step on rounding noise, which
            # AdamW turns into steps of up to lr
            assert (got[E:2 * E] - want[E:2 * E]).abs().max().item() <= 2 * steps * lr * 1.001
            got, want = torch.cat([got[:E], got[2 * E:]]), torch.cat([want[:E], want[2 * E:]])
        assert _rel(got, want) < 1e-4, (k, _rel(got, want))


# ------------------------------------------------------------------------------------------------ dropout
def _dropout_model(z, cuda):
    return _model(z, cuda, 128, 9, should_smooth_labels=True, multi_task=True).train()


def _train_once(sg, seed):
    labels, labels_clf, lmt, lcl, lmo = ho.labels(24, 9)
    torch.manual_seed(seed)
    o = sg(embedding=ho.embeddings(24, 128, 9), labels=labels, labels_clf=labels_clf, labels_multi_task=lmt,
           labels_climate=lcl, labels_month=lmo)
    sg.backward(o.loss)
    grads = {k: p.grad.clone() for k, p in sg.named_parameters() if p.grad is not None}
    for p in sg.parameters():
        p.grad = None
    return o, grads


def test_dropout_same_seed_is_bit_identical_and_another_differs(cuda, gold):
    z, _ = gold
    sg = _dropout_model(z, cuda)
    o1, g1 = _train_once(sg, 1)
    o2, g2 = _train_once(sg, 1)
    o3, g3 = _train_once(sg, 2)
    assert torch.equal(o1.loss, o2.loss) and torch.equal(o1.top5_geocells.values, o2.top5_geocells.values)
    assert g1.keys() == g2.keys() and all(torch.equal(g1[k], g2[k]) for k in g1)
    assert not torch.equal(g1["self_attn.in_proj_weight"], g3["self_attn.in_proj_weight"])


def test_dropout_keep_rate(cuda):
    """1.024e6 positional-encoding draws and 64000 attention draws at p = 0.1: keep rate within 5 sigma of 0.9."""
    from pigeon_b200 import ops
    from pigeon_b200.super_guessr import PositionalEncoder
    E, N = 256, 1000
    p = {k: v.to(cuda) for k, v in ho.synthetic_params(E, 8, 3).items()}
    a = ops.view_attention_forward(ho.embeddings(N, E, 3).to(cuda), PositionalEncoder(E).pos_encoding.to(cuda),
                                   ops.head_pack_weight(p[ho.ATTN_KEYS[0]]), p[ho.ATTN_KEYS[1]],
                                   ops.head_pack_weight(p[ho.ATTN_KEYS[2]]), p[ho.ATTN_KEYS[3]], 16, 0, 0.1, 0.1,
                                   *torch.randint(0, 2 ** 62, (2,)).tolist(), return_masks=True)
    for m in (a["mask_x"], a["mask_p"]):
        n = m.numel()
        assert abs(m.double().mean().item() - 0.9) <= 5 * math.sqrt(0.9 * 0.1 / n), (n, m.double().mean().item())
    assert a["mask_x"].numel() >= 10 ** 6


def test_dropout_gradients_match_fp64_autograd_with_the_returned_masks(cuda, gold):
    from pigeon_b200 import ops
    z, _ = gold
    sg = _dropout_model(z, cuda)
    labels, labels_clf, lmt, lcl, lmo = ho.labels(24, 9)
    torch.manual_seed(3)
    o = sg(embedding=ho.embeddings(24, 128, 9), labels=labels, labels_clf=labels_clf, labels_multi_task=lmt,
           labels_climate=lcl, labels_month=lmo)
    st = dict(sg._attn_state)
    sg.backward(o.loss)
    assert st["p_x"] == 0.1 and st["p_attn"] == 0.1
    # the masks of that forward, read back by re-running the kernel with its seed and offset
    w_in3, w_out3 = sg._packed_attn()
    sa = sg.self_attn
    emb = ho.embeddings(24, 128, 9)
    m = ops.view_attention_forward(emb.to(cuda), sg.pos_encoder.pos_encoding.detach(), w_in3, sa.in_proj_bias.detach(),
                                   w_out3, sa.out_proj.bias.detach(), 16, 0, 0.1, 0.1, st["seed"], st["offset"],
                                   return_masks=True)
    assert torch.equal(m["saved"], st["saved"])
    P = {k: v.detach().double().cpu().requires_grad_(True) for k, v in sg.state_dict().items()
         if k.startswith(("self_attn.", "cell_layer.", "multi_task_head.", "climate_layer.", "month_layer."))}
    a = ho.attention(emb.double(), sg.pos_encoder.pos_encoding.detach().double().cpu(), *[P[k] for k in ho.ATTN_KEYS],
                     mask_x=m["mask_x"].cpu(), mask_p=m["mask_p"].cpu(), p_x=0.1, p_attn=0.1)
    logits = torch.nn.functional.linear(a["cls"], P["cell_layer.weight"], P["cell_layer.bias"])
    heads = {n: (P[n + ".weight"], P[n + ".bias"]) for n in ("multi_task_head", "climate_layer", "month_layer")}
    loss = ho.classification_loss(logits, torch.tensor(z["centroids"]), labels, labels_clf, smooth=True) + \
        ho.multi_task_loss(a["cls"], heads, lmt, lcl, lmo)
    loss.backward()
    np.testing.assert_allclose(o.loss.item(), loss.item(), rtol=1e-5)
    for k, prm in sg.named_parameters():
        if k in P:
            assert _rel(prm.grad, P[k].grad) < 1e-4, (k, _rel(prm.grad, P[k].grad))


# ------------------------------------------------------------------------------------------------ through the tower
def _tower_model(z, cuda):
    from pigeon_b200 import CLIPVisionTower, VitDims, synthetic
    meta = json.loads(str(z["tower_meta"]))
    dims = VitDims(**meta["dims"])
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=meta["seed"], std=meta["std"]))
    sg = _model(z, cuda, dims.hidden, meta["seed"], base_model=tower, should_smooth_labels=True).train()
    _no_dropout(sg)
    for p in sg.parameters():
        p.requires_grad_(p.dtype == torch.float32)
    sg.lla_geocells.requires_grad_(False)
    sg.pos_encoder.pos_encoding.requires_grad_(False)
    px = torch.randn(meta["N"], 12, 336, 336, generator=torch.Generator().manual_seed(meta["seed"] + 1))
    return sg, px, meta


def _tower_step(sg, px, meta):
    labels, labels_clf, *_ = ho.labels(meta["N"], meta["seed"])
    o = sg(pixel_values=px, labels=labels, labels_clf=labels_clf)
    sg.backward(o.loss)
    return o, {k: p.grad.detach().clone() for k, p in sg.named_parameters() if p.grad is not None}


def test_tower_gradients_match_reference_and_chunking_keeps_the_positional_rows(cuda, gold):
    """The tower's backward GEMMs take bf16 operands (tests/test_gpu_train_tower.py): per-tensor relative error <= 3e-2.
    max_train_views = 4 runs one panorama per chunk; the PE row must still be the sample's index in the whole batch."""
    z, _ = gold
    sg, px, meta = _tower_model(z, cuda)
    o, grads = _tower_step(sg, px, meta)
    np.testing.assert_allclose(float(o.loss), float(z["tower_loss"]), rtol=1e-3)
    assert sg.last_pooled is None
    for key, g in grads.items():
        assert "tower_sub/" + key in z.files, key
        got = ho.sample(g.double().cpu())
        ref = torch.from_numpy(z["tower_sub/" + key]).double()
        if float(z["tower_norm/" + key]) < 1e-9:
            continue
        assert _rel(got, ref) < 3e-2, (key, _rel(got, ref))
    assert set("tower_sub/" + k for k in grads) == {k for k in z.files if k.startswith("tower_sub/")}
    sg2, _, _ = _tower_model(z, cuda)
    sg2.max_train_views = 4
    o2, grads2 = _tower_step(sg2, px, meta)
    np.testing.assert_allclose(float(o2.loss), float(o.loss), rtol=1e-5)
    for key, g in grads.items():
        assert _rel(grads2[key], g) < 1e-4, (key, _rel(grads2[key], g))


# ------------------------------------------------------------------------------------------------ integration
def test_evaluate_model_refines_the_raw_views(cuda, gold):
    """evaluation.predict_batch hands `last_pooled` to the refiner when it is set; for the hierarchical head it is None, so the
    refiner averages the raw views, as the reference's refiner does (proto_refiner.py:138-139)."""
    from pigeon_b200 import ProtoRefiner, synthetic
    from pigeon_b200.loops import evaluate_model
    z, _ = gold
    E, n, C = 128, 37, 1000
    sg = _model(z, cuda, E, 11).eval()
    bank = synthetic.synthetic_bank(C, 3000, E, seed=4, members_mean=2.0, empty_cells=3)
    ref = ProtoRefiner(topk=5, max_refinement=1e6, temperature=1.6, protos=bank).eval()
    emb = ho.embeddings(n, E, 12)
    labels, labels_clf, *_ = ho.labels(n, 12)

    class DS(torch.utils.data.Dataset):
        def __len__(self):
            return n

        def __getitem__(self, i):
            if isinstance(i, str):
                return {"labels": labels.numpy(), "labels_clf": labels_clf.numpy()}[i]
            return dict(embedding=emb[i], labels=labels[i], labels_clf=labels_clf[i])

    class Args:
        per_device_eval_batch_size = 16

    res = evaluate_model(sg, DS(), None, Args(), ref)
    # batch by batch: a sample's positional-encoding row is its index within its batch (the reference's quirk)
    lls, cells = [], []
    for lo in range(0, n, Args.per_device_eval_batch_size):
        sl = slice(lo, lo + Args.per_device_eval_batch_size)
        out = sg(embedding=emb[sl], labels=labels[sl], labels_clf=labels_clf[sl])
        _, ll, _ = ref(out.embedding, initial_preds=out.preds_LLH, candidate_cells=out.top5_geocells.indices,
                       candidate_probs=out.top5_geocells.values)
        lls.append(ll.cpu().numpy())
        cells.append(out.preds_geocell.cpu().numpy())
    assert np.array_equal(res["preds"], np.concatenate(lls))
    assert np.array_equal(res["preds_geocell"], np.concatenate(cells))


def test_hierarchical_without_panorama_is_the_single_image_head(cuda, gold):
    from pigeon_b200 import SuperGuessr
    z, _ = gold
    E, N = 128, 10
    models = []
    for hier in (True, False):
        torch.manual_seed(0)
        sg = SuperGuessr(None, panorama=False, hierarchical=hier, embed_dim=E, num_candidates=5, geocells=z["centroids"])
        w = ho.synthetic_params(E, 1000, 1)
        with torch.no_grad():                            # the attention's init draws shift cell_layer's: set it explicitly
            sg.cell_layer.weight.copy_(w["cell_layer.weight"])
            sg.cell_layer.bias.copy_(w["cell_layer.bias"])
        models.append(sg.to(cuda))
    assert hasattr(models[0], "self_attn") and not hasattr(models[1], "self_attn")
    emb = ho.embeddings(N, E, 2)
    _, labels_clf, *_ = ho.labels(N, 2)
    outs = []
    for sg in models:
        sg.eval()
        e = sg(embedding=emb, labels_clf=labels_clf)
        sg.train()
        t = sg(embedding=emb, labels_clf=labels_clf)
        sg.backward(t.loss)
        outs.append((e, t, sg.cell_layer.weight.grad.clone(), sg.cell_layer.bias.grad.clone()))
    (e1, t1, gw1, gb1), (e2, t2, gw2, gb2) = outs
    assert torch.equal(e1.top5_geocells.values, e2.top5_geocells.values) and torch.equal(e1.loss, e2.loss)
    assert torch.equal(t1.loss, t2.loss) and torch.equal(gw1, gw2) and torch.equal(gb1, gb2)
    assert all(p.grad is None for p in models[0].self_attn.parameters())
