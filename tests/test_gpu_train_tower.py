"""Fine-tune step through the vision tower (N1): backward kernels one by one against torch autograd in fp32, then the
whole tower backward and the SuperGuessr training forward against tests/golden/train_tower_*.npz — gradients the
UNMODIFIED reference model produced under torch autograd (oracle/make_golden.py).

Tolerance: the backward runs its GEMMs with bf16 operands (8-bit mantissa) and fp32 accumulation, the reference is fp32:
per-tensor relative L2 error <= 3e-2 (typically 3e-3 .. 1e-2), cosine >= 0.999."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
REL = 3e-2


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _lib():
    from pigeon_b200._lib import check, current_stream_ptr, load, ptr
    return load(), check, ptr, current_stream_ptr


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------------ building blocks
@pytest.mark.parametrize("M,N,K", [(300, 512, 200), (1000, 256, 2308), (256, 640, 1152), (4096, 1024, 577)])
def test_gemm_bf16_operands(cuda, M, N, K):
    lib, check, ptr, sp = _lib()
    g = torch.Generator().manual_seed(M + N)
    Kp = (K + 7) // 8 * 8
    a = torch.zeros(M, Kp, device=cuda, dtype=torch.bfloat16)
    w = torch.zeros(N, Kp, device=cuda, dtype=torch.bfloat16)
    a[:, :K] = (torch.randn(M, K, generator=g) * 1e-4).to(cuda, torch.bfloat16)          # gradient-sized values
    w[:, :K] = (torch.randn(N, K, generator=g) * 0.05).to(cuda, torch.bfloat16)
    a[:, K:] = 7.0                                                                         # must not be read (TMA extent = K)
    out = torch.full((M, N), float("nan"), device=cuda)
    check(lib.pg_gemm_ex(ptr(a), Kp, ptr(w), Kp, ptr(out), N, None, None, M, N, K, 3, 1, sp()), "pg_gemm_ex")
    ref = a[:, :K].double() @ w[:, :K].double().t()
    assert _rel(out, ref) < 1e-5
    # accumulate into an existing buffer from a separate residual source (out-of-place residual epilogue)
    resid = torch.randn(M, N, generator=g).to(cuda) * 1e-4
    out2 = torch.zeros(M, N, device=cuda)
    check(lib.pg_gemm_ex(ptr(a), Kp, ptr(w), Kp, ptr(out2), N, None, ptr(resid), M, N, K, 2, 1, sp()), "pg_gemm_ex")
    assert _rel(out2, ref + resid.double()) < 1e-5


def test_transpose_and_dgelu(cuda):
    lib, check, ptr, sp = _lib()
    g = torch.Generator().manual_seed(1)
    for dt, code in ((torch.float32, 0), (torch.float16, 1), (torch.bfloat16, 2)):
        src = torch.randn(577, 200, generator=g).to(cuda, dt)
        out = torch.zeros(200, 584, device=cuda, dtype=torch.bfloat16)
        check(lib.pg_transpose_to_bf16(ptr(src), code, 200, ptr(out), 584, 577, 200, sp()), "pg_transpose_to_bf16")
        assert torch.equal(out[:, :577], src.float().t().to(torch.bfloat16))
    u = (torch.randn(1000, 512, generator=g) * 3).to(cuda, torch.float16)
    dh = torch.randn(1000, 512, generator=g).to(cuda) * 1e-3
    du = torch.empty(1000, 512, device=cuda, dtype=torch.bfloat16)
    check(lib.pg_dgelu_bf16(ptr(dh), ptr(u), ptr(du), u.numel(), sp()), "pg_dgelu_bf16")
    x = u.float().requires_grad_(True)
    (x * torch.sigmoid(1.702 * x)).backward(dh)
    assert _rel(du.float(), x.grad) < 4e-3                                                 # bf16 rounding of the output


@pytest.mark.parametrize("code", [0, 1, 2])
def test_transpose_ragged_shapes_odd_strides_unaligned_source(cuda, code):
    """Rows and columns of 1, 63, 65, 577 x 4097 (partial 64 x 64 tiles), odd lds / ldo (no paired loads or stores) and a
    source one element off its pair alignment (the unpaired load path): bf16(src^T) bit for bit, nothing written outside."""
    lib, check, ptr, sp = _lib()
    dt = (torch.float32, torch.float16, torch.bfloat16)[code]
    g = torch.Generator().manual_seed(code)
    for rows in (1, 63, 65, 577):
        for cols in (1, 63, 65, 4097):
            for odd in (True, False):
                lds = cols + (1 - cols % 2 if odd else cols % 2)      # odd, or even with the source offset by one element
                ldo = rows + (1 - rows % 2 if odd else rows % 2)
                base = torch.randn(rows * lds + 1, generator=g).to(cuda, dt)
                src = base[0 if odd else 1:][:rows * lds].view(rows, lds)
                out = torch.full((cols + 1, ldo), float("nan"), device=cuda, dtype=torch.bfloat16)
                check(lib.pg_transpose_to_bf16(src.data_ptr(), code, lds, ptr(out), ldo, rows, cols, sp()),
                      "pg_transpose_to_bf16")
                ref = src[:, :cols].float().t().to(torch.bfloat16)
                assert torch.equal(out[:cols, :rows].view(torch.int16), ref.view(torch.int16)), (rows, cols, odd)
                assert torch.isnan(out[:cols, rows:].float()).all() and torch.isnan(out[cols:].float()).all()


@pytest.mark.parametrize("n_views,seq,heads", [(2, 17, 4), (3, 257, 2), (2, 577, 16), (1, 128, 2), (1, 64, 2)])
def test_attention_backward_matches_autograd(cuda, n_views, seq, heads):
    lib, check, ptr, sp = _lib()
    hidden = heads * 64
    rows = n_views * seq
    g = torch.Generator().manual_seed(seq)
    qkv = (torch.randn(rows, 3 * hidden, generator=g) * 0.8).to(cuda, torch.float16)
    d_out = (torch.randn(rows, hidden, generator=g) * 1e-5).to(cuda)                      # far below fp16's normal range
    out = torch.empty(rows, hidden, device=cuda, dtype=torch.float16)
    lse2 = torch.empty(n_views * heads, seq, device=cuda)
    check(lib.pg_attention_f16_lse(ptr(qkv), ptr(out), ptr(lse2), n_views, seq, heads, sp()), "pg_attention_f16_lse")
    # fp32 reference of the same op on the same fp16 inputs
    t = qkv.float().reshape(n_views, seq, 3, heads, 64).permute(2, 0, 3, 1, 4)            # [3, v, h, s, d]
    q, k, v = (x.clone().requires_grad_(True) for x in t)
    s = (q @ k.transpose(-1, -2)) * 0.125
    o = torch.softmax(s, dim=-1) @ v
    ref_lse2 = torch.logsumexp(s, dim=-1) * 1.4426950408889634
    assert (lse2.reshape(n_views, heads, seq) - ref_lse2).abs().max().item() < 2e-3
    o.backward(d_out.reshape(n_views, seq, heads, 64).permute(0, 2, 1, 3))
    ref = torch.stack([q.grad, k.grad, v.grad]).permute(1, 3, 0, 2, 4).reshape(rows, 3 * hidden)
    dqkv = torch.full((rows, 3 * hidden), float("nan"), device=cuda, dtype=torch.bfloat16)
    need = lib.pg_attention_backward_workspace_bytes(n_views, seq, heads)
    from pigeon_b200.vit_train import _aligned_empty
    ws = _aligned_empty(need, cuda)
    check(lib.pg_attention_backward(ptr(qkv), ptr(out), ptr(d_out), ptr(lse2), ptr(dqkv), n_views, seq, heads, ptr(ws),
                                    need, sp()), "pg_attention_backward")
    got = dqkv.float()
    assert torch.isfinite(got).all()
    for i, name in enumerate("qkv"):
        a, b = got[:, i * hidden:(i + 1) * hidden], ref[:, i * hidden:(i + 1) * hidden]
        assert _rel(a, b) < 1.5e-2, (name, _rel(a, b))


# ------------------------------------------------------------------------------------------------ whole tower vs the reference
def _load(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    return z, json.loads(str(z["meta"]))


def _model(meta, z, cuda):
    from pigeon_b200 import CLIPVisionTower, SuperGuessr, VitDims, synthetic
    dims = VitDims(**meta["dims"])
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=meta["sd_seed"], std=meta["std"]), strict=True)
    sg = SuperGuessr(tower, panorama=False, should_smooth_labels=True, num_candidates=5, geocells=z["centroids"]).to(cuda)
    g = torch.Generator().manual_seed(meta["w_seed"])
    with torch.no_grad():
        sg.cell_layer.weight.copy_(torch.randn(meta["C"], dims.hidden, generator=g) * 0.03)
        sg.cell_layer.bias.copy_(torch.randn(meta["C"], generator=g) * 0.01)
    gp = torch.Generator().manual_seed(meta["px_seed"])
    px = torch.randn(meta["n_views"], 3, dims.image_size, dims.image_size, generator=gp)
    return sg, px, dims


def _check_grads(sg, z, meta, expect_names=None):
    stride, worst = meta["stride"], {}
    scale = max(float(z[k]) for k in z.files if k.startswith("norm/"))
    for name, p in sg.named_parameters():
        key = name.replace("base_model.", "")
        if "sub/" + key not in z.files:
            continue
        if expect_names is not None and not expect_names(key):
            assert p.grad is None, f"{key} should be frozen"
            continue
        assert p.grad is not None, key
        got = p.grad.detach().reshape(-1).double().cpu()[::stride]
        ref = torch.from_numpy(z["sub/" + key]).double()
        norm = float(z["norm/" + key])
        err = (got - ref).norm().item() / max(ref.norm().item(), 1e-30)
        if norm < 1e-6 * scale:                       # k_proj.bias: mathematically zero gradient
            assert got.norm().item() < 1e-3 * scale, key
            continue
        worst[key] = err
        assert err < REL, (key, err)
        cos = torch.dot(got, ref).item() / (got.norm().item() * ref.norm().item())
        assert cos > 0.999, (key, cos)
    return worst


@pytest.mark.parametrize("name", ["train_tower_small", "train_tower_mid"])
def test_tower_backward_matches_reference_autograd(cuda, name):
    z, meta = _load(name)
    sg, px, dims = _model(meta, z, cuda)
    sg.train()
    sg.max_train_views = 4                                     # forces two chunks for the 6-view fixture
    out = sg(pixel_values=px.to(cuda), labels=torch.tensor(z["labels"]), labels_clf=torch.tensor(z["labels_clf"]))
    np.testing.assert_allclose(float(out.loss), float(z["loss"]), rtol=1e-3)
    sg.backward(out.loss)
    worst = _check_grads(sg, z, meta)
    try:                                   # measured parity, appended to a log; never fails the test
        d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "parity.log"), "a") as f:
            f.write(f"{name}: worst per-tensor relative gradient error {max(worst.values()):.3e} "
                    f"({max(worst, key=worst.get)}), median {float(np.median(list(worst.values()))):.3e}\n")
    except OSError:
        pass


def test_reference_freeze_policy_and_optimizer_step(cuda):
    """models/super_guessr.py:159-160: encoder.layers[:-1] frozen, embeddings + pre_layrnorm + last layer + head train."""
    from pigeon_b200.training import AdamW
    z, meta = _load("train_tower_mid")
    sg, px, dims = _model(meta, z, cuda)
    for p in sg.base_model.vision_model.encoder.layers[:-1].parameters():
        p.requires_grad = False
    sg.train()
    lab, clf = torch.tensor(z["labels"]), torch.tensor(z["labels_clf"])
    opt = AdamW(sg.parameters(), lr=1e-4)
    out = sg(pixel_values=px.to(cuda), labels=lab, labels_clf=clf)
    sg.backward(out.loss)
    last = f"encoder.layers.{dims.layers - 1}."
    _check_grads(sg, z, meta, expect_names=lambda k: ("encoder.layers." not in k) or (last in k))
    before = {n: p.detach().clone() for n, p in sg.named_parameters() if p.grad is not None}
    loss0 = float(out.loss)
    opt.step()
    opt.zero_grad()
    for n, p in sg.named_parameters():
        if n in before:
            assert (p.detach() - before[n]).abs().max().item() > 0, n
    out1 = sg(pixel_values=px.to(cuda), labels=lab, labels_clf=clf)     # repacked fp16 weights are the updated ones
    assert float(out1.loss) < loss0
    sg.backward(out1.loss)
    sg.eval()
    with torch.no_grad():
        ev = sg(pixel_values=px.to(cuda), labels=lab, labels_clf=clf)
    np.testing.assert_allclose(float(ev.loss), float(out1.loss), rtol=1e-4)


def test_data_parallel_gradients_match_full_batch(cuda):
    """2 ranks x half of the golden batch, NCCL gradient averaging == the reference's full-batch gradients."""
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                        "127.0.0.1", "--master-port", "29577", os.path.join(root, "tools", "ddp_train_check.py")],
                       capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]


def test_train_model_loop_with_trainable_tower(cuda):
    """`train_model` (mirror of training/train_eval_loop.py:164-253) end to end on a tiny tower: host pixel batches from a
    DataLoader, gradient accumulation, optimizer steps on tower + head, per-epoch evaluation, best-checkpoint saving."""
    import tempfile
    from pigeon_b200 import CLIPVisionTower, SuperGuessr, VitDims, synthetic
    from pigeon_b200.training import train_model
    dims = VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=2)
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=3, std=0.05), strict=True)
    Cc, n = 12, 16
    sg = SuperGuessr(tower, panorama=False, should_smooth_labels=True, num_candidates=5,
                     geocells=synthetic.synthetic_geocells(Cc, 0)).to(cuda)
    for p in sg.base_model.vision_model.encoder.layers[:-1].parameters():      # reference freeze policy
        p.requires_grad = False
    g = torch.Generator().manual_seed(8)
    px = torch.randn(n, 3, 56, 56, generator=g)
    labels = torch.tensor(synthetic.synthetic_geocells(n, 9))
    labels_clf = torch.randint(0, Cc, (n,), generator=g)

    class DS(torch.utils.data.Dataset):
        def __len__(self):
            return n

        def __getitem__(self, i):
            if isinstance(i, str):
                return {"labels": labels.numpy(), "labels_clf": labels_clf.numpy()}[i]
            return dict(pixel_values=px[i], labels=labels[i], labels_clf=labels_clf[i])

    class Args:
        learning_rate = 1e-3
        per_device_train_batch_size = 4
        per_device_eval_batch_size = 8
        num_train_epochs = 3
        gradient_accumulation_steps = 2

    before = {k: v.detach().clone() for k, v in sg.state_dict().items()}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "best.model")
        out = train_model(sg, {"train": DS(), "val": DS()}, False, False, Args(), None, patience=None, save_path=path)
        assert out is sg and os.path.exists(path)
        saved = torch.load(path, map_location="cpu")
        assert set(saved) == set(before)
    hist = sg.train_history
    assert len(hist) == 3 and all(np.isfinite(hist)) and hist[-1] < hist[0]          # the training loss goes down
    after = sg.state_dict()
    changed = [k for k in before if not torch.equal(before[k], after[k])]
    assert any("encoder.layers.1." in k for k in changed) and any("cell_layer" in k for k in changed)
    assert any("embeddings" in k for k in changed)
    assert not any("encoder.layers.0." in k for k in changed)                        # frozen layer untouched


@pytest.mark.parametrize("M,N,K,bf16", [(512, 512, 640, 1), (1024, 4096, 2308, 1), (3072, 1024, 577, 0), (256, 256, 70, 1)])
def test_gemm_tn_mn_major_operands(cuda, M, N, K, bf16):
    """pg_gemm_tn: D (+)= a^T w with a [K, M], w [K, N] — the weight-gradient product straight from row-major operands."""
    lib, check, ptr, sp = _lib()
    dt = torch.bfloat16 if bf16 else torch.float16
    g = torch.Generator().manual_seed(M + K)
    a = (torch.randn(K, M, generator=g) * 1e-3).to(cuda, dt)
    w = (torch.randn(K, N, generator=g) * 0.3).to(cuda, dt)
    ref = a.double().t() @ w.double()
    out = torch.full((M, N), float("nan"), device=cuda)
    check(lib.pg_gemm_tn(ptr(a), M, ptr(w), N, ptr(out), N, M, N, K, 0, bf16, sp()), "pg_gemm_tn")
    assert _rel(out, ref) < 1e-5
    acc0 = torch.randn(M, N, generator=g).to(cuda) * 1e-3
    out = acc0.clone()
    check(lib.pg_gemm_tn(ptr(a), M, ptr(w), N, ptr(out), N, M, N, K, 1, bf16, sp()), "pg_gemm_tn")
    assert _rel(out, acc0.double() + ref) < 1e-5
    from pigeon_b200 import PigeonB200Error
    with pytest.raises(PigeonB200Error):                       # shapes the MN-major path does not take
        check(lib.pg_gemm_tn(ptr(a), M, ptr(w), N, ptr(out), N, M, 200, K, 0, bf16, sp()), "pg_gemm_tn")


def test_tower_backward_at_real_geometry_vs_oracle(cuda):
    """ViT-L/14-336 (24 layers, 577 tokens, 1024 hidden), 2 views: pg_vit_forward_train / pg_vit_backward against
    oracle/train.tower_gradients (fp32 autograd through the oracle's restated forward, itself pinned to the reference's
    gradients by tests/test_oracle_golden.py).  Every trainable parameter of the tower is compared."""
    import time
    from oracle import train as otrain
    from pigeon_b200 import CLIPVisionTower, VitDims, synthetic
    from pigeon_b200.vit_train import TowerTrainer
    dims = VitDims()
    sd = synthetic.random_vit_state_dict(dims, seed=0)
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(sd, strict=True)
    tower.to(cuda)
    g = torch.Generator().manual_seed(11)
    px = torch.randn(2, 3, 336, 336, generator=g)
    d_emb = torch.randn(2, dims.hidden, generator=g) * 1e-4
    tr = TowerTrainer(tower, max_views=2)
    emb = tr.forward(px.to(cuda).half())
    tr.backward(d_emb.to(cuda))
    tr.finalize(1)
    t0 = time.time()
    ref_emb, ref = otrain.tower_gradients(sd, px.half().float(), d_emb, patch=dims.patch_size, heads=dims.heads,
                                          layers=dims.layers)
    assert _rel(emb.cpu(), ref_emb) < 1e-3
    worst = {}
    for name, p in tower.named_parameters():
        key = name.replace("vision_model.", "", 1)
        if key not in ref:
            continue
        assert p.grad is not None, name
        r = ref[key].double()
        if r.norm().item() < 1e-12:
            continue
        err = (p.grad.detach().cpu().double() - r).norm().item() / r.norm().item()
        if "k_proj.bias" in key:                      # mathematically zero gradient (softmax shift invariance): noise / noise
            continue
        worst[key] = err
        assert err < REL, (key, err)
    assert len(worst) >= 24 * 14
    try:
        d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "parity.log"), "a") as f:
            f.write(f"vit_large_336 tower backward (24 layers, 577 tokens, 2 views) vs fp32 CPU oracle: worst per-tensor relative "
                    f"gradient error {max(worst.values()):.3e} ({max(worst, key=worst.get)}), median "
                    f"{float(np.median(list(worst.values()))):.3e}; oracle took {time.time() - t0:.0f} s\n")
    except OSError:
        pass
