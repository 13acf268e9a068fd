"""CPU-only: the C-ABI library loads and exports every symbol the header declares; host-side logic
(bank packing, sharding, packed all-gather over gloo with world_size 2, module surface)."""
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from pigeon_b200 import _lib
    header = open(os.path.join(ROOT, "include", "pigeon_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(pg_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 18
    lib = _lib.load()
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/pigeon_b200.h but not exported"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    m = re.search(r"#define PG_ABI_VERSION (\d+)", header)
    assert m and lib.pg_abi_version() == int(m.group(1)) == _lib.ABI_VERSION


def test_no_gpu_fails_loudly():
    """On a box without CUDA the product path must raise, never fall back to CPU arithmetic."""
    if torch.cuda.is_available():
        pytest.skip("has a GPU")
    from pigeon_b200 import PigeonB200Error, SuperGuessr, ops
    with pytest.raises(PigeonB200Error):
        ops.layernorm_f16(torch.zeros(4, 128), torch.ones(128), torch.zeros(128), 1e-5)
    sg = SuperGuessr(None, panorama=True, geocells=np.zeros((8, 2))).eval()
    with pytest.raises(PigeonB200Error):
        sg(embedding=torch.zeros(2, 4, 1024), labels_clf=torch.zeros(2, dtype=torch.long))


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "pigeon_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f"{f} imports the oracle"


def test_shard_range_partitions():
    from pigeon_b200.dist import shard_range
    for total in (0, 1, 7, 256, 2048, 2049):
        for world in (1, 2, 3, 8):
            spans = [shard_range(total, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == total
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            sizes = [hi - lo for lo, hi in spans]
            assert max(sizes) - min(sizes) <= 1


def test_bank_from_arrays_matches_manual_means():
    from pigeon_b200 import bank as bank_mod
    rng = np.random.default_rng(0)
    n, D = 50, 128
    data = rng.standard_normal((n, 4, D)).astype(np.float32)
    ll = rng.uniform(-90, 90, (n, 2)).astype(np.float32)
    cells = np.array([3, 0, 3, 1, 5])                       # unsorted rows, cell 2 and 4 empty, 6 cells total
    idx = [[1, 2, 3], [4], [10, 11], [], [20, 21, 22, 23]]   # row 3 has no members -> dropped
    b = bank_mod.bank_from_arrays(cells, rng.uniform(-90, 90, (5, 2)), idx, torch.from_numpy(data), ll, num_cells=6)
    assert b["cell_off"].tolist() == [0, 1, 1, 1, 3, 3, 4]
    assert b["proto_count"].tolist() == [1, 3, 2, 4]
    assert b["member_idx"].tolist() == [4, 1, 2, 3, 10, 11, 20, 21, 22, 23]
    m = torch.from_numpy(data).mean(1)
    np.testing.assert_allclose(b["proto_emb"][1], m[[1, 2, 3]].mean(0).numpy(), rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(b["data_emb"], m.numpy())
    # the CSV `count` column, when given, is what the single-member shortcut tests (proto_refiner.py:243-244) — also where it
    # disagrees with the length of the index list
    b2 = bank_mod.bank_from_arrays(cells, rng.uniform(-90, 90, (5, 2)), idx, torch.from_numpy(data), ll, num_cells=6,
                                   proto_count=[1, 7, 2, 9, 1])
    assert b2["proto_count"].tolist() == [7, 1, 2, 1] and b2["member_idx"].tolist() == b["member_idx"].tolist()


def test_module_surface_matches_reference_signatures():
    import inspect
    from pigeon_b200 import CLIPEmbedding, ModelOutput, ProtoRefiner, SuperGuessr
    sg = list(inspect.signature(SuperGuessr.__init__).parameters)[1:12]
    assert sg == ["base_model", "panorama", "hierarchical", "should_smooth_labels", "multi_task", "heading", "yfcc",
                  "serving", "freeze_base", "num_candidates", "embed_dim"]                     # super_guessr.py:31-34
    fw = list(inspect.signature(SuperGuessr.forward).parameters)[1:]
    assert fw == ["pixel_values", "embedding", "heading", "labels", "labels_clf", "labels_multi_task", "labels_climate",
                  "labels_month", "index"]                                                      # :350-353
    pr = list(inspect.signature(ProtoRefiner.__init__).parameters)[1:9]
    assert pr == ["topk", "hedge", "max_refinement", "temperature", "proto_path", "dataset_path", "protos", "verbose"]
    pf = list(inspect.signature(ProtoRefiner.forward).parameters)[1:7]
    assert pf == ["embedding", "geo_tensor", "initial_preds", "candidate_cells", "candidate_probs", "cluster"]
    ce = list(inspect.signature(CLIPEmbedding.__init__).parameters)[1:5]
    assert ce == ["model_name", "device", "load_checkpoint", "panorama"]                        # clip_embedder.py:11-12
    assert ModelOutput._fields == ("loss", "loss_clf", "loss_reg", "loss_climate", "loss_month", "preds_LLH",
                                   "preds_geocell", "preds_mt", "preds_climate", "preds_month", "top5_geocells",
                                   "embedding")                                                 # models/utils.py:7-9
    from pigeon_b200 import loops, training
    tm = list(inspect.signature(training.train_model).parameters)[:8]
    assert tm == ["loaded_model", "dataset", "on_embeddings", "yfcc", "train_args", "metrics", "patience",
                  "should_profile"]                                                             # train_eval_loop.py:164-166
    ev = list(inspect.signature(loops.evaluate_model).parameters)[:8]
    assert ev == ["model", "dataset", "metrics", "train_args", "refiner", "yfcc", "writer", "step"]   # :35-37
    fm = list(inspect.signature(training.finetune_model).parameters)[:7]
    assert fm == ["model", "dataset", "multi_task", "heading", "yfcc", "early_stopping", "train_args"]   # train_modes.py:67-69
    fe = list(inspect.signature(training.finetune_on_embeddings).parameters)[:6]
    assert fe == ["dataset", "multi_task", "heading", "yfcc", "early_stopping", "train_args"]           # train_modes.py:110-112
    opt = list(inspect.signature(training.AdamW.__init__).parameters)[1:6]
    assert opt == ["params", "lr", "betas", "eps", "weight_decay"]                               # torch.optim.AdamW


def test_tower_state_dict_uses_hf_key_names_and_roundtrips():
    from pigeon_b200 import CLIPVisionTower, VitDims, synthetic
    dims = VitDims(image_size=56, hidden=256, heads=4, intermediate=512, layers=2)
    sd = synthetic.random_vit_state_dict(dims, seed=3)
    t = CLIPVisionTower(dims)
    t.load_state_dict(sd)
    assert set(t.state_dict()) == set(sd)
    assert "vision_model.pre_layrnorm.weight" in sd and "vision_model.encoder.layers.1.self_attn.q_proj.weight" in sd
    assert len(list(t.vision_model.encoder.layers[:-1].parameters())) == 16                     # freeze policy handle


GLOO_WORKER = textwrap.dedent("""
    import os, sys, torch, torch.distributed as dist
    sys.path.insert(0, %r)
    from pigeon_b200 import dist as pdist
    rank, world = int(sys.argv[1]), 2
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=sys.argv[2], RANK=str(rank), WORLD_SIZE="2")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B = 3
    pack = dict(emb=torch.full((B, 5), float(rank)) + torch.arange(5), idx=torch.arange(B * 2).reshape(B, 2) + 100 * rank,
                val=torch.rand(B, 2).double(), init=torch.full((B, 2), rank + 0.5, dtype=torch.float64))
    out = pdist.all_gather_rows(pack)
    assert out["emb"].shape == (2 * B, 5) and out["emb"].dtype == torch.float32
    assert torch.equal(out["emb"][:B], torch.zeros(B, 5) + torch.arange(5)) and torch.equal(out["emb"][B:], torch.ones(B, 5) + torch.arange(5))
    assert out["idx"].dtype == torch.int64 and out["idx"][B:].min() == 100 and out["idx"][:B].max() == 5
    assert out["init"].dtype == torch.float64 and out["init"][0, 0] == 0.5 and out["init"][-1, 0] == 1.5
    assert torch.equal(out["val"][rank * B:(rank + 1) * B], pack["val"])
    lo, hi = pdist.shard_range(7, rank, world)
    assert (lo, hi) == ((0, 4) if rank == 0 else (4, 7))
    dist.destroy_process_group()
    print("rank", rank, "ok")
""")


def test_packed_all_gather_gloo_world2(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(GLOO_WORKER % ROOT)
    port = str(29000 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), str(r), port], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
             for r in range(2)]
    outs = [p.communicate(timeout=120)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o


def test_shard_bank_partitions_cells_and_members():
    """bank.shard_bank: every geocell lives in exactly one shard (cell % world), prototype rows / member lists / member
    embeddings are compacted consistently, the union of the shards is the bank."""
    from pigeon_b200 import bank as bank_mod, synthetic
    full = synthetic.synthetic_bank(37, 400, 128, seed=5, members_mean=3.0, empty_cells=3)
    W = 4
    C = full["cell_off"].shape[0] - 1
    seen = np.zeros(C, np.int64)
    total_p = 0
    for r in range(W):
        sh = bank_mod.shard_bank(full, r, W)
        assert sh["cell_off"].shape == full["cell_off"].shape and sh["cell_off"][0] == 0
        total_p += sh["proto_emb"].shape[0]
        for c in range(C):
            lo, hi = sh["cell_off"][c], sh["cell_off"][c + 1]
            flo, fhi = full["cell_off"][c], full["cell_off"][c + 1]
            if c % W != r:
                assert hi == lo
                continue
            seen[c] += 1
            assert hi - lo == fhi - flo
            assert np.array_equal(sh["proto_emb"][lo:hi], full["proto_emb"][flo:fhi])
            assert np.array_equal(sh["proto_lnglat"][lo:hi], full["proto_lnglat"][flo:fhi])
            assert np.array_equal(sh["proto_count"][lo:hi], full["proto_count"][flo:fhi])
            for k in range(hi - lo):       # member lists point at the same embeddings / labels after compaction
                m_new = sh["member_idx"][sh["member_off"][lo + k]: sh["member_off"][lo + k + 1]]
                m_old = full["member_idx"][full["member_off"][flo + k]: full["member_off"][flo + k + 1]]
                assert np.array_equal(sh["data_emb"][m_new], full["data_emb"][m_old])
                assert np.array_equal(sh["data_lnglat"][m_new], full["data_lnglat"][m_old])
    assert (seen == 1).all() and total_p == full["proto_emb"].shape[0]


GLOO_MERGE_WORKER = textwrap.dedent("""
    import os, sys, torch, torch.distributed as dist
    sys.path.insert(0, %r)
    from pigeon_b200 import dist as pdist
    rank, world = int(sys.argv[1]), 2
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=sys.argv[2], RANK=str(rank), WORLD_SIZE="2")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    B, k = 5, 3
    g = torch.Generator().manual_seed(3)
    cand = torch.randint(0, 11, (B, k), generator=g)
    truth_logit = -torch.rand(B, k, generator=g)
    truth_ll = torch.rand(B, k, 2, generator=g)
    mine = (cand %% world) == rank                       # what a scan over this rank's shard returns
    bl = torch.where(mine, truth_logit, torch.full((B, k), -100000.0))
    bll = torch.where(mine[..., None], truth_ll, torch.zeros(B, k, 2))
    gathered = pdist.all_gather_rows(dict(best_logit=bl, best_lnglat=bll))
    merged = pdist.merge_partials_by_owner(gathered, cand, world)
    assert torch.equal(merged["best_logit"], truth_logit), merged["best_logit"]
    assert torch.equal(merged["best_lnglat"], truth_ll)
    dist.destroy_process_group()
    print("rank", rank, "ok")
""")


def test_owner_merge_of_sharded_partials_gloo_world2(tmp_path):
    """Cell-sharded retrieval, host side: partials of two ranks (each -100000 where it does not hold the geocell) merged by
    owner after the packed all-gather reproduce the unsharded partials bit for bit."""
    script = tmp_path / "m.py"
    script.write_text(GLOO_MERGE_WORKER % ROOT)
    port = str(31000 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), str(r), port], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
             for r in range(2)]
    outs = [p.communicate(timeout=120)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o


def test_preprocess_plan_matches_oracle_geometry():
    """pg_preprocess_workspace_bytes is pure host arithmetic (resize geometry, Pillow's kernel support, the input rows the
    vertical pass needs): its layout must follow from the oracle's restatement of the same formulas."""
    import ctypes as C
    from oracle import preprocess as op
    from pigeon_b200 import _lib
    lib = _lib.load()
    size = 336
    align = lambda x, a=256: (x + a - 1) // a * a
    shapes = [(480, 640), (500, 375), (150, 210), (336, 400), (900, 1300), (337, 336), (2000, 3000), (64, 4000)]
    desc = (_lib.Image * len(shapes))()
    inter, ks = 0, 0
    for i, (h, w) in enumerate(shapes):
        desc[i] = _lib.Image(0x1000, h, w, 3 * w)              # fake device pointer: nothing is dereferenced
        nh, nw = op.resized_shape(h, w, size)
        top, left = (nh - size) // 2, (nw - size) // 2
        kv, bv, _ = op.precompute_coeffs(h, nh)
        kh, _, _ = op.precompute_coeffs(w, nw)
        first, last = int(bv[top, 0]), int(bv[top + size - 1, 0] + bv[top + size - 1, 1])
        inter += align((last - first) * size * 3)
        ks = max(ks, kv, kh)
    n = len(shapes)
    expect = align(n * 64) + align(n * 2 * size * ks * 4) + align(n * 2 * size * 2 * 4) + inter
    assert lib.pg_preprocess_workspace_bytes(desc, n, size) == expect
    bad = (_lib.Image * 1)(_lib.Image(0x1000, 8, 40000, 120000))
    assert lib.pg_preprocess_workspace_bytes(bad, 1, size) == 0 and b"exceeds" in lib.pg_last_error()


def test_trainer_layout_and_optimizer_arguments():
    """Host logic of the fine-tune step that needs no GPU: which blocks train (reference freeze policy,
    models/super_guessr.py:159-160), partly frozen blocks are refused, AdamW validates its hyper-parameters."""
    from pigeon_b200 import CLIPVisionTower, PigeonB200Error, VitDims
    from pigeon_b200.training import AdamW
    from pigeon_b200.vit_train import TowerTrainer
    dims = VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=3)
    tower = CLIPVisionTower(dims)
    tr = TowerTrainer(tower)
    assert tr.layout() == (True, [True, True, True]) and tr.any_trainable()
    for p in tower.vision_model.encoder.layers[:-1].parameters():
        p.requires_grad = False
    assert tr.layout() == (True, [False, False, True])
    for p in tower.parameters():
        p.requires_grad = False
    assert tr.layout() == (False, [False, False, False]) and not tr.any_trainable()
    tower.vision_model.encoder.layers[1].mlp.fc2.bias.requires_grad = True
    with pytest.raises(PigeonB200Error):
        tr.layout()
    tower.vision_model.encoder.layers[1].mlp.fc2.bias.requires_grad = False
    tower.vision_model.embeddings.class_embedding.requires_grad = True
    with pytest.raises(PigeonB200Error):
        tr.layout()
    w = torch.nn.Parameter(torch.zeros(4))
    for kw in (dict(lr=-1.0), dict(betas=(1.0, 0.9)), dict(eps=-1e-8), dict(weight_decay=-0.1)):
        with pytest.raises(ValueError):
            AdamW([w], **kw)
    opt = AdamW([w, torch.nn.Parameter(torch.zeros(2), requires_grad=False)], lr=1e-3)
    assert len(opt.params) == 1
    w.grad = torch.ones(4)
    opt.zero_grad()
    assert w.grad is None
    w.grad = torch.ones(4)                               # CPU tensors: the optimizer has no CPU path
    with pytest.raises(PigeonB200Error):
        opt.step()


GLOO_GRAD_WORKER = textwrap.dedent("""
    import os, sys, numpy as np, torch, torch.distributed as dist
    sys.path.insert(0, %r)
    from pigeon_b200 import SuperGuessr
    rank, world = int(sys.argv[1]), 2
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=sys.argv[2], RANK=str(rank), WORLD_SIZE="2")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sg = SuperGuessr(None, panorama=True, multi_task=True, embed_dim=128, geocells=np.zeros((10, 2)))
    params = sg._mt_params()
    assert len(params) == 6
    grads = [torch.full_like(p, float(rank + 1)) for p in params]
    sg._publish_mt_grads(grads, world)                  # DDP-style: mean over ranks, accumulated into .grad
    sg._publish_mt_grads([torch.full_like(p, 2.0 * (rank + 1)) for p in params], world)
    for p in params:
        assert torch.allclose(p.grad, torch.full_like(p, 1.5 + 3.0)), p.grad.flatten()[:3]
    dist.destroy_process_group()
    print("rank", rank, "ok")
""")


def test_gradient_averaging_gloo_world2(tmp_path):
    script = tmp_path / "g.py"
    script.write_text(GLOO_GRAD_WORKER % ROOT)
    port = str(31000 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), str(r), port], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
             for r in range(2)]
    outs = [p.communicate(timeout=180)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o


def test_state_dict_is_a_plain_weights_file(tmp_path):
    """Checkpoints written from the mirror (`torch.save(model.state_dict())`, train_eval_loop.py:238) must load with
    `weights_only=True` and carry exactly the reference's key names — nothing but tensors may ride along."""
    from pigeon_b200 import CLIPVisionTower, SuperGuessr, VitDims, _versions, synthetic
    dims = VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=2)
    tower = CLIPVisionTower(dims)
    sg = SuperGuessr(tower, panorama=False, geocells=synthetic.synthetic_geocells(12, 0))
    v0 = tower._weights_version()
    for p in sg.parameters():
        _versions.bump(p)                                   # what AdamW.step() does after a raw-pointer update
    assert tower._weights_version() != v0
    path = tmp_path / "m.model"
    torch.save(sg.state_dict(), path)
    assert path.stat().st_size < 2 * sum(t.numel() * t.element_size() for t in sg.state_dict().values())
    sd = torch.load(path, map_location="cpu", weights_only=True)
    assert set(sd) == set(sg.state_dict())
    assert "base_model.vision_model.encoder.layers.1.mlp.fc2.weight" in sd and "cell_layer.weight" in sd and "lla_geocells" in sd


def test_repack_groups_follow_the_parameters_that_moved():
    """After an optimizer step only the groups whose parameters changed are repacked for the kernels (one encoder layer under
    the reference's last-layer fine-tune policy, train_eval_loop.py:187 + super_guessr.py:159-160)."""
    from pigeon_b200 import CLIPVisionTower, VitDims, _versions
    dims = VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=3)
    tower = CLIPVisionTower(dims)
    before = tower._group_versions()
    assert set(before) == {"embeddings", 0, 1, 2}
    for p in tower.vision_model.encoder.layers[2].parameters():
        _versions.bump(p)                                   # what pg_adamw_step's wrapper does after a raw-pointer update
    after = tower._group_versions()
    assert {g for g in after if after[g] != before[g]} == {2}
    with torch.no_grad():
        tower.vision_model.embeddings.class_embedding.add_(1.0)   # an in-place torch update bumps ._version
    assert {g for g in after if tower._group_versions()[g] != after[g]} == {"embeddings"}


def test_model_summary_text_and_partial_freeze():
    """`print(model)` is what the reference's run scripts log (models/super_guessr.py:486-501): same lines, same tabs.  A CLIP
    tower that is not frozen keeps only its last encoder layer trainable (:146-160; the pretrained-head load is skipped in
    serving mode, so this runs without a checkpoint)."""
    from pigeon_b200 import CLIPVisionTower, SuperGuessr, VitDims, synthetic
    dims = VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=3)
    sg = SuperGuessr(CLIPVisionTower(dims), panorama=True, serving=True, geocells=synthetic.synthetic_geocells(12, 0))
    assert str(sg) == ("SuperGuessr(\n\tbase_model\t= True\n\tpanorama\t= True\n\thierarchical\t= False\n"
                       "\tmulti-task\t= False\n\tyfcc\t\t= False\n\tembedding_size\t= 256\n\tinput_dim\t= 256\n"
                       "\tnum_geocells\t= 12\n\tlabel_smoothing\t= False\n\tuses_headings\t= False\n"
                       "\tfreeze_base\t= False\n\tserving\t\t= True\n)")
    frozen = SuperGuessr(CLIPVisionTower(dims), freeze_base=True, geocells=synthetic.synthetic_geocells(12, 0))
    assert not any(p.requires_grad for p in frozen.base_model.parameters())
    assert all(p.requires_grad for p in frozen.cell_layer.parameters())


def test_load_state_copies_by_name_and_reports_unknown_keys(tmp_path, capsys):
    """models/super_guessr.py:222-238."""
    from pigeon_b200 import SuperGuessr
    sg = SuperGuessr(None, panorama=True, embed_dim=16, geocells=np.zeros((5, 2)))
    sd = {k: torch.full_like(v, 0.5) for k, v in sg.state_dict().items() if v.is_floating_point()}
    sd["not_a_parameter"] = torch.zeros(1)
    path = tmp_path / "head.model"
    torch.save(sd, path)
    real_load = torch.load
    try:
        torch.load = lambda f, map_location=None, **kw: real_load(f, map_location="cpu", **kw)   # no GPU in this suite
        sg.load_state(str(path))
    finally:
        torch.load = real_load
    assert "Parameter not_a_parameter not in model's state." in capsys.readouterr().out
    assert float(sg.cell_layer.weight.detach().mean()) == 0.5


def test_docs_only_name_entry_points_that_exist():
    """DESIGN.md / INTEGRATION.md / README.md may only cite C entry points and structs the header declares
    (`pg_vit_{create,destroy}` brace groups are expanded; a trailing-underscore prefix such as `pg_profile_*` is a family)."""
    header = open(os.path.join(ROOT, "include", "pigeon_b200.h")).read()
    code = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(pg_[a-z0-9_]+)\s*\(", code)) | set(re.findall(r"typedef struct (pg_\w+)", code))
    for doc in ("DESIGN.md", "INTEGRATION.md", "README.md"):
        text = open(os.path.join(ROOT, doc)).read()
        names = set()
        for m in re.finditer(r"pg_([a-z0-9_]*)\{([a-z0-9_,]+)\}", text):
            names |= {f"pg_{m.group(1)}{alt}" for alt in m.group(2).split(",")}
        text = re.sub(r"pg_[a-z0-9_]*\{[a-z0-9_,]+\}", " ", text)
        names |= set(re.findall(r"\bpg_[a-z0-9_]+\b", text))
        unknown = {n for n in names if n not in declared and not (n.endswith("_") and any(d.startswith(n) for d in declared))}
        assert not unknown, (doc, sorted(unknown))


def test_ctypes_structs_match_the_header_layout_at_abi_4(tmp_path):
    """Every ctypes mirror in pigeon_b200/_lib.py, pg_gemm_problem included, has the size and the field offsets gcc computes
    from include/pigeon_b200.h (a reordered, missing or mistyped field would silently corrupt the arguments of the C ABI), and
    the binding is at ABI version 4, the first with pg_gemm_problem."""
    import ctypes as C
    import shutil
    import subprocess
    from pigeon_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    pairs = {"pg_vit_config": _lib.VitConfig, "pg_image": _lib.Image, "pg_vit_layer": _lib.VitLayer,
             "pg_vit_saved_layer": _lib.VitSavedLayer, "pg_vit_saved": _lib.VitSaved, "pg_vit_layer_bwd": _lib.VitLayerBwd,
             "pg_vit_grads": _lib.VitGrads, "pg_vit_weights": _lib.VitWeights, "pg_refiner_bank": _lib.RefinerBank,
             "pg_gemm_problem": _lib.GemmProblem}
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "pigeon_b200.h"', "int main(void) {"]
    for cname, cls in pairs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([gcc, "-std=c99", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True).stdout.splitlines())
    for cname, cls in pairs.items():
        assert int(got[cname]) == C.sizeof(cls), (cname, got[cname], C.sizeof(cls))
        for fname, _ in cls._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(cls, fname).offset, (cname, fname)
    assert _lib.ABI_VERSION == 4
