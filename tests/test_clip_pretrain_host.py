"""CPU-only checks of the CLIP pretraining loop's host side: the linear schedule and its lengths, the weight-decay groups,
checkpoints that HF loads, the collator, the configuration, `run.py pretrain`'s arguments and the oracle against its
golden (tests/golden/clip_pretrain.npz)."""
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def test_library_exports_the_pretraining_symbols():
    from pigeon_b200 import _lib
    lib = _lib.load()
    for name in ("pg_grad_norm_clip_workspace_bytes", "pg_grad_norm_clip", "pg_adamw_hf_step"):
        assert name in _lib.SIGNATURES and hasattr(lib, name), name
    assert lib.pg_grad_norm_clip_workspace_bytes(0) == 0 and lib.pg_grad_norm_clip_workspace_bytes(1 << 40) == 8 * 1024


@pytest.mark.parametrize("T,W", [(10, 0), (10, 3), (7, 7), (1000, 200), (200, 4), (5, 1)])
def test_linear_schedule_matches_transformers(T, W):
    from transformers import get_linear_schedule_with_warmup
    from pigeon_b200.training import linear_schedule_lambda
    ref_opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=1e-3)
    ref = get_linear_schedule_with_warmup(ref_opt, W, T)
    got_opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=1e-3)
    got = torch.optim.lr_scheduler.LambdaLR(got_opt, linear_schedule_lambda(W, T))
    for _ in range(T + 2):
        assert got.get_last_lr() == ref.get_last_lr()
        ref_opt.step(), got_opt.step()
        ref.step(), got.step()


def test_schedule_lengths():
    from pigeon_b200.training import schedule_lengths
    # 4.23.1: len(dataloader) = ceil(N / world) // batch; updates/epoch = max(len // acc, 1); T = ceil(epochs * that)
    assert schedule_lengths(28, 4, 2, 1, 2) == (7, 3, 6, 0, 2)
    assert schedule_lengths(28, 4, 2, 1, 2, warmup_ratio=0.2) == (7, 3, 6, 2, 2)
    assert schedule_lengths(1001, 32, 8, 4, 20, warmup_ratio=0.2) == (7, 1, 20, 4, 20)       # 251 per rank
    assert schedule_lengths(100_000, 32, 8, 4, 20, warmup_ratio=0.2) == (781, 97, 1940, 388, 20)
    assert schedule_lengths(100_000, 32, 8, 4, 4, warmup_ratio=0.02) == (781, 97, 388, 8, 4)
    assert schedule_lengths(100_000, 32, 8, 4, 2.5) == (781, 97, 243, 0, 3)
    assert schedule_lengths(28, 4, 2, 1, 2, max_steps=7) == (7, 3, 7, 0, 3)                  # max_steps wins over epochs
    assert schedule_lengths(28, 4, 2, 1, 2, max_steps=7, warmup_steps=3, warmup_ratio=0.5) == (7, 3, 7, 3, 3)
    assert schedule_lengths(3, 4, 2, 1, 1) == (0, 1, 1, 0, 1)


def _tiny():
    from make_clip_golden import GEOMETRIES, hf_clip
    from pigeon_b200 import CLIPModel, synthetic
    g = GEOMETRIES["tiny"]
    sd = synthetic.random_clip_state_dict(g["text"], g["vision"], seed=3, std=0.05, projection_dim=g["projection"])
    m = CLIPModel(g["text"], g["vision"], projection_dim=g["projection"])
    m.load_state_dict(sd)
    return m, hf_clip(g["text"], g["vision"], g["projection"], sd)


def test_decay_groups_match_hf_trainer():
    import clip_pretrain_oracle as O
    from pigeon_b200.training import decay_parameter_names, hf_named_parameters, optimizer_grouped_parameters
    m, hf = _tiny()
    assert [n for n, _ in hf_named_parameters(m)] == [n for n, _ in hf.named_parameters()]
    assert sorted(decay_parameter_names(m)) == sorted(O.hf_decay_parameter_names(hf))
    decay = set(decay_parameter_names(m))
    for n in ("logit_scale", "text_model.embeddings.token_embedding.weight", "vision_model.embeddings.class_embedding",
              "vision_model.embeddings.patch_embedding.weight", "text_model.embeddings.position_embedding.weight"):
        assert n in decay, n
    assert "vision_model.pre_layrnorm.weight" not in decay and "text_model.final_layer_norm.weight" not in decay
    ours = optimizer_grouped_parameters(m, 0.1)
    ref = O.hf_param_groups(hf, 0.1)
    names_m = {id(p): n for n, p in m.named_parameters()}
    names_h = {id(p): n for n, p in hf.named_parameters()}
    for go, gr in zip(ours, ref):
        assert go["weight_decay"] == gr["weight_decay"]
        assert [names_m[id(p)] for p in go["params"]] == [names_h[id(p)] for p in gr["params"]]


def test_checkpoint_round_trip_with_transformers(tmp_path):
    from transformers import CLIPModel as HFCLIPModel
    from pigeon_b200 import CLIPModel
    m, _ = _tiny()
    m.save_pretrained(str(tmp_path / "ours"))
    hf = HFCLIPModel.from_pretrained(str(tmp_path / "ours"))
    hs = hf.state_dict()
    for k, v in m.state_dict().items():
        assert torch.equal(hs[k], v), k
    hf.save_pretrained(str(tmp_path / "hf"), safe_serialization=False)
    back = CLIPModel.from_pretrained(str(tmp_path / "hf"))
    assert back.text_dims == m.text_dims and back.vision_dims == m.vision_dims
    for k, v in m.state_dict().items():
        assert torch.equal(back.state_dict()[k], v), k
    back = CLIPModel.from_pretrained(str(tmp_path / "ours"))
    for k, v in m.state_dict().items():
        assert torch.equal(back.state_dict()[k], v), k


def test_collator_pads_with_clip_eos():
    from pigeon_b200.pretrain import CLIP_PAD_TOKEN_ID, CLIPCollator
    rows = [{"input_ids": [49406, 5, 49407], "pixel_values": np.zeros((3, 4, 4), np.float32)},
            {"input_ids": torch.tensor([49406, 7, 8, 9, 49407]), "attention_mask": [1, 1, 1, 1, 1],
             "pixel_values": torch.ones(3, 4, 4)}]
    b = CLIPCollator()(rows)
    assert CLIP_PAD_TOKEN_ID == 49407
    assert b["input_ids"].tolist() == [[49406, 5, 49407, 49407, 49407], [49406, 7, 8, 9, 49407]]
    assert b["attention_mask"].tolist() == [[1, 1, 1, 0, 0], [1, 1, 1, 1, 1]]
    assert b["pixel_values"].shape == (2, 3, 4, 4)
    assert b["input_ids"].argmax(-1).tolist() == [2, 4]                 # the pooled row stays the first EOS


def test_pretrain_config_matches_reference():
    from pigeon_b200 import config
    # reference config.py:145-177 (PRETAIN_ARGS) and :112-143 (PRETAIN_ARGS_YFCC)
    common = dict(overwrite_output_dir=True, do_train=True, do_eval=True, evaluation_strategy='steps', eval_steps=50,
                  per_device_train_batch_size=32, per_device_eval_batch_size=32, gradient_accumulation_steps=8,
                  weight_decay=0.001, adam_beta1=0.9, adam_beta2=0.98, adam_epsilon=1e-06, max_grad_norm=1.0,
                  max_steps=-1, lr_scheduler_type='linear', logging_first_step=False, logging_steps=1,
                  save_strategy='steps', save_steps=50, seed=42, dataloader_drop_last=True, run_name=None, adafactor=False,
                  report_to='tensorboard', skip_memory_metrics=True, resume_from_checkpoint=None)
    want = dict(common, output_dir='saved_models/pretrained', learning_rate=1e-06, num_train_epochs=20, warmup_ratio=0.2)
    want_yfcc = dict(common, output_dir='saved_models/pretrained_yfcc', learning_rate=5e-07, num_train_epochs=4,
                     warmup_ratio=0.02)
    for ns, w in ((config.PRETAIN_ARGS, want), (config.PRETAIN_ARGS_YFCC, want_yfcc)):
        for k, v in w.items():
            assert getattr(ns, k) == v, k


def test_run_pretrain_arguments():
    sys.path.insert(0, ROOT)
    import run
    a = run.build_parser().parse_args(["pretrain", "openai/clip-vit-large-patch14-336", "-l", "data/pre", "--yfcc", "-r"])
    assert (a.mode, a.name, a.load, a.yfcc, a.resume) == ("pretrain", "openai/clip-vit-large-patch14-336", "data/pre",
                                                          True, True)
    assert run.build_parser().parse_args(["pretrain", "x", "-l", "d"]).resume is False
    r = subprocess.run([sys.executable, os.path.join(ROOT, "run.py"), "pretrain", "x"], capture_output=True, text=True,
                       cwd=ROOT)
    assert r.returncode != 0 and "-l" in r.stderr


def test_trainer_rejects_unsupported_arguments():
    from pigeon_b200.pretrain import CLIPPretrainer
    m, _ = _tiny()
    base = dict(per_device_train_batch_size=4, lr_scheduler_type="linear")
    with pytest.raises(NotImplementedError):
        CLIPPretrainer(m, SimpleNamespace(**dict(base, lr_scheduler_type="cosine")), [])
    with pytest.raises(Exception, match="max_train_views"):
        CLIPPretrainer(m, SimpleNamespace(**dict(base, per_device_train_batch_size=65)), [])


def test_oracle_reproduces_golden():
    import make_clip_pretrain_golden as G
    z = np.load(os.path.join(ROOT, "tests", "golden", "clip_pretrain.npz"))
    meta = json.loads(str(z["meta"]))
    assert meta["settings"]["max_grad_norm"] == G.SETTINGS["max_grad_norm"]
    log, snaps = G.run()
    steps = [e for e in log if "loss" in e]
    for k in ("loss", "learning_rate", "grad_norm", "epoch"):
        np.testing.assert_allclose([e[k] for e in steps], z[f"log/{k}"], rtol=2e-6, atol=0)
    np.testing.assert_allclose([e["eval_loss"] for e in log if "eval_loss" in e], z["eval/loss"], rtol=2e-6)
    for k, ps in snaps.items():
        for n, p in ps.items():
            np.testing.assert_allclose(p.reshape(-1)[::meta["stride"]].numpy(), z[f"sub/{k}/{n}"], rtol=2e-6, atol=2e-7,
                                       err_msg=n)
