"""Hierarchical panorama head, host side: the fp64 oracle (tests/hierarchical_oracle.py) against tests/golden/hierarchical.npz
(outputs of the UNMODIFIED reference, tools/make_hierarchical_golden.py), the port's parameters and seeded initial values
against the reference's, the constructor's refusals, and the C ABI's argument checks (which return before touching a device)."""
import json
import os

import numpy as np
import pytest
import torch

import hierarchical_oracle as ho

GOLD = os.path.join(os.path.dirname(__file__), "golden", "hierarchical.npz")


@pytest.fixture(scope="module")
def gold():
    z = np.load(GOLD, allow_pickle=False)
    return z, json.loads(str(z["meta"]))


def _pe(E):
    from pigeon_b200.super_guessr import PositionalEncoder
    return PositionalEncoder(E).pos_encoding.detach()


def _rel(a, b):
    a, b = torch.as_tensor(np.asarray(a), dtype=torch.float64), torch.as_tensor(np.asarray(b), dtype=torch.float64)
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _params64(E, C, seed):
    return {k: v.double().requires_grad_(True) for k, v in ho.synthetic_params(E, C, seed).items()}


@pytest.mark.parametrize("name", ["eval_a", "eval_b", "eval_c", "serve"])
def test_oracle_reproduces_reference_eval(gold, name):
    z, meta = gold
    case = meta["cases"][name]
    E, N, seed = case["E"], case["N"], int(z[f"{name}_seed"])
    p = {k: v.double() for k, v in ho.synthetic_params(E, meta["C"], seed).items()}
    cent = torch.tensor(z["centroids"])
    a = ho.attention(ho.embeddings(N, E, seed).double(), _pe(E).double(), *[p[k] for k in ho.ATTN_KEYS])
    logits, probs, pred, pred_llh, topk = ho.head(a["cls"], p["cell_layer.weight"], p["cell_layer.bias"], cent, 5)
    assert (z[f"{name}_margin"] > meta["margin"]).all()
    assert np.array_equal(topk.indices.numpy(), z[f"{name}_topk_idx"])
    assert np.array_equal(pred_llh.numpy(), z[f"{name}_preds_LLH"])
    np.testing.assert_allclose(topk.values.numpy(), z[f"{name}_topk_val"], rtol=2e-5)
    if case["serving"]:
        return
    assert np.array_equal(pred.numpy(), z[f"{name}_preds_geocell"])
    labels, labels_clf, *_ = ho.labels(N, seed)
    loss = ho.classification_loss(logits, cent, labels, labels_clf, smooth=case["smooth"])
    np.testing.assert_allclose(loss.item(), z[f"{name}_loss_clf"], rtol=2e-5)


def test_oracle_reproduces_reference_gradients(gold):
    """d loss / d every trainable parameter and d embedding of the reference (fp32 autograd, dropouts at p = 0) against fp64
    autograd through the oracle; the auxiliary heads keep the seeded nn.Linear init, taken here from the golden state."""
    z, meta = gold
    seed, E, N = int(z["grad_seed"]), 128, 24
    p = _params64(E, meta["C"], seed)
    emb = ho.embeddings(N, E, seed).double().requires_grad_(True)
    cent = torch.tensor(z["centroids"])
    labels, labels_clf, lmt, lcl, lmo = ho.labels(N, seed)
    from pigeon_b200 import SuperGuessr
    torch.manual_seed(seed)
    port = SuperGuessr(None, panorama=True, hierarchical=True, embed_dim=E, multi_task=True, should_smooth_labels=True,
                       geocells=z["centroids"])
    heads = {n: tuple(t.detach().double().requires_grad_(True) for t in (getattr(port, n).weight, getattr(port, n).bias))
             for n in ("multi_task_head", "climate_layer", "month_layer")}
    a = ho.attention(emb, _pe(E).double(), *[p[k] for k in ho.ATTN_KEYS])
    logits = torch.nn.functional.linear(a["cls"], p["cell_layer.weight"], p["cell_layer.bias"])
    loss = ho.classification_loss(logits, cent, labels, labels_clf, smooth=True) + ho.multi_task_loss(a["cls"], heads, lmt, lcl, lmo)
    loss.backward()
    np.testing.assert_allclose(loss.item(), z["grad_loss"], rtol=1e-5)
    assert _rel(ho.sample(emb.grad), z["grad/embedding"]) < 1e-4
    for k, t in p.items():
        assert _rel(ho.sample(t.grad), z["grad/" + k]) < 1e-4, k
    for n, (w, b) in heads.items():
        assert _rel(ho.sample(w.grad), z[f"grad/{n}.weight"]) < 1e-4 and _rel(ho.sample(b.grad), z[f"grad/{n}.bias"]) < 1e-4, n


def test_oracle_reproduces_reference_adamw_trajectory(gold):
    z, meta = gold
    seed, E, N, steps, lr = int(z["adam_seed"]), 128, 24, int(z["adam_steps"]), float(z["adam_lr"])
    p = _params64(E, meta["C"], seed)
    opt = torch.optim.AdamW(list(p.values()), lr=lr)
    cent = torch.tensor(z["centroids"])
    for i in range(steps):
        _, labels_clf, *_ = ho.labels(N, seed + i)
        a = ho.attention(ho.embeddings(N, E, seed + i).double(), _pe(E).double(), *[p[k] for k in ho.ATTN_KEYS])
        logits = torch.nn.functional.linear(a["cls"], p["cell_layer.weight"], p["cell_layer.bias"])
        loss = ho.classification_loss(logits, cent, labels_clf=labels_clf)
        np.testing.assert_allclose(loss.item(), z["adam_losses"][i], rtol=1e-5)
        loss.backward()
        opt.step()
        opt.zero_grad()
    for k, t in p.items():
        got, want = ho.sample(t.detach()), torch.from_numpy(z["adam/" + k]).double()
        if k == "self_attn.in_proj_bias":
            check_key_bias_steps(got, want, E, steps, lr)
            got, want = torch.cat([got[:E], got[2 * E:]]), torch.cat([want[:E], want[2 * E:]])
        assert _rel(got, want) < 1e-5, k


def check_key_bias_steps(got, want, E, steps, lr):
    """The key bias adds q0 . bk to every score of a head alike, which the softmax cancels: its exact gradient is zero and
    what either run computes is rounding noise, which AdamW normalises into steps of up to lr.  After `steps` updates the
    two runs can differ there by up to 2 * steps * lr, and no more."""
    assert (got[E:2 * E] - want[E:2 * E]).abs().max().item() <= 2 * steps * lr * 1.001


def test_state_dict_names_shapes_and_seeded_values_match_the_reference(gold):
    """torch.manual_seed(s); SuperGuessr(hierarchical=True) draws the reference's initial weights: same keys in the same order,
    same shapes, same values (pos_encoder, then self_attn, then cell_layer, then the multi-task layers)."""
    from pigeon_b200 import SuperGuessr
    z, _ = gold
    torch.manual_seed(int(z["state_seed"]))
    sg = SuperGuessr(None, panorama=True, hierarchical=True, embed_dim=int(z["state_E"]), multi_task=True,
                     geocells=z["centroids"])
    sd = sg.state_dict()
    ref = [k[len("state/"):] for k in z.files if k.startswith("state/")]
    assert list(sd) == ref
    assert {k: list(v.shape) for k, v in sd.items()} == json.loads(str(z["state_shapes"]))
    for k in ref:
        assert torch.equal(ho.sample(sd[k].cpu()), torch.from_numpy(z["state/" + k])), k
    assert not sg.pos_encoder.pos_encoding.requires_grad
    assert sg.self_attn.in_proj_weight.requires_grad and sg.self_attn.dropout == 0.1 and sg.pos_encoder.dropout.p == 0.1


def test_hierarchical_refusals(capsys):
    from pigeon_b200 import SuperGuessr
    cells = np.zeros((8, 2))
    with pytest.raises(NotImplementedError, match="hierarchical=True with heading=True"):
        SuperGuessr(None, panorama=True, hierarchical=True, heading=True, embed_dim=64, geocells=cells)
    with pytest.raises(NotImplementedError, match="single images"):
        SuperGuessr(None, panorama=False, hierarchical=True, heading=True, embed_dim=64, geocells=cells)
    capsys.readouterr()
    SuperGuessr(None, panorama=True, hierarchical=True, embed_dim=64, geocells=cells)
    assert "Number of attention heads: 16" in capsys.readouterr().out


def test_view_attention_entry_points_are_exported_and_check_their_arguments():
    from pigeon_b200 import _lib
    lib = _lib.load()
    for name in ("pg_view_attn_forward", "pg_view_attn_backward", "pg_view_attn_workspace_bytes", "pg_view_attn_saved_floats"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    assert lib.pg_view_attn_saved_floats(3, 64, 16) == 14 * 3 * 64 + 4 * 3 * 16
    fake = 1 << 20                                     # never dereferenced: every refusal below returns first

    def fwd(N, E, heads=16, pe_rows=1000, n0=0, p=0.1):
        return lib.pg_view_attn_forward(fake, N, E, heads, fake, pe_rows, n0, fake, fake, fake, fake, p, p, 1, 2, fake,
                                        1 << 40, fake, None, None, fake, None)

    for args, msg in (((4, 100), b"bad shape"), ((4, 48, 32), b"bad shape"), ((1001, 64), b"positional-encoding rows"),
                      ((10, 64, 16, 1000, 995), b"positional-encoding rows"), ((4, 64, 16, 1000, 0, 1.0), b"dropout")):
        assert fwd(*args) != 0
        assert msg in lib.pg_last_error(), (args, lib.pg_last_error())
    assert lib.pg_view_attn_backward(fake, 4, 100, 16, 0, fake, fake, fake, 0.0, 0.0, 0, 0, 0, None, None, None, None, fake,
                                     fake, 1 << 40, None) != 0
    assert b"bad shape" in lib.pg_last_error()
