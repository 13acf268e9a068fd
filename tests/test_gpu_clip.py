"""CLIP text tower, projections, image-text logits and CLIPModel.forward on the H100 against fp32 references
(tests/clip_oracle.py for HF CLIPTextTransformer / CLIPModel, torch on the same operands for the building blocks).

Budgets: 1e-3 relative (the project's fp16-operand budget) for tower outputs and embeds; the projection's split GEMM
< 2e-5 (the geocell head's bar); the fp32 logits kernels 1e-5."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

REL_TOL = 1e-3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _record(line):
    """Measured parity numbers are appended to the file named by PG_PARITY_LOG when that variable is set; never fails a
    test."""
    path = os.environ.get("PG_PARITY_LOG")
    if path:
        with open(path, "a") as f:
            f.write(line + "\n")


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _captions(lengths, vocab, seed, S=None):
    """CLIP-tokenizer layout: BOS = vocab - 2 first, EOS = vocab - 1 last, padded with EOS, attention_mask 0 on padding."""
    g = torch.Generator().manual_seed(seed)
    S = S or max(lengths)
    ids = torch.full((len(lengths), S), vocab - 1, dtype=torch.int64)
    mask = torch.zeros((len(lengths), S), dtype=torch.int64)
    for b, L in enumerate(lengths):
        ids[b, 0] = vocab - 2
        if L > 2:
            ids[b, 1:L - 1] = torch.randint(0, vocab - 2, (L - 2,), generator=g)
        mask[b, :L] = 1
    return ids, mask


# ------------------------------------------------------------------------------------------------ masked attention
def _attention_ref(qkv, n, S, heads, mask, causal):
    q, k, v = qkv.float().cpu().view(n, S, 3, heads, 64).permute(2, 0, 3, 1, 4)
    w = (q @ k.transpose(-1, -2)) / 8.0
    ok = torch.ones(n, 1, S, S, dtype=torch.bool)
    if causal:
        ok &= torch.ones(S, S, dtype=torch.bool).tril()[None, None]
    if mask is not None:
        ok &= mask.cpu().bool()[:, None, None, :]
    w = w.masked_fill(~ok, float("-inf"))
    return (torch.softmax(w, -1) @ v).transpose(1, 2).reshape(n * S, heads * 64)


@pytest.mark.parametrize("S", [1, 7, 64, 77, 130])
@pytest.mark.parametrize("mode", ["causal", "causal_padded", "interior_zero"])
def test_masked_attention(cuda, S, mode):
    from pigeon_b200 import ops
    n, heads = 3, 2
    g = torch.Generator().manual_seed(S)
    qkv = (torch.randn(n * S, 3 * heads * 64, generator=g) * 1.5).half()
    mask = None
    if mode != "causal":
        mask = torch.ones(n, S, dtype=torch.int64)
        if mode == "causal_padded":
            for b, L in enumerate([S, max(1, S // 2), max(1, S - 3)]):
                mask[b, L:] = 0
        else:
            mask[:, S // 2] = 0 if S > 1 else 1
            mask[1, 1::3] = 0
    causal = mode != "interior_zero"
    out = ops.attention_f16_masked(qkv.to(cuda), n, S, heads, mask.to(cuda) if mask is not None else None, causal=causal)
    torch.cuda.synchronize()
    ref = _attention_ref(qkv, n, S, heads, mask, causal)
    assert torch.isfinite(out).all()
    e = _rel(out, ref)
    assert e < 2e-3, (S, mode, e)


@pytest.mark.parametrize("S", [7, 77, 577])
def test_unmasked_variant_is_bit_identical(cuda, S):
    from pigeon_b200 import ops
    qkv = torch.randn(2 * S, 3 * 4 * 64, generator=torch.Generator().manual_seed(1)).half().to(cuda)
    a = ops.attention_f16(qkv, 2, S, 4)
    b = ops.attention_f16_masked(qkv, 2, S, 4, None, causal=False)
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ CLS rows
@pytest.mark.parametrize("fold", [True, False])
def test_vit_forward_cls(cuda, fold):
    from pigeon_b200 import synthetic
    from pigeon_b200.vit_engine import VitDims, VitEngine
    dims = VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=2)
    sd = synthetic.random_vit_state_dict(dims, seed=4, std=0.05)
    px = torch.randn(5, 3, 56, 56, generator=torch.Generator().manual_seed(2)).to(cuda)
    eng = VitEngine(sd, dims, device=cuda, max_views_per_pass=2, fold_layernorm=fold)
    emb, hid = eng.forward(px, return_hidden=True)
    emb2, cls = eng.forward_cls(px)
    torch.cuda.synchronize()
    assert torch.equal(emb, emb2)
    assert torch.equal(cls, hid[:, 0])


# ------------------------------------------------------------------------------------------------ text tower
def _text_tower(cuda, td, seed, std):
    from pigeon_b200 import CLIPTextTower, synthetic
    from pigeon_b200.vit_engine import VitDims
    vd = VitDims(image_size=28, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    sd = synthetic.random_clip_state_dict(td, vd, seed=seed, std=std)
    tower = CLIPTextTower(td)
    tower.load_state_dict({k: v for k, v in sd.items() if k.startswith("text_model.")})
    tower = tower.to(cuda)
    tower.max_texts_per_pass = 3
    return tower, sd


def _odd_mask(mask):
    """(float mask with 2, -1 and 1.5 in place of some of the ones after key 0, the same mask with those entries 0).  HF's
    `_expand_mask` excludes every key whose mask is not exactly 1."""
    odd = mask.double().clone()
    values = [2.0, -1.0, 1.5]
    for b in range(odd.shape[0]):
        for i, j in enumerate(range(1 + b % 2, int(mask[b].sum()), 2)):
            odd[b, j] = values[(b + i) % 3]
    return odd, torch.where(odd == 1, odd, torch.zeros_like(odd))


def _text_vs_oracle(cuda, td, lengths, seed, std, odd_mask=False):
    import clip_oracle
    tower, sd = _text_tower(cuda, td, seed, std)
    ids, mask = _captions(lengths, td.vocab, seed + 1)
    if odd_mask:
        mask, _ = _odd_mask(mask)
    out = tower(input_ids=ids.to(cuda), attention_mask=mask.to(cuda))
    torch.cuda.synchronize()
    ref_h, ref_p = clip_oracle.text_forward(sd, ids, mask, heads=td.heads, layers=td.layers, eps=td.ln_eps)
    W = sd["text_projection.weight"]
    from pigeon_b200 import ops
    te = ops.clip_project(out.pooler_output, ops.head_pack_weight(W.to(cuda)))
    ref_te = ref_p @ W.T
    te, ref_te = te / te.norm(dim=-1, keepdim=True), ref_te / ref_te.norm(dim=-1, keepdim=True)
    return _rel(out.last_hidden_state, ref_h), _rel(out.pooler_output, ref_p), _rel(te, ref_te)


def test_text_tower_tiny(cuda):
    from pigeon_b200 import TextDims
    td = TextDims(vocab=1000, max_positions=16, hidden=256, heads=4, intermediate=512, layers=2)
    e_h, e_p, e_t = _text_vs_oracle(cuda, td, [12, 5, 9, 1, 16, 2, 7], seed=3, std=0.05)
    print(f"text tower tiny rel-L2: last_hidden_state {e_h:.3e} pooled {e_p:.3e} text_embeds {e_t:.3e}")
    assert e_h < REL_TOL and e_p < REL_TOL and e_t < REL_TOL, (e_h, e_p, e_t)


def test_text_tower_excludes_mask_values_other_than_one(cuda):
    """attention_mask entries 2, -1 and 1.5 exclude their keys, as in HF: the tower matches the oracle, and both the tower
    and the trainer's forward give the bits of the same mask with those entries 0."""
    from pigeon_b200 import TextDims
    from pigeon_b200.clip_train import TextTrainer
    td = TextDims(vocab=1000, max_positions=16, hidden=256, heads=4, intermediate=512, layers=2)
    e_h, e_p, e_t = _text_vs_oracle(cuda, td, [12, 5, 9, 1, 16, 2, 7], seed=3, std=0.05, odd_mask=True)
    assert e_h < REL_TOL and e_p < REL_TOL and e_t < REL_TOL, (e_h, e_p, e_t)
    tower, _ = _text_tower(cuda, td, seed=3, std=0.05)
    ids, mask = _captions([12, 5, 9, 1, 16, 2, 7], td.vocab, 4)
    odd, zeroed = _odd_mask(mask)
    assert (odd != zeroed).any() and (odd[:, 0] == 1).all()
    ids, odd, zeroed = ids.to(cuda), odd.to(cuda), zeroed.to(cuda)
    a, b = tower(input_ids=ids, attention_mask=odd), tower(input_ids=ids, attention_mask=zeroed)
    assert torch.equal(a.last_hidden_state, b.last_hidden_state) and torch.equal(a.pooler_output, b.pooler_output)
    tt = TextTrainer(tower)
    pa = tt.forward(ids, odd).clone()
    pb = tt.forward(ids, zeroed)
    assert torch.equal(pa, pb)


def test_text_tower_large(cuda):
    """The real geometry: 12 layers of 768, 8 captions of lengths 3 ... 77 (right-padded)."""
    from pigeon_b200 import TextDims
    td = TextDims()
    e_h, e_p, e_t = _text_vs_oracle(cuda, td, [3, 77, 12, 40, 5, 66, 25, 9], seed=5, std=0.02)
    print(f"text tower CLIP-L rel-L2: last_hidden_state {e_h:.3e} pooled {e_p:.3e} text_embeds {e_t:.3e}")
    _record(f"clip_text_large (12 layers, 8 captions, lengths 3..77) vs fp32 CPU oracle: rel-L2 last_hidden_state "
            f"{e_h:.3e}, pooled {e_p:.3e}, text_embeds {e_t:.3e}")
    assert e_h < REL_TOL and e_p < REL_TOL and e_t < REL_TOL, (e_h, e_p, e_t)


# ------------------------------------------------------------------------------------------------ projection
@pytest.mark.parametrize("D,P,ln", [(1024, 768, True), (768, 768, False), (256, 384, True)])
def test_projection_split_gemm(cuda, D, P, ln):
    from pigeon_b200 import ops
    g = torch.Generator().manual_seed(D + P)
    x = torch.randn(37, D, generator=g) * 3 + 0.5
    W = torch.randn(P, D, generator=g) * 0.02
    gam, bet = (1 + 0.1 * torch.randn(D, generator=g)), 0.1 * torch.randn(D, generator=g)
    out = ops.clip_project(x.to(cuda), ops.head_pack_weight(W.to(cuda)), gam.to(cuda) if ln else None,
                           bet.to(cuda) if ln else None, 1e-5)
    x64 = x.double()
    if ln:
        x64 = torch.nn.functional.layer_norm(x64, (D,), gam.double(), bet.double(), 1e-5)
    ref = x64 @ W.double().T
    e = _rel(out, ref)
    print(f"projection D={D} P={P} ln={ln}: rel-L2 vs fp64 {e:.3e}")
    _record(f"clip_project D={D} P={P} layernorm={ln} vs fp64: rel-L2 {e:.3e}")
    assert e < 2e-5, e


# ------------------------------------------------------------------------------------------------ logits
@pytest.mark.parametrize("Ni,Nt", [(70, 50), (64, 64), (1, 3), (130, 130)])
def test_logits_probs_argmax_loss(cuda, Ni, Nt):
    from pigeon_b200 import ops
    g = torch.Generator().manual_seed(Ni * 7 + Nt)
    img = torch.randn(Ni, 768, generator=g)
    txt = torch.randn(Nt, 768, generator=g)
    scale = math.log(1 / 0.07)
    want_loss = Ni == Nt
    out = ops.clip_logits(img.to(cuda), txt.to(cuda), scale, per_text=True, probs=True, pred=True, loss=want_loss)
    torch.cuda.synchronize()
    ie, te = img / img.norm(dim=-1, keepdim=True), txt / txt.norm(dim=-1, keepdim=True)
    lpt = te @ ie.T * math.exp(scale)
    lpi = lpt.T
    assert _rel(out["logits_per_image"], lpi) <= 1e-5
    assert torch.equal(out["logits_per_text"].cpu(), out["logits_per_image"].cpu().T)
    assert _rel(out["probs"], lpi.softmax(1)) <= 1e-5
    top2 = lpi.topk(min(2, Nt), dim=1).values
    clear = (top2[:, 0] - top2[:, -1] > 1e-3) if Nt > 1 else torch.ones(Ni, dtype=torch.bool)
    assert torch.equal(out["pred"].cpu()[clear], lpi.argmax(1)[clear])
    if want_loss:
        t = torch.arange(Ni)
        ref = (torch.nn.functional.cross_entropy(lpt, t) + torch.nn.functional.cross_entropy(lpi, t)) / 2
        assert abs(out["loss"].item() - ref.item()) <= 1e-5 * abs(ref.item()), (out["loss"].item(), ref.item())


def test_logits_first_argmax_on_ties(cuda):
    from pigeon_b200 import ops
    img = torch.tensor([[1.0, 0.0], [0.0, 1.0]])
    txt = torch.tensor([[0.0, 2.0], [1.0, 0.0], [0.0, 1.0], [3.0, 0.0]])     # exact ties between captions
    out = ops.clip_logits(img.to(cuda), txt.to(cuda), 0.0, pred=True)
    assert out["pred"].cpu().tolist() == [1, 0]


# ------------------------------------------------------------------------------------------------ CLIPModel
def _model(cuda, td, vd, seed, std, projection_dim=None):
    from pigeon_b200 import CLIPModel, synthetic
    sd = synthetic.random_clip_state_dict(td, vd, seed=seed, std=std, projection_dim=projection_dim)
    m = CLIPModel(td, vd, projection_dim=projection_dim or td.hidden)
    m.load_state_dict(sd)
    return m.to(cuda).eval(), sd


def test_clip_model_matches_hf_golden_tiny(cuda):
    """The tiny geometry of tests/golden/clip.npz (HF CLIPModel outputs) through pigeon_b200.CLIPModel."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_clip_golden as mk
    g = mk.GEOMETRIES["tiny"]
    z = np.load(os.path.join(ROOT, "tests", "golden", "clip.npz"))
    m, _ = _model(cuda, g["text"], g["vision"], g["seed"], g["std"], g["projection"])
    px = mk.pixels(g["n_images"], g["vision"].image_size, g["px_seed"])
    o = m(input_ids=torch.from_numpy(z["tiny_input_ids"]).to(cuda), pixel_values=px.to(cuda),
          attention_mask=torch.from_numpy(z["tiny_attention_mask"]).to(cuda), return_loss=True)
    scale = math.exp(float(m.logit_scale.detach()))
    assert _rel(o.text_embeds, z["tiny_text_embeds"]) < REL_TOL
    assert _rel(o.image_embeds, z["tiny_image_embeds"]) < REL_TOL
    assert (o.logits_per_image.cpu() - torch.from_numpy(z["tiny_logits_per_image"])).abs().max() <= 1e-3 * scale
    assert abs(o.loss.item() - float(z["tiny_loss"])) <= 1e-3 * abs(float(z["tiny_loss"]))


def test_clip_model_forward_large(cuda):
    """Real geometry (CLIP-L/14-336 towers) on 4 images x 4 captions against the fp32 oracle, then the same through
    get_caption_probabilities / zero_shot_accuracy."""
    import clip_oracle
    from pigeon_b200 import TextDims, VitDims, get_caption_probabilities, zero_shot_accuracy
    td, vd = TextDims(), VitDims()
    m, sd = _model(cuda, td, vd, seed=31, std=0.02)
    ids, mask = _captions([77, 6, 30, 14], td.vocab, 32)
    px = torch.randn(4, 3, 336, 336, generator=torch.Generator().manual_seed(33))
    o = m(input_ids=ids.to(cuda), pixel_values=px.to(cuda), attention_mask=mask.to(cuda), return_loss=True)
    torch.cuda.synchronize()
    ref = clip_oracle.clip_forward(sd, ids, px, mask, text_heads=td.heads, text_layers=td.layers, patch=vd.patch_size,
                                   vision_heads=vd.heads, vision_layers=vd.layers, eps=td.ln_eps, return_loss=True)
    scale = math.exp(float(sd["logit_scale"]))
    e_t, e_i = _rel(o.text_embeds, ref["text_embeds"]), _rel(o.image_embeds, ref["image_embeds"])
    d_log = (o.logits_per_image.cpu() - ref["logits_per_image"]).abs().max().item()
    d_loss = abs(o.loss.item() - ref["loss"].item()) / abs(ref["loss"].item())
    print(f"CLIPModel CLIP-L/14-336: text_embeds {e_t:.3e} image_embeds {e_i:.3e} max|d logits| {d_log:.3e} "
          f"(bound {1e-3 * scale:.3e}) loss rel {d_loss:.3e}")
    _record(f"clip_model_large (4 images x 4 captions) vs fp32 CPU oracle: rel-L2 text_embeds {e_t:.3e}, image_embeds "
            f"{e_i:.3e}, max |d logits| {d_log:.3e} (exp(logit_scale) = {scale:.2f}), loss rel {d_loss:.3e}")
    assert e_t < REL_TOL and e_i < REL_TOL
    assert d_log <= 1e-3 * scale
    assert d_loss <= 1e-3
    assert torch.equal(o.logits_per_text.cpu(), o.logits_per_image.cpu().T)
    lpi = ref["logits_per_image"]
    top2 = lpi.topk(2, dim=1).values
    clear = top2[:, 0] - top2[:, 1] > 2 * 1e-3 * scale
    pred = o.logits_per_image.softmax(dim=1).argmax(dim=1).cpu()
    assert torch.equal(pred[clear], lpi.argmax(1)[clear])
    probs = get_caption_probabilities(m, px.to(cuda), ids.to(cuda), mask.to(cuda))
    assert (probs.cpu() - lpi.softmax(1)).abs().max().item() <= 1e-3 * scale
    acc = zero_shot_accuracy(m, px.to(cuda), ids.to(cuda), lpi.argmax(1), mask.to(cuda))
    assert acc == 1.0 or not bool(clear.all())


def test_clip_errors(cuda):
    from pigeon_b200 import TextDims, VitDims
    td = TextDims(vocab=1000, max_positions=16, hidden=256, heads=4, intermediate=512, layers=1)
    vd = VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    m, _ = _model(cuda, td, vd, seed=1, std=0.05)
    px = torch.randn(2, 3, 56, 56).to(cuda)
    with pytest.raises(ValueError):
        m(input_ids=torch.ones(2, 17, dtype=torch.int64, device=cuda), pixel_values=px)
    with pytest.raises(ValueError):
        m.get_text_features(torch.ones(2, 17, dtype=torch.int64, device=cuda))
    with pytest.raises(ValueError):
        m(input_ids=torch.ones(3, 4, dtype=torch.int64, device=cuda), pixel_values=px, return_loss=True)
    o = m(input_ids=torch.ones(3, 4, dtype=torch.int64, device=cuda), pixel_values=px)     # no loss: any counts
    assert o.loss is None and o.logits_per_image.shape == (2, 3)
