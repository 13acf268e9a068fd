"""Selective repacking of both towers' engines on the H100: after an in-place change of one encoder layer, or of one
embedding parameter, `engine()` keeps the same engine, replaces the packed tensors of the moved group only, and computes
what a freshly built engine computes, bit for bit.  A per-pass limit changed after the first forward reaches the engine."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _vision(cuda):
    from pigeon_b200 import CLIPVisionTower, VitDims, synthetic
    from pigeon_b200.vit_engine import VitEngine
    dims = VitDims(image_size=56, patch_size=14, hidden=256, heads=4, intermediate=512, layers=3)
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=3, std=0.05))
    tower = tower.to(cuda)
    px = torch.randn(5, 3, 56, 56, generator=torch.Generator().manual_seed(4)).to(cuda)
    return dict(tower=tower, model=tower.vision_model, emb=tower.vision_model.embeddings.class_embedding,
                limit="max_views_per_pass", run=lambda eng: eng.forward(px, return_hidden=True),
                need=lambda eng, k: eng.workspace_bytes(k),
                fresh=lambda k: VitEngine(tower.state_dict(), dims, device=cuda, max_views_per_pass=k))


def _text(cuda):
    from pigeon_b200 import CLIPTextTower, TextDims, VitDims, synthetic
    from pigeon_b200.clip_text import TextEngine
    td = TextDims(vocab=1000, max_positions=16, hidden=256, heads=4, intermediate=512, layers=3)
    vd = VitDims(image_size=28, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    sd = synthetic.random_clip_state_dict(td, vd, seed=5, std=0.05)
    tower = CLIPTextTower(td)
    tower.load_state_dict({k: v for k, v in sd.items() if k.startswith("text_model.")})
    tower = tower.to(cuda)
    ids = torch.randint(0, td.vocab, (5, 12), generator=torch.Generator().manual_seed(6)).to(cuda)
    return dict(tower=tower, model=tower.text_model, emb=tower.text_model.embeddings.token_embedding.weight,
                limit="max_texts_per_pass", run=lambda eng: eng.forward(ids, return_hidden=True),
                need=lambda eng, k: eng.workspace_bytes(k, ids.shape[1]),
                fresh=lambda k: TextEngine(tower.state_dict(), td, device=cuda, max_texts_per_pass=k))


def _assert_same_bits(a, b):
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


@pytest.mark.parametrize("make", [_vision, _text], ids=["vision", "text"])
@pytest.mark.parametrize("moved", [1, "embeddings"])
def test_only_the_moved_group_is_repacked(cuda, make, moved):
    t = make(cuda)
    tower = t["tower"]
    setattr(tower, t["limit"], 2)
    t["run"](tower.engine())
    eng, packs = tower.engine(), dict(tower.engine()._packs)
    with torch.no_grad():
        if moved == "embeddings":
            t["emb"].mul_(1.5)
        else:
            t["model"].encoder.layers[moved].mlp.fc1.weight.add_(0.01)
    assert tower.engine() is eng
    assert {g for g in packs if eng._packs[g] is not packs[g]} == {moved}
    _assert_same_bits(t["run"](eng), t["run"](t["fresh"](2)))


@pytest.mark.parametrize("make", [_vision, _text], ids=["vision", "text"])
def test_pass_limit_set_after_the_first_forward_is_used(cuda, make):
    t = make(cuda)
    tower = t["tower"]
    setattr(tower, t["limit"], 2)
    eng = tower.engine()
    t["run"](eng)
    assert eng._ws.numel() < t["need"](eng, 5)
    setattr(tower, t["limit"], 5)
    assert tower.engine() is eng and getattr(eng, t["limit"]) == 5
    out = t["run"](eng)
    assert eng._ws.numel() >= t["need"](eng, 5)           # one pass over the 5 inputs
    _assert_same_bits(out, t["run"](t["fresh"](5)))
