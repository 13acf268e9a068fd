"""CPU-only checks of the CLIP text tower / CLIPModel: the fp32 oracle (tests/clip_oracle.py) against HF CLIPModel outputs
stored in tests/golden/clip.npz (tools/make_clip_golden.py), the ctypes mirrors of the new C structs, the HF key names of
`pigeon_b200.CLIPModel`, and the no-GPU error path."""
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "clip.npz")


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).norm() / b.norm()).item()


def _inputs(name):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_clip_golden as mk
    from pigeon_b200 import synthetic
    g = mk.GEOMETRIES[name]
    z = np.load(GOLDEN)
    sd = synthetic.random_clip_state_dict(g["text"], g["vision"], seed=g["seed"], std=g["std"], projection_dim=g["projection"])
    px = mk.pixels(g["n_images"], g["vision"].image_size, g["px_seed"])
    return g, sd, px, {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + "_")}


@pytest.mark.parametrize("name", ["tiny", "large"])
def test_oracle_matches_hf_golden(name):
    import clip_oracle
    g, sd, px, z = _inputs(name)
    td, vd = g["text"], g["vision"]
    ids, mask = torch.from_numpy(z["input_ids"]), torch.from_numpy(z["attention_mask"])
    n_loss = int(z["n_loss"])
    o = clip_oracle.clip_forward(sd, ids, px, mask, text_heads=td.heads, text_layers=td.layers, patch=vd.patch_size,
                                 vision_heads=vd.heads, vision_layers=vd.layers, eps=td.ln_eps)
    assert _rel(o["text_embeds"], z["text_embeds"]) <= 2e-6
    assert _rel(o["image_embeds"], z["image_embeds"]) <= 2e-6
    assert _rel(o["logits_per_image"], z["logits_per_image"]) <= 2e-6
    assert _rel(o["logits_per_text"], z["logits_per_text"]) <= 2e-6
    t = torch.arange(n_loss)
    lpt = o["logits_per_text"][:n_loss, :n_loss]
    loss = (torch.nn.functional.cross_entropy(lpt, t) + torch.nn.functional.cross_entropy(lpt.T, t)) / 2
    assert abs(loss.item() - float(z["loss"])) <= 2e-6 * abs(float(z["loss"]))
    if name == "tiny":
        assert _rel(o["last_hidden_state"], z["last_hidden_state"]) <= 2e-6
    else:
        pos = torch.from_numpy(z["lhs_positions"])
        rows = torch.stack([o["last_hidden_state"][b, pos[b]] for b in range(pos.shape[0])])
        assert _rel(rows, z["last_hidden_state_rows"]) <= 2e-6
    # pooling pinned to 4.23.1's argmax of the ids; the fixture's captions end in EOS = vocab - 1 (the largest id)
    assert (ids.argmax(-1) == mask.sum(-1) - 1).all()


def test_golden_fixture_is_small():
    assert os.path.getsize(GOLDEN) < 1 << 20


def test_text_structs_match_the_header_layout(tmp_path):
    import ctypes as C
    import shutil
    import subprocess
    from pigeon_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    pairs = {"pg_text_config": _lib.TextConfig, "pg_text_weights": _lib.TextWeights}
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "pigeon_b200.h"', "int main(void) {"]
    for cname, cls in pairs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    r = subprocess.run([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True).stdout.splitlines())
    for cname, cls in pairs.items():
        assert int(got[cname]) == C.sizeof(cls), (cname, got[cname], C.sizeof(cls))
        for fname, _ in cls._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(cls, fname).offset, (cname, fname)


def test_clip_model_state_dict_uses_hf_key_names_and_roundtrips():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_clip_golden as mk
    from pigeon_b200 import CLIPModel, synthetic
    g = mk.GEOMETRIES["tiny"]
    td, vd = g["text"], g["vision"]
    hf = mk.hf_clip(td, vd, g["projection"], synthetic.random_clip_state_dict(td, vd, seed=1, projection_dim=g["projection"]))
    hf_keys = {k for k in hf.state_dict() if "position_ids" not in k}
    m = CLIPModel(td, vd, projection_dim=g["projection"])
    assert set(m.state_dict()) == hf_keys
    m2 = CLIPModel.from_hf(hf)
    for k, v in hf.state_dict().items():
        if "position_ids" not in k:
            assert torch.equal(m2.state_dict()[k], v), k
    m.load_state_dict(m2.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), m2.state_dict().values()))
    # the towers read the same parameters the model registers
    assert m.text_tower.text_model.final_layer_norm.weight is m.text_model.final_layer_norm.weight
    assert m.vision_tower.vision_model.post_layernorm.bias is m.vision_model.post_layernorm.bias


def test_clip_no_gpu_fails_loudly():
    if torch.cuda.is_available():
        pytest.skip("has a GPU")
    from pigeon_b200 import CLIPModel, CLIPTextTower, PigeonB200Error, TextDims, VitDims, get_caption_probabilities, ops
    td = TextDims(vocab=100, max_positions=8, hidden=256, heads=4, intermediate=512, layers=1)
    vd = VitDims(image_size=28, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    m = CLIPModel(td, vd, projection_dim=256)
    ids = torch.tensor([[98, 5, 99]])
    px = torch.zeros(1, 3, 28, 28)
    with pytest.raises(PigeonB200Error):
        m(input_ids=ids, pixel_values=px, return_loss=True)
    with pytest.raises(PigeonB200Error):
        m.get_text_features(ids)
    with pytest.raises(PigeonB200Error):
        get_caption_probabilities(m, px, ids)
    with pytest.raises(PigeonB200Error):
        CLIPTextTower(td).pooled(ids)
    with pytest.raises(PigeonB200Error):
        ops.clip_logits(torch.zeros(2, 8), torch.zeros(2, 8), 1.0)
    with pytest.raises(PigeonB200Error):
        ops.attention_f16_masked(torch.zeros(8, 3 * 64, dtype=torch.float16), 1, 8, 1, causal=True)


def test_clip_argument_errors_before_any_kernel():
    """S > max_position_embeddings and a loss over unequal image / caption counts are ValueErrors (HF fails there too,
    the latter with an indexing error), raised before anything touches a device."""
    from pigeon_b200 import CLIPModel, TextDims, VitDims
    td = TextDims(vocab=100, max_positions=8, hidden=256, heads=4, intermediate=512, layers=1)
    vd = VitDims(image_size=28, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    m = CLIPModel(td, vd, projection_dim=256)
    with pytest.raises(ValueError):
        m(input_ids=torch.ones(1, 9, dtype=torch.int64), pixel_values=torch.zeros(1, 3, 28, 28))
    with pytest.raises(ValueError):
        m(input_ids=torch.ones(2, 4, dtype=torch.int64), pixel_values=torch.zeros(1, 3, 28, 28), return_loss=True)


def test_attention_mask_admits_only_ones():
    """HF's `_expand_mask` excludes every key whose mask is not exactly 1; the kernels get that as a 0/1 int64 mask."""
    from pigeon_b200.clip_text import admissible_keys
    m = torch.tensor([[1, 0, 2, -1, 1.5, 0.5, 1], [1, 1, 1, 1, 1, 1, 0]], dtype=torch.float64)
    want = torch.tensor([[1, 0, 0, 0, 0, 0, 1], [1, 1, 1, 1, 1, 1, 0]])
    for t in (m, m.float(), m.half(), m.to(torch.int64)):
        got = admissible_keys(t)
        assert got.dtype == torch.int64 and got.is_contiguous()
        assert torch.equal(got, want if t.is_floating_point() else (m.to(torch.int64) == 1).to(torch.int64))
    assert torch.equal(admissible_keys(torch.tensor([[True, False]])), torch.tensor([[1, 0]]))
