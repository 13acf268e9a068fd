"""CPU-only checks of the CLIPModel training step: the ctypes mirrors of the new C structs, the build of the new kernels
(no register spills; the unmasked attention and GEMM kernels compile to the SASS pinned in
tests/golden/sass_sm90a_unmasked.json), the HF-autograd golden fixture, and the errors raised before any kernel runs."""
import ctypes as C
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pigeon_b200", "csrc")


def test_training_structs_match_the_header_layout(tmp_path):
    from pigeon_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    pairs = {"pg_text_saved": _lib.TextSaved, "pg_text_grads": _lib.TextGrads}
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


def test_every_source_is_built_and_exported():
    from pigeon_b200 import _build, _lib
    on_disk = {f for f in os.listdir(CSRC) if f.endswith(".cu")}
    assert on_disk <= set(_build.SOURCES), on_disk - set(_build.SOURCES)
    header = open(os.path.join(ROOT, "include", "pigeon_b200.h")).read()
    for name in ("pg_text_forward_train", "pg_text_backward_workspace_bytes", "pg_text_backward", "pg_vit_backward_cls",
                 "pg_clip_loss_grad", "pg_clip_loss_grad_workspace_bytes", "pg_attention_f16_masked_lse",
                 "pg_attention_backward_masked", "pg_layernorm_f32"):
        assert re.search(r"\b" + name + r"\(", header), name
        assert name in _lib.SIGNATURES, name


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


def test_new_kernels_do_not_spill(tmp_path):
    """-Xptxas -v of the sources holding the new kernels: no local-memory spills."""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    from pigeon_b200 import _build
    for src in ("clip_train.cu", "attention_bwd_wgmma.cu", "attention_wgmma.cu", "vit_train_capi.cu"):
        r = subprocess.run([nvcc, *_build._flags(), "-Xptxas", "-v", "-I", os.path.join(ROOT, "include"), "-c",
                            os.path.join(CSRC, src), "-o", str(tmp_path / (src + ".o"))], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        spills = [l for l in r.stderr.splitlines() if "spill" in l and not re.search(r"\b0 bytes spill stores, 0 bytes spill loads", l)]
        assert not spills, (src, spills)


def _sass_digests(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    res = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", out, re.S):
        name = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+", "ANON", m.group(1))
        res[name] = hashlib.sha256(re.sub(r"/\*[0-9a-f]{4}\*/", "", m.group(2)).encode()).hexdigest()
    return res


def test_unmasked_attention_and_gemm_sass_is_unchanged(tmp_path):
    """The masked variants are separate instantiations: the vision tower's attention forward / backward and every GEMM
    compile to the SASS they had before the training step was added (digests in tests/golden/sass_sm90a_unmasked.json)."""
    nvcc = _nvcc()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if nvcc is None or not os.path.exists(cuobjdump):
        pytest.skip("CUDA toolkit not available")
    from pigeon_b200 import _build
    pinned = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_sm90a_unmasked.json")))
    got = {}
    for f in ("attention_wgmma", "attention_bwd_wgmma", "gemm_wgmma"):
        obj = str(tmp_path / (f + ".o"))
        r = subprocess.run([nvcc, *_build._flags(), "-I", os.path.join(ROOT, "include"), "-c", os.path.join(CSRC, f + ".cu"),
                            "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        got.update({f"{f}:{k}": v for k, v in _sass_digests(obj).items()})
    for k, v in pinned.items():
        assert got.get(k) == v, k


def test_train_golden_fixture_is_small_and_complete():
    path = os.path.join(ROOT, "tests", "golden", "clip_train.npz")
    assert os.path.getsize(path) < 1 << 20
    z = np.load(path)
    for name in ("tiny", "mid"):
        keys = {k[len(name) + 5:] for k in z.files if k.startswith(name + "/sub/")}
        assert "logit_scale" in keys and "visual_projection.weight" in keys and "text_projection.weight" in keys
        assert "text_model.embeddings.token_embedding.weight" in keys
        assert "text_model.embeddings.position_embedding.weight" in keys
        assert "vision_model.post_layernorm.weight" in keys and "text_model.final_layer_norm.bias" in keys
    assert z["mid/input_ids"].shape == (8, 77)


def _tiny_model():
    from pigeon_b200 import CLIPModel, TextDims, VitDims
    td = TextDims(vocab=100, max_positions=8, hidden=256, heads=4, intermediate=512, layers=1)
    vd = VitDims(image_size=28, patch_size=14, hidden=256, heads=4, intermediate=512, layers=1)
    return CLIPModel(td, vd, projection_dim=256)


def test_training_step_on_a_cpu_model_fails_loudly():
    from pigeon_b200 import PigeonB200Error
    m = _tiny_model()
    with pytest.raises(PigeonB200Error):
        m.forward_train(torch.tensor([[98, 5, 99]]), torch.zeros(1, 3, 28, 28))
    with pytest.raises(PigeonB200Error):
        m.backward()
