"""Pretraining from image files on the GPU: `ClipImageProcessor(windows=...)` against the host route (the reference's
Pillow crop or pad, then the same processor) on every item of tests/golden/pretrain_data.npz, the window kernel per
element on both sides of its grid cap, `FilesPretrainer` against `CLIPPretrainer` on rows built from the same items,
and `run.py pretrain` from a metadata CSV end to end."""
import os
import random
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from test_pretrain_data_host import make_dataset, write_golden_tree  # noqa: E402

KEYS = ["streetview/train/0", "streetview/val/0", "yfcc/train/0", "yfcc/val/0"]


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("pretrain_data")
    write_golden_tree(root)
    return root


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("png", [False, True])
def test_windows_match_host_route_on_golden_items(cuda, tree, dtype, png):
    from pigeon_b200.preprocess import ClipImageProcessor
    from pigeon_b200.pretrain_data import read_batch
    proc = ClipImageProcessor(device=cuda, dtype=dtype, png=png)
    for key in KEYS:
        ds = make_dataset(tree, key)
        _, files, windows, fills = read_batch(ds, list(range(len(ds))))       # panorama strips share their file
        got = proc(images=files, windows=windows, fills=fills)["pixel_values"]
        host = [np.asarray(ds.item_pil(i)[0].convert("RGB")) for i in range(len(ds))]
        want = proc(images=host)["pixel_values"]
        assert torch.equal(got, want), key


def _pad(a, x0, y0, w, h, fill):
    """a[y0:y0+h, x0:x0+w] of an [H, W, 3] array, `fill` outside it."""
    out = np.empty((h, w, 3), np.uint8)
    out[:] = np.asarray(fill, np.uint8)
    H, W = a.shape[:2]
    ys, xs = max(y0, 0), max(x0, 0)
    ye, xe = min(y0 + h, H), min(x0 + w, W)
    if ye > ys and xe > xs:
        out[ys - y0:ye - y0, xs - x0:xe - x0] = a[ys:ye, xs:xe]
    return out


def test_windows_inside_outside_and_larger(cuda):
    from pigeon_b200.preprocess import ClipImageProcessor, CropWindow
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (233, 301, 3), dtype=np.uint8)
    cases = [((10, 7, 200, 150), (0, 0, 0)), ((0, 0, 301, 233), (0, 0, 0)), ((-40, 100, 250, 250), (200, 30, 90)),
             ((250, -60, 120, 90), (1, 2, 3)), ((-150, -100, 596, 596), (0, 0, 0)), ((-3, -5, 310, 240), (9, 9, 9)),
             ((400, 300, 50, 40), (255, 0, 128))]                                      # entirely outside: all fill
    for dtype in (torch.float32, torch.float16):
        proc = ClipImageProcessor(device=cuda, dtype=dtype)
        dev = torch.from_numpy(img).to(cuda)
        got = proc(images=[dev] * len(cases), windows=[CropWindow(*w) for w, _ in cases],
                   fills=[f for _, f in cases])["pixel_values"]
        want = proc(images=[_pad(img, *w, f) for w, f in cases])["pixel_values"]
        assert torch.equal(got, want)
        full = proc(images=[dev], windows=[CropWindow(0, 0, 301, 233)])["pixel_values"]
        assert torch.equal(full, proc(images=[dev])["pixel_values"])               # the no-window path's bits


@pytest.mark.parametrize("n", [65535, 65538])
def test_window_kernel_per_element_across_grid_cap(cuda, n):
    """Every output element of `n` windowed images (grid.y is capped at 65535 images) equals the unwindowed pre-processing
    of the same image padded on the host."""
    from pigeon_b200.preprocess import ClipImageProcessor
    rng = np.random.default_rng(n)
    base = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((9, 13), (16, 7), (5, 5))]
    combos = [(0, (0, 0, 13, 9), (0, 0, 0)), (1, (-3, 2, 12, 15), (7, 200, 3)), (2, (-4, -4, 13, 11), (255, 1, 2)),
              (0, (4, -6, 9, 21), (50, 60, 70)), (1, (1, 1, 5, 14), (0, 0, 0))]
    size = 8
    proc = ClipImageProcessor(size=size, device=cuda)
    want = proc(images=[_pad(base[b], *w, f) for b, w, f in combos])["pixel_values"]
    dev = [torch.from_numpy(a).to(cuda) for a in base]
    which = np.arange(n) % len(combos)
    wins = [combos[k][1] + (combos[k][2],) for k in which]
    got = proc.preprocess_device([dev[combos[k][0]] for k in which], wins)
    assert got.shape == (n, 3, size, size)
    idx = torch.from_numpy(which).to(cuda)
    assert torch.equal(got, want[idx])


def _tiny_model(cuda, seed=31):
    from make_clip_train_golden import GEOMETRIES
    from pigeon_b200 import CLIPModel, synthetic
    g = GEOMETRIES["mid"]
    m = CLIPModel(g["text"], g["vision"], projection_dim=g["projection"])
    m.load_state_dict(synthetic.random_clip_state_dict(g["text"], g["vision"], seed=seed, std=0.05,
                                                       projection_dim=g["projection"]))
    return m.to(cuda)


def _args(out_dir):
    return SimpleNamespace(output_dir=str(out_dir), per_device_train_batch_size=4, per_device_eval_batch_size=4,
                           gradient_accumulation_steps=2, num_train_epochs=1, max_steps=-1, learning_rate=2e-3,
                           adam_beta1=0.9, adam_beta2=0.98, adam_epsilon=1e-6, weight_decay=0.1, max_grad_norm=4.6,
                           warmup_ratio=0.2, warmup_steps=0, lr_scheduler_type="linear", logging_strategy="steps",
                           logging_steps=1, evaluation_strategy="no", save_strategy="no", save_steps=500, seed=42)


def _recording(cls):
    class Rec(cls):
        batches = []

        def get_train_dataloader(self):
            loader, sampler = super().get_train_dataloader()
            outer = self

            class L:
                def __len__(self):
                    return len(loader)

                def __iter__(self):
                    for b in loader:
                        outer.batches.append({k: v.detach().cpu().clone() for k, v in b.items()})
                        yield b
            return L(), sampler
    Rec.batches = []
    return Rec


def test_files_trainer_matches_rows_trainer(cuda, tree, tmp_path):
    """Same items through FilesPretrainer (files, captions drawn in sampler order, workers reading) and CLIPPretrainer
    (rows of pixel_values and input_ids built beforehand with the captions that order gives): the same batches bit for
    bit, and the same losses and parameters within the noise of two identical runs."""
    from transformers import CLIPTokenizer
    from torch.utils.data import DistributedSampler
    from pigeon_b200.preprocess import ClipImageProcessor
    from pigeon_b200.pretrain import CLIPCollator, CLIPPretrainer
    from pigeon_b200.pretrain_data import FilesCollator, FilesPretrainer
    tok = CLIPTokenizer.from_pretrained(os.path.join(str(tree), "tokenizer"))
    ds = make_dataset(tree, "streetview/train/1")
    m1 = _tiny_model(cuda)
    proc = ClipImageProcessor(size=m1.vision_dims.image_size, device=cuda)
    col = FilesCollator(proc, tok, num_workers=2)
    Files, Rows = _recording(FilesPretrainer), _recording(CLIPPretrainer)

    random.seed(5)
    t1 = Files(m1, _args(tmp_path / "a"), ds, None, col)
    loss1 = t1.train()

    random.seed(5)                                       # the captions the files route drew, in its sampler order
    sampler = DistributedSampler(ds, num_replicas=1, rank=0, shuffle=True, seed=42)
    sampler.set_epoch(0)
    order = list(sampler)[:len(ds) // 4 * 4]
    caps = {i: ds.caption(i) for i in order}
    rows = []
    for i in range(len(ds)):
        data, window, fill = ds.read(i)
        px = col.pixels([data], [window], [fill])[0].cpu()
        ids = tok(caps.get(i, ""), truncation=True)
        rows.append({"pixel_values": px, "input_ids": ids["input_ids"], "attention_mask": ids["attention_mask"]})
    m2 = _tiny_model(cuda)
    t2 = Rows(m2, _args(tmp_path / "b"), rows, None, CLIPCollator(pad_token_id=tok.pad_token_id))
    loss2 = t2.train()

    assert len(Files.batches) == len(Rows.batches) == len(ds) // 4 // 2 * 2     # the last update ends the run
    for a, b in zip(Files.batches, Rows.batches):
        for k in ("input_ids", "attention_mask", "pixel_values"):
            assert torch.equal(a[k], b[k]), k
    l1 = [e["loss"] for e in t1.state.log_history if "loss" in e]
    l2 = [e["loss"] for e in t2.state.log_history if "loss" in e]
    assert len(l1) == len(l2) >= 3
    assert np.allclose(l1, l2, rtol=1e-3) and abs(loss1 - loss2) <= 1e-3 * abs(loss2)
    for (n, p), (_, q) in zip(m1.named_parameters(), m2.named_parameters()):
        d = (p.detach().double() - q.detach().double()).norm() / max(q.detach().double().norm().item(), 1e-12)
        assert d <= 5e-2, n


def test_accuracy_is_a_share_over_whole_batches(cuda, tree):
    from transformers import CLIPTokenizer
    from pigeon_b200.preprocess import ClipImageProcessor
    from pigeon_b200.pretrain_data import FilesCollator
    tok = CLIPTokenizer.from_pretrained(os.path.join(str(tree), "tokenizer"))
    m = _tiny_model(cuda)
    ds = make_dataset(tree, "streetview/train/1")
    ds.collator = FilesCollator(ClipImageProcessor(size=m.vision_dims.image_size, device=cuda), tok)
    random.seed(0)
    acc = ds.accuracy(m, batch_size=16, trials=30)          # 36 items: two whole batches
    assert 0.0 <= acc <= 1.0 and (acc * 32) == pytest.approx(round(acc * 32))
    assert np.isnan(ds.accuracy(m, batch_size=64))


def test_run_pretrain_from_csv_end_to_end(cuda, tree, tmp_path):
    m = _tiny_model(cuda)
    m.save_pretrained(str(tmp_path / "tiny"))
    os.makedirs(tmp_path / "data")                          # the image folders config names, relative to the run
    os.symlink(os.path.join(str(tree), "streetview"), tmp_path / "data" / "streetview_outputs_cropped")
    os.symlink(os.path.join(str(tree), "panoramas"), tmp_path / "data" / "streetview_part_2_data")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "run.py"), "pretrain", "tiny", "-l",
                        os.path.join(str(tree), "data_pretrain.csv"), "-a", "-w", "2", "--tokenizer",
                        os.path.join(str(tree), "tokenizer")], cwd=str(tmp_path), capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    assert "Before traing: Accuracy" in r.stdout and "After training: Accuracy" in r.stdout
