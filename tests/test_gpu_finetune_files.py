"""Fine-tuning from the image files of a raw four-view split (`train_model(..., collate_fn=encoded_eval_collate,
processor=ClipImageProcessor())`) against fine-tuning from the same files' pixel_values, made beforehand by the same
processor and passed the way pre-processed datasets are.  With the same torch seed, two epochs with gradient
accumulation 2 and the multi-task heads, at a batch size that divides the split and at one that leaves a ragged last
batch, the model receives bit-identical inputs in every training and evaluation call.  With the tower frozen (geocell
and auxiliary heads trained) the per-epoch losses, evaluation results, saved checkpoints and parameters are
bit-identical too.  With the tower trained under the reference freeze policy the losses agree to 1e-5 and the
parameters within AdamW's step size: the tower backward sums LayerNorm and bias gradients across CTAs with atomicAdd
(csrc/train_vit.cu), so two runs of the same route differ in the last bits as well, and AdamW's normalised step can
turn that into up to about lr for entries whose gradient is rounding noise.  The files are baseline JPEGs decoded on
the GPU plus a progressive JPEG and a PNG that Pillow decodes on the host."""
import io
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
datasets = pytest.importorskip("datasets")
VIEWS = ["image", "image_2", "image_3", "image_4"]
C = 30                       # geocells of the synthetic head


@pytest.fixture(autouse=True)
def _rows_without_torchvision(monkeypatch):
    """datasets' torch formatter imports torchvision.io.VideoReader whenever torchvision is loaded (an earlier test's
    transformers import loads it), and this torchvision has none: format the rows as a process without it does."""
    monkeypatch.delitem(sys.modules, "torchvision", raising=False)


@pytest.fixture(scope="module", autouse=True)
def _keep_global_rng():
    """The runs here seed torch's global generators, which later modules' unseeded initialisations also use: leave
    them as this module found them."""
    with torch.random.fork_rng(devices=range(torch.cuda.device_count())):
        yield


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _files(n):
    """4 n encoded views: baseline JPEGs of assorted sizes, one progressive JPEG and one PNG."""
    from PIL import Image
    from pigeon_b200 import synthetic
    sizes = [(240, 320), (320, 240), (336, 336), (200, 500), (97, 131)]
    out = []
    for k in range(4 * n):
        img = Image.fromarray(synthetic.synthetic_photo(*sizes[k % len(sizes)], seed=k))
        f = io.BytesIO()
        if k == 5:
            img.save(f, "JPEG", quality=90, progressive=True)
        elif k == 10:
            img.save(f, "PNG")
        else:
            img.save(f, "JPEG", quality=88 + k % 8, subsampling=2 if k % 3 else 0)
        out.append(f.getvalue())
    return out


def _split(n, seed):
    rng = np.random.default_rng(seed)
    files = _files(n)
    data = {c: [{"bytes": files[4 * r + v], "path": None} for r in range(n)] for v, c in enumerate(VIEWS)}
    from pigeon_b200 import synthetic
    data.update(labels=synthetic.synthetic_geocells(n, seed).tolist(), labels_clf=rng.integers(0, C, n).tolist(),
                labels_multi_task=rng.normal(size=(n, 6)).tolist(), labels_climate=rng.dirichlet(np.ones(28), n).tolist(),
                labels_month=rng.integers(0, 12, n).tolist(), heading=rng.uniform(0, 360, n).tolist())
    f = {c: datasets.Image() for c in VIEWS}
    f.update(labels=datasets.Sequence(datasets.Value("float64")), labels_clf=datasets.Value("int64"),
             labels_multi_task=datasets.Sequence(datasets.Value("float32")),
             labels_climate=datasets.Sequence(datasets.Value("float32")), labels_month=datasets.Value("int64"),
             heading=datasets.Value("float32"))
    return datasets.Dataset.from_dict(data, features=datasets.Features(f)).with_format("torch"), files


class Twin(torch.utils.data.Dataset):
    """The split's rows with pixel_values instead of image columns, as a pre-processed dataset yields them."""

    def __init__(self, split, px):
        self.labels = split.remove_columns(VIEWS)
        self.px = px

    def __len__(self):
        return len(self.px)

    def __getitem__(self, i):
        if isinstance(i, str):
            return self.labels[i]
        return dict(self.labels[i], pixel_values=self.px[i])


def _model(seed, tower_trains):
    from pigeon_b200 import SuperGuessr, synthetic
    from pigeon_b200.super_guessr import CLIPVisionTower
    from pigeon_b200.vit_engine import VitDims
    dims = VitDims(image_size=336, patch_size=14, hidden=256, heads=4, intermediate=512, layers=2)
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=seed, std=0.05), strict=True)
    torch.manual_seed(seed)
    sg = SuperGuessr(tower, panorama=True, multi_task=True, should_smooth_labels=True, num_candidates=5,
                     freeze_base=not tower_trains, geocells=synthetic.synthetic_geocells(C, seed)).to("cuda")
    for p in sg.base_model.vision_model.encoder.layers[:-1].parameters():      # reference freeze policy
        p.requires_grad = False
    inputs = []

    def forward(**kw):                                   # what every training and evaluation call receives
        inputs.append({k: v.detach().cpu().clone() for k, v in kw.items()})
        return type(sg).forward(sg, **kw)
    sg.forward = forward
    return sg, inputs


@pytest.mark.parametrize("tower_trains", [False, True])
@pytest.mark.parametrize("batch", [4, 5])
def test_train_from_files_equals_train_from_pixel_values(cuda, tmp_path, monkeypatch, batch, tower_trains):
    from pigeon_b200 import benchmark, loops, training
    from pigeon_b200.preprocess import ClipImageProcessor
    splits = {"train": _split(12, 1), "val": _split(5, 2)}
    maker = ClipImageProcessor(device=cuda)
    twins = {}
    for k, (split, files) in splits.items():
        px = maker(images=files)["pixel_values"].cpu()
        twins[k] = Twin(split, px.view(len(split), 12, 336, 336))
    encoded = {k: benchmark.EvalDataset(split).encoded() for k, (split, _) in splits.items()}

    class Args:
        learning_rate = 1e-3
        per_device_train_batch_size = batch
        per_device_eval_batch_size = 3
        num_train_epochs = 2
        gradient_accumulation_steps = 2

    evals = []
    real = training.evaluate_model

    def spy(*a, **kw):
        evals[-1].append(real(*a, **kw))
        return evals[-1][-1]
    monkeypatch.setattr(training, "evaluate_model", spy)
    runs = []
    for route, ds, kw in (("pixels", twins, {}),
                          ("files", encoded, dict(collate_fn=loops.encoded_eval_collate,
                                                  processor=ClipImageProcessor(device=cuda)))):
        evals.append([])
        sg, inputs = _model(7, tower_trains)
        torch.manual_seed(11)
        path = str(tmp_path / f"{route}.model")
        training.train_model(sg, ds, False, False, Args(), None, save_path=path, **kw)
        runs.append((sg, inputs, sg.train_history, torch.load(path, map_location="cpu"), kw.get("processor")))
    (a, in_a, hist_a, saved_a, _), (b, in_b, hist_b, saved_b, proc) = runs
    assert proc.gpu_decoded > 0 and proc.host_decoded >= 2 * 2 * 2          # both routes, both epochs' train + val
    steps = 2 * (-(-12 // batch) + 2)                                         # per epoch: train batches + 2 of val
    assert len(in_a) == len(in_b) == steps
    for xa, xb in zip(in_a, in_b):
        assert sorted(xa) == sorted(xb) == ["heading", "labels", "labels_clf", "labels_climate", "labels_month",
                                            "labels_multi_task", "pixel_values"]
        for k in xa:
            assert xa[k].dtype == xb[k].dtype and torch.equal(xa[k], xb[k]), k
    sa, sb = a.state_dict(), b.state_dict()
    assert sorted(sa) == sorted(sb) == sorted(saved_a) == sorted(saved_b)
    assert len(hist_a) == 2 and np.isfinite(hist_a).all() and len(evals[0]) == len(evals[1]) == 2
    if tower_trains:
        np.testing.assert_allclose(hist_a, hist_b, rtol=1e-5)
        # AdamW's normalised step moves an entry by up to about lr whatever its gradient's size, so an entry whose
        # gradient is rounding noise can move either way on each route: at most 2 lr apart per optimizer step
        updates = 2 * (-(-(-(-12 // batch)) // 2))
        for k in sa:
            assert (sa[k].double() - sb[k].double()).abs().max() <= 2 * Args.learning_rate * updates, k
    else:
        assert hist_a == hist_b
        for ea, eb in zip(*evals):
            assert sorted(ea) == sorted(eb)
            for k in ea:
                if isinstance(ea[k], np.ndarray):
                    assert ea[k].dtype == eb[k].dtype and np.array_equal(ea[k], eb[k]), k
                else:
                    assert ea[k] == eb[k], k
        for k in sa:
            assert torch.equal(sa[k], sb[k]) and torch.equal(saved_a[k], saved_b[k]), k
    moved = _model(7, tower_trains)[0].state_dict()
    assert not torch.equal(moved["multi_task_head.weight"], sa["multi_task_head.weight"])
    fc1 = "base_model.vision_model.encoder.layers.1.mlp.fc1.weight"
    assert torch.equal(moved[fc1], sa[fc1]) != tower_trains
