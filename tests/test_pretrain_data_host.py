"""Host side of pretraining from the reference's metadata CSV and image folders (pigeon_b200.pretrain_data) against the
unmodified reference's items in tests/golden/pretrain_data.npz (tools/make_pretrain_data_golden.py): index mapping,
captions under the same `random` seeds and index orders, crop windows, Pillow-path hashes; tokenisation against
CLIPTokenizer's own padding; and `run.py pretrain` routing.  No GPU."""
import hashlib
import json
import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "pretrain_data.npz")


def write_golden_tree(root):
    """The golden's input files under `root` (CSV paths of `v` files rooted there); returns the records."""
    G = np.load(GOLD)
    off = G["offsets"]
    for k, name in enumerate(G["names"]):
        data = G["blob"][off[k]:off[k + 1]].tobytes()
        if name.endswith(".csv"):
            data = data.replace(b"@ROOT@", str(root).encode())
        path = os.path.join(str(root), str(name))
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as f:
            f.write(data)
    return json.loads(G["records"].tobytes())


def make_dataset(root, key):
    """The pretrain_data dataset of a golden record key ('streetview/train/0', 'yfcc/val/1', ...)."""
    from pigeon_b200.pretrain_data import PretrainDataset, PretrainDatasetYFCC
    kind, split, aux = key.split("/")
    r = str(root)
    if kind == "streetview":
        return PretrainDataset(split, os.path.join(r, "data_pretrain.csv"), bool(int(aux)),
                               image_path=os.path.join(r, "streetview"), image_path_2=os.path.join(r, "panoramas"))
    return PretrainDatasetYFCC(split, os.path.join(r, "data_yfcc.csv"), bool(int(aux)),
                               image_path=os.path.join(r, "yfcc"), driving_side=os.path.join(r, "driving_side.json"))


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("pretrain_data")
    return root, write_golden_tree(root)


def reference_window(item):
    """(x0, y0, width, height) of the reference's crop from its recorded torchvision / Pillow calls."""
    calls = dict((k, v) for k, v in item["crop"])
    if "box" in calls:
        x0, y0, x1, y1 = (int(round(v)) for v in calls["box"])
        return x0, y0, x1 - x0, y1 - y0
    pad_l, pad_t = (calls["pad"][0], calls["pad"][1]) if "pad" in calls else (0, 0)
    if "crop" in calls:
        top, left, h, w = calls["crop"]
        return left - pad_l, top - pad_t, w, h
    if "pad" in calls:                                  # padded to exactly the crop size
        return -pad_l, -pad_t, item["size"][0], item["size"][1]
    return None                                         # no crop (`o` items): the whole image


def test_golden_covers_every_branch(tree):
    _, records = tree
    kinds = {c[0] for r in records.values() for it in r["items"] for c in it["crop"]}
    assert kinds == {"pad", "crop", "box"}
    assert any(it["mode"] == "P" for r in records.values() for it in r["items"])
    sizes = [it["size"] for r in records.values() for it in r["items"] if any(c[0] == "box" for c in it["crop"])]
    assert any(w != h for w, h in sizes)                # Pillow's rounding of an odd float box


@pytest.mark.parametrize("key", ["streetview/train/0", "streetview/train/1", "streetview/val/0", "streetview/val/1",
                                 "yfcc/train/0", "yfcc/train/1", "yfcc/val/0", "yfcc/val/1"])
def test_items_match_reference(tree, key):
    root, records = tree
    rec = records[key]
    ds = make_dataset(root, key)
    assert len(ds) == rec["len"]
    if rec["mapping"] is not None:
        assert [list(ds._convert_to_row_index(i)) for i in range(len(ds))] == rec["mapping"]
    for run in rec["captions"]:
        random.seed(run["seed"])
        assert [ds[i][3] for i in run["order"]] == run["captions"], run["seed"]
    for i, item in enumerate(rec["items"]):
        data, window, fill, _ = ds[i]
        assert isinstance(data, bytes)
        want = reference_window(item)
        if want is None:
            from PIL import Image
            import io
            want = (0, 0) + Image.open(io.BytesIO(data)).size
        assert tuple(window[:4]) == want, (i, window, item["crop"])
        assert fill is not None
        img, _ = ds.item_pil(i)
        assert list(img.size) == item["size"] and img.mode == item["mode"]
        sha = hashlib.sha256(np.ascontiguousarray(np.asarray(img.convert("RGB"))).tobytes()).hexdigest()
        assert sha == item["sha"], i


def test_read_draws_no_random(tree):
    root, _ = tree
    ds = make_dataset(root, "streetview/train/1")
    state = random.getstate()
    for i in range(len(ds)):
        ds.read(i)
    assert random.getstate() == state


def test_panorama_strips_share_one_read(tree):
    from pigeon_b200.pretrain_data import read_batch
    root, _ = tree
    ds = make_dataset(root, "streetview/train/0")
    strips = [i for i in range(len(ds)) if ds.locate(i)[1] == "l"][:5]
    idx, files, windows, fills = read_batch(ds, strips)
    assert idx == strips and all(f is files[0] for f in files)
    assert [w.clip[0] for w in windows] == [512 * c for c in range(5)]


def test_center_crop_and_box_helpers_match_torchvision_and_pillow():
    F = pytest.importorskip("torchvision.transforms.functional")
    from PIL import Image
    from pigeon_b200.pretrain_data import center_crop_origin, square_crop_box
    rng = np.random.default_rng(0)
    for _ in range(60):
        w, h, s = (int(v) for v in rng.integers(1, 40, 3))
        img = Image.fromarray(rng.integers(1, 256, (h, w, 3), dtype=np.uint8))
        got = np.asarray(F.center_crop(img, [s, s]))
        x0, y0 = center_crop_origin(w, h, s)
        assert np.array_equal(np.asarray(img.crop((x0, y0, x0 + s, y0 + s))), got), (w, h, s)
        d = min(w, h)
        box = ((w - d) / 2, (h - d) / 2, (w + d) / 2, (h + d) / 2)
        assert np.array_equal(np.asarray(img.crop(box)), np.asarray(img.crop(square_crop_box(w, h)))), (w, h)


def test_tokens_equal_clip_tokenizer_padding(tree):
    from transformers import CLIPTokenizer
    from pigeon_b200.pretrain_data import FilesCollator
    root, records = tree
    tok = CLIPTokenizer.from_pretrained(os.path.join(str(root), "tokenizer"))
    col = FilesCollator(processor=None, tokenizer=tok)
    caps = [c for r in records.values() for run in r["captions"] for c in run["captions"]]
    caps.append("a very long caption " * 20)                    # past 77 tokens: truncated
    for k in range(0, len(caps), 13):
        chunk = caps[k:k + 13]
        got = col.tokens(chunk)
        want = tok(chunk, padding=True, truncation=True, return_tensors="pt")
        assert torch.equal(got["input_ids"], want["input_ids"]) and got["input_ids"].dtype == torch.int64
        assert torch.equal(got["attention_mask"], want["attention_mask"].long())
    assert col.tokens(caps[-1:])["input_ids"].shape[1] == 77


def test_out_of_range_index(tree):
    root, _ = tree
    ds = make_dataset(root, "yfcc/train/0")
    with pytest.raises(IndexError):
        ds[len(ds)]


def test_cli_routes_csv_to_files(monkeypatch, tmp_path):
    sys.path.insert(0, ROOT)
    import run
    from pigeon_b200 import pretrain_data
    seen = {}
    monkeypatch.setattr(pretrain_data, "pretrain_files", lambda *a, **kw: seen.update(args=a, kw=kw))
    run.main(["pretrain", "m", "-l", "meta.csv", "--yfcc", "-a", "-w", "3", "--tokenizer", "tok", "--png"])
    assert seen["args"] == ("m", "meta.csv")
    assert seen["kw"] == dict(yfcc=True, auxiliary=True, resume=False, num_workers=3, tokenizer="tok", png=True,
                              jpeg_multiscan=False)
    seen.clear()
    from pigeon_b200 import training
    monkeypatch.setattr(training, "pretrain", lambda *a, **kw: seen.update(dd=a[1]))
    from datasets import Dataset, DatasetDict
    DatasetDict(train=Dataset.from_dict({"x": [1]})).save_to_disk(str(tmp_path / "dd"))
    run.main(["pretrain", "m", "-l", str(tmp_path / "dd")])        # a directory: the pre-processed DatasetDict route
    assert "args" not in seen and "train" in seen["dd"]
    with pytest.raises(NotImplementedError, match="-l"):
        run.main(["pretrain", "m"])
