"""Generate tests/golden/pretrain_data.npz: items of the UNMODIFIED reference `PretrainDataset` and
`PretrainDatasetYFCC` (dataset_creation/pretrain/) on synthetic metadata and image files, for pigeon_b200.pretrain_data.

The reference modules are loaded through oracle/reference_shim.py (its `config`, with the image folders, metadata and
driving-side JSON pointed at a temporary directory).  `CLIPProcessor.from_pretrained`, which they call at import, is
stubbed with a tiny local CLIP BPE tokenizer (byte-level vocabulary, a few merges, model_max_length 77), written here.

The inputs cover every source and branch: `o` rows (four images each, JPEG and PNG, odd sizes), `v` files smaller than
the 596 crop on one or both sides and larger with odd margins, a `P`-mode PNG whose palette entry 0 is not black and an
`L`-mode PNG, `l` panoramas lower than the 385 crop, one whose last strip is narrower than 385, and YFCC files with odd
width and height differences (Pillow's half-to-even rounding of the float crop box).  Every optional metadata column
has NaNs; the countries include THE_LIST / PLURALS entries, 'United States Of America' and the truncated YFCC names.

Stored (only data):
  files/*        every input file (images, both CSVs with the temporary root replaced by @ROOT@, the driving-side JSON,
                 the tokenizer files) as one byte blob with names and offsets
  records        JSON: per dataset, len, the index -> (row, column) mapping, the captions of every index for several
                 seeded index orders and `random` seeds, and per item the crop the reference made (torchvision's pad
                 and crop arguments or Pillow's float box), the cropped size and mode, and SHA-256 of the RGB array

    python tools/make_pretrain_data_golden.py
"""
from __future__ import annotations

import hashlib
import importlib.util
import io
import json
import os
import random
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "pretrain_data.npz")
ORDERS = 4                      # seeded index orders per dataset (plus the identity order)


def _bytes_to_unicode():
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs, n = bs[:], 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return [chr(c) for c in cs]


def tokenizer_files():
    chars = _bytes_to_unicode()
    vocab = {}
    for c in chars + [c + "</w>" for c in chars]:
        vocab[c] = len(vocab)
    merges = [("t", "h"), ("th", "e</w>"), ("i", "n</w>"), ("o", "n</w>"), ("a", "n"), ("e", "r"), ("t", "o</w>"),
              ("o", "f</w>"), ("a", "t</w>"), ("e", "n"), ("s", "t"), ("i", "s</w>"), ("o", "r"), ("r", "e")]
    for a, b in merges:
        vocab.setdefault(a + b, len(vocab))
    vocab["<|startoftext|>"] = len(vocab)
    vocab["<|endoftext|>"] = len(vocab)
    cfg = dict(model_max_length=77, bos_token="<|startoftext|>", eos_token="<|endoftext|>", pad_token="<|endoftext|>",
               unk_token="<|endoftext|>", tokenizer_class="CLIPTokenizer")
    return {"tokenizer/vocab.json": json.dumps(vocab).encode(),
            "tokenizer/merges.txt": ("#version: 0.2\n" + "".join(f"{a} {b}\n" for a, b in merges)).encode(),
            "tokenizer/tokenizer_config.json": json.dumps(cfg).encode()}


def _photo(w, h, seed):
    """Random colours on a grid of 16 x 16 pixel cells, aligned with JPEG's blocks so that the files stay small; the
    crops, strips and resampling windows still cut through the cells at every offset."""
    rng = np.random.default_rng(seed)
    cells = rng.integers(0, 32, ((h + 15) // 16, (w + 15) // 16, 3), dtype=np.uint8) * 8
    return np.repeat(np.repeat(cells, 16, axis=0), 16, axis=1)[:h, :w]


def _encode(a, fmt, mode=None, seed=0):
    from PIL import Image
    im = Image.fromarray(a)
    if mode == "P":
        im = im.quantize(colors=64, method=Image.Quantize.MEDIANCUT)
        pal = im.getpalette()
        pal[0:3] = [200, 30, 90]                       # palette entry 0: the padding colour, not black
        im.putpalette(pal)
    elif mode == "L":
        im = im.convert("L")
    b = io.BytesIO()
    if fmt == "JPEG":
        im.save(b, "JPEG", quality=60)
    else:
        im.save(b, "PNG", optimize=True)
    return b.getvalue()


def inputs():
    """{relative name: bytes} of every input file; CSV paths of `v` files start with @ROOT@."""
    files = dict(tokenizer_files())
    nan = float("nan")
    countries = ["United States Of America", "Netherlands", "France", "Philippines", "Japan", "United Kingdom",
                 "Cayman Islands", "Brazil"]
    rows, k = [], 0

    def meta(i):
        rng = random.Random(1000 + i)
        return dict(country_name=countries[i % len(countries)],
                    geo_area=nan if i % 5 == 1 else f"Area {i}",
                    town=nan if i % 4 == 2 else f"Town{i}",
                    climate_zone=nan if i % 3 == 0 else ["Tropical rainforest climate", "Cold semi-arid climate",
                                                         "Temperate oceanic climate"][i % 3],
                    driving_right=nan if i % 6 == 4 else bool(i % 2),
                    heading=nan if i % 7 == 3 else round(rng.uniform(0, 360), 3),
                    month=nan if i % 5 == 3 else rng.randrange(12))

    o_sizes = [(320, 240), (331, 197), (257, 401), (336, 336), (500, 283), (199, 301), (640, 480), (251, 253)]
    for r in range(6):                                              # `o`: four views, JPEG and PNG
        names = []
        for c in range(4):
            w, h = o_sizes[(r * 4 + c) % len(o_sizes)]
            fmt = "PNG" if (r + c) % 3 == 0 else "JPEG"
            name = f"o_{r}_{c}.{'png' if fmt == 'PNG' else 'jpg'}"
            files["streetview/" + name] = _encode(_photo(w, h, k), fmt)
            k += 1
            names.append(name)
        rows.append(dict(image=names[0], image_2=names[1], image_3=names[2], image_4=names[3], source="o",
                         selection="val" if r == 5 else "train", **meta(len(rows))))
    v_specs = [(300, 200, "JPEG", None), (700, 500, "JPEG", None), (801, 640, "PNG", None), (400, 250, "PNG", "P"),
               (595, 601, "PNG", "L"), (1001, 597, "JPEG", None), (250, 700, "PNG", "P")]
    for i, (w, h, fmt, mode) in enumerate(v_specs):
        name = f"v_{i}.{'png' if fmt == 'PNG' else 'jpg'}"
        files["vfiles/" + name] = _encode(_photo(w, h, k), fmt, mode)
        k += 1
        rows.append(dict(image="@ROOT@/vfiles/" + name, image_2=nan, image_3=nan, image_4=nan, source="v",
                         selection="val" if i == 6 else "train", **meta(len(rows))))
    l_specs = [(2560, 300, "JPEG"), (2200, 400, "JPEG"), (2600, 211, "PNG")]
    for i, (w, h, fmt) in enumerate(l_specs):
        name = f"l_{i}.{'png' if fmt == 'PNG' else 'jpg'}"
        files["panoramas/" + name] = _encode(_photo(w, h, k), fmt)
        k += 1
        rows.append(dict(image=name, image_2=nan, image_3=nan, image_4=nan, source="l",
                         selection="val" if i == 2 else "train", **meta(len(rows))))
    import pandas as pd
    files["data_pretrain.csv"] = pd.DataFrame(rows).to_csv(index=False).encode()

    ycountries = ["United States Of America", "United States Minor Outlying Isl", "South Georgia and the South Sand",
                  "Germany", "Isle of Man", "Vatican City", "India", "Western Sahara"]
    y_sizes = [(101, 50), (102, 51), (50, 103), (64, 64), (333, 200), (200, 333), (77, 78), (150, 149), (90, 61),
               (61, 90)]
    yrows = []
    for i, (w, h) in enumerate(y_sizes):
        fmt = "PNG" if i % 3 == 1 else "JPEG"
        name = f"y_{i}.{'png' if fmt == 'PNG' else 'jpg'}"
        files["yfcc/" + name] = _encode(_photo(w, h, k), fmt)
        k += 1
        m = meta(i)
        del m["driving_right"], m["heading"], m["month"]
        m["country_name"] = ycountries[i % len(ycountries)]
        yrows.append(dict(image=name, selection="val" if i >= 8 else "train", **m))
    files["data_yfcc.csv"] = pd.DataFrame(yrows).to_csv(index=False).encode()
    files["driving_side.json"] = json.dumps({"United States": "right", "Germany": "right", "India": "left",
                                             "Isle of Man": "left"}).encode()
    return files


def write_tree(files, root):
    for name, data in files.items():
        path = os.path.join(root, name)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        if name.endswith(".csv"):
            data = data.replace(b"@ROOT@", root.encode())
        with open(path, "wb") as f:
            f.write(data)


def _sha(img) -> str:
    return hashlib.sha256(np.ascontiguousarray(np.asarray(img.convert("RGB"))).tobytes()).hexdigest()


def reference_modules(root):
    """The reference's two dataset modules, imported with config pointed at `root`."""
    from oracle import reference_shim
    reference_shim.install()
    cfg = sys.modules["config"]
    cfg.IMAGE_PATH = os.path.join(root, "streetview")
    cfg.IMAGE_PATH_2 = os.path.join(root, "panoramas")
    cfg.IMAGE_PATH_YFCC = os.path.join(root, "yfcc")
    cfg.PRETRAIN_METADATA_PATH = os.path.join(root, "data_pretrain.csv")
    cfg.PRETRAIN_METADATA_PATH_YFCC = os.path.join(root, "data_yfcc.csv")
    cfg.DRIVING_SIDE_PATH = os.path.join(root, "driving_side.json")
    import transformers
    from transformers import CLIPTokenizer
    tok = CLIPTokenizer.from_pretrained(os.path.join(root, "tokenizer"))
    transformers.CLIPProcessor.from_pretrained = classmethod(lambda cls, *a, **kw: tok)
    mods = []
    for name in ("pretrain_dataset", "pretrain_dataset_yfcc"):
        path = os.path.join(reference_shim.REF, "dataset_creation", "pretrain", f"{name}.py")
        spec = importlib.util.spec_from_file_location(f"_ref_{name}", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mods.append(mod)
    return mods


class CropLog:
    """Records the crops the reference makes: torchvision's pad / crop arguments and Pillow's crop boxes."""

    def __init__(self):
        import torchvision.transforms.functional as F
        from PIL import Image
        self.F, self.Image, self.calls = F, Image, []
        self.real = (F.pad, F.crop, Image.Image.crop)
        log = self.calls

        def pad(img, padding, *a, **kw):
            log.append(("pad", list(padding)))
            return self.real[0](img, padding, *a, **kw)

        def crop(img, top, left, height, width):
            log.append(("crop", [top, left, height, width]))
            return self.real[1](img, top, left, height, width)

        def pil_crop(im, box=None):
            if box is not None and any(isinstance(v, float) for v in box):
                log.append(("box", [float(v) for v in box]))
            return self.real[2](im, box)
        F.pad, F.crop, Image.Image.crop = pad, crop, pil_crop

    def take(self):
        out = list(self.calls)
        self.calls.clear()
        return out

    def close(self):
        self.F.pad, self.F.crop, self.Image.Image.crop = self.real


def record(ds, is_yfcc, log):
    n = len(ds)
    rec = dict(len=n, mapping=[list(ds._convert_to_row_index(i)) for i in range(n)] if not is_yfcc else None,
               items=[], captions=[])
    for i in range(n):
        log.take()
        img, _ = ds[i]
        rec["items"].append(dict(crop=log.take(), size=list(img.size), mode=img.mode, sha=_sha(img)))
    rng = np.random.default_rng(7)
    orders = [list(range(n))] + [rng.permutation(n).tolist() for _ in range(ORDERS)]
    for k, order in enumerate(orders):
        random.seed(100 + k)
        rec["captions"].append(dict(seed=100 + k, order=order, captions=[ds[i][1] for i in order]))
    return rec


def main():
    files = inputs()
    with tempfile.TemporaryDirectory() as root:
        write_tree(files, root)
        ref, ref_y = reference_modules(root)
        log = CropLog()
        try:
            records = {}
            for aux in (False, True):
                for split in ("train", "val"):
                    records[f"streetview/{split}/{int(aux)}"] = record(ref.PretrainDataset(split, auxiliary=aux), False, log)
                    records[f"yfcc/{split}/{int(aux)}"] = record(ref_y.PretrainDatasetYFCC(split, auxiliary=aux), True, log)
        finally:
            log.close()
    names = sorted(files)
    off = np.cumsum([0] + [len(files[k]) for k in names]).astype(np.int64)
    blob = np.frombuffer(b"".join(files[k] for k in names), dtype=np.uint8)
    np.savez_compressed(OUT, names=np.array(names), offsets=off, blob=blob,
                        records=np.frombuffer(json.dumps(records).encode(), dtype=np.uint8))
    print(f"wrote {OUT}: {len(names)} files, {blob.size} bytes of inputs, "
          f"{sum(len(r['items']) for r in records.values())} items")


if __name__ == "__main__":
    main()
