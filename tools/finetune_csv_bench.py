#!/usr/bin/env python
"""`run.py embed` without -l from a metadata CSV and an image folder, stage by stage, on one GPU, with the card name and
its power limit read in the same run.

The corpus is synthetic and written to a temporary directory: --rows four-view rows (80 % train, 10 % val, 10 % test) of
640x640 q90 JPEGs (one file name per view, hard links to 16 distinct encodings, so the files are read from the
page cache), with the columns the reference's metadata CSV has, and a
geocell CSV of 2000 rectangular cells over the globe.  The embedder is CLIP ViT-L/14-336 with random weights (the same
work as the trained one); the head training that follows is left out.  Each round runs the whole command once:

  * `build_s`: `finetune_data.generate_finetune_dataset` (CSV read, paths, the three splits);
  * `embed_s`: the embedding pass over every split's `image` files (read, GPU decode and pre-processing, tower), with
    `embed_images_per_s`;
  * `preprocess_s`: `dataset_preprocessing.preprocess` (geocell labels on the GPU, embedding join);
  * `save_s`: `save_to_disk` of the labelled dataset.

The first round also loads the modules and builds the kernels' state; the last is reported, with every round listed.

    python tools/finetune_csv_bench.py [--rows 2000] [--rounds 2] [--out RESULT.json]
"""
import argparse
import io
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from benchmark_eval_bench import card  # noqa: E402


def _jpeg(seed):
    from PIL import Image
    from pigeon_b200 import synthetic
    b = io.BytesIO()
    Image.fromarray(synthetic.synthetic_photo(640, 640, seed=seed)).save(b, "JPEG", quality=90)
    return b.getvalue()


def corpus(root, rows):
    """meta.csv, imgs/ and the geocell CSV under `root`."""
    import pandas as pd
    from dataset_preprocessing_data import wkt
    from pigeon_b200 import config
    os.makedirs(os.path.join(root, "imgs"))
    for s in range(16):
        with open(os.path.join(root, f"pool_{s}.jpg"), "wb") as f:
            f.write(_jpeg(s))
    rng = np.random.default_rng(0)
    views = ("image", "image_2", "image_3", "image_4")
    names = {v: [] for v in views}
    for r in range(rows):
        for j, v in enumerate(views):
            name = f"{r}_{j}.jpg"
            os.link(os.path.join(root, f"pool_{(4 * r + j) % 16}.jpg"), os.path.join(root, "imgs", name))
            names[v].append(name)
    frame = pd.DataFrame(dict(**names, lng=rng.uniform(-180, 180, rows), lat=rng.uniform(-90, 90, rows)))
    for j, c in enumerate(("elevation", "population", "temp_avg", "temp_diff", "prec_avg", "prec_diff")):
        frame[f"{c}_reg"] = rng.normal(0, 1, rows)
    frame["climate"] = rng.integers(0, 28, rows)
    frame["heading"] = rng.uniform(0, 360, rows)
    frame["month"] = rng.integers(1, 13, rows)
    frame["selection"] = np.where(np.arange(rows) % 10 < 8, "train", np.where(np.arange(rows) % 10 == 8, "val", "test"))
    frame["geo_area"] = "Area"
    frame.to_csv(os.path.join(root, "meta.csv"), index=False)
    box = lambda x0, y0, x1, y1: [[[[x0, y0], [x1, y0], [x1, y1], [x0, y1], [x0, y0]]]]
    xs, ys = np.linspace(-180, 180, 51), np.linspace(-90, 90, 41)
    cells = [box(xs[i], ys[k], xs[i + 1], ys[k + 1]) for i in range(50) for k in range(40)]
    geo = os.path.join(root, config.GEOCELL_PATH)
    os.makedirs(os.path.dirname(geo), exist_ok=True)
    pd.DataFrame(dict(lng=[(c[0][0][0][0] + c[0][0][1][0]) / 2 for c in cells],
                      lat=[(c[0][0][0][1] + c[0][0][2][1]) / 2 for c in cells],
                      polygon=[wkt(c) for c in cells])).to_csv(geo, index=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("finetune_csv_bench: needs a GPU")
    import datasets
    import run
    from pigeon_b200 import CLIPEmbedding, config, dataset_preprocessing, finetune_data, synthetic, training
    from pigeon_b200.super_guessr import CLIPVisionTower
    from pigeon_b200.vit_engine import VitDims
    gpu, power = card()
    dims = VitDims()
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=0), strict=True)
    model = CLIPEmbedding("unused", device="cuda", clip_model=tower)
    stage = {}

    def timed(name, fn):
        def wrapper(*args, **kw):
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = fn(*args, **kw)
            torch.cuda.synchronize()
            stage[name] = stage.get(name, 0.0) + time.perf_counter() - t
            return out
        return wrapper

    real = (finetune_data.generate_finetune_dataset, run.embed_images, dataset_preprocessing.preprocess,
            datasets.DatasetDict.save_to_disk, run.CLIPEmbedding, training.finetune_on_embeddings)
    finetune_data.generate_finetune_dataset = timed("build_s", real[0])
    run.embed_images = timed("embed_s", real[1])
    dataset_preprocessing.preprocess = timed("preprocess_s", real[2])
    datasets.DatasetDict.save_to_disk = timed("save_s", real[3])
    run.CLIPEmbedding = lambda *args, **kw: model
    training.finetune_on_embeddings = lambda *args, **kw: None
    rounds = []
    old = os.getcwd()
    try:
        with tempfile.TemporaryDirectory() as root:
            corpus(root, a.rows)
            os.chdir(root)
            config.METADATA_PATH, config.IMAGE_PATH = "meta.csv", "imgs"
            for r in range(a.rounds):
                stage.clear()
                t = time.perf_counter()
                run.main(["embed", "unused"])
                torch.cuda.synchronize()
                res = {k: round(v, 3) for k, v in stage.items()}
                res["total_s"] = round(time.perf_counter() - t, 3)
                res["embed_images_per_s"] = round(a.rows / stage["embed_s"], 1)
                rounds.append(res)
                print(f"round {r}: {res}", flush=True)
    finally:
        os.chdir(old)
        (finetune_data.generate_finetune_dataset, run.embed_images, dataset_preprocessing.preprocess,
         datasets.DatasetDict.save_to_disk, run.CLIPEmbedding, training.finetune_on_embeddings) = real
    result = dict(gpu=gpu, power_limit_w=power, rows=a.rows, files=4 * a.rows, embedded_images=a.rows,
                  image="640x640 q90 JPEG", tower="ViT-L/14-336 (random weights)", geocells=2000, **rounds[-1],
                  rounds=rounds)
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
