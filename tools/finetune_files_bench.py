#!/usr/bin/env python
"""Fine-tune step from image files (`train_model`'s encoded route: `loops.encoded_batches` over a raw four-view split)
against the same step from device-resident pixel_values, on one GPU, with the card name and its power limit read in the
same run.

Shape: BASELINE.json configs[3] per rank (cfg4: 128 four-view samples = 512 views per step), ViT-L/14-336 with random
weights, a 1 000-cell haversine-smoothed head, AdamW lr 2e-5, the reference freeze policy (every encoder layer but the
last frozen) and, with --all-trainable, every parameter trainable.

Corpora, each written to a temporary directory as an HF raw split (`image`..`image_4` as file paths, `labels`,
`labels_clf`; `DatasetDict.save_to_disk`) and read back through `EvalDataset(...).encoded()`:
  * `baseline640`: 640x640 baseline 4:2:0 JPEGs at q90 without restart markers (all decoded on the GPU);
  * `mix`: `benchmark_eval_bench`'s Flickr-like mix, 500x375 to 1024x768, q85-95, about 4 % progressive and 2 % PNG
    (those go to Pillow on the host).

Measured, the two step routes alternating per round in one process (--rounds rounds of one pass over the split each):
  * `resident`: the step on a fixed batch of pixel_values and labels already on the device;
  * `files`: the step fed by `encoded_batches` from a DataLoader with --workers workers reading the files, batch i+1
    decoded and pre-processed on a side stream under step i;
  * `decode`: `encoded_pixel_values` alone on collated batches already in memory (host parse and staging, GPU decode,
    Pillow for the rest, pre-processing), synchronised after each batch.
Step times are the intervals between CUDA events recorded after consecutive steps (the first step of each pass, which
has nothing to overlap its decode with, is reported separately); `enqueue_ms` is the host time to queue one resident
step, which stays far below its device time only when the step never waits for the device.  Medians over all rounds.

    python tools/finetune_files_bench.py [--samples 128] [--steps 5] [--rounds 2] [--workers 8] [--all-trainable]
"""
import argparse
import io
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from benchmark_eval_bench import card, corpus  # noqa: E402

CELLS = 1000
VIEWS = ["image", "image_2", "image_3", "image_4"]


def baseline640(n, seed=0, distinct=64):
    """n (name, bytes, kind): 640x640 q90 4:2:0 baseline JPEGs without restart markers, `distinct` seeded encodes."""
    from PIL import Image
    from pigeon_b200 import synthetic
    pool = []
    for k in range(distinct):
        f = io.BytesIO()
        Image.fromarray(synthetic.synthetic_photo(640, 640, seed * 1000 + k)).save(f, "JPEG", quality=90, subsampling=2)
        pool.append(f.getvalue())
    order = np.random.default_rng(seed).integers(0, distinct, n)
    return [(f"{i:05d}.jpg", pool[j], "baseline") for i, j in enumerate(order)]


def write_split(files, samples, tmp):
    """The files as the views of `samples` rows of an HF raw split on disk; returns the loaded train split."""
    import datasets
    from pigeon_b200 import synthetic
    img = os.path.join(tmp, "img")
    os.makedirs(img)
    paths = []
    for name, data, _ in files:
        paths.append(os.path.join(img, name))
        with open(paths[-1], "wb") as f:
            f.write(data)
    rng = np.random.default_rng(3)
    cols = {c: [{"bytes": None, "path": paths[4 * r + v]} for r in range(samples)] for v, c in enumerate(VIEWS)}
    cols.update(labels=synthetic.synthetic_geocells(samples, 4).tolist(),
                labels_clf=rng.integers(0, CELLS, samples).tolist())
    feats = {c: datasets.Image() for c in VIEWS}
    feats.update(labels=datasets.Sequence(datasets.Value("float64")), labels_clf=datasets.Value("int64"))
    split = datasets.Dataset.from_dict(cols, features=datasets.Features(feats))
    datasets.DatasetDict(train=split).save_to_disk(os.path.join(tmp, "raw"))
    return datasets.DatasetDict.load_from_disk(os.path.join(tmp, "raw"))["train"].with_format("torch")


def model(all_trainable):
    from pigeon_b200 import CLIPVisionTower, SuperGuessr, VitDims, synthetic
    from pigeon_b200.training import AdamW
    dims = VitDims()
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(synthetic.random_vit_state_dict(dims, seed=0), strict=True)
    sg = SuperGuessr(tower, panorama=True, should_smooth_labels=True, num_candidates=5,
                     geocells=synthetic.synthetic_geocells(CELLS, 0)).to("cuda")
    if not all_trainable:
        for p in sg.base_model.vision_model.encoder.layers[:-1].parameters():
            p.requires_grad = False
    sg.train()
    return sg, AdamW(sg.parameters(), lr=2e-5)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--samples", type=int, default=128, help="four-view samples per step")
    ap.add_argument("--steps", type=int, default=5, help="timed steps per pass (the split holds steps + 1 batches)")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--corpus", default="baseline640,mix")
    ap.add_argument("--all-trainable", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/finetune_files_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("finetune_files_bench: no CUDA device")
    from pigeon_b200 import benchmark, loops
    from pigeon_b200.preprocess import ClipImageProcessor
    gpu, power = card()
    B, n_rows = args.samples, args.samples * (args.steps + 1)
    base = dict(gpu=gpu, power_limit_w=power, samples=B, views=4 * B, workers=args.workers,
                policy="all trainable" if args.all_trainable else "reference freeze policy")
    lines = []

    def emit(d):
        d = dict(base, **d)
        lines.append(d)
        print(json.dumps(d), flush=True)

    sg, opt = model(args.all_trainable)
    gen = torch.Generator().manual_seed(5)
    px = torch.randn(B, 12, 336, 336, generator=gen).to("cuda")
    lab = {"labels": torch.tensor(np.random.default_rng(6).uniform(-60, 60, (B, 2)), dtype=torch.float32).cuda(),
           "labels_clf": torch.randint(0, CELLS, (B,), generator=gen).cuda()}
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def step(data):
        out = sg(**data)
        sg.backward(out.loss)
        opt.step()
        opt.zero_grad()

    def timed(batches):
        """Events after each step of one pass; returns (first step ms, later step intervals ms)."""
        marks = [ev()]
        marks[0].record()
        for data in batches:
            step(data)
            marks.append(ev())
            marks[-1].record()
        torch.cuda.synchronize()
        ms = [a.elapsed_time(b) for a, b in zip(marks, marks[1:])]
        return ms[0], ms[1:]

    for name in args.corpus.split(","):
        files = baseline640(4 * n_rows) if name == "baseline640" else corpus(4 * n_rows)
        tmp = tempfile.mkdtemp(prefix="finetune_files_bench_")
        try:
            rows = benchmark.EvalDataset(write_split(files, n_rows, tmp)).encoded()
            proc = ClipImageProcessor()
            loader = torch.utils.data.DataLoader(rows, B, shuffle=True, num_workers=args.workers,
                                                 collate_fn=loops.encoded_eval_collate)
            res = {"resident": [], "files": [], "files_first": [], "enqueue": []}
            timed(loops.encoded_batches(loader, proc))                           # warm-up: modules, workspaces, allocator
            timed([dict(lab, pixel_values=px)] * 2)
            for _ in range(args.rounds):
                _, ms = timed([dict(lab, pixel_values=px)] * (args.steps + 1))
                res["resident"] += ms
                first, ms = timed(loops.encoded_batches(loader, proc))
                res["files"] += ms
                res["files_first"].append(first)
                torch.cuda.synchronize()
                t = time.perf_counter()
                step(dict(lab, pixel_values=px))
                res["enqueue"].append((time.perf_counter() - t) * 1e3)
                torch.cuda.synchronize()
            batches = [loops.encoded_eval_collate([rows[i] for i in range(s, s + B)]) for s in range(0, n_rows, B)]
            dec = []
            for _ in range(args.rounds):
                for b in batches:
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    loops.encoded_pixel_values(b, proc)
                    torch.cuda.synchronize()
                    dec.append((time.perf_counter() - t) * 1e3)
            med = {k: statistics.median(v) for k, v in res.items()}
            kinds = {k: sum(f[2] == k for f in files) for k in ("baseline", "progressive", "png")}
            emit(dict(corpus=name, kinds=kinds, corpus_mb=round(sum(len(f[1]) for f in files) / 1e6, 1),
                      resident_ms_per_step=round(med["resident"], 1), files_ms_per_step=round(med["files"], 1),
                      files_over_resident=round(med["files"] / med["resident"], 4),
                      files_first_step_ms=round(med["files_first"], 1),
                      decode_ms_per_batch=round(statistics.median(dec), 1),
                      enqueue_ms_per_resident_step=round(med["enqueue"], 1),
                      gpu_decoded=proc.gpu_decoded, host_decoded=proc.host_decoded,
                      resident_ms=[round(x, 1) for x in res["resident"]], files_ms=[round(x, 1) for x in res["files"]],
                      decode_ms=[round(x, 1) for x in dec]))
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "finetune_files_bench.jsonl"), "a") as f:
            f.write("".join(json.dumps(d) + "\n" for d in lines))


if __name__ == "__main__":
    main()
