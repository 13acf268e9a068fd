#!/usr/bin/env python
"""CLIP pretraining step from image files (`pretrain_data.FilesPretrainer`: captions drawn and tokenised on the host,
files read by DataLoader workers, decode + crop window + pre-processing of batch i+1 on a side stream under step i)
against the same step from resident rows (`CLIPPretrainer` on rows that already hold pixel_values and input_ids), on
one GPU, with the card name and its power limit read in the same run.

Shape: the reference's PRETAIN_ARGS (32 pairs per micro-batch, gradient accumulation 8: one update = 256 pairs),
CLIP-L/14-336 towers with random weights.  The corpus is synthetic StreetView metadata written to a temporary
directory: `o` rows of four 640x640 q90 JPEGs, `v` files of 800x600 (cropped to 596, no padding) and `l` panoramas of
2560x640 (five strips, each centre-cropped to 385), 1024 items in all: one epoch is four updates.  Captions come from
the tiny BPE tokenizer of tests/golden/pretrain_data.npz: it splits most words into characters, so nearly every caption
reaches the 77-token limit, longer than CLIP's own tokenizer makes them (the text tower's work is that of 77 tokens).

Measured, the two routes alternating per round in one process (--rounds rounds of --warmup + --steps updates each):
  * `files_update_ms` / `rows_update_ms`: median interval between consecutive updates (the loop logs every update, which
    synchronises the host);
  * `pixels_ms`: decode + window + pre-processing of one 32-item batch alone, synchronised after each batch;
  * `captions_ms` / `tokens_ms`: host time to draw and to tokenise one batch's captions.

    python tools/pretrain_files_bench.py [--steps 3] [--warmup 1] [--rounds 2] [--workers 8] [--out RESULT.json]
"""
import argparse
import io
import json
import os
import random
import statistics
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from benchmark_eval_bench import card  # noqa: E402


def _jpeg(w, h, seed):
    from PIL import Image
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    a = np.stack([127 + 100 * np.sin(x / rng.uniform(9, 60) + c) * np.cos(y / rng.uniform(9, 60)) for c in range(3)], -1)
    a = np.clip(a + rng.normal(0, 12, a.shape), 0, 255).astype(np.uint8)
    b = io.BytesIO()
    Image.fromarray(a).save(b, "JPEG", quality=90)
    return b.getvalue()


def corpus(root):
    """Metadata CSV and files: 160 `o` rows (640 items), 144 `v` rows, 48 `l` rows (240 items)."""
    import pandas as pd
    from test_pretrain_data_host import write_golden_tree
    write_golden_tree(os.path.join(root, "golden"))
    for d in ("o", "v", "l"):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    pool = {(640, 640): [_jpeg(640, 640, s) for s in range(16)], (800, 600): [_jpeg(800, 600, 100 + s) for s in range(8)],
            (2560, 640): [_jpeg(2560, 640, 200 + s) for s in range(4)]}
    rows, k = [], 0
    base = dict(country_name="France", geo_area="Normandy", town="Caen", climate_zone="Temperate oceanic climate",
                driving_right=True, heading=90.0, month=5.0, selection="train")

    def put(kind, size):
        nonlocal k
        name = f"{kind}_{k}.jpg"
        with open(os.path.join(root, kind, name), "wb") as f:
            f.write(pool[size][k % len(pool[size])])
        k += 1
        return name
    for _ in range(160):
        n = [put("o", (640, 640)) for _ in range(4)]
        rows.append(dict(base, image=n[0], image_2=n[1], image_3=n[2], image_4=n[3], source="o"))
    for _ in range(144):
        rows.append(dict(base, image=os.path.join(root, "v", put("v", (800, 600))), source="v"))
    for _ in range(48):
        rows.append(dict(base, image=put("l", (2560, 640)), source="l"))
    path = os.path.join(root, "meta.csv")
    pd.DataFrame(rows).to_csv(path, index=False)
    return path


def args_for(out, updates):
    from pigeon_b200 import config
    return SimpleNamespace(**dict(vars(config.PRETAIN_ARGS), output_dir=out, num_train_epochs=1, max_steps=updates,
                                  evaluation_strategy="no", save_strategy="no", warmup_ratio=0.2))


def timed(cls):
    class T(cls):
        stamps = []

        def _maybe_log_save_evaluate(self, *a, **kw):
            out = super()._maybe_log_save_evaluate(*a, **kw)      # logging_steps=1: the loss read synchronises
            torch.cuda.synchronize()
            T.stamps.append(time.perf_counter())
            return out
    T.stamps = []
    return T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)           # warmup + steps <= 4: one epoch
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    from transformers import CLIPTokenizer
    from pigeon_b200 import CLIPModel, TextDims, VitDims, synthetic
    from pigeon_b200.preprocess import ClipImageProcessor
    from pigeon_b200.pretrain import CLIPCollator, CLIPPretrainer
    from pigeon_b200.pretrain_data import FilesCollator, FilesPretrainer, PretrainDataset, read_batch
    gpu, power = card()
    dev = torch.device("cuda:0")
    td, vd = TextDims(), VitDims()
    sd = synthetic.random_clip_state_dict(td, vd, seed=7, std=0.02, projection_dim=768)
    res = dict(gpu=gpu, power_limit_w=power, batch=32, accumulation=8, workers=a.workers, steps=a.steps,
               warmup=a.warmup, rounds=a.rounds)
    with tempfile.TemporaryDirectory() as root:
        meta = corpus(root)
        tok = CLIPTokenizer.from_pretrained(os.path.join(root, "golden", "tokenizer"))
        ds = PretrainDataset("train", meta, auxiliary=True, image_path=os.path.join(root, "o"),
                             image_path_2=os.path.join(root, "l"))
        assert len(ds) == 1024, len(ds)
        col = FilesCollator(ClipImageProcessor(device=dev), tok, num_workers=a.workers)

        # pieces of one batch, alone
        batches = [read_batch(ds, list(range(b * 32, b * 32 + 32))) for b in range(len(ds) // 32)]
        for _ in range(2):
            col.pixels(*batches[0][1:])
        torch.cuda.synchronize()
        px_ms, cap_ms, tok_ms = [], [], []
        for _ in range(2):
            for idx, files, windows, fills in batches[::2]:
                t0 = time.perf_counter()
                col.pixels(files, windows, fills)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                caps = [ds.caption(i) for i in idx]
                t2 = time.perf_counter()
                col.tokens(caps)
                t3 = time.perf_counter()
                px_ms.append(1e3 * (t1 - t0))
                cap_ms.append(1e3 * (t2 - t1))
                tok_ms.append(1e3 * (t3 - t2))
        res.update(pixels_ms=statistics.median(px_ms), captions_ms=statistics.median(cap_ms),
                   tokens_ms=statistics.median(tok_ms))

        # resident rows: the items the files route sees, pre-processed once, captions drawn in index order
        rows = []
        for idx, files, windows, fills in batches:
            px = col.pixels(files, windows, fills).cpu()
            for j, i in enumerate(idx):
                ids = tok(ds.caption(i), truncation=True)
                rows.append(dict(pixel_values=px[j], input_ids=ids["input_ids"], attention_mask=ids["attention_mask"]))
        updates = a.warmup + a.steps
        files_ms, rows_ms = [], []
        for r in range(a.rounds):
            for route in ("files", "rows"):
                m = CLIPModel(td, vd, projection_dim=768)
                m.load_state_dict(sd)
                m = m.to(dev)
                random.seed(r)
                if route == "files":
                    T = timed(FilesPretrainer)
                    tr = T(m, args_for(os.path.join(root, "out"), updates), ds, None, col)
                else:
                    T = timed(CLIPPretrainer)
                    tr = T(m, args_for(os.path.join(root, "out"), updates), rows, None,
                           CLIPCollator(pad_token_id=tok.pad_token_id))
                tr.train()
                st = T.stamps
                gaps = [1e3 * (st[i + 1] - st[i]) for i in range(a.warmup - 1 if a.warmup else 0, len(st) - 1)]
                (files_ms if route == "files" else rows_ms).extend(gaps[-a.steps:] if len(gaps) >= a.steps else gaps)
                print(route, r, [round(g, 1) for g in gaps], flush=True)
                del tr, m
                torch.cuda.empty_cache()
        res.update(files_update_ms=statistics.median(files_ms), rows_update_ms=statistics.median(rows_ms),
                   files_update_all_ms=files_ms, rows_update_all_ms=rows_ms)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
