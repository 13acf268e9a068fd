#!/usr/bin/env python
"""Entry points of the hot path with the reference's CLI (run.py:21-93): `embed`, `evaluate` and `finetune`.

    python run.py evaluate HEAD.model -l DATASET_DIR [-b BASE.model] [--yfcc] [--metrics]
    python run.py evaluate HEAD.model -l BENCHMARK -b BASE.model [--yfcc] [--metrics] [-w WORKERS]   # config.BENCHMARKS
    python run.py embed CLIP.model -l DATASET_DIR [--jpeg-multiscan] [--png]                     # image column + index
    python run.py finetune openai/clip-vit-large-patch14-336 -l DATASET_DIR [-m] [--heading] [-w WORKERS]  # (run.py:165-169)
    python run.py finetune openai/clip-vit-large-patch14-336 -l RAW_DIR [--jpeg-multiscan] [--png] [-w WORKERS]
    python run.py finetune - -l EMBEDDING_DATASET_DIR --embeddings [-m]                          # head on embeddings (:171-175)

    python run.py pretrain openai/clip-vit-large-patch14-336 -l PRETRAIN_DATASET_DIR [--yfcc] [-r]          # (run.py:154-163)

`pretrain` trains a CLIPModel contrastively with the HF Trainer loop of `pretrain.CLIPPretrainer` (PRETAIN_ARGS, or
PRETAIN_ARGS_YFCC with --yfcc; -r passes its `resume_from_checkpoint` to the trainer, as the reference does).  Its dataset is a pre-processed
`DatasetDict` with `train` and `val` splits whose rows hold pixel_values, input_ids and attention_mask; the caption synthesis
of the reference's PretrainDataset is not part of this repository.  Datasets are HF `DatasetDict`s on disk, as in the
reference (run.py:143-162); none are shipped with either repository.

`finetune` trains the tower and head (`training.finetune_model`).  A split whose rows hold encoded `image` columns
(`image`..`image_4`, with `labels`, `labels_clf` and any auxiliary label columns) and no `pixel_values` is wrapped in
`benchmark.EvalDataset`, as the reference's `EvalDataset.transform` wraps train, val and test; each batch is then decoded
and pre-processed on the GPU while the previous step trains.  Splits that hold `pixel_values` are trained on as they are.

`--png` (embed, evaluate, finetune) decodes PNG files on the GPU too, `--jpeg-multiscan` (embed, finetune) progressive
and multi-scan JPEGs; by default Pillow decodes them on the host.  The pixels are the same either way.

`--metrics` (evaluate, finetune) evaluates with `metrics.compute_geoguessr_metrics`, as the reference's evaluate.py and
train_modes.py do: the full GeoGuessr table, with Country_accuracy against config.COUNTRY_PATH.  Without it only
Geocell_accuracy is computed.

`evaluate -l NAME`, when NAME is not a directory and config.BENCHMARKS exists, evaluates the benchmark NAME listed there (a
JSON file the user supplies: {name: {"meta": CSV, "images": folder prefix}}) as the reference's run.py:158-162 does, through
`benchmark.BenchmarkDataset`.  A split whose rows hold encoded `image` columns and no `pixel_values` (the reference's raw
holdout splits) is wrapped in `benchmark.EvalDataset`.  Both are decoded and pre-processed on the GPU batch by batch.
"""
import argparse
import logging
import os

import torch

from pigeon_b200 import CLIPEmbedding, ProtoRefiner, SuperGuessr
from pigeon_b200 import config as cfg
from pigeon_b200.loops import embed_images, encoded_eval_collate, encoded_image_collate, evaluate_model

logger = logging.getLogger('run')


def evaluate(model: str, dataset, yfcc: bool, landmarks: bool = False, base_model: str = None, heading: bool = False,
             refine: bool = True, metrics=None, num_workers: int = 0, png: bool = False):
    """reference evaluation/evaluate.py:10-86.  A BenchmarkDataset or EvalDataset is read as encoded files and
    pre-processed on the GPU batch by batch (`png`: PNG files decoded on the GPU too); the model's `panorama` is the
    dataset's (the reference always builds panorama=True, which a benchmark's single view cannot take)."""
    from pigeon_b200.benchmark import BenchmarkDataset, EvalDataset
    encoded = isinstance(dataset, (BenchmarkDataset, EvalDataset))
    if encoded and base_model is None:
        raise ValueError('Evaluating images needs a base model (-b): the prediction head alone takes embeddings, not pixels.')
    embed_model = None
    if base_model is not None:
        from transformers import CLIPVisionModel
        embed_model = CLIPVisionModel.from_pretrained(cfg.CLIP_MODEL)                      # :36
        if base_model != cfg.CLIP_MODEL:
            from pigeon_b200 import load_state_dict
            load_state_dict(embed_model, torch.load(base_model, map_location='cpu'))       # :37-40
    panorama = dataset.panorama if encoded else True
    full_model = SuperGuessr(embed_model, panorama=panorama, hierarchical=False, multi_task=False, heading=heading,
                             freeze_base=True, yfcc=yfcc, num_candidates=50)               # :42-44
    full_model.to('cuda')
    # :45-46 — the PIGEOTTO head first, then `model` on top: entries `model` does not carry keep the base head's values
    full_model.load_state(cfg.CLIP_PRETRAINED_HEAD_YFCC)
    full_model.load_state(model)
    refiner = None
    if refine:                                                                             # :50-80
        proto_model_path = cfg.PROTO_MODEL_YFCC_PATH if yfcc else cfg.PROTO_MODEL_PATH
        proto_path = cfg.PROTO_PATH_YFCC if yfcc else cfg.PROTO_PATH
        dataset_path = cfg.DATASET_PATH_YFCC if yfcc else cfg.DATASET_PATH
        if landmarks:                                                                      # :57-60: YFCC + landmarks bank
            proto_path = cfg.PROTO_PATH_LANDMARKS
            proto_model_path = cfg.PROTO_MODEL_LANDMARKS_PATH
            dataset_path = [cfg.DATASET_PATH_YFCC, cfg.DATASET_PATH_LANDMARKS]
        protos = None
        try:
            protos = torch.load(proto_model_path, map_location='cpu', weights_only=False).protos
        except FileNotFoundError:
            pass
        if protos is None:
            refiner = ProtoRefiner(20, False, 10000, proto_path=proto_path, dataset_path=dataset_path, temperature=1)
            torch.save(refiner, proto_model_path)
        else:
            refiner = ProtoRefiner(40, False, 100000, proto_path=proto_path, dataset_path=dataset_path, protos=protos,
                                   temperature=0.6, verbose=False)
        print(refiner)
    if encoded:
        from pigeon_b200.preprocess import ClipImageProcessor
        return evaluate_model(full_model, dataset.encoded(), metrics, None, refiner, num_workers=num_workers,
                              collate_fn=encoded_eval_collate, processor=ClipImageProcessor(png=png))
    return evaluate_model(full_model, dataset, metrics, None, refiner, num_workers=num_workers)


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description='PIGEON hot path on H100 (pretrain / finetune / embed / evaluate)')
    p.add_argument('mode', choices=['pretrain', 'finetune', 'embed', 'evaluate'])
    p.add_argument('name', help='model / prediction-head path')
    p.add_argument('-l', '--load', default=None, help='comma-separated HF dataset directories')
    p.add_argument('-b', '--base', default=None, help='base (vision tower) checkpoint')
    p.add_argument('--refine', action='store_true', default=True)
    p.add_argument('-r', '--resume', action='store_true', help='pretrain: resume from train_args.resume_from_checkpoint (run.py:77-81)')
    p.add_argument('--yfcc', action='store_true')
    p.add_argument('--landmarks', action='store_true')
    p.add_argument('--heading', action='store_true')
    p.add_argument('-m', '--multitask', action='store_true')
    p.add_argument('--embeddings', action='store_true', help='finetune: train the head on pre-computed embeddings')
    p.add_argument('--jpeg-multiscan', action='store_true',
                   help='embed / finetune: decode progressive and multi-scan JPEGs on the GPU too (by default Pillow '
                        'decodes them)')
    p.add_argument('--png', action='store_true',
                   help='embed / evaluate / finetune: decode PNG files on the GPU too (by default Pillow decodes them)')
    p.add_argument('-w', '--workers', type=int, default=0,
                   help='evaluate / finetune: DataLoader worker processes (they read the image files of a benchmark or '
                        'raw split)')
    p.add_argument('--metrics', action='store_true',
                   help='evaluate / finetune: report compute_geoguessr_metrics (needs config.COUNTRY_PATH)')
    return p


def metrics_fn(args):
    """The `metrics` callable evaluate_model gets: compute_geoguessr_metrics with --metrics, else None."""
    if not args.metrics:
        return None
    from pigeon_b200.metrics import compute_geoguessr_metrics
    return compute_geoguessr_metrics


def is_raw_split(split) -> bool:
    """A split of encoded images (an `image` column, the reference's raw holdout and fine-tuning splits) rather than of
    pre-processed `pixel_values`."""
    columns = getattr(split, 'column_names', None) or ()
    return 'image' in columns and 'pixel_values' not in columns


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.load is None:
        raise NotImplementedError('A dataset must be given with -l (the reference regenerates it from un-shipped raw data).')
    load = args.load.split(',')[0]
    if args.mode == 'evaluate' and not os.path.isdir(load) and os.path.isfile(cfg.BENCHMARKS):   # run.py:158-162
        from pigeon_b200.benchmark import BenchmarkDataset
        print(evaluate(args.name, BenchmarkDataset(load), args.yfcc, args.landmarks, base_model=args.base,
                       heading=args.heading, refine=args.refine, metrics=metrics_fn(args), num_workers=args.workers,
                       png=args.png))
        return
    from datasets import DatasetDict
    dataset = DatasetDict.load_from_disk(load)
    if args.mode == 'pretrain':
        from pigeon_b200.training import pretrain
        pretrain(args.name, dataset.with_format('torch'), cfg.PRETAIN_ARGS_YFCC if args.yfcc else cfg.PRETAIN_ARGS,
                 resume=args.resume)
    elif args.mode == 'finetune':
        from pigeon_b200.training import finetune_model, finetune_on_embeddings
        ds = dataset.with_format('torch')
        if args.embeddings:
            finetune_on_embeddings(ds, multi_task=args.multitask, heading=args.heading, yfcc=args.yfcc,
                                   metrics=metrics_fn(args))                                                 # run.py:175
        else:
            kw = {}
            if 'train' in ds and is_raw_split(ds['train']):                  # EvalDataset.transform (eval_dataset.py:77-94)
                from pigeon_b200.benchmark import EvalDataset
                from pigeon_b200.preprocess import ClipImageProcessor
                ds = {k: EvalDataset(v).encoded() for k, v in ds.items()}
                kw = dict(collate_fn=encoded_eval_collate,
                          processor=ClipImageProcessor(jpeg_multiscan=args.jpeg_multiscan, png=args.png))
            finetune_model(args.name, ds, multi_task=args.multitask, heading=args.heading, yfcc=args.yfcc,
                           metrics=metrics_fn(args), num_workers=args.workers, **kw)                         # run.py:169
    elif args.mode == 'embed':
        kw = {}
        if args.jpeg_multiscan or args.png:
            from pigeon_b200.preprocess import ClipImageProcessor
            kw['processor'] = ClipImageProcessor(device='cuda', dtype=torch.float16, jpeg_multiscan=args.jpeg_multiscan,
                                                 png=args.png)
        model = CLIPEmbedding(args.name, load_checkpoint=True, panorama=not args.yfcc, **kw)    # run.py:126-129
        # EmbedDataset semantics (embed_dataset.py:17-22): data['image'] and data['index'] of each split; the files stay
        # encoded until the GPU decodes them
        from datasets import Image
        splits = {k: v.cast_column('image', Image(decode=False)) for k, v in dataset.items()}
        embed_images(model, splits, collate_fn=encoded_image_collate)
    else:
        split = dataset['test'] if 'test' in dataset else dataset[list(dataset.keys())[-1]]
        split = split.with_format('torch')
        if is_raw_split(split):
            from pigeon_b200.benchmark import EvalDataset
            split = EvalDataset(split)
        print(evaluate(args.name, split, args.yfcc, args.landmarks, base_model=args.base,
                       heading=args.heading, refine=args.refine, metrics=metrics_fn(args), num_workers=args.workers,
                       png=args.png))


if __name__ == '__main__':
    torch.multiprocessing.set_start_method('spawn', force=True)                           # run.py:192
    main()
