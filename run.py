#!/usr/bin/env python
"""Entry points of the hot path with the reference's CLI (run.py:21-93): `embed`, `evaluate` and `finetune`.

    python run.py evaluate HEAD.model -l DATASET_DIR [-b BASE.model] [--yfcc] [--metrics]
    python run.py evaluate HEAD.model -l BENCHMARK -b BASE.model [--yfcc] [--metrics] [-w WORKERS]   # config.BENCHMARKS
    python run.py embed CLIP.model -l DATASET_DIR [--jpeg-multiscan] [--png]                     # image column + index
    python run.py finetune openai/clip-vit-large-patch14-336 -l DATASET_DIR [-m] [--heading] [-w WORKERS]  # (run.py:165-169)
    python run.py finetune openai/clip-vit-large-patch14-336 -l RAW_DIR [--jpeg-multiscan] [--png] [-w WORKERS]
    python run.py finetune - -l EMBEDDING_DATASET_DIR --embeddings [-m]                          # head on embeddings (:171-175)
    python run.py finetune openai/clip-vit-large-patch14-336 -l A_DIR,B_DIR[,...] [-m]           # train splits joined (:143-156)

    python run.py finetune openai/clip-vit-large-patch14-336 [--yfcc | --landmarks] [-s N] [-m] [--heading]  # no -l (:112-141)
    python run.py embed CLIP.model [--yfcc | --landmarks] [-s N] [-m] [--heading]
    python run.py evaluate HEAD.model -b BASE.model [--yfcc | --landmarks] [-s N] [-t]

    python run.py pretrain openai/clip-vit-large-patch14-336 -l PRETRAIN_DATASET_DIR [--yfcc] [-r]          # (run.py:154-163)
    python run.py pretrain openai/clip-vit-large-patch14-336 -l META.csv [--yfcc] [-a] [-r] [-w WORKERS] [--tokenizer DIR]

`pretrain` trains a CLIPModel contrastively with the HF Trainer loop of `pretrain.CLIPPretrainer` (PRETAIN_ARGS, or
PRETAIN_ARGS_YFCC with --yfcc; -r passes its `resume_from_checkpoint` to the trainer, as the reference does).  Its dataset is a pre-processed
`DatasetDict` with `train` and `val` splits whose rows hold pixel_values, input_ids and attention_mask, or, when -l names a
`.csv` file, the reference's pretraining metadata (run.py:106-110): `pretrain_data.PretrainDataset` (PretrainDatasetYFCC
with --yfcc) synthesises the captions (-a adds the auxiliary sentences), CLIPTokenizer from --tokenizer (a local directory,
config.CLIP_TOKENIZER_PATH by default) tokenises them, and the image files are decoded, cropped and pre-processed on the GPU
batch by batch; -w worker processes read the files.  Datasets are HF `DatasetDict`s on disk, as in the
reference (run.py:143-162); none are shipped with either repository.

Without -l, `finetune`, `embed` and `evaluate` build their dataset as the reference does (run.py:112-141): the metadata CSV
and image folder (config.METADATA_PATH and IMAGE_PATH; METADATA_PATH_YFCC and IMAGE_PATH_YFCC with --yfcc;
METADATA_PATH_LANDMARKS and IMAGE_PATH_LANDMARKS with --landmarks) become raw splits through
`finetune_data.generate_finetune_dataset` (-s N samples N rows, seeded from torch.initial_seed()), which
`dataset_preprocessing.preprocess` labels against config.GEOCELL_PATH (GEOCELL_PATH_YFCC with --yfcc), with -m adding
the multi-task labels.  The result is saved to data/hf_new_VIT (data/hf_dataset_N with -s N), config.DATASET_PATH_YFCC
with --yfcc or config.DATASET_PATH_LANDMARKS with --landmarks, and the mode then runs on it:
- `finetune` trains from the image files of the raw splits, as below;
- `embed` first writes data/landmark_embeddings/{split}.npy and {split}_indices.npy from each split's `image` files with
  CLIPEmbedding(name, panorama=not --yfcc) (the pass `embed -l` runs; the reference leaves this call commented out and
  reads the files), `preprocess` joins them as the `embedding` column, and the head is trained on them
  (`training.finetune_on_embeddings`, run.py:171-175);
- `evaluate` takes `val`, or `test` with -t (run.py:177-179).  The reference skips that choice under --yfcc and would pass
  the whole DatasetDict; here --yfcc chooses the same way.
With -l, `evaluate` keeps its choice of `test` when the dataset has one (else the last split), so -t changes nothing
there, and `finetune --embeddings` needs -l (`embed` without -l is its counterpart).  Several -l directories,
comma-separated, are joined as in run.py:143-156: their `train` splits concatenated, `val` and `test` from the first
(`pretrain` reads the first only).

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
    p.add_argument('-l', '--load', default=None,
                   help='comma-separated HF dataset directories (several: their train splits concatenated, val / test '
                        'from the first); without -l the dataset is generated from the metadata CSV')
    p.add_argument('-b', '--base', default=None, help='base (vision tower) checkpoint')
    p.add_argument('-s', '--sample', default=None,
                   help='without -l: how many metadata rows to sample (seeded from torch.initial_seed())')
    p.add_argument('-t', '--test', action='store_true', help='evaluate without -l: the test split instead of val')
    p.add_argument('--refine', action='store_true', default=True)
    p.add_argument('-r', '--resume', action='store_true', help='pretrain: resume from train_args.resume_from_checkpoint (run.py:77-81)')
    p.add_argument('--yfcc', action='store_true')
    p.add_argument('--landmarks', action='store_true')
    p.add_argument('--heading', action='store_true')
    p.add_argument('-m', '--multitask', action='store_true')
    p.add_argument('-a', '--auxiliary', action='store_true',
                   help='pretrain from a metadata CSV: add the auxiliary caption sentences (climate, driving side, ...)')
    p.add_argument('--tokenizer', default=cfg.CLIP_TOKENIZER_PATH,
                   help='pretrain from a metadata CSV: local directory of the CLIP tokenizer files')
    p.add_argument('--embeddings', action='store_true', help='finetune: train the head on pre-computed embeddings')
    p.add_argument('--jpeg-multiscan', action='store_true',
                   help='embed / finetune / pretrain: decode progressive and multi-scan JPEGs on the GPU too (by default Pillow '
                        'decodes them)')
    p.add_argument('--png', action='store_true',
                   help='embed / evaluate / finetune / pretrain: decode PNG files on the GPU too (by default Pillow decodes them)')
    p.add_argument('-w', '--workers', type=int, default=0,
                   help='evaluate / finetune / pretrain: DataLoader worker processes (they read the image files of a '
                        'benchmark, raw split or pretraining CSV)')
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


def embedder(args):
    """CLIPEmbedding(name, load_checkpoint=True, panorama=not --yfcc) (run.py:126-129), with the GPU decoders --png and
    --jpeg-multiscan ask for."""
    kw = {}
    if args.jpeg_multiscan or args.png:
        from pigeon_b200.preprocess import ClipImageProcessor
        kw['processor'] = ClipImageProcessor(device='cuda', dtype=torch.float16, jpeg_multiscan=args.jpeg_multiscan,
                                             png=args.png)
    return CLIPEmbedding(args.name, load_checkpoint=True, panorama=not args.yfcc, **kw)


def embed_splits(model, dataset, save_dir: str = 'data/landmark_embeddings'):
    """`{split}.npy` / `{split}_indices.npy` of every split in `save_dir`, embedded from the encoded `image` column.
    EmbedDataset semantics (embed_dataset.py:17-22): data['image'] and data['index'] of each split; the files stay
    encoded until the GPU decodes them."""
    from datasets import Image
    splits = {k: v.select_columns(['image', 'index']).cast_column('image', Image(decode=False)) for k, v in dataset.items()}
    embed_images(model, splits, save_dir=save_dir, collate_fn=encoded_image_collate)


def dataset_path(args) -> str:
    """Where the dataset generated without -l is saved (run.py:103, 136-138)."""
    if args.landmarks:
        return cfg.DATASET_PATH_LANDMARKS
    if args.yfcc:
        return cfg.DATASET_PATH_YFCC
    return 'data/hf_new_VIT' if args.sample is None else f'data/hf_dataset_{args.sample}'


def require_preprocess_columns(dataset, geocells: str, embed: bool) -> None:
    """The columns `preprocess` requires of the generated splits beyond those every split has: `heading` under
    config.GEOCELL_PATH, and in `embed` mode the image columns it drops (`image_2`..`image_4` too under GEOCELL_PATH).
    Checked before the embedding pass, so that a CSV `preprocess` would reject fails before any image is embedded."""
    from pigeon_b200.dataset_preprocessing import VIEW_COLUMNS
    need = ['heading'] if geocells == cfg.GEOCELL_PATH else []
    if embed:
        need += ['image'] + (list(VIEW_COLUMNS) if geocells == cfg.GEOCELL_PATH else [])
    for name, split in dataset.items():
        missing = [c for c in need if c not in split.column_names]
        if missing:
            raise ValueError(f'split {name!r} lacks column(s) {missing}, which preprocess needs under {geocells}'
                             + (' in embed mode' if embed else ''))


def generate_dataset(args):
    """run.py:112-141: the raw splits from the metadata CSV and image folder (`finetune_data.generate_finetune_dataset`),
    labelled by `dataset_preprocessing.preprocess` and saved to `dataset_path(args)`.  In `embed` mode the embedding
    files are written first, from the raw splits, and `preprocess` joins them."""
    from pigeon_b200.dataset_preprocessing import preprocess
    from pigeon_b200.finetune_data import generate_finetune_dataset
    metadata = cfg.METADATA_PATH_YFCC if args.yfcc else cfg.METADATA_PATH
    images = cfg.IMAGE_PATH_YFCC if args.yfcc else cfg.IMAGE_PATH
    if args.landmarks:
        metadata, images = cfg.METADATA_PATH_LANDMARKS, cfg.IMAGE_PATH_LANDMARKS
    dataset = generate_finetune_dataset(sample=args.sample, metadata_path=metadata, image_path=images)
    geocells = cfg.GEOCELL_PATH_YFCC if args.yfcc else cfg.GEOCELL_PATH
    require_preprocess_columns(dataset, geocells, embed=args.mode == 'embed')
    kw = {}
    if args.mode == 'embed':
        embed_splits(embedder(args), dataset, save_dir='data/landmark_embeddings')
        kw = dict(embedder=True, embeddings_dir='data/landmark_embeddings')
    dataset = preprocess(dataset, geocells, multi_task=args.multitask, **kw)
    dataset.save_to_disk(dataset_path(args))
    return dataset


def load_datasets(loads):
    """run.py:143-156: the `train` splits of every dataset concatenated, `val` and `test` from the first."""
    from datasets import DatasetDict, concatenate_datasets
    loaded = [DatasetDict.load_from_disk(x) for x in loads]
    out = DatasetDict(train=concatenate_datasets([d['train'] for d in loaded]))
    for split in ('val', 'test'):
        if split in loaded[0]:
            out[split] = loaded[0][split]
    print('New training dataset length:', len(out['train']))
    return out


def main(argv=None):
    args = build_parser().parse_args(argv)
    loads = args.load.split(',') if args.load else []
    if args.mode == 'pretrain' and not loads:
        raise NotImplementedError('A dataset must be given with -l (the reference regenerates it from un-shipped raw data).')
    if not loads and args.mode == 'finetune' and args.embeddings:
        raise ValueError('finetune --embeddings needs -l EMBEDDING_DATASET_DIR: without -l, `run.py embed` builds the '
                         'embedding dataset and trains the head on it')
    if not loads:
        run_mode(args, generate_dataset(args), generated=True)
        return
    if len(loads) > 1 and args.mode != 'pretrain':
        run_mode(args, load_datasets(loads))
        return
    load = loads[0]
    if args.mode == 'pretrain' and load.endswith('.csv'):
        from pigeon_b200.pretrain_data import pretrain_files
        pretrain_files(args.name, load, yfcc=args.yfcc, auxiliary=args.auxiliary, resume=args.resume,
                       num_workers=args.workers, tokenizer=args.tokenizer, png=args.png,
                       jpeg_multiscan=args.jpeg_multiscan)
        return
    if args.mode == 'evaluate' and not os.path.isdir(load) and os.path.isfile(cfg.BENCHMARKS):   # run.py:158-162
        from pigeon_b200.benchmark import BenchmarkDataset
        print(evaluate(args.name, BenchmarkDataset(load), args.yfcc, args.landmarks, base_model=args.base,
                       heading=args.heading, refine=args.refine, metrics=metrics_fn(args), num_workers=args.workers,
                       png=args.png))
        return
    from datasets import DatasetDict
    run_mode(args, DatasetDict.load_from_disk(load))


def run_mode(args, dataset, generated: bool = False):
    """The mode on a loaded `DatasetDict` (run.py:164-189).  `generated`: the dataset `generate_dataset` made, on which
    `embed` trains the head on its embeddings and `evaluate` takes `val` (`test` with -t)."""
    if args.mode == 'pretrain':
        from pigeon_b200.training import pretrain
        pretrain(args.name, dataset.with_format('torch'), cfg.PRETAIN_ARGS_YFCC if args.yfcc else cfg.PRETAIN_ARGS,
                 resume=args.resume)
    elif args.mode == 'embed' and generated:
        from pigeon_b200.training import finetune_on_embeddings
        finetune_on_embeddings(dataset.with_format('torch'), multi_task=args.multitask, heading=args.heading,
                               yfcc=args.yfcc, metrics=metrics_fn(args))                                     # run.py:175
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
        embed_splits(embedder(args), dataset)
    else:
        if generated:                                                         # run.py:177-179
            split = dataset['test'] if args.test else dataset['val']
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
