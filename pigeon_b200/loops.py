"""Callers of the hot path: the evaluation loop and the bulk-embedding loop, same signatures as the reference
(training/train_eval_loop.py:35-161 `evaluate_model`; preprocessing/embed.py:16-83 `compute_embeddings`,
`embed_images`) with the per-batch body replaced by `evaluation.predict_batch` / `CLIPEmbedding.forward`.

Differences that are deliberate (SURVEY.md §8f N4): results stay on the device until the end of the loop (one D2H
copy instead of one `.cpu()` sync per batch), `accelerate` is not needed (torch.distributed + `pigeon_b200.dist`),
and TensorBoard logging is optional (`writer=None` -> no logging) because tensorboard is outside the hot path.
"""
from __future__ import annotations

import logging
from typing import Any, Callable, Optional

import numpy as np
import torch
from torch.utils.data import DataLoader

from . import dist as pdist
from .config import EMBED_BATCH_SIZE_PER_GPU, EVAL_BATCH_SIZE
from .evaluation import predict_batch

logger = logging.getLogger('evaluation')


def evaluate_model(model, dataset, metrics: Optional[Callable], train_args=None, refiner=None, yfcc: bool = False,
                   writer=None, step: int = 0, num_workers: int = 0, collate_fn=None, processor=None):
    """reference training/train_eval_loop.py:35-161.  `train_args` only needs `.per_device_eval_batch_size`.
    With `collate_fn=encoded_eval_collate` and a `processor` (preprocess.ClipImageProcessor), `dataset` yields encoded
    files (`BenchmarkDataset.encoded()`, `EvalDataset.encoded()`) and each batch is decoded and pre-processed on the
    GPU before the model sees it; without them the batches carry pixel_values, as before."""
    logger.warning('Starting evaluation ...')
    bs = getattr(train_args, 'per_device_eval_batch_size', EVAL_BATCH_SIZE)
    if (collate_fn is None) != (processor is None):
        raise ValueError('collate_fn and processor go together: the collate yields encoded files, the processor decodes them')
    eval_data = DataLoader(dataset, bs, shuffle=False, pin_memory=collate_fn is None, num_workers=num_workers,
                           collate_fn=collate_fn)
    was_training = model.training
    model.eval()
    if refiner is not None:
        refiner.eval()
    preds, cells, top_cells, top_probs, losses, n = [], [], [], [], [], 0
    with torch.no_grad():
        for data in eval_data:                                                       # :77
            if processor is not None:
                data = encoded_pixel_values(data, processor)
            ll, cell, outputs = predict_batch(model, refiner, dict(data), gather=False)
            b = ll.shape[0]
            n += b
            losses.append(outputs.loss.detach().double() * b)                        # device scalar, no sync
            preds.append(ll if refiner is not None else outputs.preds_LLH)           # :98-105
            cells.append(outputs.preds_geocell)
            top_cells.append(outputs.top5_geocells.indices)
            top_probs.append(outputs.top5_geocells.values)
    # dtype as the reference collects it: float32 from the refiner, float64 centroid coordinates without (:98-105)
    preds_np = torch.cat(preds).cpu().numpy()                                        # single D2H at the end
    cells_np = torch.cat(cells).cpu().numpy()
    top_np = torch.cat(top_cells).cpu().numpy()
    labels_lla, labels_cell = dataset['labels'], dataset['labels_clf']               # :115-120
    if not isinstance(labels_lla, np.ndarray):
        labels_lla, labels_cell = np.asarray(labels_lla), np.asarray(labels_cell)
    results = (preds_np, cells_np, None, None, None, top_np, labels_lla, labels_cell, None, None, None)   # :137-139
    eval_dict = metrics(results) if metrics is not None else {'Geocell_accuracy': float((cells_np == labels_cell).mean())}
    loss = float(torch.stack(losses).sum().item() / max(n, 1))
    if writer is not None:                                                           # :144-155
        writer.add_scalar('Loss/val', loss, step)
        for metric, value in eval_dict.items():
            writer.add_scalar(metric, value, step)
    if was_training:
        model.train()
    logger.warning('Back to training ...')
    eval_dict = dict(eval_dict, loss=loss, preds=preds_np, preds_geocell=cells_np, top_geocells=top_np)
    return -eval_dict['Geocell_accuracy'] if metrics is not None else eval_dict


def compute_embeddings(name: str, model: Any, data: DataLoader, accelerator=None, save_dir: Optional[str] = 'data/landmark_embeddings'):
    """reference preprocessing/embed.py:16-43: embed every batch, all-gather (index, output) across ranks, rank 0
    saves `{name}.npy` / `{name}_indices.npy`.  One packed all-gather per batch (`dist.all_gather_rows`)."""
    logger.warning(f'Starting {name} embedding ...')
    outs, idxs = [], []
    for pixels, index in data:
        output = model(pixels)                                                       # CLIPEmbedding.forward
        pack = pdist.all_gather_rows(dict(index=index.to(output.device), output=output))
        outs.append(pack['output'])
        idxs.append(pack['index'])
    all_outputs = [o.cpu().numpy() for o in outs]
    all_indices = [i.cpu().numpy() for i in idxs]
    rank0 = (not pdist.is_distributed()) or torch.distributed.get_rank() == 0
    if rank0 and save_dir is not None:
        import os
        os.makedirs(save_dir, exist_ok=True)
        np.save(f'{save_dir}/{name}.npy', np.concatenate(all_outputs) if all_outputs else np.zeros((0,)))
        np.save(f'{save_dir}/{name}_indices.npy', np.concatenate(all_indices) if all_indices else np.zeros((0,)))
    return all_outputs, all_indices


def raw_image_collate(batch):
    """collate_fn for datasets that yield (uint8 RGB image of any size, index): the images stay a list, the model's GPU
    pre-processor (pigeon_b200.preprocess) turns the whole batch into pixel_values in one launch."""
    images, index = zip(*batch)
    return list(images), torch.as_tensor(index)


def read_encoded(image) -> bytes:
    """The file behind an HF `Image(decode=False)` value ({'bytes', 'path'}): its bytes, or the file at its path when
    the bytes are None."""
    data = image.get('bytes')
    if data is None:
        with open(image['path'], 'rb') as f:
            data = f.read()
    return data


def encoded_image_collate(batch):
    """collate_fn for rows of an HF dataset whose `image` column is cast to `Image(decode=False)` (the reference's
    EmbedDataset rows: data['image'], data['index']): yields (list of encoded files, index).  A row's `bytes` are used,
    or its `path` is read when `bytes` is None; the model's pre-processor decodes the batch (JPEGs on the GPU)."""
    return [read_encoded(row['image']) for row in batch], torch.as_tensor([row['index'] for row in batch])


# Columns of a row that `SuperGuessr.forward` takes besides the pixels: `labels` and `labels_clf` are in every row, the
# others only in the splits that carry them (multi-task and heading fine-tuning).
LABEL_COLUMNS = ('labels', 'labels_clf', 'labels_multi_task', 'labels_climate', 'labels_month', 'heading')


def encoded_eval_collate(batch):
    """collate_fn for `EncodedRows` (pigeon_b200.benchmark: rows of a BenchmarkDataset or EvalDataset), in evaluation
    and in fine-tuning: reads every view's file of every row, row by row, and stacks each of `LABEL_COLUMNS` the rows
    carry, with the dtype the rows give it.  No CUDA work, so it may run on DataLoader workers; `encoded_pixel_values`
    turns the batch into pixel_values in the main process."""
    out = {'files': [read_encoded(im) for row in batch for im in row['images']],
           'views': len(batch[0]['images']), 'square_crop': bool(batch[0]['square_crop'])}
    for k in LABEL_COLUMNS:
        if k in batch[0]:
            out[k] = torch.as_tensor(np.stack([np.asarray(row[k]) for row in batch]))
    return out


def encoded_pixel_values(batch, processor):
    """A batch of `encoded_eval_collate` -> the model's keyword arguments: pixel_values [B, 3 * views, 336, 336] on
    the device from one processor call (JPEG decode + pre-processing for the whole batch) and the batch's label
    columns."""
    px = processor(images=batch['files'], square_crop=batch['square_crop'])['pixel_values']
    b = len(batch['files']) // batch['views']
    out = {'pixel_values': px.view(b, 3 * batch['views'], px.shape[2], px.shape[3])}
    out.update((k, batch[k]) for k in LABEL_COLUMNS if k in batch)
    return out


def encoded_batches(loader: DataLoader, processor):
    """The batches of `loader` (collate_fn=encoded_eval_collate) as the model's keyword arguments on the device, each
    decoded and pre-processed on a side stream while the current stream still runs the work queued before it was
    requested: a training loop that asks for batch i+1 after queueing step i gets the decode of i+1 under step i.

    The current stream waits on the side stream before a batch is handed out, and its tensors are recorded as used
    there, so their memory is not reused while the step reads them.  Labels go to the device on the side stream too,
    so the step's own `.to(device)` calls find them there and do not synchronise the host.  The processor's buffers
    are only touched on the side stream from the first batch on; that batch's work waits for everything queued
    before it (an evaluation that used the same processor, say)."""
    dev = processor.device
    main = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(main)
    for batch in loader:
        with torch.cuda.stream(side):
            out = encoded_pixel_values(batch, processor)
            for k, v in out.items():
                if not v.is_cuda:
                    out[k] = v.pin_memory().to(dev, non_blocking=True)
        main.wait_stream(side)
        for v in out.values():
            v.record_stream(main)
        yield out


def embed_images(loaded_model: Any, dataset, num_workers: int = 0, save_dir: Optional[str] = 'data/landmark_embeddings',
                 collate_fn=None):
    """reference preprocessing/embed.py:45-83.  `dataset` maps split name -> dataset yielding (pixels, index); with
    `collate_fn=raw_image_collate` the items may be raw uint8 images instead of CPU-pre-processed tensors, with
    `collate_fn=encoded_image_collate` rows of encoded images."""
    loaded_model.eval()
    for split in ('train', 'val', 'test'):
        if split not in dataset:
            continue
        ds = dataset[split]
        sampler = None
        if pdist.is_distributed():
            sampler = torch.utils.data.distributed.DistributedSampler(ds, shuffle=False)
        loader = DataLoader(ds, EMBED_BATCH_SIZE_PER_GPU, shuffle=False, num_workers=num_workers, sampler=sampler,
                            pin_memory=collate_fn is None, collate_fn=collate_fn)
        compute_embeddings(split, loaded_model, loader, save_dir=save_dir)
        if pdist.is_distributed():
            torch.distributed.barrier()                                              # accelerator.wait_for_everyone()
