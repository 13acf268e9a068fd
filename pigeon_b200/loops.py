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
                   writer=None, step: int = 0, num_workers: int = 0):
    """reference training/train_eval_loop.py:35-161.  `train_args` only needs `.per_device_eval_batch_size`."""
    logger.warning('Starting evaluation ...')
    bs = getattr(train_args, 'per_device_eval_batch_size', EVAL_BATCH_SIZE)
    eval_data = DataLoader(dataset, bs, shuffle=False, pin_memory=True, num_workers=num_workers)
    was_training = model.training
    model.eval()
    if refiner is not None:
        refiner.eval()
    preds, cells, top_cells, top_probs, losses, n = [], [], [], [], [], 0
    with torch.no_grad():
        for data in eval_data:                                                       # :77
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


def encoded_image_collate(batch):
    """collate_fn for rows of an HF dataset whose `image` column is cast to `Image(decode=False)` (the reference's
    EmbedDataset rows: data['image'], data['index']): yields (list of encoded files, index).  A row's `bytes` are used,
    or its `path` is read when `bytes` is None; the model's pre-processor decodes the batch (JPEGs on the GPU)."""
    files = []
    for row in batch:
        im = row['image']
        data = im.get('bytes')
        if data is None:
            with open(im['path'], 'rb') as f:
                data = f.read()
        files.append(data)
    return files, torch.as_tensor([row['index'] for row in batch])


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
