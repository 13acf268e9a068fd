"""Fine-tune loop of the reference (training/train_eval_loop.py:164-253 `train_model`) for the part of the model the
H100 path trains: the geocell head on embeddings (`on_embeddings=True`, base_model=None), the head on a frozen tower
(`freeze_base=True`), and the tower itself under the reference's policy (super_guessr.py:159-160: embeddings frozen with all
but the last encoder layer; `SuperGuessr._forward_train_tower` + `vit_train.TowerTrainer`).  Same loop shape — `output = model(**data)`, backward, gradient accumulation, AdamW step,
evaluation and best-checkpoint saving per epoch — with `accelerate`/DDP replaced by torch.distributed plumbing
(`SuperGuessr.backward` all-reduces the micro-batch gradient) and `torch.optim.AdamW` by `pg_adamw_step`.
"""
from __future__ import annotations

import logging
from typing import Any, Callable, Dict, Iterable, Optional

import torch
from torch.utils.data import DataLoader

from . import _versions
from . import dist as pdist
from ._lib import PigeonB200Error, check, current_stream_ptr, load, ptr
from .loops import evaluate_model

logger = logging.getLogger('train')


class AdamW:
    """torch.optim.AdamW(params, lr, betas, eps, weight_decay) — the optimizer of train_eval_loop.py:187 — as one fused
    CUDA kernel per parameter tensor (pg_adamw_step), fp32 state, same update order as torch's single-tensor path."""

    def __init__(self, params: Iterable[torch.nn.Parameter], lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 1e-2):
        if lr < 0 or eps < 0 or weight_decay < 0 or not (0 <= betas[0] < 1) or not (0 <= betas[1] < 1):
            raise ValueError("Invalid AdamW hyper-parameter")
        self.params = [p for p in params if p.requires_grad]
        self.lr, self.betas, self.eps, self.weight_decay = float(lr), (float(betas[0]), float(betas[1])), float(eps), float(weight_decay)
        self.state: Dict[int, dict] = {}
        self._lib = load()

    def zero_grad(self, set_to_none: bool = True) -> None:
        for p in self.params:
            if p.grad is not None:
                if set_to_none:
                    p.grad = None
                else:
                    p.grad.zero_()

    @torch.no_grad()
    def step(self) -> None:
        for p in self.params:
            if p.grad is None:
                continue
            if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous() or not p.grad.is_contiguous():
                raise PigeonB200Error("AdamW: parameters and gradients must be contiguous fp32 CUDA tensors")
            st = self.state.get(id(p))
            if st is None:
                st = self.state[id(p)] = dict(step=0, exp_avg=torch.zeros_like(p), exp_avg_sq=torch.zeros_like(p))
            st["step"] += 1
            check(self._lib.pg_adamw_step(ptr(p), ptr(p.grad), ptr(st["exp_avg"]), ptr(st["exp_avg_sq"]), p.numel(), self.lr,
                                          self.betas[0], self.betas[1], self.eps, self.weight_decay, st["step"], 1.0,
                                          current_stream_ptr()), "pg_adamw_step")
            _versions.bump(p)                                    # raw-pointer update: invalidate packed copies


def _to_batch(data: Any) -> dict:
    return dict(data) if not isinstance(data, dict) else data


def train_model(loaded_model: Any, dataset, on_embeddings: bool, yfcc: bool, train_args, metrics: Optional[Callable],
                patience: Optional[int] = None, should_profile: bool = False, save_path: Optional[str] = None,
                num_workers: int = 0):
    """reference training/train_eval_loop.py:164-253.  `train_args` needs `.learning_rate`,
    `.per_device_train_batch_size`, `.num_train_epochs`, optionally `.gradient_accumulation_steps`,
    `.per_device_eval_batch_size`.  Returns the trained model (the best one is saved to `save_path` if given)."""
    if train_args is None:
        from .config import TRAIN_ARGS as train_args
    model = loaded_model
    optimizer = AdamW(model.parameters(), lr=train_args.learning_rate)                       # :187
    train_ds = dataset['train']
    sampler = None
    if pdist.is_distributed():
        sampler = torch.utils.data.distributed.DistributedSampler(train_ds, shuffle=True)
    train_data = DataLoader(train_ds, train_args.per_device_train_batch_size, shuffle=sampler is None, sampler=sampler,
                            pin_memory=True, num_workers=num_workers)                        # :188-189
    prior_eval_loss, current_patience = None, 0
    grad_acc_steps = getattr(train_args, 'gradient_accumulation_steps', None) or 1          # :200-201
    logger.warning('Starting training ...')
    model.train()
    optimizer.zero_grad()
    history = []
    for epoch in range(int(train_args.num_train_epochs)):
        if sampler is not None:
            sampler.set_epoch(epoch)
        combined_loss = None
        for i, data in enumerate(train_data):                                                # :214
            output = model(**_to_batch(data))
            model.backward(output.loss)                                                      # :216
            l = output.loss.detach().double()
            combined_loss = l if combined_loss is None else combined_loss + l                # device scalar, no sync
            if i % grad_acc_steps == (grad_acc_steps - 1) or (i + 1) == len(train_data):     # :220-222
                optimizer.step()
                optimizer.zero_grad()
        history.append(float(combined_loss) if combined_loss is not None else float('nan'))
        eval_loss = None
        if 'val' in dataset and dataset['val'] is not None:
            eval_loss = evaluate_model(model, dataset['val'], metrics, train_args, None, yfcc, None, epoch)   # :232
            if not isinstance(eval_loss, (int, float)):
                eval_loss = -float((eval_loss['preds_geocell'] == _labels_clf(dataset['val'])).mean())
        if eval_loss is None or prior_eval_loss is None or eval_loss < prior_eval_loss:     # :235-241
            if pdist.is_distributed():
                torch.distributed.barrier()
            rank0 = (not pdist.is_distributed()) or torch.distributed.get_rank() == 0
            if save_path is not None and rank0:
                torch.save(model.state_dict(), save_path)
            prior_eval_loss, current_patience = eval_loss, 0
        else:
            current_patience += 1
        if patience is not None and current_patience == patience:                            # :247-249
            logger.warning(f'Early stopping after {patience} epochs ...')
            break
    model.train_history = history
    return model


def _labels_clf(ds):
    import numpy as np
    return np.asarray(ds['labels_clf'])


def finetune_model(model: Any, dataset, multi_task: bool, heading: bool, yfcc: bool, early_stopping: Optional[int] = None,
                   train_args=None, metrics: Optional[Callable] = None, **train_kwargs):
    """reference training/train_modes.py:67-107.  `model`: a HuggingFace model name (loaded with CLIPVisionModel, needs the
    checkpoint on disk) or an already built `SuperGuessr`."""
    from .super_guessr import SuperGuessr
    if isinstance(model, str):
        if 'clip-vit' not in model:
            raise Exception('Not a clip-vit model.')                                          # :96
        from transformers import CLIPVisionModel
        loaded = CLIPVisionModel.from_pretrained(model)
        model = SuperGuessr(loaded.base_model, panorama=True, hierarchical=False, multi_task=multi_task, heading=heading,
                            freeze_base=False, should_smooth_labels=True).to('cuda')           # :99-101
    return train_model(model, dataset, False, yfcc, train_args, metrics, early_stopping, **train_kwargs)   # :105


def finetune_on_embeddings(dataset, multi_task: bool, heading: bool, yfcc: bool, early_stopping: Optional[int] = None,
                           train_args=None, metrics: Optional[Callable] = None, **model_kwargs):
    """reference training/train_modes.py:110-133: the head (and auxiliary heads) trained on pre-computed embeddings."""
    from .super_guessr import SuperGuessr
    model = SuperGuessr(base_model=None, panorama=(yfcc == False), hierarchical=False, multi_task=multi_task,  # noqa: E712
                        heading=heading, freeze_base=True, should_smooth_labels=True, yfcc=yfcc, **model_kwargs).to('cuda')
    print(model)
    return train_model(model, dataset, True, yfcc, train_args, metrics, early_stopping)
