"""Fine-tune loop of the reference (training/train_eval_loop.py:164-253 `train_model`) for the part of the model the
H100 path trains: the geocell head on embeddings (`on_embeddings=True`, base_model=None), the head on a frozen tower
(`freeze_base=True`), and the tower itself under the reference's policy (super_guessr.py:159-160: embeddings frozen with all
but the last encoder layer; `SuperGuessr._forward_train_tower` + `vit_train.TowerTrainer`).  Same loop shape — `output = model(**data)`, backward, gradient accumulation, AdamW step,
evaluation and best-checkpoint saving per epoch — with `accelerate`/DDP replaced by torch.distributed plumbing
(`SuperGuessr.backward` all-reduces the micro-batch gradient) and `torch.optim.AdamW` by `pg_adamw_step`.
"""
from __future__ import annotations

import logging
import math
from typing import Any, Callable, Dict, Iterable, Optional

import torch
from torch.utils.data import DataLoader

from . import _versions
from . import dist as pdist
from ._lib import PigeonB200Error, check, current_stream_ptr, load, ptr
from .loops import encoded_batches, evaluate_model

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


class AdamWHF(torch.optim.Optimizer):
    """transformers.optimization.AdamW (transformers 4.23.1, `optim="adamw_hf"`, the HF Trainer's default optimizer, so the
    one reference training/train_modes.py:30-64 pretrains with) as one fused CUDA kernel per parameter tensor
    (pg_adamw_hf_step), fp32 state.  It differs from torch.optim.AdamW (`AdamW` above): eps is added to sqrt(v) before the
    bias correction is folded into the step size, and the decoupled weight decay is applied after the update.

    A torch Optimizer, so torch's LR schedulers drive `param_groups[i]["lr"]` and `state_dict()` has torch's layout
    (per parameter: `step`, `exp_avg`, `exp_avg_sq`).  `step(clip_coef=, grad_scale=)` reads each gradient as
    grad * grad_scale * clip_coef, with clip_coef an f32 CUDA scalar (from `ops.grad_norm_clip`), so no host sync."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-6, weight_decay: float = 0.0,
                 correct_bias: bool = True):
        if lr < 0 or eps < 0 or weight_decay < 0 or not (0 <= betas[0] < 1) or not (0 <= betas[1] < 1):
            raise ValueError("Invalid AdamWHF hyper-parameter")
        if not correct_bias:
            raise NotImplementedError("AdamWHF implements correct_bias=True (the HF Trainer's setting) only")
        super().__init__(params, dict(lr=float(lr), betas=(float(betas[0]), float(betas[1])), eps=float(eps),
                                      weight_decay=float(weight_decay), correct_bias=True))
        self._lib = load()

    @torch.no_grad()
    def step(self, closure=None, clip_coef: Optional[torch.Tensor] = None, grad_scale: float = 1.0):
        if closure is not None:
            raise NotImplementedError("AdamWHF.step takes no closure")
        stream = current_stream_ptr()
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous() or not p.grad.is_contiguous():
                    raise PigeonB200Error("AdamWHF: parameters and gradients must be contiguous fp32 CUDA tensors")
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p)
                    st["exp_avg_sq"] = torch.zeros_like(p)
                st["step"] += 1
                check(self._lib.pg_adamw_hf_step(ptr(p), ptr(p.grad), ptr(st["exp_avg"]), ptr(st["exp_avg_sq"]), p.numel(),
                                                 group["lr"], group["betas"][0], group["betas"][1], group["eps"],
                                                 group["weight_decay"], int(st["step"]), float(grad_scale), ptr(clip_coef),
                                                 stream), "pg_adamw_hf_step")
                _versions.bump(p)                                # raw-pointer update: invalidate packed copies
        return None


# Modules of CLIPModel that are nn.LayerNorm in HF (our towers keep them in plain holder modules).
_LAYERNORM_MODULES = ("layer_norm1", "layer_norm2", "final_layer_norm", "pre_layrnorm", "post_layernorm")
_ATTN_ORDER = {"k_proj": 0, "v_proj": 1, "q_proj": 2, "out_proj": 3}


def hf_named_parameters(model) -> list:
    """`model.named_parameters()` in the order HF CLIPModel registers them (its attention holds k, v, q, out_proj in that
    order), so that optimizer state lines up with an HF checkpoint's."""
    named, out, i = list(model.named_parameters()), [], 0
    while i < len(named):
        if ".self_attn." not in named[i][0]:
            out.append(named[i])
            i += 1
            continue
        pre = named[i][0].split(".self_attn.")[0] + ".self_attn."
        j = i
        while j < len(named) and named[j][0].startswith(pre):
            j += 1
        out += sorted(named[i:j], key=lambda kv: _ATTN_ORDER[kv[0][len(pre):].split(".")[0]])   # stable: weight, bias
        i = j
    return out


def decay_parameter_names(model) -> list:
    """The HF Trainer rule (4.23.1 `create_optimizer`): `get_parameter_names(model, [nn.LayerNorm])` minus every name
    containing "bias", restated by name.  `logit_scale`, the embeddings and `class_embedding` are decayed."""
    return [n for n, _ in hf_named_parameters(model)
            if n.rsplit(".", 1)[0].split(".")[-1] not in _LAYERNORM_MODULES and "bias" not in n]


def optimizer_grouped_parameters(model, weight_decay: float) -> list:
    """[decayed group, no-decay group] of the trainable parameters, each in HF parameter order (4.23.1 `create_optimizer`)."""
    decay = set(decay_parameter_names(model))
    named = [(n, p) for n, p in hf_named_parameters(model) if p.requires_grad]
    return [{"params": [p for n, p in named if n in decay], "weight_decay": float(weight_decay)},
            {"params": [p for n, p in named if n not in decay], "weight_decay": 0.0}]


def linear_schedule_lambda(num_warmup_steps: int, num_training_steps: int) -> Callable[[int], float]:
    """lr multiplier of `transformers.get_linear_schedule_with_warmup`: s / W during warm-up, then a linear decay to 0 at T."""
    def lr_lambda(step: int) -> float:
        if step < num_warmup_steps:
            return float(step) / float(max(1, num_warmup_steps))
        return max(0.0, float(num_training_steps - step) / float(max(1, num_training_steps - num_warmup_steps)))
    return lr_lambda


def schedule_lengths(num_examples: int, batch_size: int, grad_acc: int, world: int, epochs: float, max_steps: int = -1,
                     warmup_steps: int = 0, warmup_ratio: float = 0.0):
    """(batches per epoch per rank, updates per epoch, T, W, epochs to run) as the HF Trainer (4.23.1) derives them, with
    a DistributedSampler (ceil(N / world) samples per rank) and drop-last batches."""
    per_rank = -(-num_examples // world)
    len_dataloader = per_rank // batch_size
    updates_per_epoch = max(len_dataloader // grad_acc, 1)
    if max_steps > 0:
        total = int(max_steps)
        n_epochs = max_steps // updates_per_epoch + int(max_steps % updates_per_epoch > 0)
    else:
        total = math.ceil(epochs * updates_per_epoch)
        n_epochs = math.ceil(epochs)
    warmup = int(warmup_steps) if warmup_steps > 0 else math.ceil(total * warmup_ratio)
    return len_dataloader, updates_per_epoch, total, warmup, n_epochs


def pretrain(model: Any, dataset, train_args=None, resume: bool = False, data_collator: Optional[Callable] = None):
    """reference training/train_modes.py:30-64: contrastive pretraining of a CLIPModel with the HF Trainer's loop
    (`pretrain.CLIPPretrainer`).  `model`: a `pigeon_b200.CLIPModel`, an HF `CLIPModel`, or a local directory / HF name.
    `dataset['train']` / `dataset['val']` hold rows with pixel_values, input_ids (and attention_mask).  The validation
    accuracy at batch size 16 is printed before and after training when the split has `.accuracy`.

    Unlike the reference, which calls `trainer.train` only under `if resume:`, this always trains; `resume` resumes from
    `train_args.resume_from_checkpoint` (None = start fresh, True = the latest checkpoint in output_dir)."""
    from .clip_model import CLIPModel
    from .pretrain import CLIPPretrainer
    if train_args is None:
        from .config import PRETAIN_ARGS as train_args
    if isinstance(model, str):
        model = CLIPModel.from_pretrained(model)
    elif not isinstance(model, CLIPModel):
        model = CLIPModel.from_hf(model)
    model = model.to('cuda')
    trainer = CLIPPretrainer(model, train_args, dataset['train'], eval_dataset=dataset['val'] if 'val' in dataset else None,
                             data_collator=data_collator)
    val = dataset['val'] if 'val' in dataset else None
    if hasattr(val, 'accuracy'):
        print('Before traing: Accuracy on batch size of 16 is', val.accuracy(model, batch_size=16))
    trainer.train(resume_from_checkpoint=getattr(train_args, 'resume_from_checkpoint', None) if resume else None)
    if hasattr(val, 'accuracy'):
        print('After training: Accuracy on batch size of 16 is', val.accuracy(model, batch_size=16))
    return model


def _to_batch(data: Any) -> dict:
    return dict(data) if not isinstance(data, dict) else data


def train_model(loaded_model: Any, dataset, on_embeddings: bool, yfcc: bool, train_args, metrics: Optional[Callable],
                patience: Optional[int] = None, should_profile: bool = False, save_path: Optional[str] = None,
                num_workers: int = 0, collate_fn=None, processor=None):
    """reference training/train_eval_loop.py:164-253.  `train_args` needs `.learning_rate`,
    `.per_device_train_batch_size`, `.num_train_epochs`, optionally `.gradient_accumulation_steps`,
    `.per_device_eval_batch_size`.  Returns the trained model (the best one is saved to `save_path` if given).

    With `collate_fn=loops.encoded_eval_collate` and a `processor` (preprocess.ClipImageProcessor), the splits yield
    encoded files (`EvalDataset.encoded()`): each training batch is decoded and pre-processed on the GPU while the
    previous step runs (`loops.encoded_batches`), and `val` is evaluated the same way.  Sampling, accumulation,
    evaluation, early stopping and checkpoints are those of the pixel_values route, and so is the sequence of batches
    for a given torch seed: this route draws no random numbers of its own."""
    if (collate_fn is None) != (processor is None):
        raise ValueError('collate_fn and processor go together: the collate yields encoded files, the processor decodes them')
    if train_args is None:
        from .config import TRAIN_ARGS as train_args
    model = loaded_model
    optimizer = AdamW(model.parameters(), lr=train_args.learning_rate)                       # :187
    train_ds = dataset['train']
    sampler = None
    if pdist.is_distributed():
        sampler = torch.utils.data.distributed.DistributedSampler(train_ds, shuffle=True)
    train_data = DataLoader(train_ds, train_args.per_device_train_batch_size, shuffle=sampler is None, sampler=sampler,
                            pin_memory=collate_fn is None, num_workers=num_workers, collate_fn=collate_fn)   # :188-189
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
        batches = train_data if processor is None else encoded_batches(train_data, processor)
        for i, data in enumerate(batches):                                                   # :214
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
            eval_loss = evaluate_model(model, dataset['val'], metrics, train_args, None, yfcc, None, epoch,   # :232
                                       collate_fn=collate_fn, processor=processor)
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
    checkpoint on disk) or an already built `SuperGuessr`.  `train_kwargs` go to `train_model` (`num_workers`, and
    `collate_fn` with `processor` for splits of encoded files)."""
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
