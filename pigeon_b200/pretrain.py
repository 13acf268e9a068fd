"""The HF Trainer loop (transformers 4.23.1 `Trainer.train` / `_inner_training_loop`) that reference
training/train_modes.py:30-64 runs to pretrain CLIP into StreetCLIP, around the CLIPModel contrastive step on the H100.

    for epoch:                                          DistributedSampler(seed=args.seed) order, drop-last batches
        for step, batch:                                (resume: the first (global_step % updates_per_epoch) * acc skipped)
            model.forward_train(...); model.backward()  gradients accumulate in one flat fp32 buffer (`.grad` are views)
            if (step + 1) % acc == 0 or (steps_in_epoch <= acc and step + 1 == steps_in_epoch):
                all_reduce(flat) if world > 1            one summing collective
                pg_grad_norm_clip(flat * 1/(acc*world))  HF's loss / acc, then DDP's mean; torch's clip_grad_norm_
                AdamWHF.step(clip_coef, 1/(acc*world))   transformers.optimization.AdamW on the device, no host sync
                scheduler.step(); flat.zero_()           linear warm-up and decay
                log, then evaluate, then save            `_maybe_log_save_evaluate`

As in 4.23.1, micro-batches left over at the end of an epoch (steps_in_epoch % acc) are not stepped: their gradients and
loss carry into the first update of the next epoch.  `report_to` is ignored: the log goes to `state.log_history` (and so
to `trainer_state.json` in each checkpoint) and to the `pretrain` logger.
"""
from __future__ import annotations

import json
import logging
import os
import random
import re
from dataclasses import asdict, dataclass, field
from typing import Any, Callable, Dict, List, Optional

import numpy as np
import torch
from torch.utils.data import DataLoader, DistributedSampler

from . import dist as pdist
from ._lib import PigeonB200Error
from .training import AdamWHF, hf_named_parameters, linear_schedule_lambda, optimizer_grouped_parameters, schedule_lengths

logger = logging.getLogger('pretrain')

CLIP_PAD_TOKEN_ID = 49407       # CLIPProcessor pads with the EOS id, so the pooled row stays the first EOS
PREFIX_CHECKPOINT_DIR = "checkpoint"
TRAINER_STATE_NAME = "trainer_state.json"


class CLIPCollator:
    """The reference's `collate_fn` (train_modes.py:21-27) for rows that are already tokenised and pre-processed: stacks
    `pixel_values` and pads `input_ids` to the longest caption of the batch with `pad_token_id` (attention_mask 0)."""

    def __init__(self, pad_token_id: int = CLIP_PAD_TOKEN_ID):
        self.pad_token_id = int(pad_token_id)

    def __call__(self, rows: List[Dict[str, Any]]) -> Dict[str, torch.Tensor]:
        ids = [torch.as_tensor(r["input_ids"], dtype=torch.int64).reshape(-1) for r in rows]
        S = max(int(t.numel()) for t in ids)
        input_ids = torch.full((len(rows), S), self.pad_token_id, dtype=torch.int64)
        mask = torch.zeros((len(rows), S), dtype=torch.int64)
        for b, (r, t) in enumerate(zip(rows, ids)):
            L = t.numel()
            input_ids[b, :L] = t
            m = r.get("attention_mask")
            mask[b, :L] = 1 if m is None else torch.as_tensor(m, dtype=torch.int64).reshape(-1)[:L]
        px = torch.stack([torch.as_tensor(r["pixel_values"]) for r in rows])
        return {"input_ids": input_ids, "attention_mask": mask, "pixel_values": px}


@dataclass
class TrainerState:
    """The fields of transformers' `TrainerState` that the loop keeps (saved as trainer_state.json)."""
    epoch: float = 0.0
    global_step: int = 0
    max_steps: int = 0
    num_train_epochs: int = 0
    total_flos: float = 0.0
    log_history: List[Dict[str, float]] = field(default_factory=list)

    def save_to_json(self, path: str) -> None:
        with open(path, "w") as f:
            f.write(json.dumps(asdict(self), indent=2, sort_keys=True) + "\n")

    @classmethod
    def load_from_json(cls, path: str) -> "TrainerState":
        with open(path) as f:
            d = json.load(f)
        return cls(**{k: d[k] for k in ("epoch", "global_step", "max_steps", "num_train_epochs", "total_flos", "log_history")
                      if k in d})


def _arg(args, name, default):
    v = getattr(args, name, default)
    return default if v is None else v


def _strategy(args, *names: str, default: str = "no") -> str:
    """An IntervalStrategy / SchedulerType field as a string (TrainingArguments holds enums; the first name set wins)."""
    for name in names:
        v = getattr(args, name, None)
        if v is not None:
            return str(getattr(v, "value", v))
    return default


class CLIPPretrainer:
    """`transformers.Trainer(model, args, train_dataset, eval_dataset, data_collator)` for a `pigeon_b200.CLIPModel` on
    CUDA, reading the `TrainingArguments` fields that the reference's PRETAIN_ARGS sets (a real `TrainingArguments` works)."""

    def __init__(self, model, args, train_dataset, eval_dataset=None, data_collator: Optional[Callable] = None):
        if _strategy(args, "lr_scheduler_type", default="linear") != "linear":
            raise NotImplementedError(f"lr_scheduler_type={args.lr_scheduler_type!r}: only 'linear' is implemented")
        if _arg(args, "adafactor", False):
            raise NotImplementedError("adafactor=True: only the HF AdamW optimizer is implemented")
        self.model, self.args = model, args
        self.train_dataset, self.eval_dataset = train_dataset, eval_dataset
        self.data_collator = data_collator or CLIPCollator()
        self.state = TrainerState()
        self.optimizer: Optional[AdamWHF] = None
        self.lr_scheduler = None
        self._flat: Optional[torch.Tensor] = None
        self._norm_ws: Optional[torch.Tensor] = None
        self.batch_size = int(args.per_device_train_batch_size)
        if self.batch_size > model.max_train_views:
            raise PigeonB200Error(f"per_device_train_batch_size={self.batch_size} exceeds the model's max_train_views="
                                  f"{model.max_train_views} (a contrastive batch is not split into chunks)")

    # ------------------------------------------------------------------------------------------ data
    def _world_rank(self):
        if pdist.is_distributed():
            return torch.distributed.get_world_size(), torch.distributed.get_rank()
        return 1, 0

    def _sampler(self, dataset, shuffle: bool) -> DistributedSampler:
        world, rank = self._world_rank()
        return DistributedSampler(dataset, num_replicas=world, rank=rank, shuffle=shuffle, seed=int(_arg(self.args, "seed", 42)))

    def get_train_dataloader(self):
        sampler = self._sampler(self.train_dataset, True)
        return DataLoader(self.train_dataset, batch_size=self.batch_size, sampler=sampler, collate_fn=self.data_collator,
                          drop_last=True, num_workers=int(_arg(self.args, "dataloader_num_workers", 0))), sampler

    # ------------------------------------------------------------------------------------------ optimizer
    def _setup(self, total: int, warmup: int) -> None:
        a = self.args
        self.optimizer = AdamWHF(optimizer_grouped_parameters(self.model, float(_arg(a, "weight_decay", 0.0))),
                                 lr=float(a.learning_rate), betas=(float(_arg(a, "adam_beta1", 0.9)),
                                                                   float(_arg(a, "adam_beta2", 0.999))),
                                 eps=float(_arg(a, "adam_epsilon", 1e-8)))
        self.lr_scheduler = torch.optim.lr_scheduler.LambdaLR(self.optimizer, linear_schedule_lambda(warmup, total))
        # one flat fp32 gradient buffer; every trainable parameter's .grad is a 16-byte-aligned view into it
        params = [p for _, p in hf_named_parameters(self.model) if p.requires_grad]
        offs, n = [], 0
        for p in params:
            offs.append(n)
            n += (p.numel() + 3) // 4 * 4
        self._flat = torch.zeros(n, dtype=torch.float32, device=self.model.logit_scale.device)
        for p, o in zip(params, offs):
            p.grad = self._flat[o:o + p.numel()].view_as(p)

    def _optimizer_step(self, acc: int, world: int):
        if world > 1:
            torch.distributed.all_reduce(self._flat)
        scale = 1.0 / (acc * world)
        max_norm = float(_arg(self.args, "max_grad_norm", 0.0))
        total_norm = coef = None
        if max_norm > 0:
            from .ops import grad_norm_clip
            if self._norm_ws is None:
                self._norm_ws = torch.empty(0, dtype=torch.uint8, device=self._flat.device)
            total_norm, coef = grad_norm_clip(self._flat, max_norm, scale, self._norm_ws)
        self.optimizer.step(clip_coef=coef, grad_scale=scale)
        self.lr_scheduler.step()
        self._flat.zero_()
        return total_norm

    # ------------------------------------------------------------------------------------------ loop
    def train(self, resume_from_checkpoint=None):
        a = self.args
        world, rank = self._world_rank()
        acc = int(_arg(a, "gradient_accumulation_steps", 1))
        loader, sampler = self.get_train_dataloader()
        len_dl, upe, total, warmup, n_epochs = schedule_lengths(
            len(self.train_dataset), self.batch_size, acc, world, float(a.num_train_epochs), int(_arg(a, "max_steps", -1)),
            int(_arg(a, "warmup_steps", 0)), float(_arg(a, "warmup_ratio", 0.0)))
        if len_dl == 0:
            raise ValueError(f"the training set ({len(self.train_dataset)} rows over {world} ranks) has no full batch of "
                             f"{self.batch_size}")
        self._setup(total, warmup)
        self.state = TrainerState(max_steps=total, num_train_epochs=n_epochs)
        epochs_trained, skip = 0, 0
        if resume_from_checkpoint is True:
            resume_from_checkpoint = get_last_checkpoint(a.output_dir)
            if resume_from_checkpoint is None:
                raise ValueError(f"no checkpoint found in output_dir={a.output_dir}")
        if resume_from_checkpoint:
            self._load_checkpoint(resume_from_checkpoint)
            epochs_trained = self.state.global_step // upe
            skip = (self.state.global_step % upe) * acc
        self.model.train()
        dev = self.model.logit_scale.device
        tr_loss = torch.zeros((), dtype=torch.float64, device=dev)
        total_loss, last_logged = 0.0, self.state.global_step
        stop = self.state.global_step >= total
        for epoch in range(epochs_trained, n_epochs):
            if stop:
                break
            sampler.set_epoch(epoch)
            steps_in_epoch = len(loader)
            for step, batch in enumerate(loader):
                if skip > 0:
                    skip -= 1
                    continue
                out = self.model.forward_train(batch["input_ids"].to(dev), batch["pixel_values"].to(dev),
                                               batch["attention_mask"].to(dev) if batch.get("attention_mask") is not None
                                               else None)
                self.model.backward()
                tr_loss += out.loss.detach().double() / acc
                if (step + 1) % acc == 0 or (steps_in_epoch <= acc and step + 1 == steps_in_epoch):
                    total_norm = self._optimizer_step(acc, world)
                    self.state.global_step += 1
                    self.state.epoch = epoch + (step + 1) / steps_in_epoch
                    tr_loss, total_loss, last_logged = self._maybe_log_save_evaluate(tr_loss, total_loss, last_logged,
                                                                                     total_norm)
                    if self.state.global_step >= total:
                        stop = True
                        break
        if world > 1:
            torch.distributed.all_reduce(tr_loss)
            tr_loss /= world
        total_loss += float(tr_loss)
        train_loss = total_loss / max(self.state.global_step, 1)
        self._log({"train_loss": train_loss})
        return train_loss

    def _log(self, logs: Dict[str, float]) -> None:
        logs = dict(logs, epoch=round(self.state.epoch, 2), step=self.state.global_step)
        self.state.log_history.append(logs)
        logger.info(logs)

    def _maybe_log_save_evaluate(self, tr_loss, total_loss, last_logged, total_norm):
        a, s = self.args, self.state
        if _strategy(a, "logging_strategy", default="steps") == "steps" and s.global_step % int(_arg(a, "logging_steps", 500)) == 0:
            world, _ = self._world_rank()
            if world > 1:
                torch.distributed.all_reduce(tr_loss)
                tr_loss /= world
            tr = float(tr_loss)
            logs = {"loss": round(tr / (s.global_step - last_logged), 4),
                    "learning_rate": self.lr_scheduler.get_last_lr()[0]}
            if total_norm is not None:
                logs["grad_norm"] = float(total_norm)
            total_loss += tr
            tr_loss = torch.zeros_like(tr_loss)
            last_logged = s.global_step
            self._log(logs)
        if _strategy(a, "evaluation_strategy", "eval_strategy") == "steps" and s.global_step % int(_arg(a, "eval_steps", 500)) == 0 \
                and self.eval_dataset is not None:
            self.evaluate()
        if _strategy(a, "save_strategy") == "steps" and s.global_step % int(_arg(a, "save_steps", 500)) == 0:
            self.save_checkpoint()
        return tr_loss, total_loss, last_logged

    @torch.no_grad()
    def evaluate(self, eval_dataset=None) -> Dict[str, float]:
        """eval_loss = mean over drop-last batches of `per_device_eval_batch_size` of the inference path's
        `model(..., return_loss=True).loss` (averaged over ranks)."""
        ds = self.eval_dataset if eval_dataset is None else eval_dataset
        bs = int(_arg(self.args, "per_device_eval_batch_size", 8))
        loader = DataLoader(ds, batch_size=bs, sampler=self._sampler(ds, False), collate_fn=self.data_collator,
                            drop_last=True)
        dev = self.model.logit_scale.device
        total, count = torch.zeros((), dtype=torch.float64, device=dev), torch.zeros((), dtype=torch.float64, device=dev)
        for batch in loader:
            out = self.model(input_ids=batch["input_ids"].to(dev), pixel_values=batch["pixel_values"].to(dev),
                             attention_mask=batch["attention_mask"].to(dev), return_loss=True)
            total += out.loss.double()
            count += 1
        if pdist.is_distributed():
            torch.distributed.all_reduce(total)
            torch.distributed.all_reduce(count)
        metrics = {"eval_loss": float(total / count) if float(count) > 0 else float("nan")}
        self._log(metrics)
        return metrics

    # ------------------------------------------------------------------------------------------ checkpoints
    def save_checkpoint(self) -> str:
        """output_dir/checkpoint-{global_step}/: pytorch_model.bin + config.json (HF names), optimizer.pt, scheduler.pt,
        trainer_state.json and rng_state.pth; written by rank 0."""
        out = os.path.join(self.args.output_dir, f"{PREFIX_CHECKPOINT_DIR}-{self.state.global_step}")
        _, rank = self._world_rank()
        if rank == 0:
            self.model.save_pretrained(out)
            torch.save(self.optimizer.state_dict(), os.path.join(out, "optimizer.pt"))
            torch.save(self.lr_scheduler.state_dict(), os.path.join(out, "scheduler.pt"))
            self.state.save_to_json(os.path.join(out, TRAINER_STATE_NAME))
            torch.save({"python": random.getstate(), "numpy": np.random.get_state(), "cpu": torch.random.get_rng_state(),
                        "cuda": torch.cuda.random.get_rng_state_all()}, os.path.join(out, "rng_state.pth"))
        if pdist.is_distributed():
            torch.distributed.barrier()
        return out

    def _load_checkpoint(self, path: str) -> None:
        sd = torch.load(os.path.join(path, "pytorch_model.bin"), map_location="cpu", weights_only=True)
        sd = {k: v for k, v in sd.items() if "position_ids" not in k}
        missing, unexpected = self.model.load_state_dict(sd, strict=False)
        if missing or unexpected:
            raise PigeonB200Error(f"checkpoint {path} does not match the model: missing={missing} unexpected={unexpected}")
        self.optimizer.load_state_dict(torch.load(os.path.join(path, "optimizer.pt"), map_location="cpu",
                                                  weights_only=True))
        self.lr_scheduler.load_state_dict(torch.load(os.path.join(path, "scheduler.pt"), weights_only=True))
        self.state = TrainerState.load_from_json(os.path.join(path, TRAINER_STATE_NAME))
        rng = os.path.join(path, "rng_state.pth")
        if os.path.isfile(rng):
            r = torch.load(rng, weights_only=False)
            random.setstate(r["python"])
            np.random.set_state(r["numpy"])
            torch.random.set_rng_state(r["cpu"])
            if torch.cuda.is_available() and len(r["cuda"]) == torch.cuda.device_count():
                torch.cuda.random.set_rng_state_all(r["cuda"])


def get_last_checkpoint(folder: str) -> Optional[str]:
    """The `checkpoint-N` directory with the largest N in `folder` (transformers.trainer_utils.get_last_checkpoint)."""
    if not os.path.isdir(folder):
        return None
    found = [(int(m.group(1)), d) for d in os.listdir(folder)
             if (m := re.fullmatch(rf"{PREFIX_CHECKPOINT_DIR}-(\d+)", d)) and os.path.isdir(os.path.join(folder, d))]
    return os.path.join(folder, max(found)[1]) if found else None
