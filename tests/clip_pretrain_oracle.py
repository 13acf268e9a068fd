"""The HF Trainer of transformers 4.23.1 around HF `CLIPModel` autograd, in fp32 torch on the CPU: the checker of
`pigeon_b200.pretrain.CLIPPretrainer` (tests/golden/clip_pretrain.npz, tools/make_clip_pretrain_golden.py).

Restated here, because the installed transformers no longer has them:
  * `transformers.optimization.AdamW.step` (4.23.1, correct_bias=True), the Trainer's default optim="adamw_hf";
  * the Trainer's parameter groups (`create_optimizer`: decay = get_parameter_names(model, [nn.LayerNorm]) minus biases);
  * the inner loop of `Trainer._inner_training_loop`: loss / acc per micro-batch, an update when
    (step + 1) % acc == 0 or (steps_in_epoch <= acc and step + 1 == steps_in_epoch) -- leftover micro-batches of an epoch
    carry into the next epoch's first update -- clip_grad_norm_, optimizer step, scheduler step, zero_grad, then log /
    evaluate.
Used directly from the installed packages: `torch.nn.utils.clip_grad_norm_`, `transformers.get_linear_schedule_with_warmup`,
`transformers.trainer_pt_utils.get_parameter_names` and torch's DistributedSampler (the sample order).
"""
from __future__ import annotations

import math

import torch
from torch import nn


@torch.no_grad()
def adamw_hf_step(params, state, lr, betas, eps, weight_decay):
    """transformers/optimization.py AdamW.step, 4.23.1 (correct_bias=True), on the parameters that have a gradient."""
    beta1, beta2 = betas
    for p in params:
        if p.grad is None:
            continue
        grad = p.grad
        st = state.setdefault(p, {})
        if len(st) == 0:
            st["step"] = 0
            st["exp_avg"] = torch.zeros_like(p)
            st["exp_avg_sq"] = torch.zeros_like(p)
        exp_avg, exp_avg_sq = st["exp_avg"], st["exp_avg_sq"]
        st["step"] += 1
        exp_avg.mul_(beta1).add_(grad, alpha=(1.0 - beta1))
        exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1.0 - beta2)
        denom = exp_avg_sq.sqrt().add_(eps)
        step_size = lr
        bias_correction1 = 1.0 - beta1 ** st["step"]
        bias_correction2 = 1.0 - beta2 ** st["step"]
        step_size = step_size * math.sqrt(bias_correction2) / bias_correction1
        p.addcdiv_(exp_avg, denom, value=-step_size)
        if weight_decay > 0.0:
            p.add_(p, alpha=(-lr * weight_decay))


def hf_decay_parameter_names(model):
    """Trainer.create_optimizer (4.23.1): get_parameter_names(model, ALL_LAYERNORM_LAYERS) minus names with "bias"."""
    from transformers.trainer_pt_utils import get_parameter_names
    return [n for n in get_parameter_names(model, [nn.LayerNorm]) if "bias" not in n]


def hf_param_groups(model, weight_decay):
    decay = set(hf_decay_parameter_names(model))
    return [{"params": [p for n, p in model.named_parameters() if n in decay and p.requires_grad],
             "weight_decay": weight_decay},
            {"params": [p for n, p in model.named_parameters() if n not in decay and p.requires_grad],
             "weight_decay": 0.0}]


def train(model, train_rows, eval_rows, collate, *, batch, eval_batch, acc, epochs, lr, betas, eps, weight_decay,
          max_grad_norm, warmup_ratio, eval_steps, seed, on_step=None):
    """Runs the 4.23.1 loop on one process; returns the log history (list of dicts).  `on_step(global_step)` is called after
    each update (before logging), so the caller can snapshot parameters."""
    from torch.utils.data import DataLoader, DistributedSampler
    from transformers import get_linear_schedule_with_warmup
    sampler = DistributedSampler(train_rows, num_replicas=1, rank=0, shuffle=True, seed=seed)
    loader = DataLoader(train_rows, batch_size=batch, sampler=sampler, collate_fn=collate, drop_last=True)
    upe = max(len(loader) // acc, 1)
    total = math.ceil(epochs * upe)
    warmup = math.ceil(total * warmup_ratio)
    groups = hf_param_groups(model, weight_decay)
    opt = torch.optim.SGD(groups, lr=lr)              # only a holder of param_groups["lr"] for the schedule
    sched = get_linear_schedule_with_warmup(opt, warmup, total)
    state = {}
    params = [p for p in model.parameters()]
    model.zero_grad(set_to_none=True)
    log, tr_loss, gstep, last_logged = [], 0.0, 0, 0
    for epoch in range(math.ceil(epochs)):
        sampler.set_epoch(epoch)
        steps_in_epoch = len(loader)
        for step, b in enumerate(loader):
            model.train()
            with torch.enable_grad():
                loss = model(input_ids=b["input_ids"], pixel_values=b["pixel_values"], attention_mask=b["attention_mask"],
                             return_loss=True).loss / acc
                loss.backward()
            tr_loss += loss.item()
            if (step + 1) % acc == 0 or (steps_in_epoch <= acc and step + 1 == steps_in_epoch):
                norm = torch.nn.utils.clip_grad_norm_(params, max_grad_norm)
                for g in opt.param_groups:
                    adamw_hf_step(g["params"], state, g["lr"], betas, eps, g["weight_decay"])
                sched.step()
                model.zero_grad(set_to_none=True)
                gstep += 1
                ep = epoch + (step + 1) / steps_in_epoch
                if on_step is not None:
                    on_step(gstep)
                log.append({"loss": tr_loss / (gstep - last_logged), "learning_rate": sched.get_last_lr()[0],
                            "grad_norm": float(norm), "epoch": ep, "step": gstep})
                tr_loss, last_logged = 0.0, gstep
                if gstep % eval_steps == 0:
                    log.append({"eval_loss": evaluate(model, eval_rows, collate, eval_batch), "epoch": ep, "step": gstep})
                if gstep >= total:
                    return log
    return log


@torch.no_grad()
def evaluate(model, rows, collate, batch):
    from torch.utils.data import DataLoader
    model.eval()
    losses = [model(input_ids=b["input_ids"], pixel_values=b["pixel_values"], attention_mask=b["attention_mask"],
                    return_loss=True).loss.item()
              for b in DataLoader(rows, batch_size=batch, shuffle=False, collate_fn=collate, drop_last=True)]
    return sum(losses) / len(losses)


def golden_rows(n_rows, image_size, vocab, max_len, seed):
    """Seeded dataset rows {pixel_values [3, s, s] f32, input_ids [L] i64 (BOS, L - 2 tokens, EOS)}, lengths 2..max_len."""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for _ in range(n_rows):
        L = int(torch.randint(2, max_len + 1, (1,), generator=g))
        ids = torch.empty(L, dtype=torch.int64)
        ids[0], ids[-1] = vocab - 2, vocab - 1
        ids[1:L - 1] = torch.randint(0, vocab - 2, (L - 2,), generator=g)
        rows.append({"input_ids": ids, "pixel_values": torch.randn(3, image_size, image_size, generator=g)})
    return rows
