"""CPU oracle for SURVEY.md §8(f).1: the reference's optimizer step (AdamW with the "weight decay fix" + global-norm
gradient clipping + warm-up/decay learning-rate schedule + parameter grouping).

TEST INFRASTRUCTURE ONLY — never imported by the product package.

Restates (file:line under the reference's CLIP-ViP/src):
  optimization/adamw.py:40-103    AdamW.step: m, v EMAs; denom = sqrt(v) + eps (eps OUTSIDE the bias correction);
                                  step_size = lr * sqrt(1 - b2^t) / (1 - b1^t); p -= step_size * m / denom; THEN the
                                  decoupled decay p -= lr * wd * p (on the already updated p, with the uncorrected lr)
  pretrain/run_pretrain.py:408-411  torch.nn.utils.clip_grad_norm_(params, cfg.grad_norm): total 2-norm over all grads,
                                  coef = max_norm / (total + 1e-6) clamped to 1, grads scaled in place
  optimization/sched.py:14-24,57-79 warmup_linear / warmup_cosine / noam / constant inside get_lr_sched
  optimization/utils.py:127-153   no-decay name filter ['bias','LayerNorm.bias','LayerNorm.weight','logit_scale'] and the
                                  lr_mul_prefix "top" groups
Parity pinned: tests/golden/make_golden_adamw.py runs the reference's own AdamW / get_lr_sched / grouping and torch's
clip_grad_norm_ and asserts this file reproduces them bit-for-bit in fp32.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence, Tuple

import torch

NO_DECAY = ("bias", "LayerNorm.bias", "LayerNorm.weight", "logit_scale")     # utils.py:127


def lr_schedule(global_step: int, decay: str, learning_rate: float, num_train_steps: int, warmup_ratio: float = 0.1) -> float:
    """sched.py:57-79 (the 'multi_step' branch needs epoch bookkeeping of the driver and is not restated)."""
    warmup = int(warmup_ratio * num_train_steps)
    if decay == "linear":
        f = global_step / warmup if global_step < warmup else max(0, (num_train_steps - global_step) / (num_train_steps - warmup))
    elif decay == "cosine":
        if global_step < warmup:
            f = global_step / warmup
        else:
            f = 0.5 * (1.0 + math.cos(math.pi * (global_step - warmup) / (num_train_steps - warmup)))
    elif decay == "invsqrt":
        f = global_step / warmup if global_step <= warmup else (warmup ** 0.5) * (global_step ** -0.5)
    elif decay == "constant":
        f = 1.0
    else:
        raise ValueError(decay)
    lr = learning_rate * f
    return lr if lr > 0 else 1e-8


def param_groups(named_params: Sequence[Tuple[str, torch.Tensor]], learning_rate: float, weight_decay: float,
                 lr_mul: float = 1.0, lr_mul_prefix: str = "") -> List[dict]:
    """utils.py:124-153: four groups (top/decay, top/no-decay, rest/decay, rest/no-decay)."""
    if lr_mul_prefix == "":
        rest, top = list(named_params), []
    else:
        top = [(n, p) for n, p in named_params if lr_mul_prefix in n and p.requires_grad]
        rest = [(n, p) for n, p in named_params if lr_mul_prefix not in n and p.requires_grad]
    nd = lambda n: any(k in n for k in NO_DECAY)  # noqa: E731
    return [
        {"params": [p for n, p in top if not nd(n)], "lr": lr_mul * learning_rate, "weight_decay": weight_decay},
        {"params": [p for n, p in top if nd(n)], "lr": lr_mul * learning_rate, "weight_decay": 0.0},
        {"params": [p for n, p in rest if not nd(n)], "weight_decay": weight_decay},
        {"params": [p for n, p in rest if nd(n)], "weight_decay": 0.0},
    ]


def clip_coef(grads: Sequence[torch.Tensor], max_norm: float):
    """torch.nn.utils.clip_grad_norm_ (norm_type 2): returns (total_norm, coefficient <= 1)."""
    total = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(g.float()) for g in grads]))
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    return total, coef


def adamw_step(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, step: int, lr: float,
               betas=(0.9, 0.999), eps: float = 1e-6, weight_decay: float = 0.0, correct_bias: bool = True) -> None:
    """adamw.py:70-101, in place on p, m, v (fp32); `step` is the 1-based count AFTER the increment of :77."""
    b1, b2 = betas
    m.mul_(b1).add_(g, alpha=1.0 - b1)
    v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
    denom = v.sqrt().add_(eps)
    step_size = lr
    if correct_bias:
        step_size = step_size * math.sqrt(1.0 - b2 ** step) / (1.0 - b1 ** step)
    p.addcdiv_(m, denom, value=-step_size)
    if weight_decay > 0.0:
        p.add_(p, alpha=-lr * weight_decay)
