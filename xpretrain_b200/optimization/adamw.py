"""The reference's optimizer step on the H100: AdamW ("weight decay fix") + global-norm clipping + LR schedule + grouping.

Drop-in for CLIP-ViP/src/optimization:
  * `AdamW(params, lr, betas, eps=1e-6, weight_decay, correct_bias)` — adamw.py:11-39 constructor, same `state`
    layout (`step`, `exp_avg`, `exp_avg_sq`) so `optimizer.state_dict()` checkpoints interchange with the reference's
    (`E2E_TrainingRestorer`, load_save.py:260-327).  `step()` is ONE table-driven kernel over all parameters
    (`xp_opt_adamw_step`) instead of ~10 elementwise launches per parameter; `step(max_grad_norm=5.0)` folds
    run_pretrain.py:408-411's `clip_grad_norm_` into it (the clip coefficient is applied while reading g).
  * `clip_grad_norm_(params, max_norm)` — torch.nn.utils.clip_grad_norm_ semantics as its own call.
  * `get_lr_sched` (sched.py:57-79) and `build_e2e_optimizer_w_lr_mul` / `setup_e2e_optimizer` (utils.py:99-153): host
    arithmetic, restated here so a driver needs nothing from the reference.
After a step the parameters' version counters are bumped, so the bf16 compute copies of the model refresh themselves;
`bf16_targets` lets the step write those copies directly (no separate cast pass).
There is no CPU path: parameters must be fp32 CUDA tensors.
"""
from __future__ import annotations

import math
from typing import Dict, Iterable, Optional

import torch
from torch.optim import Optimizer

from .. import ops
from .._lib import XpError


def _check_tensor(t: torch.Tensor, what: str):
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise XpError(f"xpretrain_b200 optimizer: {what} must be contiguous fp32")


_Table = ops.OptTable          # the table's earlier name here, kept for code that still builds tables through it
_clip_tables: Dict[tuple, ops.OptTable] = {}


def clip_grad_norm_(parameters: Iterable[torch.Tensor], max_norm: float) -> torch.Tensor:
    """torch.nn.utils.clip_grad_norm_(parameters, max_norm) (2-norm), as run_pretrain.py:408-411 calls it: returns the
    total norm (0-d device tensor) and scales the gradients in place when it exceeds max_norm."""
    params = [p for p in ([parameters] if isinstance(parameters, torch.Tensor) else list(parameters)) if p.grad is not None]
    if not params:
        return torch.zeros(())
    grads = []
    for p in params:
        if not p.grad.is_contiguous():
            p.grad = p.grad.contiguous()
        _check_tensor(p.grad, "gradient")
        grads.append(p.grad)
    g_ptrs = ops.ptrs(grads)                                # CUDA tensors only: refused before any table is built
    key = (tuple(g.numel() for g in grads), grads[0].device)
    tab = _clip_tables.get(key)
    if tab is None:
        tab = _clip_tables[key] = ops.OptTable(list(key[0]), grads[0].device)
    tab.begin()["g"] = g_ptrs
    tab.upload()
    ops.opt_grad_norm(tab, max_norm)
    ops.opt_scale_grads(tab)
    return tab.norm[0].clone()


class AdamW(Optimizer):
    """adamw.py:11-103 on one fused kernel.  Extra, optional: `step(max_grad_norm=...)`, `bf16_targets`."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True):
        if lr < 0.0:
            raise ValueError("Invalid learning rate: {} - should be >= 0.0".format(lr))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError("Invalid beta parameter: {} - should be in [0.0, 1.0[".format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameter: {} - should be in [0.0, 1.0[".format(betas[1]))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {} - should be >= 0.0".format(eps))
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, correct_bias=correct_bias))
        self._tables: Dict[tuple, ops.OptTable] = {}
        self.bf16_targets: Dict[int, torch.Tensor] = {}     # id(param) -> bf16 tensor that receives the updated values
        self.last_grad_norm: Optional[torch.Tensor] = None

    @torch.no_grad()
    def step(self, closure=None, max_grad_norm: Optional[float] = None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        # one launch per distinct (betas, eps) — a single one for every configuration the reference ships
        buckets: Dict[tuple, list] = {}
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("Adam does not support sparse gradients, please consider SparseAdam instead")
                buckets.setdefault((group["betas"][0], group["betas"][1], group["eps"]), []).append((p, group))
        if max_grad_norm is not None and len(buckets) > 1:
            raise NotImplementedError("fused clipping needs all parameter groups to share betas and eps")
        for (b1, b2, eps), items in buckets.items():
            for p, _ in items:
                _check_tensor(p.data, "parameter")
                if not p.grad.is_contiguous():
                    p.grad = p.grad.contiguous()
                _check_tensor(p.grad, "gradient")
            p_ptrs = ops.ptrs(p.data for p, _ in items)     # CUDA tensors only: refused before any state changes
            g_ptrs = ops.ptrs(p.grad for p, _ in items)
            dev = items[0][0].device
            key = (b1, b2, eps, tuple(p.numel() for p, _ in items), dev)
            tab = self._tables.get(key)
            if tab is None:
                tab = self._tables[key] = ops.OptTable([p.numel() for p, _ in items], dev)
            rows = tab.begin()
            sizes, decays = [], []
            for p, group in items:
                state = self.state[p]
                if len(state) == 0:                          # adamw.py:64-70
                    state["step"] = 0
                    state["exp_avg"] = torch.zeros_like(p.data)
                    state["exp_avg_sq"] = torch.zeros_like(p.data)
                state["step"] += 1
                t = state["step"]
                step_size = group["lr"]
                if group["correct_bias"]:                    # adamw.py:85-89
                    step_size = step_size * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
                sizes.append(step_size)
                decays.append(group["lr"] * group["weight_decay"] if group["weight_decay"] > 0.0 else 0.0)
            # column-wise fills of the pinned table (one numpy assignment per field, not one tuple per parameter)
            rows["p"], rows["g"] = p_ptrs, g_ptrs
            rows["m"] = [self.state[p]["exp_avg"].data_ptr() for p, _ in items]
            rows["v"] = [self.state[p]["exp_avg_sq"].data_ptr() for p, _ in items]
            rows["p_bf16"] = [self.bf16_targets[id(p)].data_ptr() if id(p) in self.bf16_targets else 0 for p, _ in items]
            rows["step_size"], rows["decay"] = sizes, decays
            tab.upload()
            if max_grad_norm is not None:
                ops.opt_grad_norm(tab, max_grad_norm)
                self.last_grad_norm = tab.norm[0]
            ops.opt_adamw_step(tab, b1, b2, eps, clip=max_grad_norm is not None)
            torch.autograd.graph.increment_version([p for p, _ in items])   # raw-pointer writes: tell autograd / the packs
        return loss


# ------------------------------------------------------------------------------ host-side helpers
def warmup_linear(step, warmup_step, tot_step):
    if step < warmup_step:
        return step / warmup_step
    return max(0, (tot_step - step) / (tot_step - warmup_step))


def warmup_cosine(step, warmup_step, tot_step):
    if step < warmup_step:
        return step / warmup_step
    return 0.5 * (1.0 + math.cos(math.pi * (step - warmup_step) / (tot_step - warmup_step)))


def noam_schedule(step, warmup_step=4000):
    if step <= warmup_step:
        return step / warmup_step
    return (warmup_step ** 0.5) * (step ** -0.5)


def get_lr_sched(global_step, decay, learning_rate, num_train_steps, warmup_ratio=0.1, decay_epochs=(), multi_step_epoch=-1):
    """sched.py:57-79."""
    warmup_steps = int(warmup_ratio * num_train_steps)
    if decay == "linear":
        lr = learning_rate * warmup_linear(global_step, warmup_steps, num_train_steps)
    elif decay == "cosine":
        lr = learning_rate * warmup_cosine(global_step, warmup_steps, num_train_steps)
    elif decay == "invsqrt":
        lr = learning_rate * noam_schedule(global_step, warmup_steps)
    elif decay == "constant":
        lr = learning_rate
    elif decay == "multi_step":
        assert multi_step_epoch >= 0
        if global_step <= warmup_steps:
            f = global_step / warmup_steps
        else:
            ms = sorted(decay_epochs)
            f = next((0.5 ** i for i, m in enumerate(ms) if multi_step_epoch < m), 0.5 ** (len(ms) + 1))
        lr = learning_rate * f
    else:
        raise ValueError(decay)
    return lr if lr > 0 else 1e-8


NO_DECAY = ("bias", "LayerNorm.bias", "LayerNorm.weight", "logit_scale")


def build_e2e_optimizer_w_lr_mul(model_param_optimizer, learning_rate, weight_decay, lr_mul=1, lr_mul_prefix=""):
    """utils.py:124-153: [top/decay, top/no-decay, rest/decay, rest/no-decay]."""
    if lr_mul_prefix == "":
        rest, top = list(model_param_optimizer), []
    else:
        top = [(n, p) for n, p in model_param_optimizer if lr_mul_prefix in n and p.requires_grad]
        rest = [(n, p) for n, p in model_param_optimizer if lr_mul_prefix not in n and p.requires_grad]
    nd = lambda n: any(k in n for k in NO_DECAY)  # noqa: E731
    return [
        {"params": [p for n, p in top if not nd(n)], "lr": lr_mul * learning_rate, "weight_decay": weight_decay},
        {"params": [p for n, p in top if nd(n)], "lr": lr_mul * learning_rate, "weight_decay": 0.0},
        {"params": [p for n, p in rest if not nd(n)], "weight_decay": weight_decay},
        {"params": [p for n, p in rest if nd(n)], "weight_decay": 0.0},
    ]


def setup_e2e_optimizer(model, opts):
    """utils.py:99-121 for opts.optim == 'adamw' (the released configs' choice)."""
    if getattr(opts, "optim", "adamw") != "adamw":
        raise NotImplementedError("only optim='adamw' is built")
    groups = build_e2e_optimizer_w_lr_mul(list(model.named_parameters()), opts.learning_rate, opts.weight_decay,
                                          lr_mul=getattr(opts, "lr_mul", 1), lr_mul_prefix=getattr(opts, "lr_mul_prefix", ""))
    return AdamW(groups, lr=opts.learning_rate, betas=tuple(opts.betas))
