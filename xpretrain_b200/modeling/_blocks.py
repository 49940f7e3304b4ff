"""Pre-LN block pieces that TimeSformer (modeling/timesformer.py) and Swin-3D (modeling/swin3d.py) share.

Both run their blocks over token-major bf16 matrices [rows, C] with the GEMM weights `w[name]` of the model's parameter layout
(modeling/_weights.py) and the gradients written into a `grads` dict keyed by parameter name.  The LayerNorm helpers take the
kernel choice from `wide`: TimeSformer uses the row-mapped kernel, Swin-3D `layernorm_any_*` (the wide kernel above 1024
columns, which its PatchMerging norms reach).
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from .. import _lib, ops

bf16, f32 = torch.bfloat16, torch.float32


def layernorm(x, ln: nn.LayerNorm, wide: bool = False, out=None):
    """LayerNorm of the rows of x [rows, C] -> (y bf16, mean, rstd); y is written into `out` when given."""
    rows, C_ = x.shape[0], ln.weight.shape[0]
    mean = torch.empty(rows, dtype=f32, device=x.device)
    rstd = torch.empty_like(mean)
    y = torch.empty(rows, C_, dtype=bf16, device=x.device) if out is None else out
    if wide:
        ops.layernorm_any_fwd(x, y, ln.weight, ln.bias, mean, rstd, rows, C_, ln.eps)
    else:
        plain = ops.rowmap(C_)
        ops.layernorm_fwd(x, plain, y, plain, ln.weight, ln.bias, mean, rstd, rows, C_, ln.eps)
    return y, mean, rstd


def layernorm_bwd(dy, x, ln: nn.LayerNorm, mean, rstd, dres, grads, name: str, wide: bool = False):
    """Gradient of the LayerNorm input x (+ dres, the gradient the residual path carries past it); dγ / dβ are accumulated
    into grads[name + ".weight" / ".bias"]."""
    rows, C_ = x.shape[0], ln.weight.shape[0]
    dx = torch.empty(rows, C_, dtype=bf16, device=dy.device)
    gw, gb = grads[name + ".weight"], grads[name + ".bias"]
    if wide:
        ops.layernorm_any_bwd(dy, x, ln.weight, mean, rstd, dres, dx, gw, gb, rows, C_)
    else:
        plain = ops.rowmap(C_)
        ops.layernorm_bwd(dy, plain, x, plain, ln.weight, mean, rstd, dres, plain if dres is not None else None, dx, plain,
                          gw, gb, rows, C_)
    return dx


def linear_bwd(w, name: str, dy, x_in, grads, out=None, **dgrad_kw):
    """dW += dy^T x_in, db += colsum(dy), returns dx = dy W (bf16), written into `out` when given."""
    ops.linear_wgrad(dy, x_in, grads[name + ".weight"])
    ops.colsum(dy, grads[name + ".bias"])
    wt = w[name + ".weight"]
    dx = torch.empty(dy.shape[0], wt.shape[1], dtype=bf16, device=dy.device) if out is None else out
    ops.linear_dgrad(dy, wt, dx, **dgrad_kw)
    return dx


def residual_linear(w, name: str, lin: nn.Linear, a, residual, scale):
    """residual + drop_path(lin(a)): fused into the GEMM epilogue when no path is dropped, else GEMM + one row-scale pass."""
    rows, N = a.shape[0], lin.weight.shape[0]
    out = torch.empty(rows, N, dtype=bf16, device=a.device)
    if scale is None:
        ops.linear_fwd(a, w[name + ".weight"], lin.bias, out, residual=residual, ldr=N)
    else:
        tmp = torch.empty(rows, N, dtype=bf16, device=a.device)
        ops.linear_fwd(a, w[name + ".weight"], lin.bias, tmp)
        ops.rowscale(tmp, scale, out, residual=residual)
    return out


def drop_scale(dy, scale):
    """The gradient entering a drop_path'ed branch: dy times the same per-row factor (one extra pass when active)."""
    if scale is None:
        return dy
    out = torch.empty_like(dy)
    ops.rowscale(dy, scale, out)
    return out


class MlpSaved(NamedTuple):
    x: torch.Tensor                  # LayerNorm-2 input: the residual stream entering the MLP half
    mean: torch.Tensor
    rstd: torch.Tensor
    h: torch.Tensor                  # LayerNorm-2 output, fc1's input
    pre: Optional[torch.Tensor]      # fc1 pre-activation (None when nothing is saved for a backward)
    f1: torch.Tensor                 # GELU(fc1), fc2's input


def mlp_fwd(w, p: str, blk, x, save: bool, scale, wide: bool = False):
    """x + drop_path(fc2(erf-GELU(fc1(norm2(x))))) for a block with `norm2` and `mlp.fc1` / `mlp.fc2` under prefix p.
    Returns (out, MlpSaved); the record holds the half's tensors whether or not the caller keeps it."""
    I = blk.mlp.fc1.weight.shape[0]
    rows, dev = x.shape[0], x.device
    h, mean, rstd = layernorm(x, blk.norm2, wide)
    pre = torch.empty(rows, I, dtype=bf16, device=dev) if save else None
    f1 = torch.empty(rows, I, dtype=bf16, device=dev)
    ops.linear_fwd(h, w[p + "mlp.fc1.weight"], blk.mlp.fc1.bias, f1, act=_lib.ACT_GELU_ERF, aux=pre, ld_aux=I)
    out = residual_linear(w, p + "mlp.fc2", blk.mlp.fc2, f1, x, scale)
    return out, MlpSaved(x, mean, rstd, h, pre, f1)


def mlp_bwd(w, p: str, blk, dx, sv: MlpSaved, grads, scale, wide: bool = False):
    """Backward of mlp_fwd: dx is d(loss)/d(out); returns d(loss)/d(x)."""
    I = blk.mlp.fc1.weight.shape[0]
    dpre = linear_bwd(w, p + "mlp.fc2", drop_scale(dx, scale), sv.f1, grads, act=_lib.ACT_DGELU_ERF, aux=sv.pre,
                      ld_aux=I)
    dh = linear_bwd(w, p + "mlp.fc1", dpre, sv.h, grads)
    del dpre
    return layernorm_bwd(dh, sv.x, blk.norm2, sv.mean, sv.rstd, dx, grads, p + "norm2", wide)
