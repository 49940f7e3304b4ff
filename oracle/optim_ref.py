"""Float64 references and element bounds for the optimizer kernels (optim.cu).

  grad_norm_ref    the global 2-norm in float64, and the kernel's rounding bound on it
  clip_coef_f32    the clip coefficient exactly as opt_norm_finalize_kernel states it (fp32, from the kernel's norm)
  adamw_ref        one AdamW step in adamw.py's order (eps outside the bias correction, decay on the updated p) in
                   float64 from the fp32 inputs and the fp32 constants the kernel sees, with a per-element bound

Bounds are first order in u = 2^-24 (x 1.001 for the rest).  Every fp32 operation of the kernel may add u times its
result; nvcc's FMA contraction only removes roundings, so the same bound holds with or without it.

Pure torch; runs on the CPU or on a GPU."""
from __future__ import annotations

import math
from typing import Sequence

import numpy as np
import torch

F64 = torch.float64
U = 2.0 ** -24
SLACK = 1.001
CHUNK, THREADS = 8192, 256          # optim.cu OPT_CHUNK / OPT_THREADS


def f32(x: float) -> float:
    return float(np.float32(x))


def grad_norm_ref(grads: Sequence[torch.Tensor]):
    """(float64 norm, relative bound on the kernel's fp32 norm).

    opt_sumsq_kernel: per thread at most CHUNK / THREADS = 32 squared terms in a fixed-order fp32 sum (vector path:
    ((x^2 + y^2) + z^2) + w^2 then += acc; scalar path: += acc), a 5-level warp butterfly, 7 adds over the 8 warps: every
    term takes part in at most 44 additions after its product rounding, so the block partial is within 45 u of its
    exact value (relative; the terms are non-negative).  The partials are summed in double (error ~ n 2^-53, below u),
    sqrt in double, one rounding to fp32: |norm - exact| <= (45 u / 2 + u) exact."""
    s = sum(float((g.to(F64) ** 2).sum()) for g in grads)
    return math.sqrt(s), (45 * U / 2 + U) * SLACK


def clip_coef_f32(max_norm: float, norm: float) -> float:
    """norm_out[1] of opt_norm_finalize_kernel for the fp32 norm it wrote: min(1, max_norm / (norm + 1e-6f)) with one IEEE
    fp32 add and division; 1 when max_norm <= 0; NaN when the norm is NaN (clip_grad_norm_'s clamp)."""
    if not max_norm > 0:
        return 1.0
    with np.errstate(all="ignore"):
        c = np.float32(max_norm) / (np.float32(norm) + np.float32(1e-6))
    return 1.0 if c > 1 else float(c)


def adamw_ref(p, g, m, v, coef: float, beta1: float, beta2: float, eps: float, step_size: float, decay: float,
              one_minus=None):
    """One opt_adamw_kernel step on fp32 tensors p, g, m, v; step_size / decay are the fp32 values of the table row.
    Returns {"p", "m", "v"} -> (exact float64, bound float64).

    The kernel forms 1 - beta as `1.f - b` from the fp32 beta (exact: Sterbenz); adamw.py passes `1.0 - beta` computed in
    double and then rounded to fp32, which differs by up to ~1e-6 relative (0.98: 0.019999981 against 0.02).  one_minus =
    (1 - beta1, 1 - beta2) states the latter, for holding adamw.py's own arithmetic to this bound."""
    b1, b2 = f32(beta1), f32(beta2)
    c1, c2 = (f32(1.0 - b1), f32(1.0 - b2)) if one_minus is None else (f32(one_minus[0]), f32(one_minus[1]))
    coef, eps, ss, dc = f32(coef), f32(eps), f32(step_size), f32(decay)
    p, g, m, v = (t.to(F64) for t in (p, g, m, v))
    gs = g * coef
    e_gs = U * gs.abs()
    m1 = m * b1 + gs * c1
    e_m = U * (2 * (m * b1).abs() + 2 * (gs * c1).abs()) + c1 * e_gs     # two products, one add, the gs rounding
    v1 = v * b2 + gs * gs * c2
    e_v = U * (2 * (v * b2).abs() + 3 * (gs * gs * c2).abs()) + 2 * c2 * gs.abs() * e_gs
    r = v1.sqrt()
    # sqrt of a perturbed value, then its own rounding: |sqrt(v1 + d) - sqrt(v1)| <= min(sqrt|d|, |d| / (2 sqrt v1))
    e_r = torch.minimum(e_v.sqrt(), e_v / (2 * r).clamp_min(1e-300)) + U * r
    den = r + eps
    e_den = e_r + U * den
    q = m1 / den
    e_q = (e_m + q.abs() * e_den) / (den - e_den).clamp_min(1e-300) + U * q.abs()
    p1 = p - ss * q
    e_p1 = ss * e_q + U * (ss * q).abs() + U * p1.abs()
    p2 = p1 - dc * p1
    e_p2 = e_p1 * (1 + dc) + U * (dc * p1).abs() + U * p2.abs()
    return {"p": (p2, e_p2 * SLACK), "m": (m1, e_m * SLACK), "v": (v1, e_v * SLACK)}


def step_size_of(lr: float, betas, step: int, correct_bias: bool = True) -> float:
    """adamw.py:85-89 as the host computes it (double), before the table stores it as fp32."""
    if not correct_bias:
        return lr
    return lr * math.sqrt(1.0 - betas[1] ** step) / (1.0 - betas[0] ** step)
