"""High-precision references of the GEMM epilogues and the row kernels, and their bf16 arms.

Every function takes the kernels' own operands (bf16 A and B, fp32 bias, bf16 residual / saved pre-activation, the
LayerNorm stream in its storage dtype) and returns float64 tensors.  `exact` is the float64 value of the operation on those
inputs; an arm rounds exactly where the kernel does (file:line next to each point), so that `|arm - exact|` is what the
rounding of the computation itself costs.  A kernel is held to a small multiple of it slice by slice (DESIGN.md §2), and,
element by element, to the deterministic fp32 accumulation bound that `absprod` feeds.

  gemm_ref            xp_gemm: C = epilogue(alpha * A B^T) in the header's order (gemm.cu)
  layernorm_ref       xp_layernorm_add_fwd / xp_layernorm_wide_fwd (rowops.cu)
  layernorm_bwd_ref   xp_layernorm_bwd / xp_layernorm_wide_bwd (rowops.cu)
  rowscale_ref, colsum_ref, l2norm_ref, l2norm_bwd_ref, gather_rows_ref, scatter_rows_ref
  repeat_counts       how often each row of a periodic operand's base block occurs (optionally with a block_weights
                      power of two per period): the reductions over its rows (split-K wgrad via gemm_ref_counted, dgamma /
                      dbeta / dres_colsum, colsum) are computed from the base block weighted by these counts, with the same
                      bounds as on the repeated operand; wrapped_column_sums gives what a dropped or displaced read sums

Pure torch; runs on the CPU or on a GPU (where the tests compute it)."""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from oracle.embed_ref import ulp_bf16

F64 = torch.float64
ACT_NONE, ACT_QUICK_GELU, ACT_DQUICK_GELU, ACT_GELU_ERF, ACT_DGELU_ERF = 0, 1, 2, 3, 4     # include/xpretrain_b200.h
OUT_BF16, OUT_F32, OUT_F32_ATOMIC = 0, 1, 2
FP16_MAX = 65504.0


def bf(x: torch.Tensor) -> torch.Tensor:
    """Round to bf16 (nearest even), keeping the tensor's dtype."""
    return x.to(torch.bfloat16).to(x.dtype)


def f32(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).to(x.dtype)


def f16_sat(x: torch.Tensor) -> torch.Tensor:
    """cvt.rn.satfinite.f16: nearest even, values beyond fp16's range become +-65504 (NaN stays NaN)."""
    return x.clamp(-FP16_MAX, FP16_MAX).to(torch.float16).to(x.dtype)


# ------------------------------------------------------------------------------------------ activations
def quick_gelu(x):
    """transformers QuickGELUActivation (CLIP_ViP.py:389), as oracle/clipvip_oracle.py:66."""
    return x * torch.sigmoid(1.702 * x)


def quick_gelu_grad(x):
    s = torch.sigmoid(1.702 * x)
    return s * (1.0 + 1.702 * x * (1.0 - s))


def gelu(x):
    """nn.GELU() (approximate='none'): the TimeSformer / Swin-3D MLPs."""
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def act_slope_bound(act: int) -> float:
    """sup |f'| of a forward activation (how far an accumulator error can move its output)."""
    return {ACT_QUICK_GELU: 1.1, ACT_GELU_ERF: 1.13}.get(act, 1.0)


# ------------------------------------------------------------------------------------------------ GEMM
def gemm_ref(a: torch.Tensor, b: torch.Tensor, *, alpha: float = 1.0, bias: Optional[torch.Tensor] = None,
             scale_cols: int = 0, col_scale: float = 1.0, act: int = ACT_NONE, residual: Optional[torch.Tensor] = None,
             aux: Optional[torch.Tensor] = None, out_mode: int = OUT_BF16, c0: Optional[torch.Tensor] = None,
             arm: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """a [M, K], b [N, K]: the logical operands (whatever their storage layout), bf16 values.  bias fp32 [N]; residual
    bf16 [M, N]; aux bf16 [M, N], the saved pre-activation a dGELU epilogue reads; c0 the starting value of an
    XP_OUT_F32_ATOMIC output.  Returns float64 `exact` (the header's order: alpha * acc, + bias, x col_scale on columns
    < scale_cols, then the activation or the residual add), `pre` (the pre-activation a forward GELU stores) and
    `absprod` = sum_k |a_mk b_nk|.

    arm='kernel' rounds where gemm.cu does: the pre-activation to bf16 (:254, :261) and the output once, to bf16 (:324) or
    fp32 (:353).  The accumulation itself is exact here; its fp32 error is bounded separately from `absprod`.
    arm='torch_bf16' (QuickGELU only) is the reference's autocast arithmetic on a bf16 fc1 output: t = bf16(v),
    bf16(t * bf16(sigmoid(bf16(1.702 t)))), every op rounded to bf16."""
    A, B = a.to(F64), b.to(F64)
    acc = A @ B.T
    absprod = A.abs() @ B.abs().T
    v = alpha * acc
    if bias is not None:
        v = v + bias.to(F64)[None, :]
    if scale_cols:
        v = torch.cat([v[:, :scale_cols] * col_scale, v[:, scale_cols:]], dim=1)
    pre = v
    if act == ACT_QUICK_GELU:
        out = quick_gelu(v)
    elif act == ACT_GELU_ERF:
        out = gelu(v)
    elif act == ACT_DQUICK_GELU:
        out = v * quick_gelu_grad(aux.to(F64))        # the bf16 aux the kernel reads (:258-259)
    elif act == ACT_DGELU_ERF:
        out = v * gelu_grad(aux.to(F64))              # (:265-266)
    else:
        out = v if residual is None else v + residual.to(F64)
    if c0 is not None:
        out = out + c0.to(F64)
    res = {"exact": out, "pre": pre, "absprod": absprod}
    if arm is None:
        return res
    if arm == "torch_bf16":
        assert act == ACT_QUICK_GELU
        t = bf(v)
        res["out"] = bf(t * bf(torch.sigmoid(bf(1.702 * t))))
        res["pre"] = t
        return res
    assert arm == "kernel"
    res["pre"] = bf(pre)
    res["out"] = bf(out) if out_mode == OUT_BF16 else f32(out)
    return res


def block_weights(n_blocks: int, device=None) -> torch.Tensor:
    """float64 [n_blocks]: a power of two per block of rows (one period of a periodic operand), 1, 2, 4 and 8 over
    successive quarters of the blocks, exact in every storage dtype.  A wrapped 32-bit offset reads from lower addresses,
    so with weights that grow along the rows the rows it reads carry less weight than the rows it should have read: the
    sum over the rows changes, where equal periods would leave it unchanged."""
    return 2.0 ** ((4 * torch.arange(n_blocks, device=device)) // n_blocks).to(F64)


def repeat_counts(stop: int, period: int, device=None, weights: Optional[torch.Tensor] = None,
                  start: int = 0) -> torch.Tensor:
    """float64 [period]: over the rows r in [start, stop) of a periodic operand, how often residue p = r % period occurs,
    each row counted with the weight of its period, weights[r // period] (1 without weights)."""
    r = torch.arange(start, stop, device=device)
    w = torch.ones(r.numel(), dtype=F64, device=device) if weights is None else weights.to(F64).to(device)[r // period]
    return torch.zeros(period, dtype=F64, device=device).index_add_(0, r % period, w)


def wrapped_column_sums(base: torch.Tensor, rows: int, weights: Optional[torch.Tensor], wrap: int):
    """The column sums of the [rows, W] periodic operand (row r = weights[r // P] x base[r % P]) as two defects would compute
    them, the elements at flat offset >= wrap (in elements) being (a) never read, (b) read from `wrap` elements earlier, as a
    32-bit byte offset that wraps inside the buffer does.  Returns float64 [W] each: (dropped, displaced)."""
    P, W = base.shape
    x = base.to(F64)
    q, s = divmod(wrap, W)
    dev = base.device
    c = torch.arange(W, device=dev)
    late = c < s                                       # columns whose first element past `wrap` is in row q + 1
    dropped, displaced = torch.empty(W, dtype=F64, device=dev), torch.empty(W, dtype=F64, device=dev)
    src_col = (c - s) % W
    for d, cols in ((0, ~late), (1, late)):
        first = min(rows, q + d)
        head = repeat_counts(first, P, dev, weights) @ x[:, cols]
        dropped[cols] = head
        # rows [first, rows) read rows [0, rows - first) at column (c - s) mod W
        displaced[cols] = head + repeat_counts(rows - first, P, dev, weights) @ x[:, src_col[cols]]
    return dropped, displaced


def gemm_ref_counted(a: torch.Tensor, b: torch.Tensor, counts: torch.Tensor, **kw) -> Dict[str, torch.Tensor]:
    """gemm_ref over a reduction whose k-rows repeat: a [M, P], b [N, P] are the base blocks (k = 0 .. P-1) and k-row p
    occurs counts[p] times.  Equal to gemm_ref on the explicitly repeated operands: `exact` and `absprod` weight each
    product by its count (counts >= 0, so sum |a b| weights the same way)."""
    return gemm_ref(a.to(F64) * counts.to(F64)[None, :], b, **kw)


def gemm_element_bound(r: Dict[str, torch.Tensor], K_split: int, splits: int, *, alpha: float = 1.0,
                       col_scale: float = 1.0, act: int = ACT_NONE, aux: Optional[torch.Tensor] = None,
                       residual: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
                       c0: Optional[torch.Tensor] = None, out_mode: int = OUT_BF16) -> torch.Tensor:
    """Per element, the largest |got - exact| a correct kernel can show: the fp32 accumulation bound
    (K_split + splits) 2^-24 absprod carried through the epilogue's slope, the epilogue's own fp32 roundings, the
    documented MUFU approximation of the sigmoid (|d s| <= 2^-12: tanh.approx, ptx.cuh fast_sigmoid) or a few fp32 ulps of
    erff / __expf, and one bf16 ulp for a bf16 output.  A dropped or doubled k-block, split or bias moves an element by
    O(its magnitude), far above this."""
    u = 2.0 ** -24
    cs = max(1.0, abs(col_scale))                     # columns past scale_cols keep slope 1
    v = r["pre"].abs()
    acc_err = (K_split + splits) * u * abs(alpha) * r["absprod"] * cs
    side = v + (0.0 if bias is None else bias.abs().to(F64)[None, :] * cs)
    if residual is not None:
        side = side + residual.to(F64).abs()
    if c0 is not None:
        side = side + c0.to(F64).abs()
    eps = 4 * u * (side + r["exact"].abs())                           # fma, col_scale, residual / atomic adds
    if out_mode == OUT_F32_ATOMIC:
        eps = eps + splits * u * (side + r["exact"].abs())
    if act in (ACT_QUICK_GELU, ACT_GELU_ERF):
        bound = act_slope_bound(act) * (acc_err + eps)
        bound = bound + (v * 2.0 ** -12 if act == ACT_QUICK_GELU else 8 * u * (v + 1.0))
    elif act == ACT_DQUICK_GELU:
        x = aux.to(F64).abs()
        bound = (acc_err + eps) * 1.2 + v * (1.0 + 1.702 * x) * 2.0 ** -12
    elif act == ACT_DGELU_ERF:
        bound = (acc_err + eps) * 1.2 + v * 8 * u * (1.0 + aux.to(F64).abs())
    else:
        bound = acc_err + eps
    if out_mode == OUT_BF16:
        bound = bound + ulp_bf16(r["exact"].abs() + bound)
    return bound


# ------------------------------------------------------------------------------------------- LayerNorm
def stream_sum(x: torch.Tensor, add: Optional[torch.Tensor]) -> torch.Tensor:
    """The LayerNorm input the kernel normalises and stores as sum_out (rowops.cu:115-128): x (+ add) added in fp32, and for
    an fp16 stream rounded to fp16 saturating (:121-124)."""
    s = x.to(F64) if add is None else f32(x.to(F64) + add.to(F64))
    if x.dtype == torch.float16 and add is not None:
        s = f16_sat(s)
    return s


def layernorm_ref(x: torch.Tensor, add: Optional[torch.Tensor], gamma: torch.Tensor, beta: torch.Tensor, eps: float,
                  y_dtype: torch.dtype = torch.bfloat16, arm: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """Rows [R, C].  exact: the float64 LayerNorm of x + add (biased variance, as nn.LayerNorm).  arm='kernel': of the
    stream value the kernel normalises (`stream_sum`), y rounded once to y_dtype (:157-158)."""
    s = stream_sum(x, add) if arm == "kernel" else (x.to(F64) if add is None else x.to(F64) + add.to(F64))
    mean = s.mean(-1, keepdim=True)
    var = ((s - mean) ** 2).mean(-1, keepdim=True)
    rstd = (var + eps) ** -0.5
    y = (s - mean) * rstd * gamma.to(F64) + beta.to(F64)
    if arm == "kernel":
        y = y.to(y_dtype).to(F64)
    return {"sum": s, "y": y, "mean": mean.squeeze(-1), "rstd": rstd.squeeze(-1), "std": (var + eps).sqrt().squeeze(-1)}


def layernorm_bwd_ref(dy: torch.Tensor, x: torch.Tensor, gamma: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor,
                      dres: Optional[torch.Tensor] = None, arm: Optional[str] = None,
                      counts: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """dx = rstd (g - mean(g) - xhat mean(g xhat)) (+ dres), g = dy gamma, xhat = (x - mean) rstd, with the mean / rstd the
    kernel reads; with exact statistics this is autograd through nn.LayerNorm.  dgamma = sum_rows dy xhat, dbeta =
    sum_rows dy, dres_colsum = sum_rows dres, and `abs_*` the sums of the magnitudes of those terms (their fp32 bounds).
    arm='kernel' rounds dx once to bf16 (rowops.cu:259).  counts [rows]: row r stands for counts[r] identical rows in the
    column sums (dx stays per row), as repeat_counts gives for a periodic operand."""
    dy, x, gm = dy.to(F64), x.to(F64), gamma.to(F64)
    xh = (x - mean.to(F64)[:, None]) * rstd.to(F64)[:, None]
    g = dy * gm
    dx = rstd.to(F64)[:, None] * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    if dres is not None:
        dx = dx + dres.to(F64)
    w = 1.0 if counts is None else counts.to(F64)[:, None]
    res = {"dx": bf(dx) if arm == "kernel" else dx, "dgamma": (w * dy * xh).sum(0), "dbeta": (w * dy).sum(0),
           "abs_dgamma": (w * (dy * xh).abs()).sum(0), "abs_dbeta": (w * dy.abs()).sum(0)}
    if dres is not None:
        res["dres_colsum"] = (w * dres.to(F64)).sum(0)
        res["abs_dres_colsum"] = (w * dres.to(F64).abs()).sum(0)
    return res


# ------------------------------------------------------------------------------------ small row kernels
def rowscale_ref(x, scale, residual=None):
    """out = (residual or 0) + scale[r] x (rowscale_kernel, rowops.cu:451-472): one fp32 fma, one bf16 rounding.  fp32 with
    a single rounding equals the exact float64 value rounded once, except in the rare double-rounding case, so the
    reference is float64 and the test compares after the kernel's one bf16 rounding."""
    v = scale.to(F64)[:, None] * x.to(F64)
    if residual is not None:
        v = v + residual.to(F64)
    return v


def colsum_ref(x, scale=1.0, counts=None):
    """(scale x sum_rows x, |scale| x sum_rows |x|); counts [rows]: row r stands for counts[r] identical rows."""
    w = 1.0 if counts is None else counts.to(F64)[:, None]
    return scale * (w * x.to(F64)).sum(0), abs(scale) * (w * x.to(F64).abs()).sum(0)


def l2norm_ref(x):
    x = x.to(F64)
    n = x.norm(dim=-1, keepdim=True)
    return {"y": x / n, "inv_norm": 1.0 / n.squeeze(-1)}


def l2norm_bwd_ref(dy, y, inv_norm, scale=1.0):
    """dx = scale (dy - y (y . dy)) inv_norm, from the y / inv_norm the kernel reads (rowops.cu:308-322)."""
    dy, y = dy.to(F64), y.to(F64)
    s = (dy * y).sum(-1, keepdim=True)
    return scale * (dy - y * s) * inv_norm.to(F64)[:, None]


def gather_rows_ref(src, index):
    out = torch.zeros(index.numel(), src.shape[1], dtype=src.dtype, device=src.device)
    ok = index >= 0
    out[ok] = src[index[ok].long()]
    return out


def scatter_rows_ref(inp, index, dst):
    out = dst.clone()
    ok = index >= 0
    out[index[ok].long()] = inp[ok]
    return out
