"""Float64 reference and element bounds of xp_lfvila_frames_patchify_u8 (lfvila_frames.cu): decoded uint8 frames through
LF-VILA's input transform (init_transform_dict, LF-VILA/src/datasets/dataloader.py:94-121) into Swin-3D's bf16 patch
matrix.

  linear_taps / linear_matrix   torch's bilinear taps along one axis: fp32 coordinate and lambda, float64 weights
  composite_taps / axis_matrix  stage A, the crop box, stage B and the mirror along one axis: the kernel's 4 taps, and
                                their float64 matrix
  transform_ref                 the whole transform of a batch of clips, with the bound of the kernel or of torch's fp32
                                pipeline
  patchify_ref                  xp_lfvila_frames_patchify_u8's patch matrix [B*N*(Ho/8)*(Wo/8), 192]

Pure torch; runs on the CPU or on a GPU."""
from __future__ import annotations

from typing import Sequence

import torch

from oracle.embed_ref import F32, F64, SLACK, U, _im2col
from oracle.frame_resize_ref import bf16_allowed, rne_bf16  # noqa: F401  (the midpoint rule of the bf16 outputs)

# The reference transform as the pinned torchvision 0.11 runs it on `.float() / 255` frames: each Resize and the resize of
# RandomResizedCrop is F.interpolate(mode="bilinear", align_corners=False) with no antialias, crops are exact slices,
# hflip mirrors the columns, then Normalize.  Val / test: resize to (240, 428), crop (12, 22, 216, 385), resize to
# input_res.  Train: crop the frame itself (stage A is the identity), resize to input_res, maybe mirror.  The source
# coordinates and lambdas are torch's fp32 values (linear_taps); everything else is float64.
#
# Bounds, with r = sum over an output's taps of w_y w_x q / 255 (the weights are >= 0, so r is also the sum of the
# absolute terms) and m, s its channel's mean and std:
#   xp_lfvila_frames_patchify_u8  fp32 weights rounded once from float64 (1 rounding each), 4 + 4 rounded accumulation
#                                 steps, / 255, - mean, / std: at most 13 u r + 2 u |m| before / s
#                                 ->  KERNEL_GAMMA (r + |m|) / s
#   torch's fp32 pipeline         q / 255 rounded (1); per resize: lambda0 = 1 - lambda1 rounded (1 relative, as
#                                 lambda0 >= 1/2 whenever it is inexact), the row and column weights (2), the two-tap sums
#                                 of each axis (4); stage B of stage A's rounded output; - mean, / std: at most
#                                 15 u r + 2 u |m| before / s  ->  TORCH_GAMMA (r + |m|) / s
KERNEL_GAMMA = 16 * U
TORCH_GAMMA = 16 * U


def linear_taps(n_in: int, n_out: int):
    """upsample_bilinear2d (align_corners=False) along one axis: (i0, i1 [n_out] int64, lambda1 fp32 [n_out]).  scale =
    n_in / n_out in fp32, d + 0.5 in fp32, then scale * (d + 0.5) - 0.5 rounded ONCE to fp32 (the fused multiply-add of
    torch's compiled CPU loop; test_lfvila_frames_cpu pins it) and clamped at 0; i0 = floor clamped to n_in - 1, i1 its
    neighbour clamped to n_in - 1, lambda1 = coordinate - i0 clamped to [0, 1]."""
    scale = torch.tensor(n_in, dtype=F32) / torch.tensor(n_out, dtype=F32)
    real = (scale.to(F64) * (torch.arange(n_out, dtype=F32) + 0.5).to(F64) - 0.5).to(F32).clamp_min(0.0)
    i0 = torch.floor(real).to(torch.int64).clamp_max(n_in - 1)
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    return i0, i1, (real - i0.to(F32)).clamp(0.0, 1.0)


def linear_matrix(n_in: int, n_out: int) -> torch.Tensor:
    """[n_out, n_in] float64 W with resize(x) = W @ x: weights 1 - lambda1 at i0 and lambda1 at i1."""
    i0, i1, t = linear_taps(n_in, n_out)
    t = t.to(F64)
    m = torch.zeros(n_out, n_in, dtype=F64)
    rows = torch.arange(n_out)
    m.index_put_((rows, i0), 1.0 - t, accumulate=True)
    m.index_put_((rows, i1), t, accumulate=True)
    return m


def composite_taps(n_src: int, n_a: int, box0: int, length: int, n_out: int, flip: bool = False):
    """The kernel's taps along one axis: (index [n_out, 4] int64, float64 weight [n_out, 4]) = stage B's two taps over the
    box (clamped to it), each through stage A's two taps, in that order; the weights are the float64 products w_B w_A the
    kernel rounds once to fp32.  flip mirrors the output."""
    b0, b1, tb = linear_taps(length, n_out)
    a0, a1, ta = linear_taps(n_src, n_a)
    tb, ta = tb.to(F64), ta.to(F64)
    idx, w = [], []
    for b, wb in ((b0, 1.0 - tb), (b1, tb)):
        a = box0 + b
        idx += [a0[a], a1[a]]
        w += [wb * (1.0 - ta[a]), wb * ta[a]]
    idx, w = torch.stack(idx, 1), torch.stack(w, 1)
    return (idx.flip(0), w.flip(0)) if flip else (idx, w)


def axis_matrix(n_src: int, n_a: int, box0: int, length: int, n_out: int, flip: bool = False) -> torch.Tensor:
    """[n_out, n_src] float64: stage A (n_src -> n_a), the box [box0, box0 + length), stage B (length -> n_out), mirror."""
    m = linear_matrix(length, n_out) @ linear_matrix(n_src, n_a)[box0:box0 + length]
    return m.flip(0) if flip else m


def transform_ref(frames_hwc: torch.Tensor, params, stage_a, out_size, mean: Sequence[float], std: Sequence[float],
                  arithmetic: str = "kernel"):
    """uint8 [B, N, H, W, 3], params [B, 5] (top, left, h, w, flip) -> (exact float64 [B, N, 3, Ho, Wo], bound) with the
    bound of xp_lfvila_frames_patchify_u8 (arithmetic="kernel") or of torch's fp32 pipeline ("torch").  mean / std are
    rounded to fp32 first, as the C entry point and torchvision's Normalize receive them."""
    B, N, H, W, _ = frames_hwc.shape
    (Ha, Wa), (Ho, Wo) = stage_a, out_size
    dev = frames_hwc.device
    m = torch.tensor(list(mean), dtype=F32).to(F64).view(1, 3, 1, 1).to(dev)
    s = torch.tensor(list(std), dtype=F32).to(F64).view(1, 3, 1, 1).to(dev)
    gamma = KERNEL_GAMMA if arithmetic == "kernel" else TORCH_GAMMA
    exact = torch.empty(B, N, 3, Ho, Wo, dtype=F64, device=dev)
    bound = torch.empty_like(exact)
    for b, (top, left, h, w, flip) in enumerate(torch.as_tensor(params).tolist()):
        my = axis_matrix(H, Ha, top, h, Ho).to(dev)
        mx = axis_matrix(W, Wa, left, w, Wo, bool(flip)).to(dev)
        x = frames_hwc[b].permute(0, 3, 1, 2).to(F64) / 255.0
        r = my @ x @ mx.t()
        exact[b] = (r - m) / s
        bound[b] = gamma * (r + m.abs()) / s
    return exact, bound * SLACK


def patchify_ref(frames_hwc: torch.Tensor, params, stage_a, out_size, mean: Sequence[float], std: Sequence[float]):
    """xp_lfvila_frames_patchify_u8: (exact, bound) float64 [B*N*(Ho/8)*(Wo/8), 192], rows (b, d, h, w), columns
    (c, kh, kw), with the kernel's bound."""
    exact, bound = transform_ref(frames_hwc, params, stage_a, out_size, mean, std)
    Ho, Wo = out_size
    return _im2col(exact.reshape(-1, 3, Ho, Wo), 8), _im2col(bound.reshape(-1, 3, Ho, Wo), 8)
