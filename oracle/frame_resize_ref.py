"""Float64 reference and element bounds of xp_vip_resize_patchify_u8 (frame_resize.cu): decoded uint8 frames of any
size, resized, normalised and cut into the bf16 patch matrix of embed_ref.patchify_u8_ref.

  bicubic_taps / bicubic_matrices   torch's upsample_bicubic2d taps along one axis: fp32 coordinate and t, float64 weights
  resize_ref / resize_frames_ref    the resize, and the whole transform with the bound of the kernel or of torch's fp32
  resize_patchify_u8_ref            xp_vip_resize_patchify_u8 in the patch_pitch(p) layout
  rne_bf16 / bf16_allowed           float64 -> bf16 round to nearest even; the midpoint rule of a bf16 output

Pure torch; runs on the CPU or on a GPU."""
from __future__ import annotations

from typing import Sequence

import torch

from oracle.embed_ref import F32, F64, SLACK, U, _im2col, ulp_bf16

# ----------------------------------------------------------------------------------------- bicubic resize
# The reference transform of decoded frames (init_transform_dict_simple, CLIP-ViP/src/datasets/dataloader.py:209-233) as the
# pinned torchvision 0.9.0 runs it on a float tensor: F.interpolate(x / 255, size=(S, S), mode="bicubic",
# align_corners=False) with A = -0.75, border-clamped taps, no antialias and no clamp of the result; CenterCrop(S) is then
# the identity, and Normalize follows.  The source coordinate and t are torch's fp32 values (bicubic_taps); everything
# else is float64.
#
# Bounds, with r_abs = sum over the 16 taps |w_y w_x| q / 255 of an output and m, s its channel's mean and std:
#   xp_vip_resize_patchify_u8   fp32 weights rounded from float64 (1 rounding each), 4 + 4 rounded accumulation steps,
#                               / 255, - mean, / std: at most 13 u r_abs + 2 u |m| before / s  ->  KERNEL_GAMMA (r_abs + |m|) / s
#   torch's fp32 pipeline       its weights are fp32 polynomials of t: an absolute error of at most E_W each (the Horner
#                               terms of the A = -0.75 kernel stay below 8 in magnitude), on top of its own rounded sums
#                               ->  (TORCH_GAMMA (r_abs + |m|) + E_W sum over the taps (|w_y| + |w_x| + E_W) q / 255) / s
A_CUBIC = -0.75
KERNEL_GAMMA = 16 * U
TORCH_GAMMA = 32 * U
E_W = 32 * U


def bicubic_taps(n_in: int, n_out: int):
    """upsample_bicubic2d (align_corners=False) along one axis: (index [n_out, 4] int64 clamped to [0, n_in), t fp32
    [n_out], weights float64 [n_out, 4]).  scale = n_in / n_out in fp32, d + 0.5 in fp32, then scale * (d + 0.5) - 0.5
    rounded ONCE to fp32, as torch's compiled CPU loop forms it (a fused multiply-add: the product of two fp32 values is
    exact in float64, and so is the subtraction at these magnitudes).  Rounding the product and the difference separately
    moves t by an ulp of the coordinate, and misses torch 2.11's CPU output by up to 2.6 x the fp32 bound at
    240 x 320 -> 224.  Floor index clamped to n_in - 1, t to [0, 1]."""
    scale = torch.tensor(n_in, dtype=F32) / torch.tensor(n_out, dtype=F32)
    real = (scale.to(F64) * (torch.arange(n_out, dtype=F32) + 0.5).to(F64) - 0.5).to(F32)
    i = torch.floor(real).to(torch.int64).clamp_max(n_in - 1)
    t = (real - i.to(F32)).clamp(0.0, 1.0)
    x = t.to(F64)

    def near(v):
        return ((A_CUBIC + 2) * v - (A_CUBIC + 3)) * v * v + 1

    def far(v):
        return ((A_CUBIC * v - 5 * A_CUBIC) * v + 8 * A_CUBIC) * v - 4 * A_CUBIC
    w = torch.stack([far(x + 1), near(x), near(1 - x), far(2 - x)], dim=1)
    idx = (i[:, None] + torch.arange(-1, 3)[None, :]).clamp(0, n_in - 1)
    return idx, t, w


def bicubic_matrices(n_in: int, n_out: int, device=None):
    """[n_out, n_in] float64: the weights W (resize(x) = W @ x), their absolute values summed per source index, and the
    number of taps per source index (a clamped border index collects several)."""
    idx, _, w = bicubic_taps(n_in, n_out)
    rows = torch.arange(n_out)[:, None].expand(n_out, 4)
    out = []
    for v in (w, w.abs(), torch.ones_like(w)):
        m = torch.zeros(n_out, n_in, dtype=F64)
        m.index_put_((rows.reshape(-1), idx.reshape(-1)), v.reshape(-1), accumulate=True)
        out.append(m.to(device))
    return out


def resize_ref(frames_hwc: torch.Tensor, S: int):
    """uint8 [..., H, W, 3] -> float64 [F, 3, S, S]: (the bicubic resize of q / 255, r_abs, the taps' sum of
    (|w_y| + |w_x| + E_W) q / 255) — the last two for the bounds above."""
    H, W = frames_hwc.shape[-3], frames_hwc.shape[-2]
    x = frames_hwc.reshape(-1, H, W, 3).permute(0, 3, 1, 2).to(F64) / 255.0
    (wy, ay, cy), (wx, ax, cx) = bicubic_matrices(H, S, x.device), bicubic_matrices(W, S, x.device)
    r = wy @ x @ wx.t()
    r_abs = ay @ x @ ax.t()
    r_w = cy @ x @ ax.t() + ay @ x @ cx.t() + E_W * (cy @ x @ cx.t())
    return r, r_abs, r_w


def resize_frames_ref(frames_hwc: torch.Tensor, S: int, mean: Sequence[float], std: Sequence[float],
                      arithmetic: str = "kernel"):
    """The whole transform: (exact float64 [F, 3, S, S], bound) with the bound of xp_vip_resize_patchify_u8
    (arithmetic="kernel") or of torch's fp32 pipeline ("torch").  mean / std are rounded to fp32 first, as the C entry
    point and torchvision's Normalize receive them."""
    r, r_abs, r_w = resize_ref(frames_hwc, S)
    m = torch.tensor(list(mean), dtype=F32).to(F64).view(1, 3, 1, 1).to(r.device)
    s = torch.tensor(list(std), dtype=F32).to(F64).view(1, 3, 1, 1).to(r.device)
    exact = (r - m) / s
    if arithmetic == "kernel":
        bound = KERNEL_GAMMA * (r_abs + m.abs()) / s
    else:
        bound = (TORCH_GAMMA * (r_abs + m.abs()) + E_W * r_w) / s
    return exact, bound * SLACK


def resize_patchify_u8_ref(frames_hwc: torch.Tensor, S: int, p: int, mean: Sequence[float], std: Sequence[float]):
    """xp_vip_resize_patchify_u8: (exact, bound) float64 in the patch_pitch(p) layout (pad columns 0 with bound 0)."""
    exact, bound = resize_frames_ref(frames_hwc, S, mean, std)
    return _im2col(exact, p), _im2col(bound, p)


def rne_bf16(x: torch.Tensor) -> torch.Tensor:
    """float64 -> the bf16 value nearest (ties to even), as float64; one rounding (x.to(bf16) rounds through fp32)."""
    ulp = ulp_bf16(x)
    return torch.round(x.to(F64) / ulp) * ulp


def bf16_allowed(got: torch.Tensor, exact: torch.Tensor, bound: torch.Tensor):
    """The midpoint rule: got must be RNE(exact), except where exact lies within `bound` of a bf16 midpoint, where either
    neighbour passes (any bf16 value that rounds some point of [exact - bound, exact + bound]; rounding is monotone).
    -> (ok mask, mask of the elements where more than one value passes)."""
    lo, hi = rne_bf16(exact - bound), rne_bf16(exact + bound)
    g = got.to(F64)
    return (g >= lo) & (g <= hi), lo != hi
