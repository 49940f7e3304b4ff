"""Float64 references and element bounds for the embedding kernels (embed.cu, tsf_embed.cu).

Every function takes the kernels' own inputs.  Outputs that the kernel forms as "one fp32 sum, then one bf16 rounding" in a
fixed order are restated in fp32 in that order (`*_f32`) and held bit-exact.  The interpolated ViP table is held to
float64 with a derived bound, and so are the fp32-atomic backward sums, whose order depends on scheduling:

  atomic sum of n addends (the existing value counts as one), any order or tree:
      |fl(sum) - sum| <= (n - 1) * 2^-24 * sum |addends|                                    (first order; x 1.001)

  patchify_ref / patchify_u8_ref   xp_vip_patchify / xp_vip_patchify_u8: im2col into the patch_pitch(p) layout
  linear_taps                      F.interpolate(mode="linear", align_corners=False) taps and weights, float64
  vip_tables_ref                   xp_vip_embed_tables: table + the M global rows, fp32 restatement / float64 + bound
  vip_bwd_ref                      xp_vip_embed_bwd (accumulating): float64 + atomic bound
  text_fwd_ref / text_bwd_ref      xp_text_embed_fwd / _bwd
  eos_ref                          xp_eos_offsets: first maximum
  tsf_tokens_ref / tsf_untokenize_ref   xp_tsf_embed_fwd / xp_tsf_untokenize

Pure torch; runs on the CPU or on a GPU."""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
U = 2.0 ** -24                    # fp32 unit roundoff
SLACK = 1.001                     # second-order terms of the first-order bounds above


def patch_pitch(p: int) -> int:
    return (3 * p * p + 7) // 8 * 8


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |x| (the smallest normal spacing below 2^-126)."""
    e = torch.floor(torch.log2(x.abs().to(F64).clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def _im2col(x: torch.Tensor, p: int) -> torch.Tensor:
    """x [F, 3, H, W] (any dtype) -> [F*(H/p)*(W/p), patch_pitch(p)], column c*p*p + kh*p + kw, pad columns zero."""
    Fr, Cc, H, W = x.shape
    cols = x.reshape(Fr, Cc, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5).reshape(-1, Cc * p * p)
    out = torch.zeros(cols.shape[0], patch_pitch(p), dtype=x.dtype, device=x.device)
    out[:, :Cc * p * p] = cols
    return out


def patchify_ref(video: torch.Tensor, p: int) -> torch.Tensor:
    """video [..., 3, H, W] f32 / bf16 / f16 -> bf16 patch matrix: one conversion to fp32 (exact), one rounding to bf16."""
    H, W = video.shape[-2], video.shape[-1]
    return _im2col(video.reshape(-1, 3, H, W).float(), p).to(BF16)


def patchify_u8_ref(frames_hwc: torch.Tensor, p: int, mean: Sequence[float], std: Sequence[float]) -> torch.Tensor:
    """frames uint8 [..., H, W, 3] -> ((x / 255) - mean) / std in IEEE fp32 (mean / std rounded to fp32 first, as the C
    entry point receives them), then one rounding to bf16."""
    H, W = frames_hwc.shape[-3], frames_hwc.shape[-2]
    x = frames_hwc.reshape(-1, H, W, 3).permute(0, 3, 1, 2).to(F32) / torch.tensor(255.0, dtype=F32)
    m = torch.tensor(list(mean), dtype=F32, device=x.device).view(1, 3, 1, 1)
    s = torch.tensor(list(std), dtype=F32, device=x.device).view(1, 3, 1, 1)
    return _im2col((x - m) / s, p).to(BF16)


# ----------------------------------------------------------------------------------------- ViP tables
def linear_taps(n_in: int, n_out: int):
    """F.interpolate(mode="linear", align_corners=False) along one axis, float64: (i0, i1, lam) per output index, with
    out[i] = (1 - lam) in[i0] + lam in[i1].  n_in == n_out is the identity (lam = 0)."""
    i0, i1, lam = [], [], []
    for i in range(n_out):
        if n_in == n_out:
            i0.append(i); i1.append(i); lam.append(0.0)
            continue
        src = max((i + 0.5) * (n_in / n_out) - 0.5, 0.0)
        a = min(int(math.floor(src)), n_in - 1)
        i0.append(a)
        i1.append(a + (1 if a < n_in - 1 else 0))
        lam.append(src - a)
    return i0, i1, lam


def tap_matrix(n_in: int, n_out: int) -> torch.Tensor:
    """[n_out, n_in] float64 weights W with interp(x) = W @ x."""
    Wm = torch.zeros(n_out, n_in, dtype=F64)
    for t, (a, b, w) in enumerate(zip(*linear_taps(n_in, n_out))):
        Wm[t, a] += 1.0 - w
        Wm[t, b] += w
    return Wm


def weight_error(n_in: int, n_out: int) -> float:
    """Largest |w1(kernel) - lam| over the output indices.  embed.cu's linear_taps computes
    src = (i + 0.5) * (n_in / n_out) - 0.5 in fp32 with the build's fast division (<= 2 ulp) and two rounded operations;
    w1 = src - floor(src) is exact.  When src lies within that error of an integer, the kernel's floor may be the
    neighbouring index with w1 within the same error of 1: the same value, written through another tap."""
    if n_in == n_out:
        return 0.0
    r = n_in / n_out
    worst = 0.0
    for i in range(n_out):
        src = abs((i + 0.5) * r - 0.5)
        worst = max(worst, (i + 0.5) * 2 * 2.0 ** -23 * r + U * (i + 0.5) * r + U * src)
    return worst * SLACK


def vip_tables_ref(pos, temporal, cls, added, B: int, T: int, L: int, M: int, temporal_size: int):
    """xp_vip_embed_tables.  Returns (table_exact [T*L, C] f64, table_bound [T*L, C] f64 (0 where bit-exact),
    table_f32 [T*L, C] bf16 restatement (valid where the bound is 0), glob [B, M, C] bf16 restatement (always exact))."""
    pos64 = pos.to(F64)
    C = pos.shape[1]
    pos_rows = pos[1:1 + L]
    if temporal is None or T == temporal_size:
        tv = torch.zeros(T, C, dtype=F32, device=pos.device) if temporal is None else temporal[:T].to(F32)
        f32 = (tv[:, None, :] + pos_rows[None, :, :]).reshape(T * L, C)           # one fp32 add (tv + pos)
        table_f32 = f32.to(BF16)
        exact = (tv.to(F64)[:, None, :] + pos_rows.to(F64)[None, :, :]).reshape(T * L, C)
        return exact, torch.zeros(T * L, C, dtype=F64, device=pos.device), table_f32, _glob(pos, cls, added, B, M)
    Wm = tap_matrix(temporal_size, T).to(pos.device)
    t64 = temporal.to(F64)
    tv = Wm @ t64                                                                       # [T, C]
    exact = (tv[:, None, :] + pos64[1:1 + L][None]).reshape(T * L, C)
    i0, i1, lam = linear_taps(temporal_size, T)
    lam_t = torch.tensor(lam, dtype=F64, device=pos.device)[:, None]
    a, b = t64[i0], t64[i1]
    dw = weight_error(temporal_size, T)
    span = 2.0 * t64.abs().amax(dim=0, keepdim=True)                                     # any |a[k'] - a[k]| of the column
    # (1 - w1) rounding, two products, their sum, + pos: one rounding each; the weight error through any neighbouring tap
    e_tv = dw * span + U * (2 * ((1 - lam_t) * a).abs() + (lam_t * b).abs() + tv.abs())
    e32 = (e_tv[:, None, :] + U * exact.reshape(T, L, C).abs()).reshape(T * L, C) * SLACK
    bound = e32 + 0.5 * ulp_bf16(exact.abs() + e32)
    return exact, bound, None, _glob(pos, cls, added, B, M)


def _glob(pos, cls, added, B, M):
    rows = [cls.to(F32)] + ([added[m].to(F32) for m in range(M - 1)] if M > 1 else [])
    g = (torch.stack(rows) + pos[0].to(F32)[None]).to(BF16)                               # one fp32 add, one rounding
    return g[None].expand(B, M, -1).contiguous()


def _atomic_bound(n: torch.Tensor, abs_sum: torch.Tensor) -> torch.Tensor:
    return (n - 1).clamp_min(0).to(F64) * U * abs_sum * SLACK


def vip_bwd_ref(d_patch, d_global, init, B: int, T: int, L: int, M: int, temporal_size: int, counts=None):
    """xp_vip_embed_bwd on top of existing gradients init = dict(pos, temporal, cls, added) (fp32; temporal / added may be
    None).  Returns {name: (exact f64, bound f64)}.  Addends per element: the existing value, B*(rows that map to it) bf16
    values; d_temporal also rounds one weight product per frame and carries the weight error of weight_error().
    counts [B]: sample b stands for counts[b] identical samples (a periodic batch; B is then the period)."""
    C = d_patch.shape[-1]
    w = torch.ones(B, dtype=F64, device=d_patch.device) if counts is None else counts.to(F64).to(d_patch.device)
    dp = d_patch.to(F64).reshape(B, T, L, C) * w[:, None, None, None]
    dg = d_global.to(F64).reshape(B, M, C) * w[:, None, None]
    B = float(w.sum())
    out = {}
    p0 = init["pos"].to(F64)
    pos = p0.clone()
    pos[0] += dg.sum(dim=(0, 1))
    pos[1:1 + L] += dp.sum(dim=(0, 1))
    pabs = p0.abs().clone()
    pabs[0] += dg.abs().sum(dim=(0, 1))
    pabs[1:1 + L] += dp.abs().sum(dim=(0, 1))
    n = torch.ones(pos.shape[0], 1, dtype=F64)
    n[0] += B * M
    n[1:1 + L] += B * T
    out["pos"] = (pos, _atomic_bound(n.to(pos.device), pabs))
    c0 = init["cls"].to(F64)
    out["cls"] = (c0 + dg[:, 0].sum(0), _atomic_bound(torch.tensor(1.0 + B), c0.abs() + dg[:, 0].abs().sum(0)))
    if init.get("added") is not None and M > 1:
        a0 = init["added"].to(F64)
        ex = a0.clone()
        ex[:M - 1] += dg[:, 1:].sum(0)
        ab = a0.abs().clone()
        ab[:M - 1] += dg[:, 1:].abs().sum(0)
        out["added"] = (ex, _atomic_bound(torch.tensor(1.0 + B), ab))
    if init.get("temporal") is not None:
        t0 = init["temporal"].to(F64)
        Wm = tap_matrix(temporal_size, T).to(t0.device)                                 # [T, Tsz]
        per_t = dp.sum(dim=(0, 2))                                                       # [T, C]
        per_t_abs = dp.abs().sum(dim=(0, 2))
        ex = t0 + Wm.t() @ per_t
        nt = 2.0 + T * B * L                                                             # + the weight product
        ab = t0.abs() + Wm.t() @ per_t_abs
        bound = _atomic_bound(torch.tensor(nt), ab) + weight_error(temporal_size, T) * per_t_abs.sum(0, keepdim=True)
        out["temporal"] = (ex, bound)
    return out


# ----------------------------------------------------------------------------------------- text
def text_fwd_ref(ids: torch.Tensor, tok: torch.Tensor, pos: torch.Tensor, Lt: int):
    """xp_text_embed_fwd: (bf16 rows [rows, C], error flag).  Out-of-range ids flag the error and read row 0."""
    flat = ids.reshape(-1)
    bad = (flat < 0) | (flat >= tok.shape[0])
    idx = torch.where(bad, torch.zeros_like(flat), flat)
    s = torch.arange(flat.numel(), device=flat.device) % Lt
    return (tok[idx].to(F32) + pos[s].to(F32)).to(BF16), int(bad.any())


def text_bwd_ref(ids: torch.Tensor, dx: torch.Tensor, d_tok0: torch.Tensor, d_pos0: torch.Tensor, Lt: int):
    """xp_text_embed_bwd on top of existing gradients: {name: (exact f64, bound f64)}; out-of-range rows are skipped."""
    flat = ids.reshape(-1)
    ok = (flat >= 0) & (flat < d_tok0.shape[0])
    d = dx.to(F64)[ok]
    idx = flat[ok]
    s = (torch.arange(flat.numel(), device=flat.device) % Lt)[ok]
    res = {}
    for name, t0, where in (("tok", d_tok0, idx), ("pos", d_pos0, s)):
        ex = t0.to(F64).index_add(0, where, d)
        ab = t0.to(F64).abs().index_add(0, where, d.abs())
        n = torch.ones(t0.shape[0], dtype=F64, device=t0.device).index_add(
            0, where, torch.ones(where.numel(), dtype=F64, device=t0.device))
        res[name] = (ex, _atomic_bound(n[:, None], ab))
    return res


def eos_ref(ids: torch.Tensor, C: int):
    """xp_eos_offsets: (offsets int64 [B], index int32 [B]) with the FIRST maximum of each row."""
    B, Lt = ids.shape
    mx = ids.max(dim=1, keepdim=True).values
    pos = torch.arange(Lt, device=ids.device).expand(B, Lt)
    first = torch.where(ids == mx, pos, torch.full_like(pos, Lt)).min(dim=1).values
    return (torch.arange(B, device=ids.device) * Lt + first) * C, first.to(torch.int32)


# ----------------------------------------------------------------------------------------- TimeSformer
def tsf_tokens_ref(x: torch.Tensor, pos: Optional[torch.Tensor], time: Optional[torch.Tensor]) -> torch.Tensor:
    """xp_tsf_embed_fwd: x [B, T, C, HW] -> bf16 [(b, p, t), C] = bf16((x + pos[p]) + time[t]) in fp32, in that order."""
    B, T, C, HW = x.shape
    v = x.to(F32).permute(0, 3, 1, 2)                                                    # [B, HW, T, C]
    if pos is not None:
        v = v + pos.to(F32)[None, :, None, :]
    if time is not None:
        v = v + time.to(F32)[None, None, :, :]
    return v.reshape(B * HW * T, C).to(BF16)


def tsf_untokenize_ref(tok: torch.Tensor, B: int, T: int, C: int, HW: int, dtype: torch.dtype) -> torch.Tensor:
    """xp_tsf_untokenize: bf16 [(b, p, t), C] -> [B, T, C, HW] of dtype (bf16 -> fp32 -> dtype)."""
    return tok.reshape(B, HW, T, C).permute(0, 2, 3, 1).to(F32).to(dtype).contiguous()
