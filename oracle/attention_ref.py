"""High-precision references of the four attention kernel families, and their bf16 arms.

Every function takes the kernels' own operands (the fused token-major qkv buffer with q already scaled by
head_dim**-0.5, the output gradient) and returns out, lse and dq / dk / dv in float64, with `q_scale` applied to dq as the
kernels do.  With `arm=None` the result is the exact float64 value of the reference semantics on those bf16 inputs.  With
an arm, the same computation rounds to bf16 exactly where the named kernel does (file:line next to each point), so that
`|arm - exact|` is the error that rounding alone costs; a kernel is held to a small multiple of it (DESIGN.md §2).

  vip_ref   CLIPAttention.forward2 (vip_attention.cu staged, vip_attention_long.cu streamed), computed frame by frame
  text_ref  CLIPAttention.forward with the causal and padding masks (text_attention.cu)
  seg_ref   groups of rows, optionally with an additive bias slab (seg_attention.cu: temporal, spatial, window)

Pure torch; runs on the CPU or on a GPU (where the tests compute it)."""
from __future__ import annotations

from typing import Dict, Optional

import torch

F64 = torch.float64
FLT_MAX = torch.finfo(torch.float32).max


def bf(x: torch.Tensor) -> torch.Tensor:
    """Round to bf16 (nearest even), keeping the tensor's dtype."""
    return x.to(torch.bfloat16).to(x.dtype)


def sdpa(q, k, v, dout=None, *, add=None, fill=None, arm: Optional[str] = None, q_scale: float = 1.0) -> Dict:
    """Softmax attention over the last two dims: q [..., n, d], k / v [..., m, d], dout [..., n, d].
    add: additive logits (-inf for masked keys), broadcastable to [..., n, m].  fill: bool, broadcastable; those logits
    become -FLT_MAX (fp32 `s + finfo.min` rounds to finfo.min for every |s| < 2^103), while the gradient still flows
    through them as through an add.  Returns out, lse and, with dout, dq (times q_scale), dk, dv and ds = dL/dlogits;
    under an arm, dq / dk / dv / out are unrounded sums of the rounded operands (the callers round once, where the kernel
    does) and ds is rounded."""
    s = q @ k.transpose(-1, -2)
    if fill is not None:
        s = s.masked_fill(fill, -FLT_MAX)
    if add is not None:
        s = s + add
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    p = e / l
    if arm == "seg":
        o = (bf(e) @ v) / l          # unnormalised P rounded for P·V: seg_attention.cu:206-218 (sum l of unrounded P :202)
    else:
        o = p @ v                    # vip: P·V with P = hi + lo, attn_wgmma.cuh fwd_step
    res = {"out": o, "lse": (m + l.log()).squeeze(-1), "p": p}
    if dout is None:
        return res
    rounds = arm in ("vip", "seg")
    # delta = rowsum(dO * O) from the bf16 O and dO the kernels read: vip_attn_bwd_kernel, vip_attention_long.cu dot16,
    # seg_attention.cu:260-286.  text_attention.cu:121-136 forms rowsum(P * dP) in fp32, which is exact here.  The O the
    # backward reads is the stored forward output: here the exact one, rounded to bf16 (the tests feed the kernels the same).
    o_d = bf(p @ v) if rounds else o
    delta = (dout * o_d).sum(-1, keepdim=True)
    ds = p * (dout @ v.transpose(-1, -2) - delta)
    if rounds:
        # P and dS rounded as MMA operands: attn_wgmma.cuh kv_step / q_step;
        # seg_attention.cu:407-411,542-544.  ds_out stores the same rounded dS (seg_attention.cu:539).
        p, ds = bf(p), bf(ds)
    res.update(dq=(ds @ k) * q_scale, dk=ds.transpose(-1, -2) @ q, dv=p.transpose(-1, -2) @ dout, ds=ds)
    return res


def _heads(x: torch.Tensor, B: int, S: int, H: int) -> torch.Tensor:
    return x.reshape(B, S, H, -1).transpose(1, 2)          # [B*S, H*d] -> [B, H, S, d]


def _rows(x: torch.Tensor) -> torch.Tensor:
    B, H, S, d = x.shape
    return x.transpose(1, 2).reshape(B * S, H * d)


def _finish(out, lse, dq, dk, dv, arm) -> Dict:
    """Outputs as the kernels store them: bf16 out / dqkv rounded once (under an arm), fp32 lse."""
    r = bf if arm is not None else (lambda x: x)
    res = {"out": r(out), "lse": lse}
    if dq is not None:
        res["dqkv"] = r(torch.cat([dq, dk, dv], dim=1))
    return res


def vip_ref(qkv, dout, B: int, H: int, T: int, L: int, M: int, q_scale: float = 1.0, arm: Optional[str] = None) -> Dict:
    """CLIPAttention.forward2 (CLIP_ViP.py:332-381) on qkv [B*S, 3C], S = M + T*L, rows per sample [M global ; T frames of L].
    Patch queries of frame t attend to [M global keys ; the L keys of frame t]; the M global queries attend to all S keys.
    Returns out [B*S, C], lse [B, H, S] and, with dout [B*S, C], dqkv [B*S, 3C].  arm="vip": out rounded once (P stays
    hi + lo); P and dS rounded in the backward; the global rows' dq / dk / dv are fp32 sums over frames rounded once
    (vip_attention.cu, vip_attn_bwd_combine_kernel)."""
    S = M + T * L
    C = qkv.shape[1] // 3
    x = qkv.to(F64)
    q, k, v = (_heads(x[:, i * C:(i + 1) * C], B, S, H) for i in range(3))
    g = _heads(dout.to(F64), B, S, H) if dout is not None else None
    out, lse = torch.empty_like(q), q.new_empty(B, H, S)
    grads = dout is not None
    dq, dk, dv = (torch.zeros_like(q) for _ in range(3)) if grads else (None, None, None)
    a = "vip" if arm is not None else None

    glob = sdpa(q[:, :, :M], k, v, g[:, :, :M] if grads else None, arm=a, q_scale=q_scale)
    out[:, :, :M], lse[:, :, :M] = glob["out"], glob["lse"]
    if grads:
        dq[:, :, :M] += glob["dq"]
        dk += glob["dk"]
        dv += glob["dv"]
    for t in range(T):
        r = slice(M + t * L, M + (t + 1) * L)
        kk = torch.cat([k[:, :, :M], k[:, :, r]], dim=2)
        vv = torch.cat([v[:, :, :M], v[:, :, r]], dim=2)
        f = sdpa(q[:, :, r], kk, vv, g[:, :, r] if grads else None, arm=a, q_scale=q_scale)
        out[:, :, r], lse[:, :, r] = f["out"], f["lse"]
        if grads:
            dq[:, :, r] += f["dq"]
            for acc, part in ((dk, f["dk"]), (dv, f["dv"])):
                acc[:, :, :M] += part[:, :, :M]
                acc[:, :, r] += part[:, :, M:]
    if not grads:
        return _finish(_rows(out), lse, None, None, None, arm)
    return _finish(_rows(out), lse, _rows(dq), _rows(dk), _rows(dv), arm)


def text_ref(qkv, mask, dout, B: int, H: int, Lt: int, q_scale: float = 1.0, arm: Optional[str] = None) -> Dict:
    """CLIPAttention.forward (CLIP_ViP.py:266-330) with the causal mask (-inf above the diagonal) and the padding mask
    (finfo.min added to the logits of keys whose mask is 0; None = no padding).  qkv [B*Lt, 3C], mask [B, Lt].
    Also returns the probabilities [B, H, Lt, Lt].  arm="text": fp32 throughout (text_attention.cu), so only the bf16
    outputs are rounded."""
    C = qkv.shape[1] // 3
    x = qkv.to(F64)
    q, k, v = (_heads(x[:, i * C:(i + 1) * C], B, Lt, H) for i in range(3))
    g = _heads(dout.to(F64), B, Lt, H) if dout is not None else None
    causal = torch.full((Lt, Lt), float("-inf"), dtype=F64, device=x.device).triu(1)
    fill = None if mask is None else (mask == 0)[:, None, None, :]
    r = sdpa(q, k, v, g, add=causal, fill=fill, q_scale=q_scale)
    res = _finish(_rows(r["out"]), r["lse"], *((_rows(r["dq"]), _rows(r["dk"]), _rows(r["dv"])) if g is not None
                                               else (None, None, None)), arm)
    res["probs"] = r["p"]
    return res


def seg_ref(qkv, dout, rows: torch.Tensor, heads: int, head_dim: int = 64, bias: Optional[torch.Tensor] = None,
            q_scale: float = 1.0, arm: Optional[str] = None) -> Dict:
    """Attention within groups of rows: rows int [n_seq, len] lists the token rows of each sequence (a temporal group, a
    spatial frame or a window); positions attend to every position of their own sequence.  bias [nW, heads, len, len] is
    added to the logits of sequence s as bias[s % nW].  Returns out [n_rows, C], lse [heads, n_rows] and, with dout,
    dqkv [n_rows, 3C] and ds [n_seq, heads, len, len] = dL/dlogits; rows no sequence lists stay zero.
    arm="seg": the unnormalised P rounded for P·V in the forward, P and dS rounded in the backward."""
    n_rows, C = qkv.shape[0], heads * head_dim
    n_seq, n = rows.shape
    idx = rows.reshape(-1).long().to(qkv.device)
    x = qkv.to(F64)[idx]

    def split(t):                                          # [n_seq*n, heads*hd] -> [n_seq, heads, n, hd]
        return t.reshape(n_seq, n, heads, head_dim).transpose(1, 2)

    def merge(t):
        return t.transpose(1, 2).reshape(n_seq * n, C)

    q, k, v = split(x[:, :C]), split(x[:, C:2 * C]), split(x[:, 2 * C:3 * C])
    g = split(dout.to(F64)[idx, :C]) if dout is not None else None
    add = None
    if bias is not None:
        nW = bias.shape[0]
        add = bias.to(F64)[torch.arange(n_seq, device=bias.device) % nW]
    r = sdpa(q, k, v, g, add=add, arm="seg" if arm is not None else None, q_scale=q_scale)
    rd = bf if arm is not None else (lambda t: t)
    out = x.new_zeros(n_rows, C)
    out[idx] = rd(merge(r["out"]))
    lse = x.new_zeros(heads, n_rows)
    lse[:, idx] = r["lse"].transpose(0, 1).reshape(heads, -1)
    res = {"out": out, "lse": lse}
    if g is not None:
        dqkv = x.new_zeros(n_rows, 3 * C)
        dqkv[idx] = rd(torch.cat([merge(r["dq"]), merge(r["dk"]), merge(r["dv"])], dim=1))
        res.update(dqkv=dqkv, ds=r["ds"])
    return res


def temporal_rows(n_rows: int, T: int) -> torch.Tensor:
    """'(b h w) t' groups: T consecutive rows each."""
    return torch.arange(n_rows).view(-1, T)


def spatial_rows(B: int, T: int, HW: int) -> torch.Tensor:
    """'(b t) (h w)' groups: the H*W rows of frame t of sample b, T rows apart (token order (h w t))."""
    b, t, s = torch.meshgrid(torch.arange(B), torch.arange(T), torch.arange(HW), indexing="ij")
    return (b * HW * T + s * T + t).reshape(B * T, HW)
