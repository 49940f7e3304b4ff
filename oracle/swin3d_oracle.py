"""CPU oracle for BASELINE.json config #5: LF-VILA's hierarchical video encoder (Swin-3D with growing temporal windows).

TEST INFRASTRUCTURE ONLY — imported by tests/, tests/golden/make_golden_swin3d.py and tools/; never by the product package.

A functional fp32 PyTorch restatement of the reference's LF-VILA/src/models/video_encoder.py (eval mode, or training mode with
explicit DropPath factors).  Parity pinned by tests/golden/make_golden_swin3d.py against the reference's own `SwinTransformer3D`
(imported with stub `timm` / `mmcv` modules): forward and every parameter gradient to fp32 round-off.

Reference lines followed:
  SwinTransformer3D.forward   video_encoder.py:587-615  patch_embed -> 6 BasicLayers -> self.norm; `local_feat` is reset to None in
                              every loop iteration (:600), so the function returns (x, x): norm_local / local_feat_proj never
                              influence the result (their parameters receive no gradient)
  PatchEmbed3D.forward        :431-448   Conv3d kernel = stride = patch_size, channels-last, optional LayerNorm
  BasicLayer.forward          :387-407   window / shift clamped to the feature size (get_window_size :67-80), shift mask from
                              compute_mask (:309-322), blocks, optional PatchMerging
  SwinTransformerBlock3D      :209-268   norm1 -> zero pad to window multiples -> cyclic shift -> window partition -> attention ->
                              reverse -> crop; residual (+DropPath); MLP(GELU) residual (+DropPath)
  WindowAttention3D.forward   :135-164   qkv, q * head_dim**-0.5, + relative-position bias (table gathered by a fixed index), + shift
                              mask (0 / -100), softmax, proj.  Zero-padded tokens are NOT masked: their k, v equal the qkv bias.
  PatchMerging.forward        :283-306   2x2 spatial neighbours concatenated [x(0,0), x(1,0), x(0,1), x(1,1)] -> LayerNorm(4C) ->
                              Linear(4C, 2C, bias=False); odd H / W zero-padded
"""
from __future__ import annotations

from dataclasses import dataclass, field
from functools import reduce
from operator import mul
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F


@dataclass
class Swin3DCfg:                      # LF-VILA/src/configs/pretrain_stage1.yaml:1-11
    patch_size: tuple = (1, 8, 8)
    in_chans: int = 3
    embed_dim: int = 128
    depths: tuple = (2, 2, 14, 2, 2, 2)
    num_heads: tuple = (4, 8, 16, 16, 16, 32)
    stages: tuple = (0, 1, 2, 2, 2, 3)
    downsample_stages: tuple = (0, 1, 4)
    window_size: tuple = ((2, 3, 5), (4, 3, 5), (8, 3, 5), (16, 3, 5), (16, 3, 5), (32, 3, 5))
    mlp_ratio: float = 4.0
    patch_norm: bool = True
    local_window: int = 8
    eps: float = 1e-5                 # nn.LayerNorm default
    temporal_no_shifting: bool = True

    def dim(self, i: int) -> int:
        return int(self.embed_dim * 2 ** self.stages[i])


def rel_pos_index(ws) -> torch.Tensor:
    """video_encoder.py:108-122: [L, L] int64 index into the (2Wd-1)(2Wh-1)(2Ww-1)-row bias table."""
    coords = torch.stack(torch.meshgrid(torch.arange(ws[0]), torch.arange(ws[1]), torch.arange(ws[2]), indexing="ij"))
    flat = torch.flatten(coords, 1)
    rel = (flat[:, :, None] - flat[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += ws[0] - 1
    rel[:, :, 1] += ws[1] - 1
    rel[:, :, 2] += ws[2] - 1
    rel[:, :, 0] *= (2 * ws[1] - 1) * (2 * ws[2] - 1)
    rel[:, :, 1] *= 2 * ws[2] - 1
    return rel.sum(-1)


def param_shapes(cfg: Swin3DCfg) -> Dict[str, tuple]:
    """state_dict of the reference module: parameters and the relative_position_index buffers."""
    C0 = cfg.embed_dim
    sh = {"patch_embed.proj.weight": (C0, cfg.in_chans) + tuple(cfg.patch_size), "patch_embed.proj.bias": (C0,)}
    if cfg.patch_norm:
        sh["patch_embed.norm.weight"] = (C0,)
        sh["patch_embed.norm.bias"] = (C0,)
    for i, depth in enumerate(cfg.depths):
        C, ws, nh = cfg.dim(i), cfg.window_size[i], cfg.num_heads[i]
        I = int(C * cfg.mlp_ratio)
        L = reduce(mul, ws)
        for j in range(depth):
            p = f"layers.{i}.blocks.{j}."
            sh[p + "norm1.weight"] = (C,); sh[p + "norm1.bias"] = (C,)
            sh[p + "attn.relative_position_bias_table"] = ((2 * ws[0] - 1) * (2 * ws[1] - 1) * (2 * ws[2] - 1), nh)
            sh[p + "attn.relative_position_index"] = (L, L)
            sh[p + "attn.qkv.weight"] = (3 * C, C); sh[p + "attn.qkv.bias"] = (3 * C,)
            sh[p + "attn.proj.weight"] = (C, C); sh[p + "attn.proj.bias"] = (C,)
            sh[p + "norm2.weight"] = (C,); sh[p + "norm2.bias"] = (C,)
            sh[p + "mlp.fc1.weight"] = (I, C); sh[p + "mlp.fc1.bias"] = (I,)
            sh[p + "mlp.fc2.weight"] = (C, I); sh[p + "mlp.fc2.bias"] = (C,)
        if i in cfg.downsample_stages:
            sh[f"layers.{i}.downsample.reduction.weight"] = (2 * C, 4 * C)
            sh[f"layers.{i}.downsample.norm.weight"] = (4 * C,); sh[f"layers.{i}.downsample.norm.bias"] = (4 * C,)
    F_ = cfg.dim(len(cfg.depths) - 1)
    for n in ("norm", "norm_local"):
        sh[n + ".weight"] = (F_,); sh[n + ".bias"] = (F_,)
    Cl = cfg.embed_dim * 4                       # local_feat_proj = PatchMerging(dim=embed_dim * 2**2)  (:545)
    sh["local_feat_proj.reduction.weight"] = (2 * Cl, 4 * Cl)
    sh["local_feat_proj.norm.weight"] = (4 * Cl,); sh["local_feat_proj.norm.bias"] = (4 * Cl,)
    return sh


def init_state_dict(cfg: Swin3DCfg, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic synthetic weights: N(0, 0.02) matrices and bias tables (the reference's trunc_normal std, :128,:571-578) with
    non-trivial biases / LayerNorm affines so that no term is hidden."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for n, s in param_shapes(cfg).items():
        if n.endswith("relative_position_index"):
            i = int(n.split(".")[1])
            sd[n] = rel_pos_index(cfg.window_size[i])
        elif "norm" in n and n.endswith(".weight"):
            sd[n] = 1.0 + 0.1 * torch.randn(s, generator=g)
        else:
            sd[n] = 0.02 * torch.randn(s, generator=g)
    return sd


def synthetic_video(B: int, D: int, H: int, W: int, cfg: Swin3DCfg, seed: int = 1234) -> torch.Tensor:
    return torch.randn(B, cfg.in_chans, D, H, W, generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------ pieces
def clamp_window(size, window, shift):
    """get_window_size, :67-80: a window (and its shift) is clamped wherever the feature map is not larger than it."""
    ws, ss = list(window), list(shift)
    for i in range(3):
        if size[i] <= window[i]:
            ws[i], ss[i] = size[i], 0
    return tuple(ws), tuple(ss)


def window_partition(x, ws):
    B, D, H, W, C = x.shape
    x = x.view(B, D // ws[0], ws[0], H // ws[1], ws[1], W // ws[2], ws[2], C)
    return x.permute(0, 1, 3, 5, 2, 4, 6, 7).contiguous().view(-1, reduce(mul, ws), C)


def window_reverse(win, ws, B, D, H, W):
    x = win.view(B, D // ws[0], H // ws[1], W // ws[2], ws[0], ws[1], ws[2], -1)
    return x.permute(0, 1, 4, 2, 5, 3, 6, 7).contiguous().view(B, D, H, W, -1)


def shift_mask(Dp, Hp, Wp, ws, ss) -> torch.Tensor:
    """compute_mask, :309-322: [nW, L, L] with 0 where two positions of a shifted window come from the same region, else -100."""
    img = torch.zeros(1, Dp, Hp, Wp, 1)
    cnt = 0
    for d in (slice(-ws[0]), slice(-ws[0], -ss[0]), slice(-ss[0], None)):
        for h in (slice(-ws[1]), slice(-ws[1], -ss[1]), slice(-ss[1], None)):
            for w in (slice(-ws[2]), slice(-ws[2], -ss[2]), slice(-ss[2], None)):
                img[:, d, h, w, :] = cnt
                cnt += 1
    mw = window_partition(img, ws).squeeze(-1)
    m = mw.unsqueeze(1) - mw.unsqueeze(2)
    return m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)


def softmax_av(logits, v):
    """softmax(logits) @ v: the attention core, kept in one function so that a calibration arm can give it the backward
    of the attention kernels (tests/encoder_cases.py)."""
    return logits.softmax(-1) @ v


def window_attention(sd, p: str, xw, heads: int, mask: Optional[torch.Tensor]):
    """WindowAttention3D.forward, :135-164.  xw: [B*nW, N, C]."""
    B_, N, C = xw.shape
    qkv = F.linear(xw, sd[p + "qkv.weight"], sd[p + "qkv.bias"]).reshape(B_, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0] * (C // heads) ** -0.5, qkv[1], qkv[2]
    attn = q @ k.transpose(-2, -1)
    idx = sd[p + "relative_position_index"][:N, :N].reshape(-1)
    bias = sd[p + "relative_position_bias_table"][idx].reshape(N, N, -1).permute(2, 0, 1)
    attn = attn + bias.unsqueeze(0)
    if mask is not None:
        nW = mask.shape[0]
        attn = (attn.view(B_ // nW, nW, heads, N, N) + mask.unsqueeze(1).unsqueeze(0)).view(-1, heads, N, N)
    out = softmax_av(attn, v).transpose(1, 2).reshape(B_, N, C)
    return F.linear(out, sd[p + "proj.weight"], sd[p + "proj.bias"])


def block_forward(sd, p: str, x, heads: int, window, shift, mask, cfg: Swin3DCfg, drop=None):
    """SwinTransformerBlock3D.forward, :248-268.  x: [B, D, H, W, C]; drop = (f_attn [B], f_mlp [B]) DropPath factors or None."""
    B, D, H, W, C = x.shape
    ws, ss = clamp_window((D, H, W), window, shift)
    h = F.layer_norm(x, (C,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], cfg.eps)
    pd, pb, pr = (ws[0] - D % ws[0]) % ws[0], (ws[1] - H % ws[1]) % ws[1], (ws[2] - W % ws[2]) % ws[2]
    h = F.pad(h, (0, 0, 0, pr, 0, pb, 0, pd))
    _, Dp, Hp, Wp, _ = h.shape
    shifted = any(s > 0 for s in ss)
    if shifted:
        h = torch.roll(h, shifts=(-ss[0], -ss[1], -ss[2]), dims=(1, 2, 3))
    aw = window_attention(sd, p + "attn.", window_partition(h, ws), heads, mask if shifted else None)
    h = window_reverse(aw.view(-1, *(ws + (C,))), ws, B, Dp, Hp, Wp)
    if shifted:
        h = torch.roll(h, shifts=ss, dims=(1, 2, 3))
    h = h[:, :D, :H, :W, :]
    if drop is not None:
        h = h * drop[0].view(B, 1, 1, 1, 1)
    x = x + h
    m = F.layer_norm(x, (C,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], cfg.eps)
    m = F.linear(F.gelu(F.linear(m, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])), sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    if drop is not None:
        m = m * drop[1].view(B, 1, 1, 1, 1)
    return x + m


def patch_merging(sd, p: str, x, cfg: Swin3DCfg):
    """PatchMerging.forward, :283-306."""
    B, D, H, W, C = x.shape
    if H % 2 == 1 or W % 2 == 1:
        x = F.pad(x, (0, 0, 0, W % 2, 0, H % 2))
    x = torch.cat([x[:, :, 0::2, 0::2, :], x[:, :, 1::2, 0::2, :], x[:, :, 0::2, 1::2, :], x[:, :, 1::2, 1::2, :]], -1)
    x = F.layer_norm(x, (4 * C,), sd[p + "norm.weight"], sd[p + "norm.bias"], cfg.eps)
    return F.linear(x, sd[p + "reduction.weight"])


def patch_embed(sd, video, cfg: Swin3DCfg):
    """PatchEmbed3D.forward, :431-448 (sizes divisible by the patch: the reference's padding branch is not exercised)."""
    x = F.conv3d(video, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=cfg.patch_size)
    x = x.permute(0, 2, 3, 4, 1).contiguous()
    if cfg.patch_norm:
        x = F.layer_norm(x, (cfg.embed_dim,), sd["patch_embed.norm.weight"], sd["patch_embed.norm.bias"], cfg.eps)
    return x


def draw_drop_masks(cfg: Swin3DCfg, B: int, drop_path_rate: float, device=None, dtype=torch.float32):
    """Training-mode DropPath factors in the reference's draw order: per block (rate linspace(0, rate, sum(depths))[k], :519)
    first the attention branch (:260), then the MLP branch (:245,:266), each floor(keep + U[0,1)) / keep of shape [B]."""
    rates = [r.item() for r in torch.linspace(0, drop_path_rate, sum(cfg.depths))]
    out = []
    for r in rates:
        if r == 0.0:
            out.append(None)
            continue
        keep = 1 - r
        out.append(tuple(((keep + torch.rand((B, 1, 1, 1, 1), dtype=dtype, device=device)).floor_() / keep).reshape(B)
                         for _ in range(2)))
    return out


def swin3d_forward(sd, video, cfg: Swin3DCfg, drop_masks: Optional[List] = None, return_stages: bool = False):
    """SwinTransformer3D.forward, :587-615.  video: [B, 3, D, H, W].  Returns x [B, D, H', W', C_last] (the reference returns the
    pair (x, x))."""
    x = patch_embed(sd, video, cfg)
    stages_out = [x]
    k = 0
    for i, depth in enumerate(cfg.depths):
        B, D, H, W, C = x.shape
        window = cfg.window_size[i]
        shift = [w // 2 for w in window]
        if cfg.temporal_no_shifting:
            shift[0] = 0
        ws, ss = clamp_window((D, H, W), window, shift)
        Dp, Hp, Wp = -(-D // ws[0]) * ws[0], -(-H // ws[1]) * ws[1], -(-W // ws[2]) * ws[2]
        mask = shift_mask(Dp, Hp, Wp, ws, ss).to(device=x.device, dtype=x.dtype)
        for j in range(depth):
            blk_shift = (0, 0, 0) if j % 2 == 0 else tuple(shift)
            x = block_forward(sd, f"layers.{i}.blocks.{j}.", x, cfg.num_heads[i], window, blk_shift, mask, cfg,
                              None if drop_masks is None else drop_masks[k])
            k += 1
        if i in cfg.downsample_stages:
            x = patch_merging(sd, f"layers.{i}.downsample.", x, cfg)
        stages_out.append(x)
    x = F.layer_norm(x, (x.shape[-1],), sd["norm.weight"], sd["norm.bias"], cfg.eps)
    return (x, stages_out) if return_stages else x


def flops_per_sample(cfg: Swin3DCfg, D: int, H: int, W: int, include_dead_local_proj: bool = False) -> float:
    """Forward FLOPs (2 per MAC) of one sample, counted like torch's FlopCounterMode does on the reference (matmuls only;
    window attention over the padded windows).  include_dead_local_proj adds the `local_feat_proj` reduction the reference
    executes at the first layer whose temporal window exceeds `local_window` and then throws away (:598-603) — with it the
    totals are BASELINE.md §2's 327.14 / 313.63 GFLOP; the useful work is 2.1 GFLOP less."""
    d, h, w = D // cfg.patch_size[0], H // cfg.patch_size[1], W // cfg.patch_size[2]
    total = 2.0 * d * h * w * cfg.embed_dim * cfg.in_chans * reduce(mul, cfg.patch_size)
    dead_done = False
    for i, depth in enumerate(cfg.depths):
        C, I = cfg.dim(i), int(cfg.dim(i) * cfg.mlp_ratio)
        if include_dead_local_proj and not dead_done and cfg.window_size[i][0] > cfg.local_window:
            dead_done = True
            total += 2.0 * d * (-(-h // 2)) * (-(-w // 2)) * 4 * C * 2 * C
        ws, _ = clamp_window((d, h, w), cfg.window_size[i], (0, 0, 0))
        dp, hp, wp = -(-d // ws[0]) * ws[0], -(-h // ws[1]) * ws[1], -(-w // ws[2]) * ws[2]
        n_real, n_pad, L = d * h * w, dp * hp * wp, reduce(mul, ws)
        per_block = 2.0 * n_pad * C * 4 * C + 4.0 * n_pad * L * C + 2.0 * n_real * 2 * C * I   # qkv+proj on padded windows, attn, MLP
        total += depth * per_block
        if i in cfg.downsample_stages:
            h, w = -(-h // 2), -(-w // 2)
            total += 2.0 * d * h * w * 4 * C * 2 * C
    return total
