"""LF-VILA's hierarchical video encoder (Swin-3D with growing temporal windows) on the H100 kernels — BASELINE.json config #5.

Drop-in for `SwinTransformer3D` of LF-VILA/src/models/video_encoder.py:450-620 as `LFVILA_Pretrain` builds it from
`VideoEncoder` (configs/pretrain_stage1.yaml:1-11): same constructor arguments, same `state_dict()` (parameters and the
`relative_position_index` buffers), same `forward(x[B,3,D,H,W]) -> (x, x)` with x `[B, D, H', W', C]`.

The module tree only holds parameters; forward/backward run as ONE autograd.Function over token-major bf16 matrices
`[B*D*H*W, C]` (rows in the reference's channels-last (b, d, h, w) order):
  * PatchEmbed3D (:431-448): im2col (`xp_vip_patchify`; for uint8 frames `xp_lfvila_frames_patchify_u8`, which fuses the
    LF-VILA datasets' resize / crop / flip / Normalize in) + wgmma GEMM + LayerNorm;
  * every block (:209-268): LayerNorm -> fused-qkv GEMM -> window attention -> proj GEMM (+residual) -> LayerNorm -> MLP GEMMs
    (erf-GELU epilogue, +residual).  The reference's F.pad / torch.roll / window_partition / window_reverse / crop copies (:214-243)
    do not exist: the attention kernel (`xp_seg_attention_*` in its indexed mode) reads and writes token rows through an index
    table obtained by applying the reference's own pad/roll/partition to an index tensor once per feature-map shape.  Zero-padded
    window positions are extra all-zero input rows of the qkv GEMM, so their k, v equal the qkv bias exactly as in the reference,
    and their gradient reaches that bias;
  * relative-position bias (+ the 0/-100 shift mask) is a [window types, heads, L, L] fp32 slab added to the logits in the
    kernel; its gradient is the column sum over windows of the kernel's dL/dlogits output, scattered back to the table;
  * PatchMerging (:283-306): row gather by an index table (2x2 neighbours, odd sizes zero-padded) -> LayerNorm(4C) (a wide kernel
    above 1024 columns) -> GEMM;
  * DropPath (timm): per-sample factors drawn with the reference's torch.rand calls (shape, order), applied by `xp_rowscale_bf16`.
`local_feat` is reset in every iteration of the reference's layer loop (:600), so `norm_local` / `local_feat_proj` never influence
the returned pair; they are kept as parameters (state_dict compatibility) and their dead computation is skipped.
There is no CPU path.
"""
from __future__ import annotations

from functools import reduce
from operator import mul
from typing import Dict, NamedTuple, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib, ops
from ._blocks import drop_scale, layernorm, layernorm_bwd, linear_bwd, mlp_bwd, mlp_fwd, residual_linear
from ._weights import ParamLayout, matrix_weight, param_layout
from .lfvila_frames import INPUT_RES, Crops, eval_crops

bf16, f32 = torch.bfloat16, torch.float32
HEAD_DIM = 32


# ------------------------------------------------------------------------------ parameter containers
class _WindowAttention3D(nn.Module):
    def __init__(self, dim, window_size, num_heads):
        super().__init__()
        ws = window_size
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * ws[0] - 1) * (2 * ws[1] - 1) * (2 * ws[2] - 1), num_heads))
        coords = torch.stack(torch.meshgrid(torch.arange(ws[0]), torch.arange(ws[1]), torch.arange(ws[2]), indexing="ij"))
        flat = torch.flatten(coords, 1)                                   # video_encoder.py:108-122
        rel = (flat[:, :, None] - flat[:, None, :]).permute(1, 2, 0).contiguous()
        rel[:, :, 0] += ws[0] - 1
        rel[:, :, 1] += ws[1] - 1
        rel[:, :, 2] += ws[2] - 1
        rel[:, :, 0] *= (2 * ws[1] - 1) * (2 * ws[2] - 1)
        rel[:, :, 1] *= 2 * ws[2] - 1
        self.register_buffer("relative_position_index", rel.sum(-1))
        self.qkv = nn.Linear(dim, dim * 3, bias=True)
        self.proj = nn.Linear(dim, dim)


class _Mlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)


class _Block(nn.Module):
    def __init__(self, dim, num_heads, window_size, mlp_ratio):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn = _WindowAttention3D(dim, window_size, num_heads)
        self.norm2 = nn.LayerNorm(dim)
        self.mlp = _Mlp(dim, int(dim * mlp_ratio))


class _PatchMerging(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)
        self.norm = nn.LayerNorm(4 * dim)


class _BasicLayer(nn.Module):
    def __init__(self, dim, depth, num_heads, window_size, mlp_ratio, downsample):
        super().__init__()
        self.blocks = nn.ModuleList([_Block(dim, num_heads, window_size, mlp_ratio) for _ in range(depth)])
        self.downsample = _PatchMerging(dim) if downsample else None


class _PatchEmbed3D(nn.Module):
    def __init__(self, patch_size, in_chans, embed_dim, norm):
        super().__init__()
        self.proj = nn.Conv3d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)
        self.norm = nn.LayerNorm(embed_dim) if norm else None


class SwinTransformer3D(nn.Module):
    """Constructor mirrors video_encoder.py:473-498."""

    def __init__(self, pretrained=None, pretrained2d=True, patch_size=[1, 8, 8], in_chans=3, embed_dim=128,
                 depths=[2, 2, 14, 2, 2, 2], num_heads=[4, 8, 16, 16, 16, 32], stages=[0, 1, 2, 2, 2, 3],
                 downsample_stages=[0, 1, 4],
                 window_size=[[2, 3, 5], [4, 3, 5], [8, 3, 5], [16, 3, 5], [16, 3, 5], [32, 3, 5]], mlp_ratio=4.,
                 qkv_bias=True, qk_scale=None, drop_rate=0., attn_drop_rate=0., drop_path_rate=0.2, norm_layer=nn.LayerNorm,
                 patch_norm=False, frozen_stages=-1, local_window=4, use_checkpoint=False, temporal_no_shifting=True):
        super().__init__()
        if pretrained is not None:
            raise TypeError("pretrained checkpoints are loaded by the caller (load_state_dict): pass pretrained=None")
        if qk_scale is not None or drop_rate or attn_drop_rate or not qkv_bias or norm_layer is not nn.LayerNorm or frozen_stages >= 0:
            raise NotImplementedError("qk_scale / dropout / qkv_bias=False / custom norm / frozen stages are not used by LF-VILA "
                                      "and are not built")
        if list(patch_size)[0] != 1 or in_chans != 3:
            raise NotImplementedError("patch_size[0] must be 1 and in_chans 3 (the LF-VILA configuration)")
        for i in range(len(depths)):
            if int(embed_dim * 2 ** stages[i]) != num_heads[i] * HEAD_DIM:
                raise ValueError("the window-attention kernels are built for head_dim 32 (dim == 32 * num_heads)")
        self.num_layers, self.embed_dim, self.patch_norm = len(depths), embed_dim, patch_norm
        self.depths, self.num_heads, self.stages = list(depths), list(num_heads), list(stages)
        self.downsample_stages, self.window_size = list(downsample_stages), [list(w) for w in window_size]
        self.patch_size, self.local_window, self.temporal_no_shifting = list(patch_size), local_window, temporal_no_shifting
        self.drop_path_rate, self.mlp_ratio, self.eps = float(drop_path_rate), mlp_ratio, 1e-5
        self.patch_embed = _PatchEmbed3D(tuple(patch_size), in_chans, embed_dim, patch_norm)
        self.layers = nn.ModuleList([
            _BasicLayer(int(embed_dim * 2 ** stages[i]), depths[i], num_heads[i], self.window_size[i], mlp_ratio,
                        i in downsample_stages) for i in range(self.num_layers)])
        self.num_features = int(embed_dim * 2 ** stages[-1])
        self.norm = nn.LayerNorm(self.num_features)
        self.norm_local = nn.LayerNorm(self.num_features)                 # never reaches the output (:600)
        self.local_feat_proj = _PatchMerging(embed_dim * 2 ** 2)         # idem (:545)
        self._tables: Dict[tuple, tuple] = {}
        self.forced_drop_masks = None
        self.init_weights()

    def init_weights(self, pretrained=None):
        """video_encoder.py:564-585: trunc_normal(0.02) Linear weights and bias tables, zero biases, unit LayerNorms."""
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, nn.LayerNorm):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
            elif isinstance(m, _WindowAttention3D):
                nn.init.trunc_normal_(m.relative_position_bias_table, std=.02)

    def _declare_layout(self) -> ParamLayout:
        """bf16 copies of the GEMM weights, one gradient group; `norm_local` / `local_feat_proj` are left out."""
        return ParamLayout(self, exclude=("norm_local.", "local_feat_proj."), cast=matrix_weight)

    def draw_drop_masks(self, B: int, device, dtype):
        """Per block: the attention-branch factor then the MLP-branch factor, each floor(keep + U[0,1)) / keep of shape [B]
        (timm DropPath as SwinTransformerBlock3D applies it, :245,:260), rates linspace(0, drop_path_rate, sum(depths)) (:519)."""
        out = []
        for r in [v.item() for v in torch.linspace(0, self.drop_path_rate, sum(self.depths))]:
            if r == 0.0:
                out.append(None)
                continue
            keep = 1 - r
            out.append(tuple(((keep + torch.rand((B, 1, 1, 1, 1), dtype=dtype, device=device)).floor_() / keep).reshape(B).float()
                             for _ in range(2)))
        return out

    def forward(self, x: torch.Tensor, only_local: bool = False, crops: Optional[Crops] = None,
                out_size: Tuple[int, int] = INPUT_RES):
        """x: the transformed float video [B, 3, D, H, W], or decoder's uint8 frames [B, D, H, W, 3], which are transformed
        as LF-VILA's datasets do (modeling/lfvila_frames.py) to out_size while their patches are extracted: with `crops`
        (train_crops while training), or the val / test transform when crops is None."""
        if not x.is_cuda:
            raise _lib.XpError("xpretrain_b200 SwinTransformer3D needs CUDA tensors on an H100: there is no CPU path")
        if only_local:
            raise NotImplementedError("only_local=True (the early local_feat return, :604-605) is not built")
        u8 = None
        if x.dtype == torch.uint8:
            if x.dim() != 5 or x.shape[-1] != 3:
                raise ValueError(f"uint8 video must be decoded frames [B, D, H, W, 3] (got {list(x.shape)})")
            if self.patch_size[1:] != [8, 8] or out_size[0] % 8 or out_size[1] % 8:
                raise ValueError(f"uint8 video needs the 8 x 8 patch and an output size divisible by it (got patch "
                                 f"{self.patch_size[1:]}, out_size {tuple(out_size)})")
            u8 = (eval_crops(x.shape[0]) if crops is None else crops, tuple(out_size))
        elif crops is not None:
            raise ValueError("crops apply to uint8 frames [B, D, H, W, 3]; float video is already transformed")
        masks = None
        if self.training and self.drop_path_rate > 0:
            masks = self.forced_drop_masks if self.forced_drop_masks is not None else \
                self.draw_drop_masks(x.shape[0], x.device, f32 if u8 else x.dtype)
        # torch.is_grad_enabled() of the caller: Function.forward always runs under no_grad, and needs_input_grad reflects
        # requires_grad even then, so without it evaluation under torch.no_grad() would keep every activation to the end
        out = _Swin3DFunction.apply(self, masks, torch.is_grad_enabled(), u8, x, *param_layout(self).params)
        return out, out


# ------------------------------------------------------------------------------------ shape bookkeeping
def _clamp_window(size, window, shift):
    ws, ss = list(window), list(shift)
    for i in range(3):
        if size[i] <= window[i]:
            ws[i], ss[i] = size[i], 0
    return tuple(ws), tuple(ss)


def _window_partition_ids(ids, ws):
    B, D, H, W = ids.shape
    x = ids.view(B, D // ws[0], ws[0], H // ws[1], ws[1], W // ws[2], ws[2])
    return x.permute(0, 1, 3, 5, 2, 4, 6).contiguous().view(-1, reduce(mul, ws))


def _shift_mask(Dp, Hp, Wp, ws, ss):
    """compute_mask, video_encoder.py:309-322 (same slices, including their behaviour for zero shifts)."""
    img = torch.zeros(1, Dp, Hp, Wp)
    cnt = 0
    for d in (slice(-ws[0]), slice(-ws[0], -ss[0]), slice(-ss[0], None)):
        for h in (slice(-ws[1]), slice(-ws[1], -ss[1]), slice(-ss[1], None)):
            for w in (slice(-ws[2]), slice(-ws[2], -ss[2]), slice(-ss[2], None)):
                img[:, d, h, w] = cnt
                cnt += 1
    mw = _window_partition_ids(img, ws)
    m = mw.unsqueeze(1) - mw.unsqueeze(2)
    return m.masked_fill(m != 0, -100.0).masked_fill(m == 0, 0.0)


def _layer_geometry(model: SwinTransformer3D, i: int, B: int, D: int, H: int, W: int, device):
    """Index tables of layer i for a [B, D, H, W] token grid (cached per shape): the reference's pad / roll / partition applied to
    the token indices.  Returns dict(ws, n_real, n_pad, idx[0] (plain blocks), idx[1] (shifted blocks), mask or None)."""
    key = ("layer", i, B, D, H, W, str(device))
    geo = model._tables.get(key)
    if geo is not None:
        return geo
    window = model.window_size[i]
    shift = [w // 2 for w in window]
    if model.temporal_no_shifting:
        shift[0] = 0
    ws, ss = _clamp_window((D, H, W), window, shift)
    pd, pb, pr = (ws[0] - D % ws[0]) % ws[0], (ws[1] - H % ws[1]) % ws[1], (ws[2] - W % ws[2]) % ws[2]
    n_real = B * D * H * W
    ids = torch.arange(n_real, dtype=torch.int64).view(B, D, H, W)
    ids = F.pad(ids, (0, pr, 0, pb, 0, pd), value=-1)                     # :219 (channels-last x: W, H, D padded at the end)
    n_pad = int((ids < 0).sum())
    ids[ids < 0] = n_real + torch.arange(n_pad)                          # every padded position gets its own all-zero input row
    Dp, Hp, Wp = ids.shape[1:]
    plain = _window_partition_ids(ids, ws).to(torch.int32).to(device)
    shifted_any = any(s > 0 for s in ss)
    if shifted_any:
        rolled = torch.roll(ids, shifts=(-ss[0], -ss[1], -ss[2]), dims=(1, 2, 3))      # :223
        shifted = _window_partition_ids(rolled, ws).to(torch.int32).to(device)
        mask = _shift_mask(Dp, Hp, Wp, ws, ss).to(device)               # [nW, L, L]
    else:
        shifted, mask = plain, None
    geo = dict(ws=ws, ss=ss, n_real=n_real, n_pad=n_pad, idx=(plain, shifted), mask=mask, L=reduce(mul, ws))
    model._tables[key] = geo
    return geo


def _merge_index(model: SwinTransformer3D, B: int, D: int, H: int, W: int, device):
    """PatchMerging.forward :289-301 on token indices: [B*D*H2*W2*4] int32 (x0, x1, x2, x3 order), -1 for the odd-size padding."""
    key = ("merge", B, D, H, W, str(device))
    ent = model._tables.get(key)
    if ent is None:
        ids = torch.arange(B * D * H * W, dtype=torch.int64).view(B, D, H, W)
        if H % 2 == 1 or W % 2 == 1:
            ids = F.pad(ids, (0, W % 2, 0, H % 2), value=-1)
        cat = torch.stack([ids[:, :, 0::2, 0::2], ids[:, :, 1::2, 0::2], ids[:, :, 0::2, 1::2], ids[:, :, 1::2, 1::2]], -1)
        ent = (cat.reshape(-1).to(torch.int32).to(device), cat.shape[2], cat.shape[3])
        model._tables[key] = ent
    return ent


# --------------------------------------------------------------------------------------------- blocks
class _WindowSaved(NamedTuple):
    x: torch.Tensor          # LayerNorm-1 input [n_real, C]
    mean: torch.Tensor
    rstd: torch.Tensor
    h: torch.Tensor          # LayerNorm-1 output + the zero rows of the padded window positions [n_real + n_pad, C]
    qkv: torch.Tensor
    a: torch.Tensor          # attention output, real + padded rows
    lse: torch.Tensor
    bias: torch.Tensor       # relative-position bias (+ shift mask) slab [nW, heads, L, L]


def _block_fwd(w, p: str, blk: _Block, x, geo, shifted: bool, heads: int, save: bool, scales, B: int):
    """SwinTransformerBlock3D.forward :248-268 on tokens x [n_real, C]."""
    C_ = x.shape[1]
    dev = x.device
    n_real, n_pad, L = geo["n_real"], geo["n_pad"], geo["L"]
    n_ext = n_real + n_pad
    s_a, s_m = scales if scales is not None else (None, None)
    # norm1; the padded window positions are extra zero rows (F.pad after the norm, :219)
    h = torch.empty(n_ext, C_, dtype=bf16, device=dev)
    if n_pad:
        h[n_real:].zero_()
    _, mean1, rstd1 = layernorm(x, blk.norm1, wide=True, out=h)
    qkv = torch.empty(n_ext, 3 * C_, dtype=bf16, device=dev)
    ops.linear_fwd(h, w[p + "attn.qkv.weight"], blk.attn.qkv.bias, qkv, scale_cols=C_,
                   col_scale=HEAD_DIM ** -0.5)                            # q * scale (:145), bias included
    # relative-position bias (+ shift mask) slab [nW, heads, L, L]
    tab = blk.attn.relative_position_bias_table.detach()
    ridx = blk.attn.relative_position_index[:L, :L].reshape(-1)
    bias = tab[ridx].view(L, L, heads).permute(2, 0, 1)                   # :149-150
    mask = geo["mask"] if shifted else None
    bias = (bias.unsqueeze(0) + mask.unsqueeze(1) if mask is not None else bias.unsqueeze(0)).float().contiguous()
    idx = geo["idx"][1 if shifted else 0]
    a = torch.empty(n_ext, C_, dtype=bf16, device=dev)
    lse = torch.empty(heads, n_ext, dtype=f32, device=dev)
    desc = ops.window_desc(n_ext, heads, HEAD_DIM, 3 * C_, C_, idx, bias)
    ops.seg_attention_fwd(qkv, a, lse, desc)
    # proj on the real rows (the crop of :242-243), residual + drop_path (:260)
    x1 = residual_linear(w, p + "attn.proj", blk.attn.proj, a[:n_real], x, s_a)
    out, mlp = mlp_fwd(w, p, blk, x1, save, s_m, wide=True)
    return out, ((_WindowSaved(x, mean1, rstd1, h, qkv, a, lse, bias), mlp) if save else None)


def _block_bwd(w, p: str, blk: _Block, dx, saved, geo, shifted: bool, heads: int, grads, scales):
    win, mlp = saved
    C_ = dx.shape[1]
    dev = dx.device
    n_real, n_pad, L = geo["n_real"], geo["n_pad"], geo["L"]
    n_ext = n_real + n_pad
    s_a, s_m = scales if scales is not None else (None, None)
    dx1 = mlp_bwd(w, p, blk, dx, mlp, grads, s_m, wide=True)
    # ---- x1 = x + drop_path(proj(window_attention(LN(x))))
    da = torch.empty(n_ext, C_, dtype=bf16, device=dev)
    if n_pad:
        da[n_real:].zero_()                                               # outputs at padded positions are cropped away
    linear_bwd(w, p + "attn.proj", drop_scale(dx1, s_a), win.a[:n_real], grads, out=da[:n_real])
    idx = geo["idx"][1 if shifted else 0]
    ds = torch.empty(idx.shape[0], heads, L, L, dtype=bf16, device=dev)
    dqkv = torch.empty(n_ext, 3 * C_, dtype=bf16, device=dev)
    delta = torch.empty(heads, n_ext, dtype=f32, device=dev)
    desc = ops.window_desc(n_ext, heads, HEAD_DIM, 3 * C_, C_, idx, win.bias, ds_out=ds)
    ops.seg_attention_bwd(win.qkv, win.a, da, win.lse, delta, dqkv, desc, HEAD_DIM ** -0.5)
    # relative-position bias table: sum dL/dlogits over all windows, scatter through the fixed index (:149)
    if (heads * L * L) % 8 == 0:
        dbias = torch.zeros(heads * L * L, dtype=f32, device=dev)
        ops.colsum(ds.view(idx.shape[0], heads * L * L), dbias)
    else:                                                                # odd tiny windows: the column-sum kernel wants 16-byte rows
        dbias = ds.view(idx.shape[0], heads * L * L).float().sum(0)
    ridx = blk.attn.relative_position_index[:L, :L].reshape(-1)
    grads[p + "attn.relative_position_bias_table"].index_add_(0, ridx, dbias.view(heads, L * L).t())
    del ds
    # qkv Linear over real + padded rows (padded inputs are zero: they only reach the bias)
    dh = linear_bwd(w, p + "attn.qkv", dqkv, win.h, grads)
    return layernorm_bwd(dh[:n_real], win.x, blk.norm1, win.mean, win.rstd, dx1, grads, p + "norm1", wide=True)


# ------------------------------------------------------------------------------------------- function
class _Swin3DFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model: SwinTransformer3D, masks, grad_mode: bool, u8, video: torch.Tensor, *params):
        # u8: None for float video [B, 3, D, H, W]; (crops, (Ho, Wo)) for uint8 frames [B, D, H, W, 3]
        ph, pw = model.patch_size[1], model.patch_size[2]
        if u8 is None:
            B, Cin, D, Hin, Win = video.shape
            if Cin != 3 or Hin % ph or Win % pw:
                raise ValueError("video must be [B, 3, D, H, W] with H, W divisible by the patch size")
        else:
            (B, D), (Hin, Win) = video.shape[:2], u8[1]
        save = grad_mode and any(ctx.needs_input_grad[5:])
        w = param_layout(model)
        w.refresh()
        dev = video.device
        C0 = model.embed_dim
        # ---- PatchEmbed3D (:431-448): frames x (h, w) patches, rows already in (b, d, h, w) order
        H, W = Hin // ph, Win // pw
        rows = B * D * H * W
        K0 = 3 * ph * pw
        patches = torch.empty(rows, K0, dtype=bf16, device=dev)
        if ph != pw:
            raise NotImplementedError("square spatial patches only")
        if u8 is None:
            frames = video.permute(0, 2, 1, 3, 4).contiguous()           # [B, D, 3, H, W]
            ops.vip_patchify(frames, patches, ph)
        else:
            ops.lfvila_frames_patchify_u8(video, u8[0].params, u8[0].stage_a, u8[1], patches, ph)
        w0 = w["patch_embed.proj.weight"].view(C0, K0)
        tok = torch.empty(rows, C0, dtype=bf16, device=dev)
        ops.linear_fwd(patches, w0, model.patch_embed.proj.bias, tok)
        pe_saved = None
        if model.patch_embed.norm is not None:
            tok_n, pm, pr = layernorm(tok, model.patch_embed.norm, wide=True)
            pe_saved = (tok, pm, pr)
            tok = tok_n
        # ---- layers
        per_sample = None
        layer_saved, geos, k = [], [], 0
        for i, layer in enumerate(model.layers):
            heads = model.num_heads[i]
            geo = _layer_geometry(model, i, B, D, H, W, dev)
            blocks_saved = []
            for j, blk in enumerate(layer.blocks):
                scales = None
                if masks is not None and masks[k] is not None:
                    per_sample = D * H * W
                    scales = tuple(m.repeat_interleave(per_sample).contiguous() for m in masks[k])
                shifted = (j % 2 == 1) and any(s > 0 for s in geo["ss"])
                tok, sv = _block_fwd(w, f"layers.{i}.blocks.{j}.", blk, tok, geo, shifted, heads, save, scales, B)
                blocks_saved.append((sv, shifted, scales))
                k += 1
            merge_saved = None
            if layer.downsample is not None:
                C_ = tok.shape[1]
                midx, H2, W2 = _merge_index(model, B, D, H, W, dev)
                n_out = B * D * H2 * W2
                cat = torch.empty(n_out, 4 * C_, dtype=bf16, device=dev)
                ops.gather_rows(tok, midx, cat, C_)
                catn, mm, mr = layernorm(cat, layer.downsample.norm, wide=True)
                red = torch.empty(n_out, 2 * C_, dtype=bf16, device=dev)
                ops.linear_fwd(catn, w[f"layers.{i}.downsample.reduction.weight"], None, red)
                merge_saved = (cat, mm, mr, catn, midx, rows, C_)
                tok, H, W, rows = red, H2, W2, n_out
            layer_saved.append((blocks_saved, merge_saved))
            geos.append(geo)
        Cl = tok.shape[1]
        outn, fm, fr = layernorm(tok, model.norm, wide=True)
        out = outn.view(B, D, H, W, Cl).to(f32 if u8 else video.dtype)
        if save:
            ctx.model, ctx.geos = model, geos
            ctx.saved = (patches, pe_saved, layer_saved, (tok, fm, fr))
            ctx.dims = (B, D, H, W, Cl)
        return out

    @staticmethod
    def backward(ctx, d_out):
        model, geos = ctx.model, ctx.geos
        w = param_layout(model)
        patches, pe_saved, layer_saved, (tok_last, fm, fr) = ctx.saved
        B, D, H, W, Cl = ctx.dims
        dev = d_out.device
        grads: Dict[str, torch.Tensor] = {}
        w.alloc_grads("", grads)
        dy = d_out.reshape(B * D * H * W, Cl).to(bf16).contiguous()
        dtok = layernorm_bwd(dy, tok_last, model.norm, fm, fr, None, grads, "norm", wide=True)
        for i in reversed(range(model.num_layers)):
            layer = model.layers[i]
            blocks_saved, merge_saved = layer_saved[i]
            if merge_saved is not None:
                cat, mm, mr, catn, midx, rows_in, C_ = merge_saved
                n_out = cat.shape[0]
                name = f"layers.{i}.downsample."
                ops.linear_wgrad(dtok, catn, grads[name + "reduction.weight"])
                dcatn = torch.empty(n_out, 4 * C_, dtype=bf16, device=dev)
                ops.linear_dgrad(dtok, w[name + "reduction.weight"], dcatn)
                dcat = layernorm_bwd(dcatn, cat, layer.downsample.norm, mm, mr, None, grads, name + "norm", wide=True)
                dtok = torch.empty(rows_in, C_, dtype=bf16, device=dev)
                ops.scatter_rows(dcat, midx, dtok, C_)                    # every input row occurs exactly once
            heads = model.num_heads[i]
            for j in reversed(range(len(layer.blocks))):
                sv, shifted, scales = blocks_saved[j]
                dtok = _block_bwd(w, f"layers.{i}.blocks.{j}.", layer.blocks[j], dtok, sv, geos[i], shifted, heads, grads,
                                  scales)
                blocks_saved[j] = None
        # ---- PatchEmbed3D
        C0 = model.embed_dim
        if pe_saved is not None:
            tok0, pm, pr = pe_saved
            dtok = layernorm_bwd(dtok, tok0, model.patch_embed.norm, pm, pr, None, grads, "patch_embed.norm", wide=True)
        ops.linear_wgrad(dtok, patches, grads["patch_embed.proj.weight"].view(C0, -1))
        ops.colsum(dtok, grads["patch_embed.proj.bias"])
        ctx.saved = None
        return (None, None, None, None, None) + w.grads_out(grads, ctx.needs_input_grad[5:])
