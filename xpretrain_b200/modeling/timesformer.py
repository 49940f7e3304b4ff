"""HD-VILA's TimeSformer on the H100 kernels — BASELINE.json config #4.

Drop-in for `TimeSformer` of hd-vila/src/modeling/timesformer.py:421-525 as `HDVILA.__init__` builds it
(e2e_model.py:53-55): same constructor arguments, same `state_dict()` names and shapes (`pos_embed`, `time_embed`,
`blocks.N.{norm1,attn.qkv,attn.proj,temporal_norm1,temporal_attn.qkv,temporal_attn.proj,temporal_fc,norm2,mlp.fc1,
mlp.fc2}`, and the never-applied `norm`), same `forward(x[B,T,C,H,W]) -> [B,T,C,H,W]`.

All three attention types of the reference's `Block` (:181) are built:
  * 'divided_space_time' (HD-VILA's): temporal then spatial attention per block, as described below;
  * 'joint_space_time': one dense attention over the H*W*T tokens of each clip (:202-205); the blocks have no
    temporal_norm1 / temporal_attn / temporal_fc (:187-191);
  * 'space_only': dense attention within each frame and no `time_embed` (:440, :501), then the frame mean (:519-522).
    The reference's output path only runs at T = 1 (at T > 1 the mean over T is followed by reshape(B, T, H, W, C),
    which raises), so only T = 1 is built, where the '(b t) (h w)' token order equals '(h w t)'; T > 1 raises
    RuntimeError before any launch.
The two dense types run `xp_dense_attention_*` (TMA + wgmma) on the same fused qkv buffer.

The module tree only holds parameters.  forward/backward run as ONE autograd.Function over token-major bf16 matrices
`[B*H*W*T, C]` in the reference's `(h w t)` row order:
  * every Linear is the wgmma GEMM (`xp_gemm`) with bias / q-scale / erf-GELU / residual epilogues,
  * both attentions are `xp_seg_attention_*` reading the fused qkv buffer through strides — the six einops rearranges
    per block of timesformer.py:210-219 never materialise,
  * LayerNorm fwd/bwd are the row kernels shared with CLIP-ViP.
  * stochastic depth (DropPath, timesformer.py:98-121) in training mode: the per-group keep factors are drawn with the
    reference's own torch.rand calls (same shapes and order, so the same seed drops the same paths) and applied by a
    row-scale kernel on the three residual branches (one extra elementwise pass each; eval mode fuses the residual add
    into the GEMM epilogue).
There is no CPU path.
"""
from __future__ import annotations

import math
from typing import Dict, List

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib, ops
from .clip_vip import _alloc_flat

bf16, f32 = torch.bfloat16, torch.float32
ATTENTION_TYPES = ('divided_space_time', 'space_only', 'joint_space_time')


class _TsfAttention(nn.Module):
    def __init__(self, dim: int, qkv_bias: bool):
        super().__init__()
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)     # timesformer.py:151
        self.proj = nn.Linear(dim, dim)


class _TsfMlp(nn.Module):
    def __init__(self, dim: int, hidden: int):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)


class _TsfBlock(nn.Module):
    def __init__(self, dim: int, hidden: int, qkv_bias: bool, eps: float, divided: bool = True):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=eps)
        self.attn = _TsfAttention(dim, qkv_bias)
        if divided:                                           # timesformer.py:187-191
            self.temporal_norm1 = nn.LayerNorm(dim, eps=eps)
            self.temporal_attn = _TsfAttention(dim, qkv_bias)
            self.temporal_fc = nn.Linear(dim, dim)
        self.norm2 = nn.LayerNorm(dim, eps=eps)
        self.mlp = _TsfMlp(dim, hidden)


class TimeSformer(nn.Module):
    """Constructor mirrors timesformer.py:424-427 (only the arguments HD-VILA uses change behaviour)."""

    def __init__(self, depth=12, num_frames=7, H=10, W=16, embed_dim=768, num_heads=12, mlp_ratio=4., qkv_bias=True,
                 qk_scale=None, drop_rate=0., attn_drop_rate=0., drop_path_rate=0.1, norm_layer=None,
                 attention_type='divided_space_time', timesformer_type='new', dropout=0.):
        super().__init__()
        if attention_type not in ATTENTION_TYPES:      # timesformer.py:182
            raise ValueError(f"attention_type must be one of {ATTENTION_TYPES}, got {attention_type!r}")
        if embed_dim != num_heads * 64:
            raise ValueError("the attention kernels are built for head_dim 64 (embed_dim == 64 * num_heads)")
        if qk_scale is not None or drop_rate or attn_drop_rate or dropout or not qkv_bias:
            raise NotImplementedError("qk_scale / dropout / qkv_bias=False are not used by HD-VILA and are not built")
        self.depth, self.H, self.W, self.embed_dim, self.num_heads = depth, H, W, embed_dim, num_heads
        self.num_features = embed_dim
        self.attention_type, self.timesformer_type = attention_type, timesformer_type
        self.drop_path_rate = float(drop_path_rate)
        self.eps = 1e-6 if norm_layer is None else getattr(norm_layer, "keywords", {}).get("eps", 1e-5)
        self.pos_embed = nn.Parameter(torch.zeros(1, H * W, embed_dim))
        if attention_type != 'space_only':              # timesformer.py:440
            self.time_embed = nn.Parameter(torch.zeros(1, num_frames, embed_dim))
        hidden = int(embed_dim * mlp_ratio)
        divided = attention_type == 'divided_space_time'
        self.blocks = nn.ModuleList([_TsfBlock(embed_dim, hidden, qkv_bias, self.eps, divided) for _ in range(depth)])
        self.norm = nn.LayerNorm(embed_dim, eps=self.eps)   # constructed, never applied (timesformer.py:451)
        self._cache: Dict[str, list] = {}
        self.forced_drop_masks = None     # tests: per-block (m_t, m_s, m_m) factors instead of fresh random draws
        self._init_weights()

    def _init_weights(self):
        """timesformer.py:453-473: trunc_normal(0.02) weights, zero biases, unit LayerNorms, temporal_fc of blocks > 0 zeroed
        (divided_space_time only, :458-466)."""
        nn.init.trunc_normal_(self.pos_embed, std=.02)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, nn.LayerNorm):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        for i, blk in enumerate(self.blocks):
            if i > 0 and self.attention_type == 'divided_space_time':
                nn.init.zeros_(blk.temporal_fc.weight)
                nn.init.zeros_(blk.temporal_fc.bias)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {'pos_embed', 'time_embed'}

    def draw_drop_masks(self, B: int, T: int, H: int, W: int, device, dtype):
        """Stochastic-depth factors of one training forward (timesformer.py:98-113): block i (rate
        linspace(0, drop_path_rate, depth)[i], :445) draws, in this order, floor(keep + U[0,1)) / keep per temporal group
        (b h w) (:212), per spatial group (b t) (:218) and per sample (:225) — the same torch.rand calls, shapes and
        order as the reference, so an identically seeded run drops the same paths.  'joint_space_time' and 'space_only'
        (:202-205) draw two factors per sample of the blocks' batch, B and B*T respectively: attention, then MLP."""
        groups = (B * H * W, B * T, B) if self.attention_type == 'divided_space_time' else \
            (B, B) if self.attention_type == 'joint_space_time' else (B * T, B * T)
        masks = []
        for r in [v.item() for v in torch.linspace(0, self.drop_path_rate, self.depth)]:
            if r == 0.0:
                masks.append(None)
                continue
            keep = 1 - r
            masks.append(tuple(((keep + torch.rand((n, 1, 1), dtype=dtype, device=device)).floor_() / keep).reshape(n).float()
                               for n in groups))
        return masks

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.attention_type == 'space_only' and x.shape[1] != 1:
            raise RuntimeError("attention_type='space_only' runs at T = 1 only: the reference's frame mean is followed "
                               "by reshape(B, T, H, W, C), which fails for T > 1 (timesformer.py:519-522)")
        if not x.is_cuda:
            raise _lib.XpError("xpretrain_b200 TimeSformer needs CUDA tensors on an H100: there is no CPU path")
        masks = None
        if self.training and self.drop_path_rate > 0:
            B, T, _, H, W = x.shape
            masks = self.forced_drop_masks if self.forced_drop_masks is not None else \
                self.draw_drop_masks(B, T, H, W, x.device, x.dtype)
        names, params = zip(*[(n, p) for n, p in self.named_parameters() if not n.startswith("norm.")])
        return _TimeSformerFunction.apply(self, list(names), masks, x, *params)


# ----------------------------------------------------------------------------------- helpers
def _w(model, name: str, p: torch.Tensor) -> torch.Tensor:
    """bf16 compute copy of a GEMM weight (refreshed for the whole model at the start of every forward)."""
    return model._cache[name]


def refresh_weights(model) -> None:
    """Re-cast every GEMM weight (parameters with >= 2 dims that `_w` serves) with ONE launch on every forward: in-place
    `p.data` updates of the reference optimizers do not move `_version`, so no validity test is used (modeling/_weights.py)."""
    from ._weights import WeightMirror
    cache = model._cache
    named = [(n, p) for n, p in model.named_parameters() if p.dim() >= 2 and n.endswith("weight")]
    dev = named[0][1].device
    if cache.get("__device__") != dev:
        cache.clear()
        cache["__device__"] = dev
        cache["__mirror__"] = WeightMirror()
        for n, p in named:
            cache[n] = torch.empty(p.shape, dtype=bf16, device=dev)
    cache["__mirror__"].refresh([(p, cache[n]) for n, p in named])


def _tables(model: TimeSformer, T: int, H: int, W: int, pos_param=None, time_param=None):
    """pos [H*W, C] / time [T, C] fp32 as the forward adds them: bilinear / linear interpolation of the learned tables
    when the grid or the frame count differs (timesformer.py:487-494, 504-508).  Parameter preprocessing on tiny
    tensors (torch); with `pos_param`/`time_param` given it is differentiable (used to pull table gradients back).
    time is None for 'space_only', which has no time table (:501)."""
    C_ = model.embed_dim
    pos = model.pos_embed.detach() if pos_param is None else pos_param
    if H != model.H or W != model.W:
        grid = pos[0].unsqueeze(0).transpose(1, 2).reshape(1, C_, model.H, model.W)
        pos = F.interpolate(grid, size=(H, W), mode='bilinear').flatten(2).transpose(1, 2)
    if not hasattr(model, "time_embed"):
        return pos[0].float().contiguous(), None
    time = model.time_embed.detach() if time_param is None else time_param
    if T != time.shape[1]:
        time = F.interpolate(time.transpose(1, 2), size=T, mode='linear').transpose(1, 2)
    return pos[0].float().contiguous(), time[0].float().contiguous()


def _ln(x, ln: nn.LayerNorm, rows: int, C_: int, eps: float):
    plain = ops.rowmap(C_)
    mean = torch.empty(rows, dtype=f32, device=x.device)
    rstd = torch.empty_like(mean)
    y = torch.empty(rows, C_, dtype=bf16, device=x.device)
    ops.layernorm_fwd(x, plain, y, plain, ln.weight, ln.bias, mean, rstd, rows, C_, eps)
    return y, mean, rstd


def _attn_fwd(model, pre: str, att: _TsfAttention, h, desc, rows: int, C_: int):
    dev = h.device
    qkv = torch.empty(rows, 3 * C_, dtype=bf16, device=dev)
    # (q k^T) * head_dim**-0.5 (timesformer.py:165): 0.125 is a power of two, folding it into q (bias included) is exact
    ops.linear_fwd(h, _w(model, pre + "qkv.weight", att.qkv.weight), att.qkv.bias, qkv, scale_cols=C_, col_scale=0.125)
    a = torch.empty(rows, C_, dtype=bf16, device=dev)
    lse = torch.empty(model.num_heads, rows, dtype=f32, device=dev)
    if isinstance(desc, _lib.XpDenseAttn):
        ops.dense_attention_fwd(qkv, a, lse, desc)
    else:
        ops.seg_attention_fwd(qkv, a, lse, desc)
    return qkv, a, lse


def _row_scales(masks, B: int, T: int, HW: int):
    """Per-token-row DropPath factors (rows ordered (b, p, t)) from the per-group factors of one block."""
    if masks is None:
        return None
    m_t, m_s, m_m = masks
    return (m_t.repeat_interleave(T).contiguous(),
            m_s.view(B, 1, T).expand(B, HW, T).reshape(-1).contiguous(),
            m_m.repeat_interleave(HW * T).contiguous())


def _residual_linear(model, name: str, lin: nn.Linear, a, residual, scale, rows: int, C_: int):
    """residual + drop_path(lin(a)): fused into the GEMM epilogue when no path is dropped, else GEMM + one row-scale pass."""
    out = torch.empty(rows, C_, dtype=bf16, device=a.device)
    if scale is None:
        ops.linear_fwd(a, _w(model, name + ".weight", lin.weight), lin.bias, out, residual=residual, ldr=C_)
    else:
        tmp = torch.empty(rows, C_, dtype=bf16, device=a.device)
        ops.linear_fwd(a, _w(model, name + ".weight", lin.weight), lin.bias, tmp)
        ops.rowscale(tmp, scale, out, residual=residual)
    return out


def _block_fwd(model: TimeSformer, i: int, x, descs, rows: int, save: bool, scales=None):
    """timesformer.py:207-226.  x: [rows, C] bf16 tokens, (h w t) order.  scales: per-row DropPath factors
    (temporal, spatial, mlp) of this block or None."""
    blk = model.blocks[i]
    C_, I = model.embed_dim, blk.mlp.fc1.weight.shape[0]
    dev, p = x.device, f"blocks.{i}."
    d_t, d_s = descs
    s_t, s_s, s_m = scales if scales is not None else (None, None, None)
    # ---- temporal attention -> proj -> drop_path -> temporal_fc -> residual (:209-214)
    ln_t, mean_t, rstd_t = _ln(x, blk.temporal_norm1, rows, C_, model.eps)
    qkv_t, a_t, lse_t = _attn_fwd(model, p + "temporal_attn.", blk.temporal_attn, ln_t, d_t, rows, C_)
    p_t = torch.empty(rows, C_, dtype=bf16, device=dev)
    ops.linear_fwd(a_t, _w(model, p + "temporal_attn.proj.weight", blk.temporal_attn.proj.weight),
                   blk.temporal_attn.proj.bias, p_t)
    if s_t is not None:
        ops.rowscale(p_t, s_t, p_t)          # in place: the saved p_t is the dropped one, as temporal_fc consumed it
    xt = torch.empty(rows, C_, dtype=bf16, device=dev)
    ops.linear_fwd(p_t, _w(model, p + "temporal_fc.weight", blk.temporal_fc.weight), blk.temporal_fc.bias, xt,
                   residual=x, ldr=C_)
    # ---- spatial attention -> proj -> residual (:216-224)
    ln_s, mean_s, rstd_s = _ln(xt, blk.norm1, rows, C_, model.eps)
    qkv_s, a_s, lse_s = _attn_fwd(model, p + "attn.", blk.attn, ln_s, d_s, rows, C_)
    x2 = _residual_linear(model, p + "attn.proj", blk.attn.proj, a_s, xt, s_s, rows, C_)
    # ---- MLP with exact-erf GELU (:225, :132-138)
    ln_m, mean_m, rstd_m = _ln(x2, blk.norm2, rows, C_, model.eps)
    pre = torch.empty(rows, I, dtype=bf16, device=dev) if save else None
    f1 = torch.empty(rows, I, dtype=bf16, device=dev)
    ops.linear_fwd(ln_m, _w(model, p + "mlp.fc1.weight", blk.mlp.fc1.weight), blk.mlp.fc1.bias, f1,
                   act=_lib.ACT_GELU_ERF, aux=pre, ld_aux=I)
    out = _residual_linear(model, p + "mlp.fc2", blk.mlp.fc2, f1, x2, s_m, rows, C_)
    saved = (x, mean_t, rstd_t, ln_t, qkv_t, a_t, lse_t, p_t, xt, mean_s, rstd_s, ln_s, qkv_s, a_s, lse_s, x2, mean_m,
             rstd_m, ln_m, pre, f1) if save else None
    return out, saved


def _dense_block_fwd(model: TimeSformer, i: int, x, desc, rows: int, save: bool, scales=None):
    """timesformer.py:202-205 ('joint_space_time' / 'space_only'): x + drop_path(attn(norm1(x))), then the MLP.  The
    attention is dense within each sequence of `desc`; scales: per-row DropPath factors (attention, mlp) or None."""
    blk = model.blocks[i]
    C_, I = model.embed_dim, blk.mlp.fc1.weight.shape[0]
    dev, p = x.device, f"blocks.{i}."
    s_a, s_m = scales if scales is not None else (None, None)
    ln_a, mean_a, rstd_a = _ln(x, blk.norm1, rows, C_, model.eps)
    qkv, a, lse = _attn_fwd(model, p + "attn.", blk.attn, ln_a, desc, rows, C_)
    x2 = _residual_linear(model, p + "attn.proj", blk.attn.proj, a, x, s_a, rows, C_)
    ln_m, mean_m, rstd_m = _ln(x2, blk.norm2, rows, C_, model.eps)
    pre = torch.empty(rows, I, dtype=bf16, device=dev) if save else None
    f1 = torch.empty(rows, I, dtype=bf16, device=dev)
    ops.linear_fwd(ln_m, _w(model, p + "mlp.fc1.weight", blk.mlp.fc1.weight), blk.mlp.fc1.bias, f1,
                   act=_lib.ACT_GELU_ERF, aux=pre, ld_aux=I)
    out = _residual_linear(model, p + "mlp.fc2", blk.mlp.fc2, f1, x2, s_m, rows, C_)
    saved = (x, mean_a, rstd_a, ln_a, qkv, a, lse, x2, mean_m, rstd_m, ln_m, pre, f1) if save else None
    return out, saved


def _linear_bwd(model, name: str, lin: nn.Linear, dy, x_in, grads, need_dx: bool = True, **dgrad_kw):
    """dW += dy^T x_in, db += colsum(dy), returns dx = dy W (bf16)."""
    ops.linear_wgrad(dy, x_in, grads[name + ".weight"])
    ops.colsum(dy, grads[name + ".bias"])
    if not need_dx:
        return None
    dx = torch.empty(dy.shape[0], lin.weight.shape[1], dtype=bf16, device=dy.device)
    ops.linear_dgrad(dy, _w(model, name + ".weight", lin.weight), dx, **dgrad_kw)
    return dx


def _block_bwd(model: TimeSformer, i: int, dx, saved, descs, grads, rows: int, scales=None):
    (x, mean_t, rstd_t, ln_t, qkv_t, a_t, lse_t, p_t, xt, mean_s, rstd_s, ln_s, qkv_s, a_s, lse_s, x2, mean_m, rstd_m,
     ln_m, pre, f1) = saved
    blk = model.blocks[i]
    C_, I = model.embed_dim, blk.mlp.fc1.weight.shape[0]
    dev, p = dx.device, f"blocks.{i}."
    d_t, d_s = descs
    plain = ops.rowmap(C_)
    delta = torch.empty(model.num_heads, rows, dtype=f32, device=dev)

    def ln_bwd(dy, x_in, ln, name, mean, rstd, dres):
        out = torch.empty(rows, C_, dtype=bf16, device=dev)
        ops.layernorm_bwd(dy, plain, x_in, plain, ln.weight, mean, rstd, dres, plain, out, plain,
                          grads[name + ".weight"], grads[name + ".bias"], rows, C_)
        return out

    def attn_bwd(pre_name, att, qkv, a, da, lse, h_in, desc):
        dqkv = torch.empty(rows, 3 * C_, dtype=bf16, device=dev)
        ops.seg_attention_bwd(qkv, a, da, lse, delta, dqkv, desc, 0.125)
        return _linear_bwd(model, pre_name + "qkv", att.qkv, dqkv, h_in, grads)

    s_t, s_s, s_m = scales if scales is not None else (None, None, None)

    def dropped(dy, s):     # gradient entering a drop_path'ed branch: the same per-row factor (one extra pass when active)
        if s is None:
            return dy
        out = torch.empty_like(dy)
        ops.rowscale(dy, s, out)
        return out

    # ---- out = x2 + drop_path(fc2(gelu(fc1(LN(x2)))))
    dpre = _linear_bwd(model, p + "mlp.fc2", blk.mlp.fc2, dropped(dx, s_m), f1, grads, act=_lib.ACT_DGELU_ERF, aux=pre,
                       ld_aux=I)
    dln_m = _linear_bwd(model, p + "mlp.fc1", blk.mlp.fc1, dpre, ln_m, grads)
    del dpre
    dx2 = ln_bwd(dln_m, x2, blk.norm2, p + "norm2", mean_m, rstd_m, dx)
    # ---- x2 = xt + drop_path(proj(attn_s(LN(xt))))
    da_s = _linear_bwd(model, p + "attn.proj", blk.attn.proj, dropped(dx2, s_s), a_s, grads)
    dln_s = attn_bwd(p + "attn.", blk.attn, qkv_s, a_s, da_s, lse_s, ln_s, d_s)
    dxt = ln_bwd(dln_s, xt, blk.norm1, p + "norm1", mean_s, rstd_s, dx2)
    # ---- xt = x + temporal_fc(drop_path(proj_t(attn_t(LN(x)))))   (the saved p_t is already the dropped one)
    dp_t = _linear_bwd(model, p + "temporal_fc", blk.temporal_fc, dxt, p_t, grads)
    if s_t is not None:
        ops.rowscale(dp_t, s_t, dp_t)
    da_t = _linear_bwd(model, p + "temporal_attn.proj", blk.temporal_attn.proj, dp_t, a_t, grads)
    dln_t = attn_bwd(p + "temporal_attn.", blk.temporal_attn, qkv_t, a_t, da_t, lse_t, ln_t, d_t)
    return ln_bwd(dln_t, x, blk.temporal_norm1, p + "temporal_norm1", mean_t, rstd_t, dxt)


def _dense_block_bwd(model: TimeSformer, i: int, dx, saved, desc, grads, rows: int, scales=None):
    x, mean_a, rstd_a, ln_a, qkv, a, lse, x2, mean_m, rstd_m, ln_m, pre, f1 = saved
    blk = model.blocks[i]
    C_, I = model.embed_dim, blk.mlp.fc1.weight.shape[0]
    dev, p = dx.device, f"blocks.{i}."
    plain = ops.rowmap(C_)
    s_a, s_m = scales if scales is not None else (None, None)

    def ln_bwd(dy, x_in, ln, name, mean, rstd, dres):
        out = torch.empty(rows, C_, dtype=bf16, device=dev)
        ops.layernorm_bwd(dy, plain, x_in, plain, ln.weight, mean, rstd, dres, plain, out, plain,
                          grads[name + ".weight"], grads[name + ".bias"], rows, C_)
        return out

    def dropped(dy, s):
        if s is None:
            return dy
        out = torch.empty_like(dy)
        ops.rowscale(dy, s, out)
        return out

    # ---- out = x2 + drop_path(fc2(gelu(fc1(LN(x2)))))
    dpre = _linear_bwd(model, p + "mlp.fc2", blk.mlp.fc2, dropped(dx, s_m), f1, grads, act=_lib.ACT_DGELU_ERF, aux=pre,
                       ld_aux=I)
    dln_m = _linear_bwd(model, p + "mlp.fc1", blk.mlp.fc1, dpre, ln_m, grads)
    del dpre
    dx2 = ln_bwd(dln_m, x2, blk.norm2, p + "norm2", mean_m, rstd_m, dx)
    # ---- x2 = x + drop_path(proj(attn(LN(x))))
    da = _linear_bwd(model, p + "attn.proj", blk.attn.proj, dropped(dx2, s_a), a, grads)
    dqkv = torch.empty(rows, 3 * C_, dtype=bf16, device=dev)
    delta = torch.empty(model.num_heads, rows, dtype=f32, device=dev)
    ops.dense_attention_bwd(qkv, a, da, lse, delta, dqkv, desc, 0.125)
    dln_a = _linear_bwd(model, p + "attn.qkv", blk.attn.qkv, dqkv, ln_a, grads)
    return ln_bwd(dln_a, x, blk.norm1, p + "norm1", mean_a, rstd_a, dx2)


class _TimeSformerFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model: TimeSformer, names: List[str], masks, x: torch.Tensor, *params):
        B, T, C_, H, W = x.shape
        if C_ != model.embed_dim:
            raise ValueError(f"expected {model.embed_dim} channels, got {C_}")
        HW, rows = H * W, B * H * W * T
        save = any(ctx.needs_input_grad[3:])
        refresh_weights(model)
        x = x.contiguous()
        pos_tab, time_tab = _tables(model, T, H, W)
        tok = torch.empty(rows, C_, dtype=bf16, device=x.device)
        ops.tsf_embed_fwd(x, pos_tab, time_tab, tok, B, T, C_, HW)
        if model.attention_type == 'divided_space_time':
            descs = (ops.temporal_desc(rows, T, model.num_heads, 3 * C_, C_),
                     ops.spatial_desc(B, T, HW, model.num_heads, 3 * C_, C_))
            scales = [_row_scales(None if masks is None else masks[i], B, T, HW) for i in range(model.depth)]
            block_fwd = _block_fwd
        else:
            # one sequence per clip ('b (h w t) m', joint) or per frame ('(b t) (h w) m', space_only at T = 1)
            seq_len = HW * T if model.attention_type == 'joint_space_time' else HW
            descs = ops.dense_desc(rows, model.num_heads, 3 * C_, C_, n_seq=rows // seq_len, seq_len=seq_len)
            scales = [None if masks is None or masks[i] is None else
                      tuple(m.repeat_interleave(seq_len).contiguous() for m in masks[i]) for i in range(model.depth)]
            block_fwd = _dense_block_fwd
        saved = []
        for i in range(model.depth):
            tok, sv = block_fwd(model, i, tok, descs, rows, save, scales[i])
            saved.append(sv)
        out = torch.empty(B, T, C_, H, W, dtype=x.dtype, device=x.device)   # timesformer.py:523 (values; contiguous)
        ops.tsf_untokenize(tok, out, B, T, C_, HW)
        if save:
            ctx.model, ctx.names, ctx.saved, ctx.descs, ctx.scales = model, names, saved, descs, scales
            ctx.dims = (B, T, C_, H, W)
            ctx.x_dtype = x.dtype
        return out

    @staticmethod
    def backward(ctx, d_out):
        model, names, saved, descs = ctx.model, ctx.names, ctx.saved, ctx.descs
        B, T, C_, H, W = ctx.dims
        HW, rows = H * W, B * H * W * T
        dev = d_out.device
        dtok = torch.empty(rows, C_, dtype=bf16, device=dev)
        ops.tsf_embed_fwd(d_out.contiguous(), None, None, dtok, B, T, C_, HW)
        grads: Dict[str, torch.Tensor] = {}
        for i in reversed(range(model.depth)):
            shapes = {n: tuple(p.shape) for n, p in model.blocks[i].named_parameters(prefix=f"blocks.{i}")}
            _alloc_flat(shapes, grads, dev)
            block_bwd = _block_bwd if model.attention_type == 'divided_space_time' else _dense_block_bwd
            dtok = block_bwd(model, i, dtok, saved[i], descs, grads, rows, ctx.scales[i])
            saved[i] = None
        dx = None
        if ctx.needs_input_grad[3]:
            dx = torch.empty(B, T, C_, H, W, dtype=ctx.x_dtype, device=dev)
            ops.tsf_untokenize(dtok, dx, B, T, C_, HW)
        # table gradients: column sums of the token gradient over the broadcast dimensions
        has_time = hasattr(model, "time_embed")       # not in 'space_only'
        if has_time:
            d_time_tab = torch.zeros(T * C_, dtype=f32, device=dev)
            ops.colsum(dtok.view(B * HW, T * C_), d_time_tab)
        d_pos_full = torch.zeros(HW * T * C_, dtype=f32, device=dev)
        ops.colsum(dtok.view(B, HW * T * C_), d_pos_full)
        d_pos_tab = d_pos_full.view(HW, T, C_).sum(1)
        with torch.enable_grad():   # pull them back through the (tiny, linear) table interpolation
            pp = model.pos_embed.detach().requires_grad_(True)
            if has_time:
                tp = model.time_embed.detach().requires_grad_(True)
                pos_tab, time_tab = _tables(model, T, H, W, pp, tp)
                grads["pos_embed"], grads["time_embed"] = torch.autograd.grad(
                    [pos_tab, time_tab], [pp, tp], [d_pos_tab, d_time_tab.view(T, C_)])
            else:
                pos_tab, _ = _tables(model, T, H, W, pp)
                grads["pos_embed"], = torch.autograd.grad([pos_tab], [pp], [d_pos_tab])
        ctx.saved = None
        return (None, None, None, dx) + tuple(grads[n] if ctx.needs_input_grad[4 + j] else None for j, n in enumerate(names))
