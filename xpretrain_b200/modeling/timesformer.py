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
from typing import Dict, NamedTuple, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib, ops
from ._blocks import MlpSaved, drop_scale, layernorm, layernorm_bwd, linear_bwd, mlp_bwd, mlp_fwd, residual_linear
from ._weights import ParamLayout, matrix_weight, param_layout

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

    def _declare_layout(self) -> ParamLayout:
        """bf16 copies of the GEMM weights, one gradient group per block; the never-applied `norm` is left out, and the
        pos_embed / time_embed gradients come from the table interpolation's own backward."""
        return ParamLayout(self, exclude=("norm.",), cast=matrix_weight,
                           group=lambda op: ".".join(op.split(".")[:2]) if op.startswith("blocks.") else None)

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
        # torch.is_grad_enabled() of the caller: Function.forward always runs under no_grad, and needs_input_grad reflects
        # requires_grad even then, so without it evaluation under torch.no_grad() would keep every activation to the end
        return _TimeSformerFunction.apply(self, masks, torch.is_grad_enabled(), x, *param_layout(self).params)


# ----------------------------------------------------------------------------------- helpers
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


def _row_scales(masks, B: int, T: int, HW: int):
    """Per-token-row DropPath factors (rows ordered (b, p, t)) from the per-group factors of one block."""
    if masks is None:
        return None
    m_t, m_s, m_m = masks
    return (m_t.repeat_interleave(T).contiguous(),
            m_s.view(B, 1, T).expand(B, HW, T).reshape(-1).contiguous(),
            m_m.repeat_interleave(HW * T).contiguous())


class _AttnSaved(NamedTuple):
    x: torch.Tensor          # LayerNorm input
    mean: torch.Tensor
    rstd: torch.Tensor
    h: torch.Tensor          # LayerNorm output, the qkv GEMM's input
    qkv: torch.Tensor        # fused [rows, 3C], q pre-scaled
    a: torch.Tensor          # attention output
    lse: torch.Tensor


class _BlockSaved(NamedTuple):
    temporal: Optional[_AttnSaved]      # divided_space_time only
    p_t: Optional[torch.Tensor]         # temporal proj output after drop_path: temporal_fc's input
    attn: _AttnSaved
    mlp: MlpSaved


def _attn_fwd(model: TimeSformer, w, i: int, half: str, x, desc) -> _AttnSaved:
    """LayerNorm -> fused qkv GEMM -> attention of block i's temporal (half 'temporal_') or spatial / dense (half '') part.
    The kernel follows the descriptor: seg attention (temporal, spatial) or dense attention (joint, space-only)."""
    blk, p = model.blocks[i], f"blocks.{i}.{half}attn."
    att = getattr(blk, half + "attn")
    rows, C_ = x.shape
    dev = x.device
    h, mean, rstd = layernorm(x, getattr(blk, half + "norm1"))
    qkv = torch.empty(rows, 3 * C_, dtype=bf16, device=dev)
    # (q k^T) * head_dim**-0.5 (timesformer.py:165): 0.125 is a power of two, folding it into q (bias included) is exact
    ops.linear_fwd(h, w[p + "qkv.weight"], att.qkv.bias, qkv, scale_cols=C_, col_scale=0.125)
    a = torch.empty(rows, C_, dtype=bf16, device=dev)
    lse = torch.empty(model.num_heads, rows, dtype=f32, device=dev)
    if isinstance(desc, _lib.XpDenseAttn):
        ops.dense_attention_fwd(qkv, a, lse, desc)
    else:
        ops.seg_attention_fwd(qkv, a, lse, desc)
    return _AttnSaved(x, mean, rstd, h, qkv, a, lse)


def _attn_bwd(model: TimeSformer, w, i: int, half: str, da, sv: _AttnSaved, desc, grads, dres):
    """Backward of _attn_fwd from the gradient of the attention output; dres is the gradient carried by the residual path
    around this part.  Returns the gradient of the part's input."""
    blk, p = model.blocks[i], f"blocks.{i}.{half}"
    rows, C_ = da.shape
    dqkv = torch.empty(rows, 3 * C_, dtype=bf16, device=da.device)
    delta = torch.empty(model.num_heads, rows, dtype=f32, device=da.device)
    if isinstance(desc, _lib.XpDenseAttn):
        ops.dense_attention_bwd(sv.qkv, sv.a, da, sv.lse, delta, dqkv, desc, 0.125)
    else:
        ops.seg_attention_bwd(sv.qkv, sv.a, da, sv.lse, delta, dqkv, desc, 0.125)
    dh = linear_bwd(w, p + "attn.qkv", dqkv, sv.h, grads)
    return layernorm_bwd(dh, sv.x, getattr(blk, half + "norm1"), sv.mean, sv.rstd, dres, grads, p + "norm1")


def _block_fwd(model: TimeSformer, w, i: int, x, descs, save: bool, scales=None):
    """timesformer.py:207-226.  x: [rows, C] bf16 tokens, (h w t) order.  descs: (temporal, spatial) attention descriptors
    of 'divided_space_time', or (None, dense) for 'joint_space_time' / 'space_only' (:202-205), whose blocks have no temporal
    part.  scales: per-row DropPath factors (temporal, attention, mlp) of this block or None."""
    blk, p = model.blocks[i], f"blocks.{i}."
    C_ = model.embed_dim
    d_t, d_a = descs
    s_t, s_a, s_m = scales if scales is not None else (None, None, None)
    temporal = p_t = None
    if d_t is not None:
        # ---- temporal attention -> proj -> drop_path -> temporal_fc -> residual (:209-214)
        temporal = _attn_fwd(model, w, i, "temporal_", x, d_t)
        p_t = torch.empty(x.shape[0], C_, dtype=bf16, device=x.device)
        ops.linear_fwd(temporal.a, w[p + "temporal_attn.proj.weight"], blk.temporal_attn.proj.bias, p_t)
        if s_t is not None:
            ops.rowscale(p_t, s_t, p_t)          # in place: the saved p_t is the dropped one, as temporal_fc consumed it
        xt = torch.empty(x.shape[0], C_, dtype=bf16, device=x.device)
        ops.linear_fwd(p_t, w[p + "temporal_fc.weight"], blk.temporal_fc.bias, xt, residual=x, ldr=C_)
        x = xt
    # ---- spatial / dense attention -> proj -> drop_path -> residual (:216-224, :202-204)
    attn = _attn_fwd(model, w, i, "", x, d_a)
    x2 = residual_linear(w, p + "attn.proj", blk.attn.proj, attn.a, x, s_a)
    # ---- MLP with exact-erf GELU (:225, :132-138)
    out, mlp = mlp_fwd(w, p, blk, x2, save, s_m)
    return out, (_BlockSaved(temporal, p_t, attn, mlp) if save else None)


def _block_bwd(model: TimeSformer, w, i: int, dx, saved: _BlockSaved, descs, grads, scales=None):
    blk, p = model.blocks[i], f"blocks.{i}."
    s_t, s_a, s_m = scales if scales is not None else (None, None, None)
    dx2 = mlp_bwd(w, p, blk, dx, saved.mlp, grads, s_m)
    # ---- x2 = xt + drop_path(proj(attn(LN(xt))))
    da = linear_bwd(w, p + "attn.proj", drop_scale(dx2, s_a), saved.attn.a, grads)
    dxt = _attn_bwd(model, w, i, "", da, saved.attn, descs[1], grads, dx2)
    if saved.temporal is None:
        return dxt
    # ---- xt = x + temporal_fc(drop_path(proj_t(attn_t(LN(x)))))   (the saved p_t is already the dropped one)
    dp_t = linear_bwd(w, p + "temporal_fc", dxt, saved.p_t, grads)
    if s_t is not None:
        ops.rowscale(dp_t, s_t, dp_t)
    da_t = linear_bwd(w, p + "temporal_attn.proj", dp_t, saved.temporal.a, grads)
    return _attn_bwd(model, w, i, "temporal_", da_t, saved.temporal, descs[0], grads, dxt)


class _TimeSformerFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model: TimeSformer, masks, grad_mode: bool, x: torch.Tensor, *params):
        B, T, C_, H, W = x.shape
        if C_ != model.embed_dim:
            raise ValueError(f"expected {model.embed_dim} channels, got {C_}")
        HW, rows = H * W, B * H * W * T
        save = grad_mode and any(ctx.needs_input_grad[3:])
        w = param_layout(model)
        w.refresh()
        x = x.contiguous()
        pos_tab, time_tab = _tables(model, T, H, W)
        tok = torch.empty(rows, C_, dtype=bf16, device=x.device)
        ops.tsf_embed_fwd(x, pos_tab, time_tab, tok, B, T, C_, HW)
        if model.attention_type == 'divided_space_time':
            descs = (ops.temporal_desc(rows, T, model.num_heads, 3 * C_, C_),
                     ops.spatial_desc(B, T, HW, model.num_heads, 3 * C_, C_))
            scales = [_row_scales(None if masks is None else masks[i], B, T, HW) for i in range(model.depth)]
        else:
            # one sequence per clip ('b (h w t) m', joint) or per frame ('(b t) (h w) m', space_only at T = 1)
            seq_len = HW * T if model.attention_type == 'joint_space_time' else HW
            descs = (None, ops.dense_desc(rows, model.num_heads, 3 * C_, C_, n_seq=rows // seq_len, seq_len=seq_len))
            scales = [None if masks is None or masks[i] is None else
                      (None,) + tuple(m.repeat_interleave(seq_len).contiguous() for m in masks[i]) for i in range(model.depth)]
        saved = []
        for i in range(model.depth):
            tok, sv = _block_fwd(model, w, i, tok, descs, save, scales[i])
            saved.append(sv)
        out = torch.empty(B, T, C_, H, W, dtype=x.dtype, device=x.device)   # timesformer.py:523 (values; contiguous)
        ops.tsf_untokenize(tok, out, B, T, C_, HW)
        if save:
            ctx.model, ctx.saved, ctx.descs, ctx.scales = model, saved, descs, scales
            ctx.dims = (B, T, C_, H, W)
            ctx.x_dtype = x.dtype
        return out

    @staticmethod
    def backward(ctx, d_out):
        model, saved, descs = ctx.model, ctx.saved, ctx.descs
        w = param_layout(model)
        B, T, C_, H, W = ctx.dims
        HW, rows = H * W, B * H * W * T
        dev = d_out.device
        dtok = torch.empty(rows, C_, dtype=bf16, device=dev)
        ops.tsf_embed_fwd(d_out.contiguous(), None, None, dtok, B, T, C_, HW)
        grads: Dict[str, torch.Tensor] = {}
        for i in reversed(range(model.depth)):
            w.alloc_grads(f"blocks.{i}", grads)
            dtok = _block_bwd(model, w, i, dtok, saved[i], descs, grads, ctx.scales[i])
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
        return (None, None, None, dx) + w.grads_out(grads, ctx.needs_input_grad[4:])
