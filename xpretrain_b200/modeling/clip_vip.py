"""H100-native CLIP-ViP dual encoder (video tower with video-proxy tokens + CLIP text tower).

Drop-in for the reference's `CLIPModel` on the VidCLIP path (CLIP-ViP/src/modeling/CLIP_ViP.py): the
module tree below exists only to hold parameters under the reference's exact `state_dict()` names
(SURVEY.md §8b: `vision_model.pre_layrnorm` spelling included, q/k/v kept as separate parameters), so
released checkpoints, `named_parameters()`-driven weight-decay groups and `load_state_dict_with_mismatch`
work unchanged.  None of these nn.Modules' own forward() is ever called: forward and backward run in one
`torch.autograd.Function` that drives the hand-written sm_90a kernels through the C ABI (xpretrain_b200.ops).
There is no eager / CPU fallback.

With `config.vision_type` other than "ViP" the same class is the per-frame CLIP model VidCLIP builds from CLIP-ViP/src/modeling/
CLIP.py (VidCLIP.py:14-23,54-65): plain CLIPVisionEmbeddings, every frame a sequence of its own, and the frame-mean head
(xp_frame_pool_fwd / _bwd) in place of the single L2 normalisation of the video feature.

Reference call stack replaced (SURVEY.md §3.2):
  CLIPModel.forward            CLIP_ViP.py:1089-1172
  CLIPVisionTransformer.forward :861-903, CLIPVisionViPEmbeddings.forward :168-197
  CLIPTextTransformer.forward  :726-786, CLIPTextEmbeddings.forward :210-227
  CLIPEncoderLayer.forward     :445-460, CLIPAttention.forward2 :332-381 / .forward :266-330, CLIPMLP.forward :392-396
"""
from __future__ import annotations

from dataclasses import dataclass, field
from types import SimpleNamespace
from typing import Dict, Optional

import torch
import torch.nn as nn

from .. import _lib, ops
from ._weights import ParamLayout, param_layout

bf16, f32 = torch.bfloat16, torch.float32


@dataclass
class TowerConfig:
    hidden_size: int
    num_attention_heads: int
    num_hidden_layers: int
    intermediate_size: int


@dataclass
class ClipVipConfig:
    """openai/clip-vit-base-patch16 hyper-parameters + `vision_additional_config` (VidCLIP.py:11-27)."""

    vision: TowerConfig = field(default_factory=lambda: TowerConfig(768, 12, 12, 3072))
    text: TowerConfig = field(default_factory=lambda: TowerConfig(512, 8, 12, 2048))
    image_size: int = 224
    patch_size: int = 16
    projection_dim: int = 512
    vocab_size: int = 49408
    max_position_embeddings: int = 77
    layer_norm_eps: float = 1e-5
    residual_fp32: bool = True          # keep the residual stream out of bf16 (as the reference does under bf16 autocast)
    residual_dtype: str = "fp32"        # its storage type: "fp32", or "fp16" (apex-O2-like: bf16's HBM cost, 8x finer rounding)
    temporal_size: int = 12
    if_use_temporal_embed: int = 1
    add_cls_num: int = 3
    logit_scale_init_value: float = 4.60
    # `vision_additional_config.type` (VidCLIP.py:14-23): "ViP" is the video-proxy tower; any other value builds the
    # per-frame CLIP model of CLIP.py, whose video feature is the mean of its frames' normalised features
    vision_type: str = "ViP"

    @property
    def num_patches(self) -> int:
        return (self.image_size // self.patch_size) ** 2

    @property
    def per_frame(self) -> bool:
        return self.vision_type != "ViP"

    @property
    def num_global_tokens(self) -> int:
        """Rows in front of each sequence's patch rows: CLS + the proxy tokens (ViP), or the CLS row alone (per frame)."""
        return 1 if self.per_frame else 1 + self.add_cls_num


# ----------------------------------------------------------------------- parameter containers
class _Attention(nn.Module):
    def __init__(self, width, heads):
        super().__init__()
        self.scale = float(width // heads) ** -0.5          # CLIPAttention.scale = head_dim ** -0.5 (CLIP_ViP.py:245)
        self.k_proj = nn.Linear(width, width)
        self.v_proj = nn.Linear(width, width)
        self.q_proj = nn.Linear(width, width)
        self.out_proj = nn.Linear(width, width)


class _MLP(nn.Module):
    def __init__(self, width, inner):
        super().__init__()
        self.fc1 = nn.Linear(width, inner)
        self.fc2 = nn.Linear(inner, width)


class _EncoderLayer(nn.Module):
    def __init__(self, tc: TowerConfig, eps):
        super().__init__()
        self.self_attn = _Attention(tc.hidden_size, tc.num_attention_heads)
        self.layer_norm1 = nn.LayerNorm(tc.hidden_size, eps=eps)
        self.mlp = _MLP(tc.hidden_size, tc.intermediate_size)
        self.layer_norm2 = nn.LayerNorm(tc.hidden_size, eps=eps)


class _Encoder(nn.Module):
    def __init__(self, tc: TowerConfig, eps):
        super().__init__()
        self.layers = nn.ModuleList([_EncoderLayer(tc, eps) for _ in range(tc.num_hidden_layers)])
        # CLIPEncoder.gradient_checkpointing (CLIP_ViP.py:626,676-690): in training mode the tower keeps only each block's
        # input and recomputes the block during the backward (_layer_fwd's `keep_input` / `upto_fc1`)
        self.gradient_checkpointing = False


class _VisionViPEmbeddings(nn.Module):
    def __init__(self, cfg: ClipVipConfig):
        super().__init__()
        w = cfg.vision.hidden_size
        self.added_cls = nn.Parameter(torch.randn(cfg.add_cls_num, w))
        self.class_embedding = nn.Parameter(torch.randn(w))
        self.patch_embedding = nn.Conv2d(3, w, kernel_size=cfg.patch_size, stride=cfg.patch_size, bias=False)
        self.position_embedding = nn.Embedding(cfg.num_patches + 1, w)
        self.register_buffer("position_ids", torch.arange(cfg.num_patches + 1).expand((1, -1)))
        if cfg.if_use_temporal_embed:
            self.temporal_embedding = nn.Parameter(torch.zeros(1, cfg.temporal_size, w))


class _VisionEmbeddings(nn.Module):
    """CLIPVisionEmbeddings of the per-frame model (CLIP.py:113-140): a CLS row and the patch rows of one frame, plus
    position_embedding[0..L]; no proxy tokens and no temporal table."""

    def __init__(self, cfg: ClipVipConfig):
        super().__init__()
        w = cfg.vision.hidden_size
        self.class_embedding = nn.Parameter(torch.randn(w))
        self.patch_embedding = nn.Conv2d(3, w, kernel_size=cfg.patch_size, stride=cfg.patch_size, bias=False)
        self.position_embedding = nn.Embedding(cfg.num_patches + 1, w)
        self.register_buffer("position_ids", torch.arange(cfg.num_patches + 1).expand((1, -1)))


class _VisionTransformer(nn.Module):
    def __init__(self, cfg: ClipVipConfig):
        super().__init__()
        self.embeddings = _VisionEmbeddings(cfg) if cfg.per_frame else _VisionViPEmbeddings(cfg)
        self.pre_layrnorm = nn.LayerNorm(cfg.vision.hidden_size, eps=cfg.layer_norm_eps)  # sic (reference spelling)
        self.encoder = _Encoder(cfg.vision, cfg.layer_norm_eps)
        self.post_layernorm = nn.LayerNorm(cfg.vision.hidden_size, eps=cfg.layer_norm_eps)


class _TextEmbeddings(nn.Module):
    def __init__(self, cfg: ClipVipConfig):
        super().__init__()
        self.token_embedding = nn.Embedding(cfg.vocab_size, cfg.text.hidden_size)
        self.position_embedding = nn.Embedding(cfg.max_position_embeddings, cfg.text.hidden_size)
        self.register_buffer("position_ids", torch.arange(cfg.max_position_embeddings).expand((1, -1)))


class _TextTransformer(nn.Module):
    def __init__(self, cfg: ClipVipConfig):
        super().__init__()
        self.embeddings = _TextEmbeddings(cfg)
        self.encoder = _Encoder(cfg.text, cfg.layer_norm_eps)
        self.final_layer_norm = nn.LayerNorm(cfg.text.hidden_size, eps=cfg.layer_norm_eps)


class CLIPModel(nn.Module):
    """Same constructor argument style, attribute names and output keys as the reference CLIPModel."""

    supports_gradient_checkpointing = True      # CLIPPreTrainedModel, CLIP_ViP.py:478

    def __init__(self, config: ClipVipConfig):
        super().__init__()
        self.config = config
        self.vision_model = _VisionTransformer(config)
        self.text_model = _TextTransformer(config)
        self.visual_projection = nn.Linear(config.vision.hidden_size, config.projection_dim, bias=False)
        self.text_projection = nn.Linear(config.text.hidden_size, config.projection_dim, bias=False)
        self.logit_scale = nn.Parameter(torch.ones([]) * config.logit_scale_init_value)
        self._init_weights()
        self._packs: Dict[str, object] = {}        # the overlap streams and the p = 14 padded patch weight, per device

    @torch.no_grad()
    def _init_weights(self):
        """CLIPPreTrainedModel._init_weights, CLIP_ViP.py:481-522 (initializer_factor 1, initializer_range 0.02)."""
        cfg = self.config
        te = self.text_model.embeddings
        te.token_embedding.weight.normal_(0.0, 0.02)
        te.position_embedding.weight.normal_(0.0, 0.02)
        ve = self.vision_model.embeddings
        ve.class_embedding.normal_(0.0, cfg.vision.hidden_size ** -0.5)
        ve.patch_embedding.weight.normal_(0.0, 0.02)
        ve.position_embedding.weight.normal_(0.0, 0.02)
        for tower, tc in ((self.vision_model, cfg.vision), (self.text_model, cfg.text)):
            in_std = tc.hidden_size ** -0.5 * (2 * tc.num_hidden_layers) ** -0.5
            for layer in tower.encoder.layers:
                for lin in (layer.self_attn.q_proj, layer.self_attn.k_proj, layer.self_attn.v_proj):
                    lin.weight.normal_(0.0, in_std)
                layer.self_attn.out_proj.weight.normal_(0.0, tc.hidden_size ** -0.5)
                layer.mlp.fc1.weight.normal_(0.0, (2 * tc.hidden_size) ** -0.5)
                layer.mlp.fc2.weight.normal_(0.0, in_std)
        self.text_projection.weight.normal_(0.0, cfg.text.hidden_size ** -0.5)
        self.visual_projection.weight.normal_(0.0, cfg.vision.hidden_size ** -0.5)
        for m in self.modules():
            if isinstance(m, nn.LayerNorm):
                m.bias.zero_()
                m.weight.fill_(1.0)
            if isinstance(m, nn.Linear) and m.bias is not None:
                m.bias.zero_()

    def _declare_layout(self) -> ParamLayout:
        """q/k/v of each encoder layer stacked into one [3C, C] operand and one fp32 [3C] bias; bf16 copies of the encoder
        GEMM weights, the patch embedding and the two projections.  One gradient group per encoder layer, and one per tower
        for the rest and its projection.  logit_scale is left out: the loss differentiates it."""
        fuse = {}
        for tower, tc in (("vision_model", self.config.vision), ("text_model", self.config.text)):
            for i in range(tc.num_hidden_layers):
                a = f"{tower}.encoder.layers.{i}.self_attn."
                for kind in ("weight", "bias"):
                    fuse[a + "qkv." + kind] = [a + x + "_proj." + kind for x in "qkv"]
        gemm = ("qkv.weight", "qkv.bias", "out_proj.weight", "fc1.weight", "fc2.weight", "patch_embedding.weight",
                "projection.weight")
        return ParamLayout(self, exclude=("logit_scale",), fuse=fuse, cast=lambda n, p: n.endswith(gemm), group=_grad_group)

    # ------------------------------------------------------------------------------ public API
    def forward(self, input_ids=None, pixel_values=None, attention_mask=None, return_loss=False, **_unused):
        """CLIPModel.forward, CLIP_ViP.py:1089-1172 (return_loss is accepted and ignored, as VidCLIP passes False).
        Per-frame model: images [N, 3, H, W] give CLIP.py's per-image features; video [B, T, 3, H, W] gives the feature
        VidCLIP.py:54-65 forms from them, normalise(mean_t normalise(projection of frame t))."""
        image_embeds, text_embeds = _run(self, pixel_values, input_ids, attention_mask)
        return {"image_embeds": image_embeds, "text_embeds": text_embeds}

    def get_image_features(self, pixel_values=None, if_norm=None, **_unused):
        """CLIP_ViP.py:1043-1085: projected (and, if if_norm, L2-normalised) video features.  Per-frame model: CLIP.py:943-985,
        the unnormalised projection of every image (or frame); like CLIP.py it takes no `if_norm`."""
        if self.config.per_frame and if_norm is not None:
            raise TypeError("get_image_features() got an unexpected keyword argument 'if_norm'")
        image_embeds, _ = _run(self, pixel_values, None, None, normalize=bool(if_norm))
        return image_embeds

    def get_text_features(self, input_ids=None, attention_mask=None, if_norm=None, **_unused):
        """CLIP_ViP.py:992-1041.  Per-frame model: CLIP.py:900-941, which takes no `if_norm`."""
        if self.config.per_frame and if_norm is not None:
            raise TypeError("get_text_features() got an unexpected keyword argument 'if_norm'")
        _, text_embeds = _run(self, None, input_ids, attention_mask, normalize=bool(if_norm))
        return text_embeds

    # ------------------------------------------------------------------- gradient checkpointing
    def gradient_checkpointing_enable(self, gradient_checkpointing_kwargs=None):
        """Set `gradient_checkpointing` on both encoders, as the reference's `_set_gradient_checkpointing` does
        (CLIP_ViP.py:524-526).  A tower in training mode then keeps only each block's input (one [rows, C] tensor in the
        residual stream's storage type) and reruns the block's forward kernels, through fc1, before the block's backward.
        Results are bit-identical to a run without checkpointing.  `gradient_checkpointing_kwargs` is accepted so Hugging
        Face call sites work and has no effect: the recompute runs inside this model's own backward, not through
        `torch.utils.checkpoint`."""
        for enc in (self.vision_model.encoder, self.text_model.encoder):
            enc.gradient_checkpointing = True

    def gradient_checkpointing_disable(self):
        """Clear `gradient_checkpointing` on both encoders: every block keeps its whole forward state again."""
        for enc in (self.vision_model.encoder, self.text_model.encoder):
            enc.gradient_checkpointing = False

    @property
    def is_gradient_checkpointing(self) -> bool:
        return any(getattr(m, "gradient_checkpointing", False) for m in self.modules())


def _grad_group(op: str) -> str:
    """Gradient group of an operand: its encoder layer ("<tower>.encoder.layers.<i>."), else its tower."""
    if ".encoder.layers." in op:
        return ".".join(op.split(".")[:4]) + "."
    return "text_model" if op.startswith(("text_model.", "text_projection.")) else "vision_model"


# --------------------------------------------------------------------------- encoder layers
def _residual_fp32(model) -> bool:
    """The residual stream is kept OUT of bf16 (as under the reference's bf16 autocast, where only the Linear / matmul inputs are
    rounded): the block outputs stay bf16 branch tensors and the add happens in fp32 inside the next LayerNorm kernel.
    `model.config.residual_fp32 = False` (or XP_RESIDUAL_BF16=1) selects the round-1 path: bf16 stream, add in the GEMM epilogue."""
    import os
    return bool(getattr(model.config, "residual_fp32", True)) and os.environ.get("XP_RESIDUAL_BF16") != "1"


def _stream_dtype(model) -> torch.dtype:
    """Storage type of the residual stream between the fused add + LayerNorm kernels: fp32 (default), or fp16
    (`config.residual_dtype = "fp16"` / XP_RESIDUAL_DTYPE=fp16): 11 mantissa bits instead of bf16's 8 at bf16's HBM cost — the
    precision the reference itself trains in under apex O2 (run_pretrain.py:234-236); values saturate at +-65504."""
    import os
    name = os.environ.get("XP_RESIDUAL_DTYPE") or getattr(model.config, "residual_dtype", "fp32")
    return torch.float16 if str(name) in ("fp16", "float16", "half") else f32


def _layer_fwd(x, pend, layer, w: ParamLayout, p: str, eps: float, attn_fwd, rows: int, save: bool, stream_dt,
               keep_input: bool = False, upto_fc1: bool = False):
    """One pre-LN residual block (CLIP_ViP.py:445-460).  x: residual stream [rows, C] in `stream_dt` (fp32 / fp16), or bf16 when
    stream_dt is None (round-1 path); pend: the previous block's bf16 branch output that still has to be added to it.
    Returns (x_out, pend_out, saved): saved is the tuple _layer_bwd reads when `save`; otherwise, with `keep_input`, the
    LayerNorm-1 input alone (x + pend as the fused add stored it), the checkpoint from which a plain call with `save` and
    `upto_fc1` rebuilds that tuple bit for bit.  `upto_fc1` stops after fc1 + QuickGELU and returns (None, None, saved): the
    backward never reads fc2's output."""
    fp32res = stream_dt is not None
    C_, I = layer.mlp.fc1.weight.shape[1], layer.mlp.fc1.weight.shape[0]
    dev = x.device
    plain = ops.rowmap(C_)
    mean1 = torch.empty(rows, dtype=f32, device=dev); rstd1 = torch.empty_like(mean1)
    h = torch.empty(rows, C_, dtype=bf16, device=dev)
    ln1, ln2 = layer.layer_norm1, layer.layer_norm2
    if pend is not None:        # x <- x + pend in fp32, fused into layer_norm1
        xs = torch.empty(rows, C_, dtype=stream_dt, device=dev)
        ops.layernorm_fwd(x, plain, h, plain, ln1.weight, ln1.bias, mean1, rstd1, rows, C_, eps, add=pend, addmap=plain,
                          sum_out=xs, summap=plain)
        x = xs
    else:
        ops.layernorm_fwd(x, plain, h, plain, ln1.weight, ln1.bias, mean1, rstd1, rows, C_, eps)
    qkv = torch.empty(rows, 3 * C_, dtype=bf16, device=dev)
    # q = (h Wq^T + bq) * head_dim**-0.5 : the scale multiplies the bias too (CLIP_ViP.py:341 / :269)
    ops.linear_fwd(h, w[p + "self_attn.qkv.weight"], w[p + "self_attn.qkv.bias"], qkv, scale_cols=C_,
                   col_scale=layer.self_attn.scale)
    a = torch.empty(rows, C_, dtype=bf16, device=dev)
    att_saved = attn_fwd(qkv, a)
    mean2 = torch.empty(rows, dtype=f32, device=dev); rstd2 = torch.empty_like(mean2)
    h2 = torch.empty(rows, C_, dtype=bf16, device=dev)
    if fp32res:
        y1 = torch.empty(rows, C_, dtype=bf16, device=dev)
        # branch only: the add is in layer_norm2
        ops.linear_fwd(a, w[p + "self_attn.out_proj.weight"], layer.self_attn.out_proj.bias, y1)
        x1 = torch.empty(rows, C_, dtype=stream_dt, device=dev)
        ops.layernorm_fwd(x, plain, h2, plain, ln2.weight, ln2.bias, mean2, rstd2, rows, C_, eps, add=y1, addmap=plain,
                          sum_out=x1, summap=plain)
        del y1
    else:
        x1 = torch.empty(rows, C_, dtype=bf16, device=dev)
        ops.linear_fwd(a, w[p + "self_attn.out_proj.weight"], layer.self_attn.out_proj.bias, x1, residual=x, ldr=C_)
        ops.layernorm_fwd(x1, plain, h2, plain, ln2.weight, ln2.bias, mean2, rstd2, rows, C_, eps)
    pre = torch.empty(rows, I, dtype=bf16, device=dev) if save else None
    f1 = torch.empty(rows, I, dtype=bf16, device=dev)
    ops.linear_fwd(h2, w[p + "mlp.fc1.weight"], layer.mlp.fc1.bias, f1, act=_lib.ACT_QUICK_GELU, aux=pre, ld_aux=I)
    saved = (x, mean1, rstd1, h, qkv, att_saved, a, x1, mean2, rstd2, h2, pre, f1) if save else (x if keep_input else None)
    if upto_fc1:
        return None, None, saved
    out = torch.empty(rows, C_, dtype=bf16, device=dev)
    if fp32res:
        ops.linear_fwd(f1, w[p + "mlp.fc2.weight"], layer.mlp.fc2.bias, out)       # branch; added by the next LayerNorm
        return x1, out, saved
    ops.linear_fwd(f1, w[p + "mlp.fc2.weight"], layer.mlp.fc2.bias, out, residual=x1, ldr=C_)
    return out, None, saved


def _pooled_ln(x, pend, rmap, ln, B: int, C_: int, eps: float):
    """LayerNorm of B selected rows (CLS / EOS, picked by `rmap`) of the final hidden state x (+ pend) -> (pooled bf16 [B, C],
    mean, rstd, (saved LayerNorm input, its row map))."""
    dev = x.device
    plain = ops.rowmap(C_)
    pooled = torch.empty(B, C_, dtype=bf16, device=dev)
    mean = torch.empty(B, dtype=f32, device=dev); rstd = torch.empty_like(mean)
    if pend is None:
        ops.layernorm_fwd(x, rmap, pooled, plain, ln.weight, ln.bias, mean, rstd, B, C_, eps)
        return pooled, mean, rstd, (x, rmap)
    rows_in = torch.empty(B, C_, dtype=torch.float16 if x.dtype == torch.float16 else f32, device=dev)
    ops.layernorm_fwd(x, rmap, pooled, plain, ln.weight, ln.bias, mean, rstd, B, C_, eps, add=pend, addmap=rmap, sum_out=rows_in,
                      summap=plain)
    return pooled, mean, rstd, (rows_in, plain)


def _colsum(x: torch.Tensor, out: torch.Tensor, aux) -> None:
    """Bias gradient = column sum of x (HBM-bound).  With an auxiliary stream it runs UNDER the tensor-bound GEMMs that follow
    (its 256-thread CTAs co-reside with the persistent GEMM CTAs); the caller joins the stream before the gradients are used.
    The caller drops x only after that join (_join_aux), so that x's memory returns to the current stream's pool in stream
    order behind the column sum.  (`x.record_stream(aux)` would defer the reuse until the allocator sees the aux event
    complete: with the host running ahead of the GPU, each layer's dpre / dqkv blocks then stayed unusable, the pool grew to
    the whole card and allocation retries — cudaFree of every cached block plus a device synchronise — made the step time
    vary by tens of percent.)"""
    if aux is None:
        ops.colsum(x, out)
        return
    aux.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(aux):
        ops.colsum(x, out)


def _join_aux(aux) -> None:
    """The current stream waits for the work queued on aux so far (a device-side wait, no host synchronise)."""
    if aux is not None:
        torch.cuda.current_stream().wait_stream(aux)


def _layer_bwd(dx, saved, layer, w: ParamLayout, grads: Dict[str, torch.Tensor], prefix: str, attn_bwd, rows: int,
               aux=None):
    """Backward of one block; dx [rows, C] bf16 is d(loss)/d(block output).  Returns d(block input)."""
    (x, mean1, rstd1, h, qkv, att_saved, a, x1, mean2, rstd2, h2, pre, f1) = saved
    C_, I = layer.mlp.fc1.weight.shape[1], layer.mlp.fc1.weight.shape[0]
    dev = dx.device
    plain = ops.rowmap(C_)
    g = lambda n: grads[prefix + n]  # noqa: E731
    # ---- x_out = x1 + fc2(quick_gelu(fc1(LN2(x1))))
    ops.linear_wgrad(dx, f1, g("mlp.fc2.weight"))
    dpre = torch.empty(rows, I, dtype=bf16, device=dev)
    ops.linear_dgrad(dx, w[prefix + "mlp.fc2.weight"], dpre, act=_lib.ACT_DQUICK_GELU, aux=pre, ld_aux=I)
    _colsum(dpre, g("mlp.fc1.bias"), aux)
    ops.linear_wgrad(dpre, h2, g("mlp.fc1.weight"))
    dh2 = torch.empty(rows, C_, dtype=bf16, device=dev)
    ops.linear_dgrad(dpre, w[prefix + "mlp.fc1.weight"], dh2)
    _join_aux(aux)          # dpre's column sum is complete: its memory may return to this stream's pool (see _colsum)
    del dpre
    dx1 = torch.empty(rows, C_, dtype=bf16, device=dev)
    # LN2 backward streams dx as the residual-branch gradient: its column sum (= fc2.bias gradient) comes out of the same pass
    ops.layernorm_bwd(dh2, plain, x1, plain, layer.layer_norm2.weight, mean2, rstd2, dx, plain, dx1, plain,
                      g("layer_norm2.weight"), g("layer_norm2.bias"), rows, C_, dres_colsum=g("mlp.fc2.bias"))
    # ---- x1 = x + out_proj(attn(qkv(LN1(x))))
    ops.linear_wgrad(dx1, a, g("self_attn.out_proj.weight"))
    da = dh2  # reuse
    ops.linear_dgrad(dx1, w[prefix + "self_attn.out_proj.weight"], da)
    dqkv = torch.empty(rows, 3 * C_, dtype=bf16, device=dev)
    attn_bwd(qkv, a, da, att_saved, dqkv)
    _colsum(dqkv, g("self_attn.qkv.bias"), aux)
    ops.linear_wgrad(dqkv, h, g("self_attn.qkv.weight"))
    dh = da
    ops.linear_dgrad(dqkv, w[prefix + "self_attn.qkv.weight"], dh)
    _join_aux(aux)          # the qkv bias gradient is complete, and dqkv may be released
    del dqkv
    dxin = torch.empty(rows, C_, dtype=bf16, device=dev)
    ops.layernorm_bwd(dh, plain, x, plain, layer.layer_norm1.weight, mean1, rstd1, dx1, plain, dxin, plain,
                      g("layer_norm1.weight"), g("layer_norm1.bias"), rows, C_, dres_colsum=g("self_attn.out_proj.bias"))
    return dxin


def _grads_ready(model, flat: torch.Tensor) -> None:
    """A gradient group (one encoder layer, or a tower's remaining parameters) is final: hand its flat buffer to
    `model.grad_ready_hook` (e.g. utils.distributed.OverlappedGradAverager, which starts an async NCCL all-reduce
    that overlaps with the rest of the backward pass — the hvd.DistributedOptimizer hooks of run_pretrain.py:226-228)."""
    hook = getattr(model, "grad_ready_hook", None)
    if hook is not None:
        hook(flat)


# ------------------------------------------------------------------------------ encoder stack
def _block_saved(sv, i: int):
    """Block i's saved tensors for its backward, released from `sv`.  A checkpointed tower kept only the block's input:
    rebuild the rest now by rerunning the block's forward kernels from it, on the stream and under the SM limit of the backward."""
    s, sv.layers[i] = sv.layers[i], None
    return s if sv.recompute is None else sv.recompute(i, s)


def _encoder_fwd(model: CLIPModel, tower: str, pool_ln: str, w: ParamLayout, x_in: list, rows: int, B: int, attn_fwd,
                 pool_rows, wproj, save: bool, ckpt: bool, stream_dt, timer=None):
    """A tower's encoder layers, then its pooled LayerNorm (`pool_ln`) of the B rows picked by the row map `pool_rows()`
    returns after the layers, and the projection `wproj`.  x_in: a list holding the only reference to the embedded rows, so
    that layer 0 releases them unless it saves them.  ckpt (with save): keep each block's input only; `recompute` rebuilds
    the rest per block in the backward.  timer: a list receiving ("fwd", start, end) CUDA events around each block.
    Returns (proj fp32 [B, projection_dim], saved): saved (None without `save`) holds what _encoder_bwd reads."""
    eps = model.config.layer_norm_eps
    tw = getattr(model, tower)
    layers = tw.encoder.layers
    x = x_in.pop()
    layer_saved = []
    pend = None
    for i, layer in enumerate(layers):
        if timer is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        x, pend, sv = _layer_fwd(x, pend, layer, w, f"{tower}.encoder.layers.{i}.", eps, attn_fwd, rows, save and not ckpt,
                                 stream_dt, keep_input=ckpt)
        if timer is not None:
            e1.record()
            timer.append(("fwd", e0, e1))
        layer_saved.append(sv)
    rmap = pool_rows()
    pooled, meanp, rstdp, post_in = _pooled_ln(x, pend, rmap, getattr(tw, pool_ln), B, x.shape[1], eps)
    proj = torch.empty(B, model.config.projection_dim, dtype=f32, device=x.device)
    ops.linear_fwd(pooled, wproj, None, proj, out_mode=_lib.OUT_F32)
    if not save:
        return proj, None
    recompute = None
    if ckpt:
        def recompute(i, xin):
            return _layer_fwd(xin, None, layers[i], w, f"{tower}.encoder.layers.{i}.", eps, attn_fwd, rows, True, stream_dt,
                              upto_fc1=True)[2]
    return proj, SimpleNamespace(B=B, rows=rows, layers=layer_saved, x_last=(x, pend), pool_map=rmap, post_in=post_in,
                                 pooled=pooled, meanp=meanp, rstdp=rstdp, recompute=recompute)


def _encoder_bwd(model: CLIPModel, tower: str, pool_ln: str, proj: str, w: ParamLayout, sv, dproj_bf16, grads, flats,
                 attn_bwd, aux=None, timer=None):
    """Backward of _encoder_fwd from dproj_bf16 [B, proj] (the gradient of the un-normalised projection output): the
    projection, the pooled LayerNorm, then the layers in reverse, each handing its finished gradient group (its buffer in
    `flats`) to `_grads_ready`.  aux: the stream of the layers' bias column sums (_colsum); timer: ("bwd", start, end) events
    per block.
    Returns the gradient of the embedded rows [rows, C] bf16."""
    tw = getattr(model, tower)
    C_, B, rows = getattr(tw, pool_ln).weight.shape[0], sv.B, sv.rows
    dev = dproj_bf16.device
    ops.linear_wgrad(dproj_bf16, sv.pooled, grads[proj + ".weight"])
    dpooled = torch.empty(B, C_, dtype=bf16, device=dev)
    ops.linear_dgrad(dproj_bf16, w[proj + ".weight"], dpooled)
    dx = torch.zeros(rows, C_, dtype=bf16, device=dev)  # only the pooled rows receive gradient from the head
    ln = f"{tower}.{pool_ln}."
    ops.layernorm_bwd(dpooled, ops.rowmap(C_), sv.post_in[0], sv.post_in[1], getattr(tw, pool_ln).weight, sv.meanp, sv.rstdp,
                      None, None, dx, sv.pool_map, grads[ln + "weight"], grads[ln + "bias"], B, C_)
    for i in reversed(range(len(tw.encoder.layers))):
        prefix = f"{tower}.encoder.layers.{i}."
        if timer is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        dx = _layer_bwd(dx, _block_saved(sv, i), tw.encoder.layers[i], w, grads, prefix, attn_bwd, rows, aux)
        if timer is not None:
            e1.record()
            timer.append(("bwd", e0, e1))
        _grads_ready(model, flats[prefix])
    return dx


# ------------------------------------------------------------------------------ vision tower
def frame_input_path(dtype: torch.dtype, H: int, W: int, image_size: int) -> str:
    """Which patch extraction takes frames of `dtype` and size H x W into a tower of `image_size`: "patchify_u8" (uint8 at
    the input resolution: /255 + Normalize fused in), "resize_u8" (uint8 of another size: the reference's bicubic Resize
    fused in as well) or "patchify" (float frames, already transformed).  Float frames of another size raise ValueError:
    the reference transform is the caller's there, and the patch matrix is sized for image_size."""
    if dtype == torch.uint8:
        return "patchify_u8" if (H, W) == (image_size, image_size) else "resize_u8"
    if (H, W) != (image_size, image_size):
        raise ValueError(f"{dtype} frames must be {image_size} x {image_size} (got {H} x {W}); uint8 decoder frames of any "
                         f"size are resized on the GPU")
    return "patchify"


def _frame_path(cfg: ClipVipConfig, video: torch.Tensor) -> str:
    """The layout checks of the vision input, then frame_input_path; raises ValueError before anything is launched."""
    if cfg.per_frame and video.dim() not in (4, 5):
        raise ValueError("the per-frame model takes images [N, 3, H, W] or video [B, T, 3, H, W] (uint8: channels-last)")
    u8 = video.dtype == torch.uint8
    if u8 and ((video.dim() != 5 and not cfg.per_frame) or video.shape[-1] != 3):
        raise ValueError("uint8 video must be channels-last [B, T, H, W, 3] (decoder layout)")
    return frame_input_path(video.dtype, video.shape[-3 if u8 else -2], video.shape[-2 if u8 else -1], cfg.image_size)


def _vision_fwd(model: CLIPModel, video: torch.Tensor, save: bool, ckpt: bool = False):
    """ckpt (with save): keep each block's input only (gradient checkpointing); the backward rebuilds the rest per block.
    The per-frame model folds the frames into the batch (CLIP.py sees [B*T, 3, H, W]): B*T sequences of one frame and one
    global (CLS) row each, where the proxy-token attention is exactly dense attention over 1 + L rows."""
    cfg = model.config
    vm = model.vision_model
    emb = vm.embeddings
    path = _frame_path(cfg, video)
    if cfg.per_frame:
        B, T = video.numel() // (video.shape[-3] * video.shape[-2] * video.shape[-1]), 1
    else:
        B, T = video.shape[0], video.shape[1]
    C_, L, M = cfg.vision.hidden_size, cfg.num_patches, cfg.num_global_tokens
    H = cfg.vision.num_attention_heads
    S = M + T * L
    rows = B * S
    dev = video.device
    w = param_layout(model)
    eps = cfg.layer_norm_eps
    Kp = 3 * cfg.patch_size * cfg.patch_size
    ldp = ops.patch_pitch(cfg.patch_size)    # patch-matrix row pitch: Kp rounded up to 8 columns, pad columns zero

    patches = torch.empty(B * T * L, ldp, dtype=bf16, device=dev)
    mean, std = getattr(model, "pixel_mean", ops.CLIP_MEAN), getattr(model, "pixel_std", ops.CLIP_STD)
    if path == "patchify_u8":      # raw decoder frames: the reference's /255 + Normalize is fused into the patch extraction
        ops.vip_patchify_u8(video.contiguous(), patches, cfg.patch_size, mean, std)
    elif path == "resize_u8":      # ... and its bicubic Resize to image_size as well
        ops.vip_resize_patchify_u8(video.contiguous(), patches, cfg.image_size, cfg.patch_size, mean, std)
    else:
        ops.vip_patchify(video.contiguous(), patches, cfg.patch_size)
    table = torch.empty(T * L, C_, dtype=bf16, device=dev)
    x0 = torch.empty(rows, C_, dtype=bf16, device=dev)
    temporal = emb.temporal_embedding if cfg.if_use_temporal_embed and not cfg.per_frame else None
    added = None if cfg.per_frame else emb.added_cls       # M = 1: the kernel reads no added_cls row
    ops.vip_embed_tables(emb.position_embedding.weight, temporal, emb.class_embedding, added, table, x0, B, T, L,
                         M, C_, cfg.temporal_size)
    wp = w["vision_model.embeddings.patch_embedding.weight"].view(C_, Kp)
    if ldp != Kp:   # e.g. p = 14: the GEMM's B operand needs the same 16-byte row pitch as the patch matrix
        wpad = model._packs.get("pad:patch")
        if wpad is None or wpad.shape != (C_, ldp) or wpad.device != dev:
            wpad = model._packs["pad:patch"] = torch.zeros(C_, ldp, dtype=bf16, device=dev)
        wpad[:, :Kp].copy_(wp)
        wp = wpad
    # conv-as-GEMM; epilogue adds the periodic [T*L, C] position+temporal table and writes past the M global rows
    ops.gemm(patches, wp, x0, M=B * T * L, N=C_, K=Kp, lda=ldp, ldb=ldp, ldc=C_, residual=table, ldr=C_, r_group=T * L,
             r_group_stride=0, c_group=T * L, c_group_stride=S * C_, c_offset=M * C_)
    # pre_layrnorm (CLIP_ViP.py:881) in two launches so that its statistics are stored compactly per half
    # (patch rows / global rows), the layout its backward and the embedding backward consume
    pmap = ops.rowmap(C_, group=T * L, group_stride=S * C_)
    gmap = ops.rowmap(C_, group=M, group_stride=S * C_)
    mean0p = torch.empty(B * T * L, dtype=f32, device=dev); rstd0p = torch.empty_like(mean0p)
    mean0g = torch.empty(B * M, dtype=f32, device=dev); rstd0g = torch.empty_like(mean0g)
    stream_dt = _stream_dtype(model) if _residual_fp32(model) else None
    x = torch.empty(rows, C_, dtype=stream_dt if stream_dt is not None else bf16, device=dev)
    ln0 = vm.pre_layrnorm
    ops.layernorm_fwd(x0, pmap, x, pmap, ln0.weight, ln0.bias, mean0p, rstd0p, B * T * L, C_, eps, x_off=M * C_,
                      y_off=M * C_)
    ops.layernorm_fwd(x0, gmap, x, gmap, ln0.weight, ln0.bias, mean0g, rstd0g, B * M, C_, eps)
    x_in = [x]
    del x

    ws = ops.vip_attention_workspace(B, H, T, M, dev)

    def attn_fwd(qkv, out):
        lse = torch.empty(B, H, S, dtype=f32, device=dev)
        ops.vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C_)
        return lse

    # pooled = post_layernorm(last_hidden[:, 0])  (CLIP_ViP.py:891-893): CLS rows picked by the row map
    proj, saved = _encoder_fwd(model, "vision_model", "post_layernorm", w, x_in, rows, B, attn_fwd,
                               lambda: ops.rowmap(C_, group=1, group_stride=S * C_), w["visual_projection.weight"], save,
                               ckpt, stream_dt, timer=getattr(model, "block_timer", None))  # bench.py: metric 2 of BASELINE.json
    if saved is not None:
        saved.T, saved.S, saved.patches, saved.x0, saved.ws = T, S, patches, x0, ws
        saved.stats0 = (mean0p, rstd0p, mean0g, rstd0g)
    return proj, saved


def _vision_bwd(model: CLIPModel, dproj_bf16: torch.Tensor, sv, grads: Dict[str, torch.Tensor], flats):
    """dproj_bf16 [B, proj] = gradient w.r.t. the un-normalised projection output."""
    cfg = model.config
    vm = model.vision_model
    C_, L, M = cfg.vision.hidden_size, cfg.num_patches, cfg.num_global_tokens
    H = cfg.vision.num_attention_heads
    B, T, S = sv.B, sv.T, sv.S
    dev = dproj_bf16.device
    plain = ops.rowmap(C_)

    def attn_bwd(qkv, a, da, lse, dqkv):
        ops.vip_attention_bwd(qkv, a, da, lse, dqkv, sv.ws, B, H, T, L, M, C_, float(C_ // H) ** -0.5)

    dx = _encoder_bwd(model, "vision_model", "post_layernorm", "visual_projection", param_layout(model), sv, dproj_bf16,
                      grads, flats, attn_bwd, aux=_overlap_stream(model, dev, "overlap_colsum"),
                      timer=getattr(model, "block_timer", None))
    # pre_layrnorm backward, written as two compact halves: patch rows [B, T*L, C] and global rows [B, M, C]
    d_patch = torch.empty(B * T * L, C_, dtype=bf16, device=dev)
    d_glob = torch.empty(B * M, C_, dtype=bf16, device=dev)
    pmap = ops.rowmap(C_, group=T * L, group_stride=S * C_)
    gmap = ops.rowmap(C_, group=M, group_stride=S * C_)
    gw, gb = grads["vision_model.pre_layrnorm.weight"], grads["vision_model.pre_layrnorm.bias"]
    mean0p, rstd0p, mean0g, rstd0g = sv.stats0
    ops.layernorm_bwd(dx, pmap, sv.x0, pmap, vm.pre_layrnorm.weight, mean0p, rstd0p, None, None, d_patch, plain, gw, gb,
                      B * T * L, C_, dy_off=M * C_, x_off=M * C_)
    ops.layernorm_bwd(dx, gmap, sv.x0, gmap, vm.pre_layrnorm.weight, mean0g, rstd0g, None, None, d_glob, plain, gw, gb,
                      B * M, C_)
    emb = "vision_model.embeddings."
    ops.vip_embed_bwd(d_patch, d_glob, grads[emb + "position_embedding.weight"],
                      grads.get(emb + "temporal_embedding"), grads[emb + "class_embedding"], grads.get(emb + "added_cls"),
                      B, T, L, M, C_, cfg.temporal_size)
    Kp = 3 * cfg.patch_size * cfg.patch_size
    if sv.patches.shape[1] == Kp:
        ops.linear_wgrad(d_patch, sv.patches, grads[emb + "patch_embedding.weight"].view(C_, Kp))
    else:           # padded pitch (xp_gemm needs N % 8 == 0): the GEMM fills [C, pitch], the Kp real columns are the gradient
        dw = torch.zeros(C_, sv.patches.shape[1], dtype=f32, device=dev)
        ops.linear_wgrad(d_patch, sv.patches, dw)
        grads[emb + "patch_embedding.weight"].view(C_, Kp).add_(dw[:, :Kp])


# -------------------------------------------------------------------------------- text tower
def _text_fwd(model: CLIPModel, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor], save: bool,
              ckpt: bool = False):
    cfg = model.config
    B, Lt = input_ids.shape
    C_, H = cfg.text.hidden_size, cfg.text.num_attention_heads
    rows = B * Lt
    dev = input_ids.device
    te = model.text_model.embeddings
    if Lt > cfg.max_position_embeddings:      # the reference fails in position_ids[:, :seq_length] + embedding add (CLIP_ViP.py:217-225)
        raise ValueError(f"text length {Lt} exceeds max_position_embeddings {cfg.max_position_embeddings}")
    ids = input_ids.contiguous().to(torch.int64)
    mask = attention_mask.contiguous().to(torch.int64) if attention_mask is not None else None
    x = torch.empty(rows, C_, dtype=bf16, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.text_embed_fwd(ids, te.token_embedding.weight, te.position_embedding.weight, x, Lt, err)
    if getattr(model, "validate_ids", False) and int(err.item()) != 0:   # opt-in: costs a device sync per forward
        raise IndexError("text_input_ids contains a token id outside [0, vocab_size) (nn.Embedding would raise, CLIP_ViP.py:222)")

    def attn_fwd(qkv, out):
        probs = torch.empty(B, H, Lt, Lt, dtype=f32, device=dev)
        ops.text_attention_fwd(qkv, mask, out, probs, B, H, Lt, C_)
        return probs

    stream_dt = _stream_dtype(model) if _residual_fp32(model) else None
    if stream_dt is not None:
        x = x.to(stream_dt)          # [B*Lt, 512]: the token + position embeddings enter the stream in its storage type
    x_in = [x]
    del x
    eos = None

    def eos_rows():     # final_layer_norm is per-row, so it is applied to the pooled EOS row only (first argmax of the ids, :776)
        nonlocal eos
        eos = torch.empty(B, dtype=torch.int64, device=dev)
        ops.eos_offsets(ids, eos, None, C_)
        return ops.rowmap(C_, offsets=eos)

    w = param_layout(model)
    proj, saved = _encoder_fwd(model, "text_model", "final_layer_norm", w, x_in, rows, B, attn_fwd, eos_rows,
                               w["text_projection.weight"], save, ckpt, stream_dt)
    if saved is not None:
        saved.Lt, saved.ids, saved.eos, saved.err = Lt, ids, eos, err
    return proj, saved


def _text_bwd(model: CLIPModel, dproj_bf16: torch.Tensor, sv, grads: Dict[str, torch.Tensor], flats):
    cfg = model.config
    C_, H = cfg.text.hidden_size, cfg.text.num_attention_heads
    B, Lt = sv.B, sv.Lt

    def attn_bwd(qkv, a, da, probs, dqkv):
        ops.text_attention_bwd(qkv, da, probs, dqkv, B, H, Lt, C_, float(C_ // H) ** -0.5)

    dx = _encoder_bwd(model, "text_model", "final_layer_norm", "text_projection", param_layout(model), sv, dproj_bf16,
                      grads, flats, attn_bwd)
    ops.text_embed_bwd(sv.ids, dx, grads["text_model.embeddings.token_embedding.weight"],
                       grads["text_model.embeddings.position_embedding.weight"], Lt, C_, cfg.vocab_size)


# ------------------------------------------------------------------- the autograd.Function
class _ClipVipFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model: CLIPModel, video, input_ids, attention_mask, normalize, grad_mode, *params):
        # grad_mode = torch.is_grad_enabled() of the caller (Function.forward itself always runs under no_grad, and
        # needs_input_grad reflects requires_grad even then): evaluation must not keep the activations alive
        w = param_layout(model)
        need = {n: r for n, r in zip(w.names, ctx.needs_input_grad[6:])}
        save = grad_mode and any(need.values())
        ctx.model = model
        w.refresh()
        ctx.normalize = normalize
        ctx.vis = ctx.txt = None
        dev = params[0].device

        def run_tower(which):
            # gradient checkpointing applies in training mode only (the reference's `self.gradient_checkpointing and
            # self.training`), and only to a tower that saves anything for the backward at all
            if which == "vis":
                tower_save = save and any(r for n, r in need.items() if n.startswith(("vision_model.", "visual_projection.")))
                enc = model.vision_model.encoder
                proj, sv = _vision_fwd(model, video, tower_save, tower_save and enc.gradient_checkpointing and enc.training)
            else:
                # a frozen text tower (VidCLIP.freeze_text_encoder) keeps nothing and runs no backward
                tower_save = save and any(r for n, r in need.items() if n.startswith(("text_model.", "text_projection.")))
                enc = model.text_model.encoder
                proj, sv = _text_fwd(model, input_ids, attention_mask, tower_save,
                                     tower_save and enc.gradient_checkpointing and enc.training)
            # per-frame model, video input: the frame-mean head (VidCLIP.py:62-65) over each video's T frame projections
            pool_t = video.shape[1] if which == "vis" and model.config.per_frame and video.dim() == 5 else 0
            if normalize and pool_t:
                feat = torch.empty(proj.shape[0] // pool_t, proj.shape[1], dtype=f32, device=dev)
                inv = (torch.empty(proj.shape[0], dtype=f32, device=dev), torch.empty(feat.shape[0], dtype=f32, device=dev))
                ops.frame_pool_fwd(proj, feat, inv[0], inv[1], pool_t)
            elif normalize:
                feat = torch.empty_like(proj)
                inv = torch.empty(proj.shape[0], dtype=f32, device=dev)
                ops.l2norm_fwd(proj, feat, inv)
            else:
                feat, inv = proj, None
            if sv is not None:
                sv.feat, sv.inv = feat, inv
                sv.pool = (proj, pool_t) if normalize and pool_t else None
                setattr(ctx, which, sv)
            return feat

        none = torch.empty(0, device=dev)
        side = _overlap_stream(model, dev, "overlap_text_tower") if (video is not None and input_ids is not None) else None
        ctx.side = side
        if side is None:
            vis = run_tower("vis") if video is not None else none
            txt = run_tower("txt") if input_ids is not None else none
        else:
            # The text tower (~300 launches of microsecond kernels, SURVEY.md §2.3 K11) runs on a side stream under the vision
            # tower: its small grids fill the SMs that the persistent vision kernels leave idle in their last wave.
            # Issue order: vision first.  After a host sync (a driver reading loss.item() every step) the GPU would otherwise sit on
            # microsecond text kernels while the host is still enqueueing them; queued behind ~600 vision launches they still
            # start while the vision tower is executing.
            main = torch.cuda.current_stream()
            side.wait_stream(main)
            vis = run_tower("vis")
            with torch.cuda.stream(side):
                txt = run_tower("txt")
            main.wait_stream(side)
            txt.record_stream(main)
        return vis, txt

    @staticmethod
    def backward(ctx, d_vis, d_txt):
        model: CLIPModel = ctx.model
        dev = model.logit_scale.device
        w = param_layout(model)
        grads: Dict[str, torch.Tensor] = {}        # operand name -> gradient view
        flats: Dict[str, torch.Tensor] = {}        # gradient group -> its flat buffer
        jobs = (("vision_model", ctx.vis, d_vis, _vision_bwd), ("text_model", ctx.txt, d_txt, _text_bwd))
        main = torch.cuda.current_stream()
        side = ctx.side if (ctx.vis is not None and ctx.txt is not None and d_vis is not None and d_txt is not None) else None
        # data-parallel runs: leave `model.nccl_sm_reserve` SMs to the NCCL kernels of the overlapped gradient all-reduce for
        # the duration of the backward pass only (the forward has no collective in flight and keeps every SM)
        reserve = int(getattr(model, "nccl_sm_reserve", 0) or 0)
        if reserve > 0:
            ops.set_sm_limit(torch.cuda.get_device_properties(dev).multi_processor_count - reserve)
        if side is not None:
            side.wait_stream(main)            # before any vision-backward launch: the text backward only needs d_txt
        for tower, sv, dfeat, bwd in jobs:
            if sv is None or dfeat is None:
                continue
            on_side = side is not None and tower == "text_model"
            if on_side:        # text backward on the side stream, under the vision backward (issued after it, see forward)
                dfeat.record_stream(side)
                with torch.cuda.stream(side):
                    _tower_backward(model, ctx, w, tower, sv, dfeat, bwd, grads, flats, dev)
                continue
            _tower_backward(model, ctx, w, tower, sv, dfeat, bwd, grads, flats, dev)
        if side is not None:
            main.wait_stream(side)
            for k, t in flats.items():      # allocated in the side stream's pool, consumed by autograd on the main stream
                if k.startswith("text_model"):
                    t.record_stream(main)
        hook = getattr(model, "grad_ready_hook", None)
        if hook is not None and hasattr(hook, "finish"):
            hook.finish()      # stream-ordered wait: autograd's accumulation below sees the averaged values
        if reserve > 0:
            ops.set_sm_limit(0)
        ctx.vis = ctx.txt = None
        return (None, None, None, None, None, None) + w.grads_out(grads, ctx.needs_input_grad[6:])


def _tower_backward(model, ctx, w: ParamLayout, tower, sv, dfeat, bwd, grads, flats, dev):
    for key in w.groups:
        if key.startswith(tower):
            flats[key] = w.alloc_grads(key, grads)
    pool = getattr(sv, "pool", None)
    if pool is not None:        # frame-mean head: d(video feature) [B, P] -> d(frame projections) [B*T, P]
        proj, pool_t = pool
        dproj = torch.empty(proj.shape, dtype=bf16, device=dev)
        ops.frame_pool_bwd(dfeat.contiguous().to(f32), sv.feat, proj, sv.inv[0], sv.inv[1], dproj, pool_t)
    else:
        dproj = torch.empty(dfeat.shape, dtype=bf16, device=dev)
        dfeat = dfeat.contiguous().to(f32)
        if ctx.normalize:
            ops.l2norm_bwd(dfeat, sv.feat, sv.inv, dproj)
        else:
            dproj.copy_(dfeat)
    bwd(model, dproj, sv, grads, flats)
    _grads_ready(model, flats[tower])


def _overlap_stream(model: CLIPModel, dev, option: str):
    """The model's stream for one overlap, created once per device: `option` "overlap_text_tower" runs the text tower on it
    under the vision tower, "overlap_colsum" the HBM-bound bias column sums of the vision backward under its GEMMs.  None
    when `model.<option>` is False or XP_NO_OVERLAP=1."""
    import os
    if not getattr(model, option, True) or os.environ.get("XP_NO_OVERLAP") == "1":
        return None
    st = model._packs.get(option)
    if st is None or st.device != dev:
        st = model._packs[option] = torch.cuda.Stream(device=dev)
    return st


def _run(model: CLIPModel, video, input_ids, attention_mask, normalize: bool = True):
    if not model.logit_scale.is_cuda:
        raise _lib.XpError("xpretrain_b200.CLIPModel must live on a CUDA (H100) device: there is no CPU path")
    if video is not None:
        _frame_path(model.config, video)
    vis, txt = _ClipVipFunction.apply(model, video, input_ids, attention_mask, normalize, torch.is_grad_enabled(),
                                      *param_layout(model).params)
    return (vis if video is not None else None), (txt if input_ids is not None else None)
