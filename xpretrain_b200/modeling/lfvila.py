"""LF-VILA's long-form video classification model (COIN, LVU) on the H100 kernels.

Drop-in for `LFVILA_Video_Classification` of LF-VILA/src/models/lfvila_video_classification.py:16-68: the same constructor
`(args, config)` (`config.VideoEncoder`, `config.bert_config` read for `hidden_size`, `config.DATA.classification_labels`),
the same `state_dict()` (`video_encoder.*` of modeling/swin3d.py, `video_global_proj.*`, `video_frame_proj.*`,
`classifier.*`; the max-pool holds nothing), and the same `forward(video_frames, labels) -> dict(video_global_feat,
video_frame_feat, prediction, loss, acc)`.  `forward` also takes decord's uint8 frames `[B, N, H, W, 3]` and an optional
`crops=` (modeling/lfvila_frames.py): the datasets' transform to `config.DATA.input_res` then runs on the GPU.

The encoder call is modeling/swin3d.py's, unchanged.  The head after it runs as ONE autograd.Function:
  * xp_lfvila_pool_fwd: MaxPool2d((2, 3), stride 1) over each frame's Hp x Wp grid, the frame means `video_frame_feat`
    [B*N, C] and the clip means `video_feat` [B, C] (mean over all N * X window maxima, :40) in fp32 with bf16 copies,
    the arg-max window position saved as a byte; its backward gathers over the windows covering each element;
  * video_global_proj / video_frame_proj: the wgmma GEMM (bf16 operands, fp32 out, bias in the epilogue);
  * xp_lfvila_normalize_*: F.normalize (x / max(||x||, 1e-12)) and its gradient, below the clamp included;
  * classifier: the same GEMM on a weight padded with zero rows to a multiple of 8 labels (the GEMM's N alignment), the
    logits written with that padded pitch;
  * xp_lfvila_ce_*: nn.CrossEntropyLoss and `acc` (first-index argmax) with a fixed reduction order.
Outputs are fp32 whatever the video dtype (fp16 video, the trainer's --fp16 input, runs the encoder on fp16 input and the
pool on its fp16 output).  There is no CPU path.
"""
from __future__ import annotations

import json
from typing import Dict, Optional

import torch
import torch.nn as nn

from .. import _lib, ops
from ._weights import ParamLayout, param_layout
from .lfvila_frames import INPUT_RES, Crops
from .swin3d import SwinTransformer3D

bf16, f32 = torch.bfloat16, torch.float32


def _get(obj, key, default=None):
    if isinstance(obj, dict):
        return obj.get(key, default)
    return getattr(obj, key, default)


class LFVILA_Video_Classification(nn.Module):
    """Constructor mirrors lfvila_video_classification.py:17-29."""

    def __init__(self, args, config):
        super().__init__()
        self.cfg = config
        self.video_encoder = SwinTransformer3D(**dict(_get(config, "VideoEncoder")))
        with open(_get(config, "bert_config")) as f:       # BertConfig.from_json_file: only hidden_size is used
            hidden = int(json.load(f).get("hidden_size", 768))
        if hidden != self.video_encoder.num_features:
            raise ValueError(f"bert_config hidden_size {hidden} must equal the video encoder's num_features "
                             f"{self.video_encoder.num_features} (the projections take the encoder output)")
        self.video_global_proj = nn.Linear(hidden, hidden)
        self.video_frame_proj = nn.Linear(hidden, hidden)
        self.n_labels = int(_get(_get(config, "DATA"), "classification_labels"))
        self.input_res = tuple(int(v) for v in _get(_get(config, "DATA"), "input_res", INPUT_RES))   # uint8 input only
        self.classifier = nn.Linear(hidden, self.n_labels)

    def _declare_layout(self) -> ParamLayout:
        """The head's parameters (the encoder has its own layout): bf16 copies of the three weights, the classifier's and
        its fp32 bias padded with zero rows to a multiple of 8 labels (the GEMM's N alignment); one gradient group."""
        return ParamLayout(self, exclude=("video_encoder.",), cast=lambda n, p: n.endswith(".weight") or n == "classifier.bias",
                           pad8=("classifier.weight", "classifier.bias"))

    def forward(self, video_frames: torch.Tensor, labels=None, crops: Optional[Crops] = None):
        """video_frames: the transformed float video [B, 3, N, H, W], or decoder's uint8 frames [B, N, H, W, 3], transformed
        to config.DATA.input_res as LF-VILA's datasets do: with `crops` (lfvila_frames.train_crops) while training, the
        val / test transform when crops is None."""
        if not isinstance(labels, torch.Tensor):
            # nn.CrossEntropyLoss()(logits, labels) raises this for labels=None (:58-59)
            raise TypeError(f"cross_entropy_loss(): argument 'target' (position 2) must be Tensor, not "
                            f"{type(labels).__name__}")
        if not video_frames.is_cuda:
            raise _lib.XpError("xpretrain_b200 LFVILA_Video_Classification needs CUDA tensors on an H100: there is no "
                               "CPU path")
        if labels.dtype != torch.int64 or labels.dim() != 1 or labels.shape[0] != video_frames.shape[0]:
            raise ValueError(f"labels must be int64 class indices of shape [{video_frames.shape[0]}] (got {labels.dtype} "
                             f"{list(labels.shape)})")
        video_embd, _ = self.video_encoder(video_frames, crops=crops, out_size=self.input_res)      # [B, N, H, W, C]
        g, fr, pred, loss, acc = _HeadFunction.apply(self, torch.is_grad_enabled(), video_embd,
                                                     labels.to(video_embd.device), *param_layout(self).params)
        return dict(video_global_feat=g, video_frame_feat=fr, prediction=pred, loss=loss, acc=acc)


class _HeadFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model: LFVILA_Video_Classification, grad_mode: bool, x: torch.Tensor, labels: torch.Tensor, *params):
        # grad_mode = torch.is_grad_enabled() of the caller: evaluation keeps nothing for a backward
        ctx.set_materialize_grads(False)
        B, N, Hp, Wp, C = x.shape
        dev = x.device
        X = max(Hp - 1, 0) * max(Wp - 2, 0)
        w = param_layout(model)
        w.refresh()
        n, n_pad = model.n_labels, w["classifier.weight"].shape[0]
        frame_raw = torch.empty(B * N, C, dtype=f32, device=dev)
        frame_bf = torch.empty(B * N, C, dtype=bf16, device=dev)
        global_raw = torch.empty(B, C, dtype=f32, device=dev)
        global_bf = torch.empty(B, C, dtype=bf16, device=dev)
        argmax = torch.empty(B, N, X, C, dtype=torch.uint8, device=dev)
        ops.lfvila_pool_fwd(x, frame_raw, frame_bf, global_raw, global_bf, argmax)
        gproj = torch.empty(B, C, dtype=f32, device=dev)
        ops.linear_fwd(global_bf, w["video_global_proj.weight"], model.video_global_proj.bias, gproj, out_mode=_lib.OUT_F32)
        fproj = torch.empty(B * N, C, dtype=f32, device=dev)
        ops.linear_fwd(frame_bf, w["video_frame_proj.weight"], model.video_frame_proj.bias, fproj, out_mode=_lib.OUT_F32)
        gfeat, gfeat_bf, gnorm = torch.empty_like(gproj), torch.empty(B, C, dtype=bf16, device=dev), gproj.new_empty(B)
        ops.lfvila_normalize_fwd(gproj, gfeat, gfeat_bf, gnorm)
        ffeat, fnorm = torch.empty_like(fproj), fproj.new_empty(B * N)
        ops.lfvila_normalize_fwd(fproj, ffeat, None, fnorm)
        del gproj, fproj
        logits = torch.empty(B, n_pad, dtype=f32, device=dev)
        ops.linear_fwd(gfeat_bf, w["classifier.weight"], w["classifier.bias"], logits, out_mode=_lib.OUT_F32)
        pred = torch.empty(B, n, dtype=f32, device=dev)
        lse, loss, acc = logits.new_empty(B), logits.new_empty(()), logits.new_empty(1)
        ops.lfvila_ce_fwd(logits, n, labels, pred, lse, loss, acc)
        ctx.mark_non_differentiable(acc)
        ctx.saved = None
        if grad_mode and any(ctx.needs_input_grad[2:]):
            ctx.model, ctx.x_meta = model, (x.shape, x.dtype)
            ctx.saved = (argmax, frame_bf, global_bf, gfeat, gfeat_bf, gnorm, ffeat, fnorm, logits, lse, labels)
        return gfeat, ffeat.view(B, N, C), pred, loss, acc

    @staticmethod
    def backward(ctx, d_gfeat, d_ffeat, d_pred, d_loss, _d_acc):
        model = ctx.model
        argmax, frame_bf, global_bf, gfeat, gfeat_bf, gnorm, ffeat, fnorm, logits, lse, labels = ctx.saved
        ctx.saved = None
        (B, N, Hp, Wp, C), xdt = ctx.x_meta
        dev = logits.device
        w = param_layout(model)
        n, n_pad = model.n_labels, w["classifier.weight"].shape[0]
        grads: Dict[str, torch.Tensor] = {}
        w.alloc_grads("", grads)                  # the classifier's padded: the GEMMs write n_pad rows
        d_global = d_frame = None
        # classifier, from the loss and / or a gradient of `prediction`
        d_class = None
        if d_loss is not None or d_pred is not None:
            dlog = torch.empty(B, n_pad, dtype=bf16, device=dev)
            ops.lfvila_ce_bwd(logits, n, lse, labels, d_loss, d_pred, dlog)
            ops.linear_wgrad(dlog, gfeat_bf, grads["classifier.weight"])
            ops.colsum(dlog, grads["classifier.bias"])
            d_class = torch.empty(B, C, dtype=f32, device=dev)
            ops.linear_dgrad(dlog, w["classifier.weight"], d_class, out_mode=_lib.OUT_F32)
        # video_global_proj + normalize, from the classifier and / or a gradient of `video_global_feat`
        if d_class is not None or d_gfeat is not None:
            dg = torch.empty(B, C, dtype=bf16, device=dev)
            ops.lfvila_normalize_bwd(d_class, None if d_gfeat is None else d_gfeat.to(f32).contiguous(), gfeat, gnorm, dg)
            ops.linear_wgrad(dg, global_bf, grads["video_global_proj.weight"])
            ops.colsum(dg, grads["video_global_proj.bias"])
            d_global = torch.empty(B, C, dtype=f32, device=dev)
            ops.linear_dgrad(dg, w["video_global_proj.weight"], d_global, out_mode=_lib.OUT_F32)
        # video_frame_proj + normalize, from a gradient of `video_frame_feat` (no loss uses it)
        if d_ffeat is not None:
            df = torch.empty(B * N, C, dtype=bf16, device=dev)
            ops.lfvila_normalize_bwd(d_ffeat.to(f32).reshape(B * N, C).contiguous(), None, ffeat, fnorm, df)
            ops.linear_wgrad(df, frame_bf, grads["video_frame_proj.weight"])
            ops.colsum(df, grads["video_frame_proj.bias"])
            d_frame = torch.empty(B * N, C, dtype=f32, device=dev)
            ops.linear_dgrad(df, w["video_frame_proj.weight"], d_frame, out_mode=_lib.OUT_F32)
        dx = None
        if ctx.needs_input_grad[2]:
            dx = torch.empty(B, N, Hp, Wp, C, dtype=xdt, device=dev)
            ops.lfvila_pool_bwd(d_frame, d_global, argmax, dx)
        return (None, None, dx, None) + w.grads_out(grads, ctx.needs_input_grad[4:])
