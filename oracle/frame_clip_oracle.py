"""CPU oracle for the per-frame CLIP video model — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A functional fp32 / fp64 restatement of the vision model VidCLIP builds when `vision_additional_config.type` is not
"ViP" (CLIP-ViP/src/modeling/VidCLIP.py:14-23,54-65 over CLIP-ViP/src/modeling/CLIP.py): every frame runs through a
plain CLIP ViT on its own, each frame's CLS feature is projected and L2-normalised, the frames are averaged and the
average is normalised again.  The text tower, the loss and the state_dict naming are those of clipvip_oracle.

Parity pinned: `tests/golden/make_golden_frame_clip.py` checks this module against the reference's own CLIP.py to fp32
round-off and writes the goldens that `tests/test_frame_clip_cpu.py` replays.
"""
from __future__ import annotations

from typing import Dict

import torch

from . import clipvip_oracle as O

Tensor = torch.Tensor

VIP_ONLY_KEYS = ("vision_model.embeddings.added_cls", "vision_model.embeddings.temporal_embedding")


def frame_embeddings(sd: Dict[str, Tensor], images: Tensor, cfg: O.ClipVipCfg,
                     pre: str = "vision_model.embeddings.") -> Tensor:
    """CLIPVisionEmbeddings.forward, CLIP.py:132-140.  images [N,3,H,W] -> [N, 1 + L, C]: the CLS row, then the patch rows
    in row-major grid order, plus position_embedding[0..L]."""
    N, C, H, W = images.shape
    w = sd[pre + "patch_embedding.weight"]
    p = cfg.patch
    x = images.reshape(N, C, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5).reshape(N, -1, C * p * p)
    patches = x @ w.reshape(w.shape[0], -1).t()                       # [N, L, width]
    cls = sd[pre + "class_embedding"].expand(N, 1, -1)
    return torch.cat([cls, patches], dim=1) + sd[pre + "position_embedding.weight"].unsqueeze(0)


def frame_vision_tower(sd: Dict[str, Tensor], images: Tensor, cfg: O.ClipVipCfg) -> Tensor:
    """CLIPVisionTransformer.forward, CLIP.py:770-801: dense pre-LN blocks over 1 + L rows; post_layernorm of the CLS row."""
    x = O.layer_norm(frame_embeddings(sd, images, cfg), sd, "vision_model.pre_layrnorm", cfg.ln_eps)
    for i in range(cfg.vision.layers):
        x = O.encoder_layer(sd, x, f"vision_model.encoder.layers.{i}.", cfg.vision.heads, cfg.ln_eps, None, None)
    return O.layer_norm(x[:, 0], sd, "vision_model.post_layernorm", cfg.ln_eps)


def frame_mean_head(proj: Tensor, B: int, T: int) -> Tensor:
    """VidCLIP.py:62-65: normalise each frame's projection, average the T frames of each video, normalise again."""
    return O.l2_normalize(O.l2_normalize(proj).reshape(B, T, -1).mean(1))


def frame_clip_forward(sd: Dict[str, Tensor], video: Tensor, input_ids: Tensor, attention_mask: Tensor,
                       cfg: O.ClipVipCfg) -> Dict[str, Tensor]:
    """VidCLIP.forward with a non-ViP type (VidCLIP.py:54-68): video [B,T,3,H,W] -> vis_features [B, P]; text_features is
    CLIP.py's normalised text_embeds."""
    B, T = video.shape[:2]
    proj = O.linear(frame_vision_tower(sd, video.reshape(B * T, *video.shape[2:]), cfg), sd, "visual_projection")
    txt = O.l2_normalize(O.linear(O.text_tower(sd, input_ids, attention_mask, cfg), sd, "text_projection"))
    return {"vis_features": frame_mean_head(proj, B, T), "text_features": txt}


def run_reduced_precision(sd: Dict[str, Tensor], video: Tensor, input_ids: Tensor, attention_mask: Tensor,
                          cfg: O.ClipVipCfg, device, mode: str):
    """Calibration arm: this restatement under torch.autocast(bf16) ('autocast') or with every floating tensor in bf16
    ('pure'), as clipvip_oracle.run_reduced_precision.  Returns (vis, txt, loss, {name: grad}) as fp32 CPU values."""
    dt = torch.bfloat16 if mode == "pure" else torch.float32
    dev = torch.device(device)
    sdg = {k: (v.detach().to(dev, dt, copy=True).requires_grad_(True) if v.is_floating_point() else v.to(dev))
           for k, v in sd.items()}
    with torch.autocast(dev.type, dtype=torch.bfloat16, enabled=(mode == "autocast")):
        o = frame_clip_forward(sdg, video.to(dev, dt), input_ids.to(dev), attention_mask.to(dev), cfg)
        loss = O.nce_learnable_temp_loss(o["vis_features"].float(), o["text_features"].float(), sdg["logit_scale"].float())
    loss.backward()
    grads = {k: t.grad.detach().float().cpu() for k, t in sdg.items() if t.is_floating_point() and t.grad is not None}
    return o["vis_features"].detach().float().cpu(), o["text_features"].detach().float().cpu(), float(loss.detach()), grads


def init_state_dict(cfg: O.ClipVipCfg, seed: int = 0, dtype=torch.float32) -> Dict[str, Tensor]:
    """clipvip_oracle.init_state_dict without the ViP tower's added_cls and temporal_embedding: the names of CLIP.py's
    CLIPModel.state_dict() (CLIP.py:113-140 embeddings), with the init statistics of CLIP.py:391-434."""
    sd = O.init_state_dict(cfg, seed=seed, dtype=dtype)
    for k in VIP_ONLY_KEYS:
        del sd[k]
    return sd


def flops_per_pair(cfg: O.ClipVipCfg, T: int, Lt: int) -> Dict[str, float]:
    """Algorithmic FLOPs (2 per MAC) per video-text pair: T dense frames of S = 1 + L rows each."""
    C, mlp, L = cfg.vision.width, cfg.vision.mlp, cfg.patches
    S = 1 + L
    d = C // cfg.vision.heads
    block = 2 * S * C * 3 * C + cfg.vision.heads * 2 * 2 * S * S * d + 2 * S * C * C + 2 * 2 * S * C * mlp
    patch = 2 * L * (3 * cfg.patch * cfg.patch) * C
    vproj = 2 * C * cfg.proj_dim
    Ct, mt = cfg.text.width, cfg.text.mlp
    tblock = 2 * Lt * Ct * 3 * Ct + cfg.text.heads * 2 * 2 * Lt * Lt * (Ct // cfg.text.heads) + 2 * Lt * Ct * Ct \
        + 2 * 2 * Lt * Ct * mt
    tproj = 2 * Ct * cfg.proj_dim
    fwd = T * (patch + cfg.vision.layers * block + vproj) + cfg.text.layers * tblock + tproj
    bwd = 2 * fwd - T * patch          # the patch embedding has no dgrad (the input needs no gradient)
    return {"fwd": float(fwd), "train": float(fwd + bwd), "frame_block_fwd": float(block)}
