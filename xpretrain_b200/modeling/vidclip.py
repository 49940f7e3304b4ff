"""VidCLIP wrapper with the reference's constructor, forward signature and output keys
(CLIP-ViP/src/modeling/VidCLIP.py:8-103), over the H100-native CLIPModel."""
from __future__ import annotations

import copy
import json
import os

import torch
import torch.nn as nn

from .clip_vip import CLIPModel, ClipVipConfig, TowerConfig


def _get(obj, key, default=None):
    if obj is None:
        return default
    if isinstance(obj, dict):
        return obj.get(key, default)
    return getattr(obj, key, default)


def config_from_args(args) -> ClipVipConfig:
    """Build the model config the way VidCLIP.__init__ does (VidCLIP.py:11-13): the CLIP hyper-parameters come from
    `args.clip_config` (a local HF-style config.json / directory if it exists, else the built-in hyper-parameters of the
    name: "openai/clip-vit-large-patch14" / "-patch14-336" (ViT-L/14 at 224 / 336 px), "...patch32" (ViT-B/32), and
    otherwise the ViT-B/16 defaults of "openai/clip-vit-base-patch16" — there is no network) and the ViP additions from
    `args.clip_vision_additional_config`.  Its `type` picks the vision model (VidCLIP.py:14-23): "ViP" (the default) is
    the video-proxy tower; any other value is the per-frame CLIP model of CLIP.py, which ignores temporal_size,
    add_cls_num and if_use_temporal_embed."""
    src = _get(args, "clip_config")
    cfg = copy.deepcopy(src) if isinstance(src, ClipVipConfig) else ClipVipConfig()
    path = None
    if isinstance(src, str):
        path = src if os.path.isfile(src) else os.path.join(src, "config.json")
    if path and os.path.isfile(path):
        with open(path) as f:
            hf = json.load(f)
        t, v = hf.get("text_config", {}), hf.get("vision_config", {})
        cfg.text = TowerConfig(t.get("hidden_size", 512), t.get("num_attention_heads", 8), t.get("num_hidden_layers", 12),
                               t.get("intermediate_size", 2048))
        cfg.vision = TowerConfig(v.get("hidden_size", 768), v.get("num_attention_heads", 12),
                                 v.get("num_hidden_layers", 12), v.get("intermediate_size", 3072))
        cfg.image_size = v.get("image_size", 224)
        cfg.patch_size = v.get("patch_size", 16)
        cfg.projection_dim = hf.get("projection_dim", 512)
        cfg.vocab_size = t.get("vocab_size", 49408)
        cfg.max_position_embeddings = t.get("max_position_embeddings", 77)
    elif isinstance(src, str) and "clip-vit-large-patch14" in src:
        # openai/clip-vit-large-patch14 and openai/clip-vit-large-patch14-336 (their Hugging Face config.json)
        cfg.vision = TowerConfig(1024, 16, 24, 4096)
        cfg.text = TowerConfig(768, 12, 12, 3072)
        cfg.patch_size = 14
        cfg.image_size = 336 if src.rstrip("/").endswith("-336") else 224
        cfg.projection_dim = 768
    elif isinstance(src, str) and "patch32" in src:
        cfg.patch_size = 32
    add = _get(args, "clip_vision_additional_config")
    cfg.vision_type = str(_get(add, "type", cfg.vision_type))
    cfg.temporal_size = int(_get(add, "temporal_size", 12))
    cfg.if_use_temporal_embed = int(_get(add, "if_use_temporal_embed", 1))
    cfg.add_cls_num = int(_get(add, "add_cls_num", 3))
    cfg.logit_scale_init_value = float(_get(add, "logit_scale_init_value", 4.60))
    return cfg


class VidCLIP(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.vision_additional_config = _get(args, "clip_vision_additional_config")
        cfg = config_from_args(args)
        self.clipmodel = CLIPModel(cfg)
        weights = _get(args, "clip_weights")
        if weights and os.path.exists(str(weights)):
            # VidCLIP.py:14-18 loads plain OpenAI-CLIP weights; the ViP tower's added_cls / temporal_embedding keep their
            # init, and the per-frame model takes every key of such a checkpoint
            path = weights if os.path.isfile(weights) else os.path.join(weights, "pytorch_model.bin")
            sd = torch.load(path, map_location="cpu")
            sd = {k[len("clipmodel."):] if k.startswith("clipmodel.") else k: v for k, v in sd.items()}
            own = self.clipmodel.state_dict()
            self.clipmodel.load_state_dict({k: v for k, v in sd.items() if k in own and own[k].shape == v.shape},
                                           strict=False)
        self.clipmodel.logit_scale.data.fill_(cfg.logit_scale_init_value)   # VidCLIP.py:25-27

    def overload_logit_scale(self, overload_logit_scale):
        self.clipmodel.logit_scale.data.fill_(overload_logit_scale)

    def forward(self, video, text_input_ids, text_input_mask, image=None, caption_ids=None, caption_masks=None):
        """video [B, T, C, H, W]; text_input_ids / text_input_mask [B, L] (VidCLIP.py:32-81)."""
        if image is not None and self.clipmodel.config.per_frame:
            # the reference's per-frame CLIP model is handed a 5-D image tensor here and fails inside Conv2d
            raise ValueError("the per-frame CLIP model (vision_additional_config.type != 'ViP') has no image/caption branch")
        out = self.clipmodel(input_ids=text_input_ids, attention_mask=text_input_mask, pixel_values=video,
                             return_loss=False)
        results = {"text_features": out["text_embeds"], "vis_features": out["image_embeds"]}
        if image is not None:
            B, img_num, C, H, W = image.shape
            L = caption_ids.shape[-1]
            out = self.clipmodel(input_ids=caption_ids.reshape(-1, L), attention_mask=caption_masks.reshape(-1, L),
                                 pixel_values=image.reshape(-1, 1, C, H, W), return_loss=False)
            results["img_features"] = out["image_embeds"]
            results["cap_features"] = out["text_embeds"]
        return results

    def forward_video(self, video):
        return self.clipmodel.get_image_features(pixel_values=video, if_norm=True)

    def forward_text(self, text_input_ids, text_input_mask):
        return self.clipmodel.get_text_features(input_ids=text_input_ids, attention_mask=text_input_mask, if_norm=True)

    def freeze_text_encoder(self, freeze_text_proj):
        freeze_list = [self.clipmodel.text_model]
        if freeze_text_proj:
            freeze_list.append(self.clipmodel.text_projection)
        for m in freeze_list:
            m.eval()
            for param in m.parameters():
                param.requires_grad = False
