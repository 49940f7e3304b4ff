"""CPU oracle of LF-VILA's video classification model (COIN / LVU): the head of
LF-VILA/src/models/lfvila_video_classification.py on top of the unchanged Swin-3D oracle (oracle/swin3d_oracle.py).

TEST INFRASTRUCTURE ONLY — imported by tests/, tests/golden/make_golden_lfvila_cls.py and tools/; never by the product package.

A functional fp32 PyTorch restatement.  Parity pinned by tests/golden/make_golden_lfvila_cls.py against the reference's own
`LFVILA_Video_Classification` (imported with stub `timm` / `mmcv` / BERT modules): outputs, loss and every parameter
gradient to fp32 round-off.

Reference lines followed:
  downsample_video_embd   :32-43  MaxPool2d((2, 3), stride (1, 1)) over each frame's [H, W] grid (channels first), the frame
                                  mean over the X pooled positions and the clip mean over all N * X of them (one mean)
  forward                 :46-68  video_global_proj / video_frame_proj, each followed by F.normalize(dim=-1); classifier on
                                  the normalised global feature; nn.CrossEntropyLoss; acc = (argmax == labels).float().mean
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle import swin3d_oracle as SO

HEAD = ("video_global_proj", "video_frame_proj", "classifier")


def param_shapes(cfg: SO.Swin3DCfg, n_labels: int) -> Dict[str, tuple]:
    """state_dict of the reference module: the encoder under `video_encoder.`, then the three Linear layers."""
    sh = {"video_encoder." + k: v for k, v in SO.param_shapes(cfg).items()}
    C = cfg.dim(len(cfg.depths) - 1)
    for name, out in (("video_global_proj", C), ("video_frame_proj", C), ("classifier", n_labels)):
        sh[name + ".weight"] = (out, C)
        sh[name + ".bias"] = (out,)
    return sh


def init_state_dict(cfg: SO.Swin3DCfg, n_labels: int, seed: int = 0) -> Dict[str, torch.Tensor]:
    """The Swin-3D oracle's weights (seed) under `video_encoder.`; head weights N(0, 0.02) and biases N(0, 0.02) (seed + 1)."""
    sd = {"video_encoder." + k: v for k, v in SO.init_state_dict(cfg, seed=seed).items()}
    g = torch.Generator().manual_seed(seed + 1)
    for k, s in param_shapes(cfg, n_labels).items():
        if not k.startswith("video_encoder."):
            sd[k] = 0.02 * torch.randn(s, generator=g)
    return sd


def synthetic_labels(B: int, n_labels: int, seed: int = 7) -> torch.Tensor:
    """Labels covering every class when B >= n_labels (a permutation of the classes, repeated)."""
    perm = torch.randperm(n_labels, generator=torch.Generator().manual_seed(seed))
    return perm.repeat((B + n_labels - 1) // n_labels)[:B].clone()


def pool(video_embd):
    """downsample_video_embd, :32-43: video_embd [B, N, H, W, C] -> (video_feat [B, C], video_frame_feat [B, N, C])."""
    B, N, H, W, C = video_embd.shape
    x = F.max_pool2d(video_embd.permute(0, 1, 4, 2, 3).reshape(B * N, C, H, W), (2, 3), stride=(1, 1))
    x = x.permute(0, 2, 3, 1).reshape(B, N, -1, C)
    return x.mean(dim=[1, 2]), x.mean(dim=2)


def head_forward(sd, video_embd, labels):
    """forward, :49-68, after the encoder."""
    g, fr = pool(video_embd)
    g = F.normalize(F.linear(g, sd["video_global_proj.weight"], sd["video_global_proj.bias"]), dim=-1)
    fr = F.normalize(F.linear(fr, sd["video_frame_proj.weight"], sd["video_frame_proj.bias"]), dim=-1)
    logits = F.linear(g, sd["classifier.weight"], sd["classifier.bias"])
    loss = F.cross_entropy(logits, labels)
    acc = (logits.max(dim=-1)[1] == labels).float().mean(dim=0, keepdim=True)
    return dict(video_global_feat=g, video_frame_feat=fr, prediction=logits, loss=loss, acc=acc)


def lfvila_cls_forward(sd, video, labels, cfg: SO.Swin3DCfg, drop_masks=None):
    """LFVILA_Video_Classification.forward on video [B, 3, N, H, W]; drop_masks as swin3d_oracle.draw_drop_masks."""
    enc = {k[len("video_encoder."):]: v for k, v in sd.items() if k.startswith("video_encoder.")}
    return head_forward(sd, SO.swin3d_forward(enc, video, cfg, drop_masks=drop_masks), labels)
