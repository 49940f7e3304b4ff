"""LF-VILA's input transform (init_transform_dict, LF-VILA/src/datasets/dataloader.py:94-121) as crop boxes for uint8 frames.

Every LF-VILA dataset hands decord's `[N, H, W, 3]` uint8 batch to
    val / test  Resize([240, 428]) + CenterCrop([216, 385]) + Resize(input_res) + Normalize(ImageNet)
    train       RandomResizedCrop(input_res, scale=(0.8, 1.0)) + RandomHorizontalFlip() + ColorJitter(0, 0, 0) + Normalize
after `.float() / 255`.  Both are "resize the frame to stage_a, crop a box, resize the box to input_res, maybe mirror",
which `ops.lfvila_frames_patchify_u8` runs fused into Swin-3D's patch extraction.  This module only says where the boxes
are: `eval_crops` the fixed centre crop, `train_crops` the reference's random draws, taken from torch's CPU generator in
the order the `train` Compose takes them, so that a given seed gives the reference's boxes and flips.  `center_crop` of
init_transform_dict is unused there, and no LF-VILA caller passes a non-zero ColorJitter, so neither exists here.
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional, Tuple

import torch

STAGE_A = (240, 428)                                        # Resize([240, 428])
CENTER_CROP = (int(240 * 0.9), int(428 * 0.9))              # CenterCrop: (216, 385)
RANDCROP_SCALE = (0.8, 1.0)
RANDCROP_RATIO = (3.0 / 4.0, 4.0 / 3.0)                     # RandomResizedCrop's default ratio
INPUT_RES = (192, 320)                                      # input_res of the released configs


class Crops(NamedTuple):
    """Per clip, a box (top, left, h, w) in stage-A coordinates and a flip flag: CPU int32 [B, 5]; and the stage-A size
    (Ha, Wa) the frames are resized to before the crop ((H, W) itself for training crops: stage A is the identity)."""
    params: torch.Tensor
    stage_a: Tuple[int, int]


def eval_crops(B: int) -> Crops:
    """The val / test transform: Resize([240, 428]), then CenterCrop's box (top = round(24 / 2), left = round(43 / 2))."""
    (Ha, Wa), (h, w) = STAGE_A, CENTER_CROP
    top, left = int(round((Ha - h) / 2.0)), int(round((Wa - w) / 2.0))
    return Crops(torch.tensor([[top, left, h, w, 0]], dtype=torch.int32).repeat(B, 1), STAGE_A)


def _random_resized_crop(H: int, W: int, generator: Optional[torch.Generator]):
    """RandomResizedCrop.get_params(scale=(0.8, 1.0), ratio=(3/4, 4/3)) on an H x W image: 10 tries, then the central
    fallback; the same draws, in the same order, from the same generator."""
    area = H * W
    log_ratio = torch.log(torch.tensor(RANDCROP_RATIO))
    for _ in range(10):
        target_area = area * torch.empty(1).uniform_(RANDCROP_SCALE[0], RANDCROP_SCALE[1], generator=generator).item()
        aspect_ratio = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1], generator=generator)).item()
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if 0 < w <= W and 0 < h <= H:
            i = torch.randint(0, H - h + 1, size=(1,), generator=generator).item()
            j = torch.randint(0, W - w + 1, size=(1,), generator=generator).item()
            return i, j, h, w
    in_ratio = float(W) / float(H)
    if in_ratio < min(RANDCROP_RATIO):
        w, h = W, int(round(W / min(RANDCROP_RATIO)))
    elif in_ratio > max(RANDCROP_RATIO):
        h, w = H, int(round(H * max(RANDCROP_RATIO)))
    else:
        w, h = W, H
    return (H - h) // 2, (W - w) // 2, h, w


def train_crops(B: int, H: int, W: int, generator: Optional[torch.Generator] = None) -> Crops:
    """The train transform's random draws for B clips of H x W frames, clip after clip: RandomResizedCrop's box,
    RandomHorizontalFlip's `torch.rand(1) < 0.5`, and the `torch.randperm(4)` the identity ColorJitter still draws.
    generator=None draws from torch's default CPU generator, as the reference's dataloader workers do."""
    rows = []
    for _ in range(B):
        i, j, h, w = _random_resized_crop(H, W, generator)
        flip = bool(torch.rand(1, generator=generator) < 0.5)
        torch.randperm(4, generator=generator)
        rows.append([i, j, h, w, int(flip)])
    return Crops(torch.tensor(rows, dtype=torch.int32).reshape(B, 5), (H, W))
