"""Writes tests/golden/lfvila_frames_u8.pt: LF-VILA's input transform of decoded uint8 clips, as the reference runs it.

The transform is the reference's own `init_transform_dict(input_res)` (LF-VILA/src/datasets/dataloader.py:94-121),
imported from a checkout of microsoft/XPretrain named by XP_REFERENCE_ROOT, applied as
VideoClassificationDataset does (video_classification_dataset.py:84-96): `frames.float() / 255`, permuted to
[N, C, H, W], then `transform(video)`.  The modules the reference imports next to it but the transform does not use
(jsonlines, decord, easydict, lmdb, tensorboardX) are stubbed.  Its Resize and RandomResizedCrop get antialias=False: the
pinned torchvision 0.11 had no antialias on tensors, the installed one defaults to it.

Each case: seeded uint8 clips [B, N, H, W, 3] (stored), and for `val` and for `train` the fp32 output [B, N, 3, 192, 320]
sampled at 2048 seeded flat positions plus its float64 sum.  `train` runs clip after clip after torch.manual_seed(SEED),
and records the box RandomResizedCrop.get_params returned and whether hflip ran.  Sources: 48 x 64 and 61 x 97
(upscales, odd), 280 x 100 (stage A downscales rows and upscales columns), 60 x 900 (the reverse, by 2.1), and 8 x 200 /
200 x 8, whose aspect ratios send every RandomResizedCrop try to its central fallback.

    XP_REFERENCE_ROOT=<checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_lfvila_frames.py
"""
import os
import sys
from unittest import mock

import torch
import torchvision.transforms as T
import torchvision.transforms.functional as TF

SOURCES = [(48, 64), (61, 97), (280, 100), (60, 900), (8, 200), (200, 8)]
B, N, INPUT_RES, SEED, SAMPLES = 2, 1, [192, 320], 1234, 2048


def reference_transforms():
    for name in ("jsonlines", "decord", "easydict", "lmdb", "tensorboardX"):
        sys.modules.setdefault(name, mock.MagicMock(name=name))       # imported at module level, never called here
    sys.path.insert(0, os.path.join(os.environ["XP_REFERENCE_ROOT"], "LF-VILA"))
    from src.datasets.dataloader import init_transform_dict
    tfs = init_transform_dict(INPUT_RES)
    for split in ("train", "val"):
        for t in tfs[split].transforms:
            if isinstance(t, (T.Resize, T.RandomResizedCrop)):
                t.antialias = False
    return tfs


def clips_for(H, W, seed):
    return torch.randint(0, 256, (B, N, H, W, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def sampled(out, seed):
    idx = torch.randint(0, out.numel(), (SAMPLES,), generator=torch.Generator().manual_seed(seed + 1))
    return {"index": idx.to(torch.int32), "values": out.reshape(-1)[idx].clone(), "sum": float(out.double().sum())}


def main():
    tfs = reference_transforms()
    draws = []
    get_params, hflip = T.RandomResizedCrop.get_params, TF.hflip

    def recorded_get_params(img, scale, ratio):
        box = get_params(img, scale, ratio)
        draws.append(list(box) + [0])
        return box

    def recorded_hflip(img):
        draws[-1][4] = 1
        return hflip(img)
    T.RandomResizedCrop.get_params = staticmethod(recorded_get_params)
    TF.hflip = recorded_hflip
    cases = []
    for k, (H, W) in enumerate(SOURCES):
        seed = 2000 + k
        clips = clips_for(H, W, seed)
        case = {"H": H, "W": W, "seed": seed, "clips": clips}
        for split in ("val", "train"):
            torch.manual_seed(SEED)
            del draws[:]
            out = torch.stack([tfs[split](c.permute(0, 3, 1, 2).float() / 255) for c in clips])
            assert out.dtype == torch.float32 and out.shape == (B, N, 3, *INPUT_RES)
            case[split] = sampled(out, seed + (0 if split == "val" else 100))
            if split == "train":
                case["train"]["draws"] = torch.tensor(draws, dtype=torch.int32)
        cases.append(case)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lfvila_frames_u8.pt")
    meta = {"seed": SEED, "input_res": INPUT_RES, "mean": (0.485, 0.456, 0.406), "std": (0.229, 0.224, 0.225),
            "torch": torch.__version__}
    torch.save({"meta": meta, "cases": cases}, path)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
