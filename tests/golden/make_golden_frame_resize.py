"""Writes tests/golden/frame_resize_u8.pt: the reference transform of decoded uint8 frames, as torchvision runs it.

init_transform_dict_simple (CLIP-ViP/src/datasets/dataloader.py:209-233) composes, for every split,
    Resize(input_res, interpolation=BICUBIC) + CenterCrop(input_res) + Normalize(mean, std)
on the float frames `img_array.permute(0, 3, 1, 2).float() / 255.` (dataset_pretrain_stage1_all_source.py:182), with
input_res = (S, S).  It is rebuilt here from the installed torchvision, with antialias=False: the pinned torchvision 0.9.0
had no antialias on tensors, and runs the same F.interpolate(mode="bicubic", align_corners=False).

Each case: seeded frames [2, H, W, 3] (torch.randint on the CPU generator, pinned by a checksum), the transformed fp32
tensor [2, 3, S, S] sampled at 2048 seeded flat positions, and its float64 sum.  Sources: 240 x 320 (the retrieval
configs' video_res), 360 x 640, 100 x 150 (upscaling), 239 x 317 (odd) and 1 x 1, each into S = 224 and 336.

    python tests/golden/make_golden_frame_resize.py
"""
import os

import torch
from torchvision import transforms

MEAN, STD = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)   # dataloader.py:210-211
SOURCES = [(240, 320), (360, 640), (100, 150), (239, 317), (1, 1)]
SIZES = [224, 336]
FRAMES, SAMPLES = 2, 2048


def frames_for(H, W, seed):
    return torch.randint(0, 256, (FRAMES, H, W, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def sample_index(n, seed):
    return torch.randint(0, n, (SAMPLES,), generator=torch.Generator().manual_seed(seed + 1))


def reference_transform(frames, S):
    tf = transforms.Compose([
        transforms.Resize((S, S), interpolation=transforms.InterpolationMode.BICUBIC, antialias=False),
        transforms.CenterCrop((S, S)),
        transforms.Normalize(mean=MEAN, std=STD),
    ])
    return tf(frames.permute(0, 3, 1, 2).float() / 255.)


def main():
    cases = []
    for k, (H, W) in enumerate(SOURCES):
        for S in SIZES:
            seed = 1000 + 10 * k + S
            frames = frames_for(H, W, seed)
            out = reference_transform(frames, S)
            assert out.dtype == torch.float32 and out.shape == (FRAMES, 3, S, S)
            idx = sample_index(out.numel(), seed)
            cases.append({"H": H, "W": W, "S": S, "seed": seed, "frames_sum": int(frames.long().sum()),
                          "index": idx.to(torch.int32), "values": out.reshape(-1)[idx].clone(),
                          "sum": float(out.double().sum())})
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "frame_resize_u8.pt")
    torch.save({"meta": {"mean": MEAN, "std": STD, "frames": FRAMES, "torch": torch.__version__}, "cases": cases}, path)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
