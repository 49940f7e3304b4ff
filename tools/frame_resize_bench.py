"""Decoded uint8 frames resized on the GPU (xp_vip_resize_patchify_u8) against the reference's CPU transform.

  kernel   CUDA-event time of 64 x 12 frames at 240 x 320 and at 720 x 1280 into 224 (p = 16), against the bytes-moved
           bound at the H100 SXM data sheet's 3.35 TB/s (the uint8 frames read once, the bf16 patch matrix written once)
  step     one training step of the bench model (ViP B/16, 12 + 12 layers, B = 64, T = 12) through the module, host frames
           to backward: uint8 240 x 320 frames (resized on the GPU) against float 224 x 224 frames already transformed
  cpu      the reference transform of one 12-frame sample (/255, Resize([224, 224], BICUBIC) + CenterCrop + Normalize, as
           init_transform_dict_simple composes it), one thread of this host's CPU, at 240 x 320 and 360 x 640

    python tools/frame_resize_bench.py [--out frame_resize_bench.json]
Prints one JSON line; the card's name and power limit are read in the same run.
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import harness  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def kernel_time(dev, H, W, frames=64 * 12, S=224, p=16, iters=50):
    from xpretrain_b200 import ops
    video = torch.randint(0, 256, (frames, H, W, 3), dtype=torch.uint8, device=dev)
    out = torch.empty(frames * (S // p) ** 2, ops.patch_pitch(p), dtype=torch.bfloat16, device=dev)
    ms = harness.window_ms(lambda: ops.vip_resize_patchify_u8(video, out, S, p), iters, 5)
    nbytes = video.numel() + out.numel() * 2
    return {"frames": frames, "src": f"{H}x{W}", "ms": round(ms, 4), "bytes_read_MB": round(video.numel() / 1e6, 1),
            "bytes_written_MB": round(out.numel() * 2 / 1e6, 1), "bound_ms": round(nbytes / HBM_BYTES_PER_S * 1e3, 4),
            "share_of_bound": round(nbytes / HBM_BYTES_PER_S * 1e3 / ms, 3)}


def step_times(dev, B=64, T=12, steps=5, warmup=2):
    from oracle import clipvip_oracle as O
    from xpretrain_b200.modeling.clip_vip import CLIPModel, ClipVipConfig
    cfg = O.ClipVipCfg()
    model = CLIPModel(ClipVipConfig())
    model.load_state_dict(O.init_state_dict(cfg, seed=0), strict=False)
    model = model.to(dev).train()
    _, ids, mask = O.synthetic_batch(B, T, 32, cfg, seed=1, ragged_text=True)
    ids, mask = ids.to(dev), mask.to(dev)
    g = torch.Generator().manual_seed(2)
    inputs = {"uint8_240x320": torch.randint(0, 256, (B, T, 240, 320, 3), generator=g, dtype=torch.uint8).pin_memory(),
              "float_224": torch.randn(B, T, 3, 224, 224, generator=g).pin_memory()}

    def step(host):
        video = host.to(dev, non_blocking=True)
        out = model(input_ids=ids, pixel_values=video, attention_mask=mask)
        (out["image_embeds"].sum() + out["text_embeds"].sum()).backward()
        model.zero_grad(set_to_none=True)

    for name in inputs:
        for _ in range(warmup):
            step(inputs[name])
    times = {name: [] for name in inputs}
    for _ in range(steps):                      # alternate the two inputs so that both see the same host noise
        for name, host in inputs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(host)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3)
    res = {name: {"median_ms": round(sorted(t)[len(t) // 2], 2), "min_ms": round(min(t), 2),
                  "h2d_MB": round(inputs[name].numel() * inputs[name].element_size() / 1e6, 1)} for name, t in times.items()}
    del model
    torch.cuda.empty_cache()
    return res


def cpu_transform_ms(H, W, T=12, reps=5):
    from torchvision import transforms
    tf = transforms.Compose([transforms.Resize((224, 224), interpolation=transforms.InterpolationMode.BICUBIC,
                                               antialias=False),
                             transforms.CenterCrop((224, 224)),
                             transforms.Normalize(mean=(0.48145466, 0.4578275, 0.40821073),
                                                  std=(0.26862954, 0.26130258, 0.27577711))])
    frames = torch.randint(0, 256, (T, H, W, 3), dtype=torch.uint8)
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        tf(frames.permute(0, 3, 1, 2).float() / 255.)
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            tf(frames.permute(0, 3, 1, 2).float() / 255.)
            t.append((time.perf_counter() - t0) * 1e3)
    finally:
        torch.set_num_threads(threads)
    return round(sorted(t)[len(t) // 2], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    harness.require_gpu()
    dev = torch.device("cuda", 0)
    res = {"kernel": [kernel_time(dev, 240, 320), kernel_time(dev, 720, 1280)],
           "step_b64_t12": step_times(dev),
           "cpu_transform_ms_per_12_frame_sample_1_thread": {"240x320": cpu_transform_ms(240, 320),
                                                             "360x640": cpu_transform_ms(360, 640)}}
    line = harness.emit(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
