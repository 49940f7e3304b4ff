"""LF-VILA's input transform on the GPU (xp_lfvila_frames_patchify_u8) against the reference's CPU transform.

  kernel   CUDA-event time of 16 clips x 32 frames from 360 x 640, 720 x 1280 and 1080 x 1920 into 192 x 320, for val
           and for train (train_crops), against the bytes-moved bound at the H100 SXM data sheet's 3.35 TB/s: the source
           rows the taps touch read once (stage A skips rows when it downscales by more than 2), the bf16 patch matrix
           written once
  model    LFVILA_Video_Classification (coin_cls.yaml: released encoder, 180 labels), 16 x 32 frames: training-step and
           no-grad evaluation clips/s fed uint8 360 x 640 frames (transformed on the GPU; train_crops drawn every step)
           against float 192 x 320 video already transformed, both resident on the GPU, alternated step by step
  cpu      the reference transform of one 32-frame clip (/255, then init_transform_dict's val or train Compose), one
           thread of this host's CPU, at 360 x 640 and 720 x 1280

    python tools/lfvila_frames_bench.py [--out lfvila_frames_bench.json]
Prints one JSON line; the card's name and power limit are read in the same run.  A measurement tool: it executes oracle/
on purpose; nothing in the product imports it.
"""
import argparse
import json
import os
import sys
import tempfile
import time
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import lfvila_cls_oracle as L  # noqa: E402
from oracle import lfvila_frames_ref as R  # noqa: E402
from oracle import swin3d_oracle as SO  # noqa: E402
from tools import harness  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
B, N, OUT = 16, 32, (192, 320)


def touched_bytes(crops, H, W):
    """Source bytes the kernel must read (rows any row tap touches, whole) + the bf16 patch matrix it writes."""
    rows = 0
    for top, left, h, w, flip in crops.params.tolist():
        idx, _ = R.composite_taps(H, crops.stage_a[0], top, h, OUT[0])
        rows += int(torch.unique(idx).numel())
    return rows * N * W * 3 + B * N * OUT[0] * OUT[1] * 3 * 2


def kernel_time(dev, H, W, mode, iters=20):
    from xpretrain_b200 import ops
    from xpretrain_b200.modeling import lfvila_frames as LF
    clips = torch.randint(0, 256, (B, N, H, W, 3), dtype=torch.uint8, device=dev)
    crops = LF.eval_crops(B) if mode == "val" else LF.train_crops(B, H, W, generator=torch.Generator().manual_seed(0))
    out = torch.empty(B * N * (OUT[0] // 8) * (OUT[1] // 8), 192, dtype=torch.bfloat16, device=dev)
    ms = harness.window_ms(lambda: ops.lfvila_frames_patchify_u8(clips, crops.params, crops.stage_a, OUT, out), iters, 3)
    nbytes = touched_bytes(crops, H, W)
    return {"mode": mode, "src": f"{H}x{W}", "frames": B * N, "ms": round(ms, 4), "input_MB": round(clips.numel() / 1e6, 1),
            "moved_MB": round(nbytes / 1e6, 1), "bound_ms": round(nbytes / HBM_BYTES_PER_S * 1e3, 4),
            "share_of_bound": round(nbytes / HBM_BYTES_PER_S * 1e3 / ms, 3)}


def model_rates(dev, steps=5, warmup=2, n=180):
    from xpretrain_b200.modeling import LFVILA_Video_Classification
    from xpretrain_b200.modeling import lfvila_frames as LF
    cfg = SO.Swin3DCfg()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "bert_large_config.json")
        with open(path, "w") as f:
            json.dump({"hidden_size": 1024}, f)
        enc = dict(patch_size=[1, 8, 8], embed_dim=128, depths=[2, 2, 14, 2, 2, 2], downsample_stages=[0, 1, 4],
                   stages=[0, 1, 2, 2, 2, 3], num_heads=[4, 8, 16, 16, 16, 32],
                   window_size=[[2, 3, 5], [4, 3, 5], [8, 3, 5], [16, 3, 5], [16, 3, 5], [32, 3, 5]], patch_norm=True,
                   local_window=8)
        model = LFVILA_Video_Classification(None, SimpleNamespace(
            VideoEncoder=enc, bert_config=path, DATA=SimpleNamespace(classification_labels=n, input_res=list(OUT))))
    model.load_state_dict(L.init_state_dict(cfg, n, seed=0))
    model = model.to(dev)
    labels = L.synthetic_labels(B, n).to(dev)
    inputs = {"uint8_360x640": torch.randint(0, 256, (B, N, 360, 640, 3), dtype=torch.uint8, device=dev),
              "float_192x320": SO.synthetic_video(B, N, *OUT, cfg, seed=1).to(dev)}

    def train(x):
        crops = LF.train_crops(B, 360, 640) if x.dtype == torch.uint8 else None
        model.zero_grad(set_to_none=True)
        model(x, labels, crops=crops)["loss"].backward()

    def evaluate(x):
        with torch.no_grad():
            model(x, labels)

    res = {}
    for phase, fn, train_mode in (("train", train, True), ("eval_no_grad", evaluate, False)):
        model.train(train_mode)
        for x in inputs.values():
            for _ in range(warmup):
                fn(x)
        times = {k: [] for k in inputs}
        for _ in range(steps):
            for k, x in inputs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(x)
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
        res[phase] = {k: {"median_ms": round(sorted(t)[len(t) // 2] * 1e3, 2),
                          "clips_per_s": round(B / sorted(t)[len(t) // 2], 1)} for k, t in times.items()}
    del model
    torch.cuda.empty_cache()
    return res


def cpu_transform_ms(H, W, mode, reps=3):
    from torchvision import transforms as T
    from xpretrain_b200 import ops
    norm = T.Normalize(ops.IMAGENET_MEAN, ops.IMAGENET_STD)
    if mode == "val":
        tf = T.Compose([T.Resize([240, 428], antialias=False), T.CenterCrop([216, 385]), T.Resize(list(OUT), antialias=False),
                        norm])
    else:
        tf = T.Compose([T.RandomResizedCrop(list(OUT), scale=(0.8, 1.0), antialias=False), T.RandomHorizontalFlip(),
                        T.ColorJitter(0, 0, 0), norm])
    frames = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8)
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        t = []
        for _ in range(reps + 1):
            t0 = time.perf_counter()
            tf((frames.float() / 255).permute(0, 3, 1, 2))       # video_classification_dataset.py:84-92
            t.append((time.perf_counter() - t0) * 1e3)
    finally:
        torch.set_num_threads(threads)
    t = sorted(t[1:])
    return round(t[len(t) // 2], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    harness.require_gpu()
    dev = torch.device("cuda", 0)
    res = {"kernel_16x32": [kernel_time(dev, H, W, mode) for H, W in ((360, 640), (720, 1280), (1080, 1920))
                            for mode in ("val", "train")],
           "model_16x32_180_labels": model_rates(dev),
           "cpu_transform_ms_per_32_frame_clip_1_thread": {f"{mode} {H}x{W}": cpu_transform_ms(H, W, mode)
                                                           for H, W in ((360, 640), (720, 1280)) for mode in ("val", "train")}}
    line = harness.emit(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
