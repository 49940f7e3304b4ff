"""The per-frame CLIP video model (vision_additional_config.type != "ViP") against the CLIP-ViP model on one GPU: the
training step (forward + fused gather_nce_loss + backward) at B = 64 videos x 12 frames at 224 px with 32 text tokens,
openai/clip-vit-base-patch16 widths.  Prints one JSON line per item:

  1. the GPU's name, power limit and maximum SM clock, read in the same call as the timings;
  2. per round, the per-frame model and the ViP model timed one after the other (the rounds alternate the two, so that a
     clock or power change on a shared GPU affects both): ms per step (CUDA events after warm-up), pairs/s, peak memory;
  3. the oracle (oracle/frame_clip_oracle.py, the reference algorithm in PyTorch eager) under bf16 autocast at the
     largest of the candidate batches that fits, as the eager comparison.

    python tools/frame_clip_bench.py [--steps 5] [--warmup 2] [--rounds 2] [--batch 64] [--checkpointing]
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from xpretrain_b200.modeling import VidCLIP  # noqa: E402
from xpretrain_b200.optimization.loss import gather_nce_loss  # noqa: E402

T, LT, SIZE = 12, 32, 224
GIB = 2 ** 30


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def build_model(dev, kind):
    add = SimpleNamespace(type=kind, temporal_size=12, if_use_temporal_embed=1, logit_scale_init_value=4.60, add_cls_num=3)
    torch.manual_seed(0)
    model = VidCLIP(SimpleNamespace(clip_config="openai/clip-vit-base-patch16", clip_weights="",
                                    clip_vision_additional_config=add))
    return model.to(dev)


def inputs(dev, B):
    g = torch.Generator().manual_seed(1234)
    video = torch.randn(B, T, 3, SIZE, SIZE, generator=g)
    ids = torch.randint(1, 49406, (B, LT), generator=g)
    ids[:, -1] = 49407
    return video.to(dev), ids.to(dev), torch.ones(B, LT, dtype=torch.long, device=dev)


def time_step(model, batch, steps, warmup):
    cm = model.clipmodel
    params = list(model.parameters())

    def step():
        for p in params:
            p.grad = None
        out = model(video=batch[0], text_input_ids=batch[1], text_input_mask=batch[2])
        loss = gather_nce_loss(out["vis_features"], out["text_features"], cm.logit_scale)
        loss.backward()
        return loss

    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(warmup):
        loss = step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    B = batch[0].shape[0]
    return {"B": B, "ms_per_step": round(ms, 2), "pairs_per_s": round(B / ms * 1e3, 2),
            "peak_gib": round(torch.cuda.max_memory_allocated() / GIB, 2), "loss_finite": bool(torch.isfinite(loss).item())}


def time_eager(model, B, steps=2):
    """The oracle's forward + loss + backward in PyTorch eager under bf16 autocast, fp32 weights, on the same weights."""
    from oracle import clipvip_oracle as O
    from oracle import frame_clip_oracle as F
    dev = next(model.parameters()).device
    sdg = {k: (v.detach().clone().requires_grad_(True) if v.is_floating_point() else v)
           for k, v in model.clipmodel.state_dict().items()}
    video, ids, mask = inputs(dev, B)
    ocfg = O.ClipVipCfg()

    def step():
        for v in sdg.values():
            if v.is_floating_point():
                v.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            o = F.frame_clip_forward(sdg, video, ids, mask, ocfg)
            loss = O.nce_learnable_temp_loss(o["vis_features"].float(), o["text_features"].float(), sdg["logit_scale"].float())
        loss.backward()

    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return {"B": B, "ms_per_step": round(ms, 1), "pairs_per_s": round(B / ms * 1e3, 2),
            "peak_gib": round(torch.cuda.max_memory_allocated() / GIB, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--checkpointing", action="store_true")
    ap.add_argument("--eager-batches", default="32,16,8,4,2")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("frame_clip_bench.py needs a GPU")
    dev = torch.device("cuda", 0)
    ident = gpu_identity()
    print(json.dumps({"item": "gpu", **ident}), flush=True)
    models = {"per_frame": build_model(dev, "meanP"), "vip": build_model(dev, "ViP")}
    for m in models.values():
        if args.checkpointing:
            m.clipmodel.gradient_checkpointing_enable()
        m.train()
    batch = inputs(dev, args.batch)
    for r in range(args.rounds):
        for kind, model in models.items():
            res = time_step(model, batch, args.steps, args.warmup)
            print(json.dumps({"item": "step", "model": kind, "round": r, "T": T, "text_tokens": LT,
                              "checkpointing": args.checkpointing, **res, **ident}), flush=True)
    vip = models.pop("vip")
    del vip, batch
    torch.cuda.empty_cache()
    model = models["per_frame"]
    eager = None
    for B in (int(b) for b in args.eager_batches.split(",")):
        try:
            eager = time_eager(model, B)
            break
        except torch.OutOfMemoryError:
            torch.cuda.empty_cache()
    print(json.dumps({"item": "eager_autocast", "what": "per-frame oracle forward + loss + backward, PyTorch eager, bf16 "
                      "autocast", "T": T, **(eager or {"fits": False}), **ident}), flush=True)


if __name__ == "__main__":
    main()
