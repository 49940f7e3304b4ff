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
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import harness  # noqa: E402

T, LT, SIZE = 12, 32, 224
NAME = "openai/clip-vit-base-patch16"


def time_step(model, batch, steps, warmup):
    last = {}

    def step():
        last["loss"], _ = harness.clip_train_step(model, batch)

    torch.cuda.empty_cache()
    ms, peak = harness.peak_gib(lambda: harness.window_ms(step, steps, warmup))
    B = batch[0].shape[0]
    return {"B": B, "ms_per_step": round(ms, 2), "pairs_per_s": round(B / ms * 1e3, 2),
            "peak_gib": round(peak, 2), "loss_finite": bool(torch.isfinite(last["loss"]).item())}


def time_eager(model, B, steps=2):
    """The oracle's forward + loss + backward in PyTorch eager under bf16 autocast, fp32 weights, on the same weights."""
    from oracle import clipvip_oracle as O
    from oracle import frame_clip_oracle as F
    ocfg = O.ClipVipCfg()
    batch = harness.clip_batch(next(model.parameters()).device, B, T, SIZE, LT)
    step = harness.eager_oracle_step(model, batch, lambda sd, video, ids, mask: F.frame_clip_forward(sd, video, ids, mask, ocfg))
    torch.cuda.empty_cache()
    ms, peak = harness.peak_gib(lambda: harness.window_ms(step, steps, 1))
    return {"B": B, "ms_per_step": round(ms, 1), "pairs_per_s": round(B / ms * 1e3, 2), "peak_gib": round(peak, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--checkpointing", action="store_true")
    ap.add_argument("--eager-batches", default="32,16,8,4,2")
    args = ap.parse_args()
    harness.require_gpu()
    dev = torch.device("cuda", 0)
    harness.emit({"item": "gpu"})
    models = {"per_frame": harness.clip_model(dev, NAME, "meanP"), "vip": harness.clip_model(dev, NAME)}
    for m in models.values():
        if args.checkpointing:
            m.clipmodel.gradient_checkpointing_enable()
        m.train()
    batch = harness.clip_batch(dev, args.batch, T, SIZE, LT)
    for r in range(args.rounds):
        for kind, model in models.items():
            res = time_step(model, batch, args.steps, args.warmup)
            harness.emit({"item": "step", "model": kind, "round": r, "T": T, "text_tokens": LT,
                          "checkpointing": args.checkpointing, **res})
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
    harness.emit({"item": "eager_autocast", "what": "per-frame oracle forward + loss + backward, PyTorch eager, bf16 "
                  "autocast", "T": T, **(eager or {"fits": False})})


if __name__ == "__main__":
    main()
