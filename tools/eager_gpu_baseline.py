"""PyTorch-eager GPU baseline for the bench workload (BASELINE.md §3 "same-box GPU eager baseline").

The reference itself is not needed on the GPU machine: this times its pinned restatement
(oracle/clipvip_oracle.py: the same torch ops in the same order as CLIP_ViP.py / loss.py) on the H100 under
torch.autocast(bfloat16) — the reference cannot run `.to(bfloat16)` (SURVEY.md §8c), autocast is its working
bf16 mode.  fwd + InfoNCE + bwd, CUDA-event timed, B = 64 (falls back to 32 / 16 if eager runs out of memory).
This is a measurement tool (it executes oracle/ on purpose); nothing in the product imports it.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import clipvip_oracle as O  # noqa: E402
from tools import harness  # noqa: E402


def run(B, steps=5, warmup=2):
    dev = torch.device("cuda", 0)
    cfg = O.ClipVipCfg()
    sd = {k: (v.to(dev).requires_grad_(True) if v.is_floating_point() else v.to(dev))
          for k, v in O.init_state_dict(cfg, seed=0).items()}
    video, ids, mask = O.synthetic_batch(B, 12, 32, cfg, seed=1234)
    video, ids, mask = video.to(dev), ids.to(dev), mask.to(dev)

    def step():
        for v in sd.values():
            if v.is_floating_point():
                v.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = O.clip_vip_forward(sd, video, ids, mask, cfg)
            loss = O.nce_learnable_temp_loss(out["vis_features"].float(), out["text_features"].float(), sd["logit_scale"])
        loss.backward()
        return loss

    ms, peak = harness.peak_gib(lambda: harness.window_ms(step, steps, warmup))
    return {"impl": "pytorch-eager (oracle port of the reference) under bf16 autocast", "batch": B, "ms_per_step": round(ms, 2),
            "pairs_per_s": round(B / ms * 1e3, 2), "max_mem_gb": round(peak, 1)}


def main():
    harness.require_gpu()
    for B in (64, 32, 16):
        try:
            harness.emit(run(B))
            break
        except torch.OutOfMemoryError:
            harness.emit({"batch": B, "error": "out of memory in eager"})
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
