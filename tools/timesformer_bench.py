"""Timing of BASELINE.json config #4 (HD-VILA TimeSformer, depth 4, dim 1024, 16 heads) on one H100.

fwd + bwd of the module (synthetic feature maps, a weighted-sum loss), CUDA-event timed, for the three shapes BASELINE.md §2
lists; beside it the reference algorithm in PyTorch eager (the pinned oracle, bf16 autocast) on the same GPU.
A measurement tool: it executes oracle/ on purpose; nothing in the product imports it.
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import timesformer_oracle as TO  # noqa: E402
from tools import harness  # noqa: E402


def main():
    harness.require_gpu()
    from xpretrain_b200.modeling.timesformer import TimeSformer

    dev = torch.device("cuda", 0)
    cfg = TO.TimeSformerCfg()
    sd = TO.init_state_dict(cfg, seed=0)
    model = TimeSformer(depth=cfg.depth, num_frames=cfg.num_frames, H=cfg.H, W=cfg.W, embed_dim=cfg.embed_dim,
                        num_heads=cfg.num_heads, drop_path_rate=0.0)
    model.load_state_dict(sd)
    model = model.to(dev).train()
    sdo = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
    peak = 989.0          # NVIDIA H100 SXM data sheet, dense bf16 (a 700 W card); MEASURED_PEAKS.json overrides it
    try:
        with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")) as f:
            mp = json.load(f)
        peak = float(mp.get("bf16_tflops_sustained", mp.get("bf16_dense_tflops_sustained", peak)))
    except (OSError, ValueError):
        pass
    for (B, T, H, W, what) in ((16, 7, 10, 16, "reference-native grid, 8 videos x 2 clips"),
                               (16, 8, 7, 7, "config #4: 8 frames x 448^2 -> 7x7 grid (both interpolations)"),
                               (4, 8, 28, 28, "stress grid 28x28")):
        x = TO.synthetic_input(B, T, H, W, cfg, seed=1).to(dev).requires_grad_(True)
        w_out = torch.randn(B, T, cfg.embed_dim, H, W, device=dev) / (B * T * H * W) ** 0.5

        def ours():
            x.grad = None
            for p in model.parameters():
                p.grad = None
            (model(x) * w_out).sum().backward()

        def eager():
            xo = x.detach().requires_grad_(True)
            for v in sdo.values():
                v.grad = None
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = TO.timesformer_forward(sdo, xo, cfg)
            (out.float() * w_out).sum().backward()

        ms = harness.window_ms(ours, 10, 3)
        ms_e = harness.window_ms(eager, 5, 2)
        fl = 3.0 * TO.flops_per_sample(cfg, T, H, W) * B
        harness.emit({"shape": [B, T, cfg.embed_dim, H, W], "what": what, "ms_fwd_bwd": round(ms, 3),
                      "samples_per_s": round(B / ms * 1e3, 1), "tflops": round(fl / ms / 1e9, 1),
                      "frac_of_sustained_peak": round(fl / ms / 1e9 / peak, 3),
                      "eager_bf16_ms": round(ms_e, 3), "speedup_vs_eager": round(ms_e / ms, 2)})


if __name__ == "__main__":
    main()
