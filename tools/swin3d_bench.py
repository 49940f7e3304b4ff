"""Timing of BASELINE.json config #5 (LF-VILA Swin-3D video encoder, released VideoEncoder config) on one H100.

fwd + bwd of the module (synthetic video, a weighted-sum loss, DropPath off), CUDA-event timed, at BASELINE.json's
[8,3,32,224,224] and the reference-native 192x320; beside it the reference algorithm in PyTorch eager (the pinned oracle, bf16
autocast) on the same GPU.  A measurement tool: it executes oracle/ on purpose; nothing in the product imports it.

    python tools/swin3d_bench.py [--graph]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import swin3d_oracle as SO  # noqa: E402
from tools import harness  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graph", action="store_true", help="also time the step replayed from CUDA graphs")
    args = ap.parse_args()
    harness.require_gpu()
    from xpretrain_b200.modeling.swin3d import SwinTransformer3D

    dev = torch.device("cuda", 0)
    cfg = SO.Swin3DCfg()
    sd = SO.init_state_dict(cfg, seed=0)
    model = SwinTransformer3D(patch_norm=True, local_window=8, drop_path_rate=0.0)
    model.load_state_dict(sd)
    model = model.to(dev).train()
    sdo = {k: (v.to(dev).requires_grad_(True) if v.is_floating_point() else v.to(dev)) for k, v in sd.items()}
    peak = 989.0          # NVIDIA H100 SXM data sheet, dense bf16 (a 700 W card); MEASURED_PEAKS.json overrides it
    try:
        with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")) as f:
            peak = float(json.load(f).get("bf16_tflops_sustained", peak))
    except (OSError, ValueError):
        pass
    for (B, D, H, W, what) in ((8, 32, 224, 224, "BASELINE.json config #5: 8 x 32 frames x 224^2 (windows padded 28->30)"),
                               (8, 32, 192, 320, "reference-native 192x320 (no window padding)")):
        video = SO.synthetic_video(B, D, H, W, cfg, seed=1).to(dev)
        with torch.no_grad():
            shape = model.eval()(video)[0].shape
        model.train()
        w_out = torch.randn(shape, device=dev) / (shape[1] * shape[2] * shape[3] * shape[4]) ** 0.5

        def ours():
            for p in model.parameters():
                p.grad = None
            (model(video)[0] * w_out).sum().backward()

        def eager():
            for v in sdo.values():
                if v.is_floating_point():
                    v.grad = None
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = SO.swin3d_forward(sdo, video, cfg)
            (out.float() * w_out).sum().backward()

        ms = harness.window_ms(ours, 5, 2)
        ms_graph, graph_note = None, None
        if args.graph:
            # the 24 blocks issue ~1300 small launches per step: replay them from CUDA graphs (torch.cuda.make_graphed_callables
            # captures this module's forward and backward, all launched on the capture stream through the C ABI)
            class First(torch.nn.Module):
                def __init__(self, m):
                    super().__init__()
                    self.m = m

                def forward(self, v):
                    return self.m(v)[0]
            try:
                gm = torch.cuda.make_graphed_callables(First(model), (video,), num_warmup_iters=3, allow_unused_input=True)

                def graphed():
                    for p in model.parameters():
                        p.grad = None
                    (gm(video) * w_out).sum().backward()
                ref_out = model(video)[0].detach()
                got = gm(video).detach()
                graph_note = f"graphed output rel diff {float((got - ref_out).norm() / ref_out.norm()):.1e}"
                ms_graph = harness.window_ms(graphed, 5, 2)
            except Exception as exc:  # noqa: BLE001 - report, do not hide
                graph_note = f"capture failed: {type(exc).__name__}: {str(exc)[:200]}"
        try:
            ms_e = harness.window_ms(eager, 3, 1)
        except torch.OutOfMemoryError:
            ms_e = None
            torch.cuda.empty_cache()
        fl = 3.0 * SO.flops_per_sample(cfg, D, H, W) * B
        harness.emit({"shape": [B, 3, D, H, W], "what": what, "ms_fwd_bwd": round(ms, 3),
                      "samples_per_s": round(B / ms * 1e3, 1), "tflops": round(fl / ms / 1e9, 1),
                      "frac_of_sustained_peak": round(fl / ms / 1e9 / peak, 3),
                      "cuda_graph_ms": None if ms_graph is None else round(ms_graph, 3), "cuda_graph_note": graph_note,
                      "eager_bf16_ms": None if ms_e is None else round(ms_e, 3),
                      "speedup_vs_eager": None if ms_e is None else round(ms_e / ms, 2)})


if __name__ == "__main__":
    main()
