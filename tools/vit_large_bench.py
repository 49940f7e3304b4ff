"""CLIP-ViP with ViT-L/14 towers on one GPU: the training step (forward + fused gather_nce_loss + backward, gradient
checkpointing on, 12 frames, 32 text tokens) at 224 px (openai/clip-vit-large-patch14, L = 256 patches per frame) and at
336 px (openai/clip-vit-large-patch14-336, L = 576).  Prints one JSON line per item:

  1. the GPU's name, power limit and maximum SM clock, read in the same call as the timings;
  2. per resolution, the largest batch of the candidates that fits: ms per step (CUDA events after warm-up), pairs/s,
     peak memory, and the GEMM rate of one step (CUDA events around every xp_gemm launch, FLOPs from the shapes);
  3. the proxy-token attention kernels alone at each step's shape and, as a reference rate, the staged kernel at the
     ViT-B/16 shape (B = 64, 12 heads, L = 196): forward and backward ms per layer, with FLOPs from the shapes
     (forward per head: 4 * 64 * (T * L * (M + L) + M * (M + T * L)); 1.474 GFLOP per (sample, layer) for B/16,
     3.32 for L/14 at 224 px, 16.5 at 336 px; backward counted as 2.5 x forward);
  4. the oracle (oracle/clipvip_oracle.py, the reference algorithm in PyTorch eager) under bf16 autocast at a small
     batch, as the eager comparison.

    python tools/vit_large_bench.py [--steps 4] [--warmup 2] [--b224 96,64,48,32] [--b336 40,32,24,16]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import harness  # noqa: E402
from xpretrain_b200 import ops  # noqa: E402

T, LT, M = 12, 32, 4
NAMES = {224: "openai/clip-vit-large-patch14", 336: "openai/clip-vit-large-patch14-336"}


def attn_fwd_flops(H, T_, L, M_):
    return H * 4 * 64 * (T_ * L * (M_ + L) + M_ * (M_ + T_ * L))


def time_step(model, B, size, steps, warmup):
    dev = next(model.parameters()).device
    batch = harness.clip_batch(dev, B, T, size, LT)
    last = {}

    def step():
        last["loss"], _ = harness.clip_train_step(model, batch)

    torch.cuda.empty_cache()
    ms, peak = harness.peak_gib(lambda: harness.window_ms(step, steps, warmup))
    # GEMM rate: CUDA events around every GEMM launch of one more step (text tower on the main stream, so that kernels on
    # side streams are not charged each other's time)
    cm = model.clipmodel
    cm.overlap_text_tower = cm.overlap_colsum = False
    rec = []
    ops.set_gemm_timer(rec)
    harness.clip_train_step(model, batch)
    torch.cuda.synchronize()
    ops.set_gemm_timer(None)
    cm.overlap_text_tower = cm.overlap_colsum = True
    g_ms = sum(a.elapsed_time(b) for (_, a, b) in rec)
    g_flops = sum(f for (f, _, _) in rec)
    return {"B": B, "ms_per_step": round(ms, 2), "pairs_per_s": round(B / ms * 1e3, 2), "peak_gib": round(peak, 2),
            "loss_finite": bool(torch.isfinite(last["loss"]).item()), "gemm_launches_per_step": len(rec),
            "gemm_ms_per_step": round(g_ms, 2), "gemm_tflops": round(g_flops / (g_ms * 1e-3) / 1e12, 1) if g_ms > 0 else None}


def time_attention(dev, B, H, L, iters=10):
    C, S = 64 * H, M + T * L
    g = torch.Generator(device="cpu").manual_seed(0)
    qkv = (torch.randn(B * S, 3 * C, generator=g) * 0.8).to(dev).to(torch.bfloat16)
    qkv[:, :C] *= 0.35
    out = torch.empty(B * S, C, dtype=torch.bfloat16, device=dev)
    dout = torch.randn(B * S, C, generator=g).to(dev).to(torch.bfloat16)
    lse = torch.empty(B, H, S, device=dev)
    dqkv = torch.empty(B * S, 3 * C, dtype=torch.bfloat16, device=dev)
    ws = ops.vip_attention_workspace(B, H, T, M, dev)
    f_ms = harness.window_ms(lambda: ops.vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C), iters, 3)
    b_ms = harness.window_ms(lambda: ops.vip_attention_bwd(qkv, out, dout, lse, dqkv, ws, B, H, T, L, M, C, 0.125), iters, 3)
    ff = attn_fwd_flops(H, T, L, M) * B
    return {"B": B, "H": H, "T": T, "L": L, "M": M, "kernel": "staged" if M + L <= 208 else "streamed",
            "gflop_fwd_per_sample_layer": round(attn_fwd_flops(H, T, L, M) / 1e9, 3),
            "fwd_ms_per_layer": round(f_ms, 3), "bwd_ms_per_layer": round(b_ms, 3),
            "fwd_tflops": round(ff / f_ms / 1e9, 1), "bwd_tflops": round(2.5 * ff / b_ms / 1e9, 1)}


def time_eager(model, size, B, steps=2):
    """The oracle's forward + loss + backward in PyTorch eager under bf16 autocast, fp32 weights (the reference's mixed
    precision), on the same weights."""
    from oracle import clipvip_oracle as O
    cfg = model.clipmodel.config
    ocfg = O.ClipVipCfg(vision=O.TowerCfg(1024, 16, cfg.vision.num_hidden_layers, 4096),
                        text=O.TowerCfg(768, 12, cfg.text.num_hidden_layers, 3072), image_size=size, patch=14, proj_dim=768)
    batch = harness.clip_batch(next(model.parameters()).device, B, T, size, LT)
    step = harness.eager_oracle_step(model, batch, lambda sd, video, ids, mask: O.clip_vip_forward(sd, video, ids, mask, ocfg))
    torch.cuda.empty_cache()
    ms, peak = harness.peak_gib(lambda: harness.window_ms(step, steps, 1))
    return {"B": B, "ms_per_step": round(ms, 1), "pairs_per_s": round(B / ms * 1e3, 2), "peak_gib": round(peak, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--b224", default="96,64,48,32")
    ap.add_argument("--b336", default="40,32,24,16")
    ap.add_argument("--eager-b224", type=int, default=4)
    ap.add_argument("--eager-b336", type=int, default=2)
    args = ap.parse_args()
    harness.require_gpu()
    dev = torch.device("cuda", 0)
    harness.emit({"item": "gpu"})
    cands = {224: [int(b) for b in args.b224.split(",")], 336: [int(b) for b in args.b336.split(",")]}
    eager_b = {224: args.eager_b224, 336: args.eager_b336}
    fitted = {}
    for size in (224, 336):
        model = harness.clip_model(dev, NAMES[size], seed_temporal=True)
        model.clipmodel.gradient_checkpointing_enable()
        model.train()
        res = None
        for B in cands[size]:
            try:
                res = time_step(model, B, size, args.steps, args.warmup)
                break
            except torch.OutOfMemoryError:
                torch.cuda.empty_cache()
                harness.emit({"item": f"step_{size}px", "B": B, "fits": False})
        fitted[size] = res["B"] if res else None
        harness.emit({"item": f"step_{size}px", "model": NAMES[size], "T": T, "text_tokens": LT, "checkpointing": True,
                      **(res or {"fits": False})})
        torch.cuda.empty_cache()
        model.clipmodel.gradient_checkpointing_disable()
        try:
            eager = time_eager(model, size, eager_b[size])
        except torch.OutOfMemoryError:
            eager = {"B": eager_b[size], "fits": False}
        harness.emit({"item": f"eager_autocast_{size}px", "what": "oracle forward + loss + backward, PyTorch eager, "
                      "bf16 autocast", "T": T, **eager})
        del model
        torch.cuda.empty_cache()
    for size, L in ((224, 256), (336, 576)):
        if fitted[size]:
            harness.emit({"item": f"attention_{size}px", **time_attention(dev, fitted[size], 16, L)})
    harness.emit({"item": "attention_vit_b16_reference", **time_attention(dev, 64, 12, 196)})


if __name__ == "__main__":
    main()
