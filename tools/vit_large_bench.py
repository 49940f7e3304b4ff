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
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from xpretrain_b200 import ops  # noqa: E402
from xpretrain_b200.modeling import VidCLIP  # noqa: E402
from xpretrain_b200.optimization.loss import gather_nce_loss  # noqa: E402

T, LT, M = 12, 32, 4
NAMES = {224: "openai/clip-vit-large-patch14", 336: "openai/clip-vit-large-patch14-336"}
GIB = 2 ** 30


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def attn_fwd_flops(H, T_, L, M_):
    return H * 4 * 64 * (T_ * L * (M_ + L) + M_ * (M_ + T_ * L))


def build_model(dev, size):
    add = SimpleNamespace(type="ViP", temporal_size=12, if_use_temporal_embed=1, logit_scale_init_value=4.60, add_cls_num=3)
    torch.manual_seed(0)
    model = VidCLIP(SimpleNamespace(clip_config=NAMES[size], clip_weights="", clip_vision_additional_config=add))
    with torch.no_grad():
        model.clipmodel.vision_model.embeddings.temporal_embedding.normal_(0, 0.02)
    return model.to(dev)


def inputs(dev, B, size):
    g = torch.Generator().manual_seed(1234)
    video = torch.randn(B, T, 3, size, size, generator=g)
    ids = torch.randint(1, 49406, (B, LT), generator=g)
    ids[:, -1] = 49407
    return video.to(dev), ids.to(dev), torch.ones(B, LT, dtype=torch.long, device=dev)


def step_fn(model, batch):
    cm = model.clipmodel
    params = list(model.parameters())

    def step():
        for p in params:
            p.grad = None
        out = model(video=batch[0], text_input_ids=batch[1], text_input_mask=batch[2])
        loss = gather_nce_loss(out["vis_features"], out["text_features"], cm.logit_scale)
        loss.backward()
        return loss
    return step


def time_step(model, B, size, steps, warmup):
    dev = next(model.parameters()).device
    batch = inputs(dev, B, size)
    step = step_fn(model, batch)
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
    peak = torch.cuda.max_memory_allocated()
    # GEMM rate: CUDA events around every GEMM launch of one more step (text tower on the main stream, so that kernels on
    # side streams are not charged each other's time)
    cm = model.clipmodel
    cm.overlap_text_tower = cm.overlap_colsum = False
    rec = []
    ops.set_gemm_timer(rec)
    step()
    torch.cuda.synchronize()
    ops.set_gemm_timer(None)
    cm.overlap_text_tower = cm.overlap_colsum = True
    g_ms = sum(a.elapsed_time(b) for (_, a, b) in rec)
    g_flops = sum(f for (f, _, _) in rec)
    return {"B": B, "ms_per_step": round(ms, 2), "pairs_per_s": round(B / ms * 1e3, 2), "peak_gib": round(peak / GIB, 2),
            "loss_finite": bool(torch.isfinite(loss).item()), "gemm_launches_per_step": len(rec),
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

    def timeit(fn):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    f_ms = timeit(lambda: ops.vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C))
    b_ms = timeit(lambda: ops.vip_attention_bwd(qkv, out, dout, lse, dqkv, ws, B, H, T, L, M, C, 0.125))
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
    dev = next(model.parameters()).device
    sdg = {k: (v.detach().clone().requires_grad_(True) if v.is_floating_point() else v)
           for k, v in model.clipmodel.state_dict().items()}
    video, ids, mask = inputs(dev, B, size)

    def step():
        for v in sdg.values():
            if v.is_floating_point():
                v.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            o = O.clip_vip_forward(sdg, video, ids, mask, ocfg)
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
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--b224", default="96,64,48,32")
    ap.add_argument("--b336", default="40,32,24,16")
    ap.add_argument("--eager-b224", type=int, default=4)
    ap.add_argument("--eager-b336", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("vit_large_bench.py needs a GPU")
    dev = torch.device("cuda", 0)
    ident = gpu_identity()
    print(json.dumps({"item": "gpu", **ident}), flush=True)
    cands = {224: [int(b) for b in args.b224.split(",")], 336: [int(b) for b in args.b336.split(",")]}
    eager_b = {224: args.eager_b224, 336: args.eager_b336}
    fitted = {}
    for size in (224, 336):
        model = build_model(dev, size)
        model.clipmodel.gradient_checkpointing_enable()
        model.train()
        res = None
        for B in cands[size]:
            try:
                res = time_step(model, B, size, args.steps, args.warmup)
                break
            except torch.OutOfMemoryError:
                torch.cuda.empty_cache()
                print(json.dumps({"item": f"step_{size}px", "B": B, "fits": False}), flush=True)
        fitted[size] = res["B"] if res else None
        print(json.dumps({"item": f"step_{size}px", "model": NAMES[size], "T": T, "text_tokens": LT, "checkpointing": True,
                          **(res or {"fits": False}), **ident}), flush=True)
        torch.cuda.empty_cache()
        model.clipmodel.gradient_checkpointing_disable()
        try:
            eager = time_eager(model, size, eager_b[size])
        except torch.OutOfMemoryError:
            eager = {"B": eager_b[size], "fits": False}
        print(json.dumps({"item": f"eager_autocast_{size}px", "what": "oracle forward + loss + backward, PyTorch eager, "
                          "bf16 autocast", "T": T, **eager, **ident}), flush=True)
        del model
        torch.cuda.empty_cache()
    for size, L in ((224, 256), (336, 576)):
        if fitted[size]:
            print(json.dumps({"item": f"attention_{size}px", **time_attention(dev, fitted[size], 16, L), **ident}), flush=True)
    print(json.dumps({"item": "attention_vit_b16_reference", **time_attention(dev, 64, 12, 196), **ident}), flush=True)


if __name__ == "__main__":
    main()
