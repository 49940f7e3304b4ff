"""Timing of HD-VILA's TimeSformer with attention_type='joint_space_time' (depth 4, dim 1024, 16 heads) on one H100, and of
the dense attention kernel alone.

  model      fwd + bwd of the module at batch 16 on three grids (T x H x W = 8 x 7 x 7, 7 x 10 x 16, 8 x 28 x 28), CUDA-event
             timed, beside the pinned oracle in PyTorch eager under bf16 autocast on the same GPU (the batch is halved
             until the eager run fits in memory; the batch used is printed)
  attention  xp_dense_attention_* (TMA + wgmma) against xp_seg_attention_* run dense (seg_len = seq_len, the mma.sync kernel)
             at the same shapes, fwd and bwd, alternating the two kernels call by call; TF/s counts 4 N^2 d per head and
             sequence forward and 2.5 x that backward
Prints one JSON line per measurement, starting with the card's name, power limit and clocks.
A measurement tool: it executes oracle/ on purpose; nothing in the product imports it.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import timesformer_oracle as TO  # noqa: E402
from oracle import timesformer_variants_oracle as V  # noqa: E402
from tools import harness  # noqa: E402

GRIDS = ((8, 7, 7), (7, 10, 16), (8, 28, 28))


def model_bench(dev, B=16):
    from xpretrain_b200.modeling.timesformer import TimeSformer

    kind = 'joint_space_time'
    cfg = TO.TimeSformerCfg()
    sd = V.init_state_dict(cfg, kind, seed=0)
    model = TimeSformer(depth=cfg.depth, num_frames=cfg.num_frames, H=cfg.H, W=cfg.W, embed_dim=cfg.embed_dim,
                        num_heads=cfg.num_heads, drop_path_rate=0.0, attention_type=kind)
    model.load_state_dict(sd)
    model = model.to(dev).train()
    sdo = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
    for (T, H, W) in GRIDS:
        x = TO.synthetic_input(B, T, H, W, cfg, seed=1).to(dev).requires_grad_(True)
        w_out = torch.randn(B, T, cfg.embed_dim, H, W, device=dev) / (B * T * H * W) ** 0.5

        def ours():
            x.grad = None
            for p in model.parameters():
                p.grad = None
            (model(x) * w_out).sum().backward()

        ms = harness.window_ms(ours, 5, 2)
        fl = 3.0 * V.flops_per_sample(cfg, T, H, W, kind) * B
        rec = {"what": "joint model fwd+bwd", "grid_THW": [T, H, W], "batch": B, "ms": round(ms, 2),
               "clips_per_s": round(B / ms * 1e3, 1), "model_tflops": round(fl / ms / 1e9, 1)}
        be = B
        while be >= 1:
            xe = x[:be].detach()
            we = w_out[:be]

            def eager():
                xo = xe.detach().requires_grad_(True)
                for v in sdo.values():
                    v.grad = None
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    out = V.timesformer_forward(sdo, xo, cfg, kind)
                (out.float() * we).sum().backward()
            try:
                ms_e = harness.window_ms(eager, 3, 1)
                rec.update(eager_batch=be, eager_ms=round(ms_e, 2), eager_clips_per_s=round(be / ms_e * 1e3, 1))
                break
            except torch.OutOfMemoryError:
                torch.cuda.empty_cache()
                be //= 2
        if "eager_clips_per_s" in rec:
            rec["speedup_vs_eager"] = round(rec["clips_per_s"] / rec["eager_clips_per_s"], 2)
        harness.emit(rec)
        del x
        torch.cuda.empty_cache()


def attention_bench(dev, B=16, heads=16, rounds=3):
    from xpretrain_b200 import ops

    C = 64 * heads
    for (T, H, W) in GRIDS:
        N = T * H * W
        rows = B * N
        g = torch.Generator(device=dev).manual_seed(0)
        qkv = torch.randn(rows, 3 * C, device=dev, generator=g).to(torch.bfloat16)
        dout = torch.randn(rows, C, device=dev, generator=g).to(torch.bfloat16)
        out = torch.empty(rows, C, dtype=torch.bfloat16, device=dev)
        lse = torch.empty(heads, rows, device=dev)
        delta = torch.empty(heads, rows, device=dev)
        dqkv = torch.empty(rows, 3 * C, dtype=torch.bfloat16, device=dev)
        dd = ops.dense_desc(rows, heads, 3 * C, C, n_seq=B, seq_len=N)
        sd = ops.seg_desc(rows, heads, 3 * C, C, n_seq=B, seq_len=N, seg_len=N, inner=1, outer_stride=N,
                          inner_stride=0, tok_stride=1)
        kernels = {
            "dense_wgmma": (lambda: ops.dense_attention_fwd(qkv, out, lse, dd),
                            lambda: ops.dense_attention_bwd(qkv, out, dout, lse, delta, dqkv, dd, 0.125)),
            "seg_mma_sync": (lambda: ops.seg_attention_fwd(qkv, out, lse, sd),
                             lambda: ops.seg_attention_bwd(qkv, out, dout, lse, delta, dqkv, sd, 0.125)),
        }
        steps = max(2, int(2e12 // (4 * N * N * 64 * heads * B)) + 1)
        res = {k: {"fwd": [], "bwd": []} for k in kernels}
        for _ in range(rounds):                 # alternate the two kernels, call by call
            for name, (f, b) in kernels.items():
                f()
                res[name]["fwd"].append(harness.window_ms(f, steps, 1))
                res[name]["bwd"].append(harness.window_ms(b, steps, 1))
        fl = 4.0 * N * N * 64 * heads * B
        for name in kernels:
            fwd, bwd = min(res[name]["fwd"]), min(res[name]["bwd"])
            harness.emit({"what": "attention", "kernel": name, "grid_THW": [T, H, W], "N": N, "batch": B,
                          "heads": heads, "fwd_ms": round(fwd, 3), "fwd_tflops": round(fl / fwd / 1e9, 1),
                          "bwd_ms": round(bwd, 3), "bwd_tflops": round(2.5 * fl / bwd / 1e9, 1),
                          "fwd_ms_all": [round(v, 3) for v in res[name]["fwd"]],
                          "bwd_ms_all": [round(v, 3) for v in res[name]["bwd"]]})
        del qkv, dout, out, dqkv
        torch.cuda.empty_cache()


def main():
    harness.require_gpu()
    dev = torch.device("cuda", 0)
    harness.emit({})
    attention_bench(dev)
    model_bench(dev)


if __name__ == "__main__":
    main()
