"""CLIP-ViP training step (forward + fused gather_nce_loss + backward, ViT-B/16, 12 + 12 layers, 32 text tokens) with
gradient checkpointing off and on.  Prints one JSON line per case:

  1. B = 64, T = 12: off and on alternately, twice each; ms per step (CUDA events), pairs/s, peak memory, and the loss,
     features and gradients of the last step of each mode compared against each other.
  2. B = 128, T = 12, checkpointing on.
  3. B = 64, T = 32 (the ActivityNet frame count), checkpointing on.

For each case the activations saved for the backward are also predicted from the shapes, with and without checkpointing;
cases 2 and 3 are not run without checkpointing (they do not fit in 80 GB).

    python tools/checkpoint_bench.py [--steps 5] [--warmup 2]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import harness  # noqa: E402

LT = 32


def saved_bytes(cfg, B, T, Lt, ckpt):
    """Bytes a training forward keeps for the backward (fp32 residual stream), from the shapes."""
    C, I, H, n = cfg.vision.hidden_size, cfg.vision.intermediate_size, cfg.vision.num_attention_heads, cfg.vision.num_hidden_layers
    L, M = cfg.num_patches, 1 + cfg.add_cls_num
    rows = B * (M + T * L)
    # per block: x, h, qkv, a, x1, h2 (4+2+6+2+4+2 = 20 B per channel), fc1 pre-activation and output, LN statistics, LSE
    block = rows * 4 * C if ckpt else rows * (20 * C + 4 * I + 16 + 4 * H)
    vis = n * block + B * T * L * 3 * cfg.patch_size ** 2 * 2 + rows * (2 * C + 8 + 6 * C) + B * H * T * M * 3 * 64 * 4
    Ct, It, Ht, nt = cfg.text.hidden_size, cfg.text.intermediate_size, cfg.text.num_attention_heads, cfg.text.num_hidden_layers
    rt = B * Lt
    tblock = rt * 4 * Ct if ckpt else rt * (20 * Ct + 4 * It + 16) + B * Ht * Lt * Lt * 4
    return vis + nt * tblock + rt * 6 * Ct


def run(model, batch, ckpt, steps, warmup):
    """(ms per step, peak GiB above the allocation before the first step, outputs of the last step)."""
    cm = model.clipmodel
    (cm.gradient_checkpointing_enable if ckpt else cm.gradient_checkpointing_disable)()
    last = {}

    def step():
        loss, out = harness.clip_train_step(model, batch)
        last.update(loss=loss.detach(), vis=out["vis_features"].detach(), txt=out["text_features"].detach())

    for p in model.parameters():
        p.grad = None
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    ms, peak = harness.peak_gib(lambda: harness.window_ms(step, steps, warmup))
    last["grads"] = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    cm.gradient_checkpointing_disable()
    return ms, peak - base / harness.GIB, last


def compare(a, b):
    """Loss and features must be equal; gradients differ by the order of fp32 atomics.  Each gradient's largest difference is
    taken relative to its largest value, k_proj.bias's relative to its layer's q/k/v bias (its exact value is zero, so its own
    largest value is rounding residue)."""
    ga, worst, at = a["grads"], 0.0, None
    for n, g in ga.items():
        names = [n.replace("k_proj", p) for p in ("q_proj", "k_proj", "v_proj")] if n.endswith("k_proj.bias") else [n]
        scale = max(float(ga[m].abs().max()) for m in names)
        if scale > 0 and float((b["grads"][n] - g).abs().max()) / scale > worst:
            worst, at = float((b["grads"][n] - g).abs().max()) / scale, n
    return {"loss_equal": bool(torch.equal(a["loss"], b["loss"])), "vis_features_equal": bool(torch.equal(a["vis"], b["vis"])),
            "text_features_equal": bool(torch.equal(a["txt"], b["txt"])), "grad_max_rel_diff": worst, "at": at}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    harness.require_gpu()
    dev = torch.device("cuda", 0)
    model = harness.clip_model(dev, "openai/clip-vit-base-patch16", seed_temporal=True)
    cfg = model.clipmodel.config
    gib = harness.GIB

    B, T = 64, 12
    batch = harness.clip_batch(dev, B, T, 224, LT)
    res = {"off": [], "on": []}
    outs = {}
    for mode in ("off", "on", "off", "on"):
        ms, peak, last = run(model, batch, mode == "on", args.steps, args.warmup)
        res[mode].append({"ms_per_step": round(ms, 2), "pairs_per_s": round(B / ms * 1e3, 1), "peak_gib": round(peak, 2)})
        outs.setdefault(mode, []).append(last)
    cmp_modes = compare(outs["off"][-1], outs["on"][-1])
    cmp_runs = compare(outs["off"][0], outs["off"][-1])      # the same mode twice: the run-to-run spread of the atomics
    del outs
    harness.emit({"case": "B64_T12_off_vs_on", "B": B, "T": T, "runs": res,
                  "predicted_saved_gib": {"off": round(saved_bytes(cfg, B, T, LT, False) / gib, 2),
                                          "on": round(saved_bytes(cfg, B, T, LT, True) / gib, 2)},
                  "off_vs_on": cmp_modes, "off_vs_off": cmp_runs})
    del batch

    for B, T in ((128, 12), (64, 32)):
        batch = harness.clip_batch(dev, B, T, 224, LT)
        ms, peak, last = run(model, batch, True, args.steps, args.warmup)
        finite = bool(torch.isfinite(last["loss"]).item()) and all(bool(torch.isfinite(g).all()) for g in last["grads"].values())
        del last, batch
        harness.emit({"case": f"B{B}_T{T}_on", "B": B, "T": T, "ms_per_step": round(ms, 2),
                      "pairs_per_s": round(B / ms * 1e3, 1), "peak_gib": round(peak, 2), "finite": finite,
                      "predicted_saved_gib": {"off": round(saved_bytes(cfg, B, T, LT, False) / gib, 2),
                                              "on": round(saved_bytes(cfg, B, T, LT, True) / gib, 2)}})


if __name__ == "__main__":
    main()
