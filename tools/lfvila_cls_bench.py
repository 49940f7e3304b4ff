"""Timing of LF-VILA's video classification model (coin_cls.yaml: released encoder, 180 labels) on one H100.

At the released geometry, 16 clips x 32 frames x 192 x 320 per GPU: the training step (forward + backward of the
cross-entropy loss, DropPath at the encoder's default 0.2) and its clips/s, no-grad evaluation clips/s, the peak memory of
each, the head's share of the step (the pool, projections, normalisations, classifier and loss, forward and backward, from
torch.profiler's kernel times), and beside it the reference algorithm in PyTorch eager (the pinned oracle, bf16 autocast) on
the same GPU at the largest batch that fits.  The card's name and power limit are read in the same run.  A measurement
tool: it executes oracle/ on purpose; nothing in the product imports it.

    python tools/lfvila_cls_bench.py [--batch 16] [--steps 5] [--warmup 2]
"""
import argparse
import json
import os
import sys
import tempfile
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import lfvila_cls_oracle as L  # noqa: E402
from oracle import swin3d_oracle as SO  # noqa: E402
from tools import harness  # noqa: E402

# the head's own kernels (pool, normalise, loss) by name; its GEMMs and column sums share kernels with the encoder, so the
# head's whole share is the step's kernel time minus the encoder's (head_ms)
HEAD_KERNELS = ("lfvila_",)


def head_ms(model, video, labels):
    """Device time of the head in one training step: the encoder alone (forward + backward of a weighted sum of its output)
    is subtracted from the whole step, both as sums of kernel times from torch.profiler."""
    enc_out = model.video_encoder(video)[0]
    w = torch.randn(enc_out.shape, device=video.device, dtype=enc_out.dtype)
    del enc_out

    def step():
        model.zero_grad(set_to_none=True)
        model(video, labels)["loss"].backward()

    def encoder():
        model.zero_grad(set_to_none=True)
        (model.video_encoder(video)[0] * w).sum().backward()

    total, named = harness.profiled_kernel_ms(step, HEAD_KERNELS)
    enc, _ = harness.profiled_kernel_ms(encoder)
    return total, enc, named


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--labels", type=int, default=180)
    a = ap.parse_args()
    harness.require_gpu()
    from xpretrain_b200.modeling import LFVILA_Video_Classification

    dev = torch.device("cuda", 0)
    cfg = SO.Swin3DCfg()
    B, D, H, W, n = a.batch, 32, 192, 320, a.labels
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "bert_large_config.json")
        with open(path, "w") as f:
            json.dump({"hidden_size": 1024}, f)
        enc = dict(patch_size=[1, 8, 8], embed_dim=128, depths=[2, 2, 14, 2, 2, 2], downsample_stages=[0, 1, 4],
                   stages=[0, 1, 2, 2, 2, 3], num_heads=[4, 8, 16, 16, 16, 32],
                   window_size=[[2, 3, 5], [4, 3, 5], [8, 3, 5], [16, 3, 5], [16, 3, 5], [32, 3, 5]], patch_norm=True,
                   local_window=8)
        model = LFVILA_Video_Classification(None, SimpleNamespace(VideoEncoder=enc, bert_config=path,
                                                                  DATA=SimpleNamespace(classification_labels=n)))
    sd = L.init_state_dict(cfg, n, seed=0)
    model.load_state_dict(sd)
    model = model.to(dev)
    video = SO.synthetic_video(B, D, H, W, cfg, seed=1).to(dev)
    labels = L.synthetic_labels(B, n).to(dev)

    def train_step():
        model.zero_grad(set_to_none=True)
        model(video, labels)["loss"].backward()

    def evaluate():
        with torch.no_grad():
            model(video, labels)

    model.train()
    ms_train = harness.window_ms(train_step, a.steps, a.warmup)
    _, peak_train = harness.peak_gib(train_step)
    model.eval()
    ms_eval = harness.window_ms(evaluate, a.steps, a.warmup)
    _, peak_eval = harness.peak_gib(evaluate)
    model.train()
    total, enc_ms, named = head_ms(model, video, labels)
    res = {"what": f"LFVILA_Video_Classification, coin_cls.yaml, {B} x 3 x {D} x {H} x {W}, {n} labels",
           "train_ms_per_step": round(ms_train, 2), "train_clips_per_s": round(B / ms_train * 1e3, 2),
           "train_peak_gib": round(peak_train, 2), "eval_ms": round(ms_eval, 2),
           "eval_clips_per_s": round(B / ms_eval * 1e3, 2), "eval_peak_gib": round(peak_eval, 2),
           "profiled_step_kernel_ms": round(total, 2), "profiled_encoder_kernel_ms": round(enc_ms, 2),
           "head_kernel_ms": round(total - enc_ms, 3), "head_share_of_step": round((total - enc_ms) / total, 4),
           "head_named_kernels_ms": round(named, 3)}
    harness.emit(res)
    del model
    torch.cuda.empty_cache()

    # the reference algorithm in eager PyTorch, bf16 autocast, at the largest batch (halving from B) that fits
    sdo = {k: (v.to(dev).requires_grad_(True) if v.is_floating_point() else v.to(dev)) for k, v in sd.items()}
    eb = B
    while eb >= 1:
        try:
            v = SO.synthetic_video(eb, D, H, W, cfg, seed=1).to(dev)
            lab = L.synthetic_labels(eb, n).to(dev)

            def eager():
                for t in sdo.values():
                    if t.is_floating_point():
                        t.grad = None
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    out = L.lfvila_cls_forward(sdo, v, lab, cfg)
                out["loss"].float().backward()
            ms_e = harness.window_ms(eager, max(2, a.steps // 2), 1)
            harness.emit({"what": "reference algorithm, eager PyTorch + bf16 autocast (oracle/lfvila_cls_oracle.py)",
                          "batch": eb, "train_ms_per_step": round(ms_e, 2),
                          "train_clips_per_s": round(eb / ms_e * 1e3, 2),
                          "speedup_clips_per_s": round((B / ms_train) / (eb / ms_e), 2)})
            break
        except torch.OutOfMemoryError:
            for t in sdo.values():
                if t.is_floating_point():
                    t.grad = None
            torch.cuda.empty_cache()
            eb //= 2


if __name__ == "__main__":
    main()
