"""Forward + backward time of every built contrastive loss (build_loss_func names) against the oracle restatement of the
same loss in eager PyTorch fp32 on the same GPU, plus kernel launches per call.  Prints one JSON line.

    python tools/loss_bench.py [--sizes 128,512,1024] [--dim 512] [--iters 200] [--warmup 20]
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import loss_family_oracle as LF  # noqa: E402
from tools import harness  # noqa: E402
from xpretrain_b200 import ops  # noqa: E402
from xpretrain_b200.optimization.loss import _LOSSES, build_loss_func  # noqa: E402

TEMP = 0.05


def features(name, N, d, dev):
    g = torch.Generator().manual_seed(N + d)
    n_args = 2 if name in ("NCEContrastiveLoss", "NCELearnableTempDSLLoss", "NCELearnableTempLoss") else 4
    base = F.normalize(torch.randn(N, d, generator=g), dim=-1)
    return [F.normalize(torch.randn(N, d, generator=g) + 0.5 * base, dim=-1).to(dev) for _ in range(n_args)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="128,512,1024")
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    harness.require_gpu()
    dev = torch.device("cuda", 0)
    rows = []
    for N in (int(x) for x in args.sizes.split(",")):
        for name in sorted(_LOSSES):
            feats = [f.requires_grad_(True) for f in features(name, N, args.dim, dev)]
            ls = torch.tensor(4.6, device=dev, requires_grad=True)
            fn = build_loss_func({"loss_name": name, "temp": TEMP})
            extra = [] if name == "NCEContrastiveLoss" else [ls]

            def ours():
                fn(*feats, *extra).backward()

            def eager():
                LF.nce_family_loss(name, feats, TEMP if name == "NCEContrastiveLoss" else ls).backward()

            ours()
            torch.cuda.synchronize()
            ops.reset_launch_count()
            ours()
            torch.cuda.synchronize()
            launches = ops.launch_count()
            t_ours = harness.window_ms(ours, args.iters, args.warmup)
            t_eager = harness.window_ms(eager, args.iters, args.warmup)
            rows.append({"loss": name, "N": N, "d": args.dim, "ours_ms": round(t_ours, 4), "eager_fp32_ms": round(t_eager, 4),
                         "speedup": round(t_eager / t_ours, 2), "launches_per_call": launches})
    harness.emit({"metric": "contrastive_loss_fwd_bwd_ms", "iters": args.iters, "warmup": args.warmup, "results": rows})


if __name__ == "__main__":
    main()
