"""CUDA-event timing of the window-attention kernels (config #5) at the per-stage shapes of the released LF-VILA VideoEncoder
for a batch of 8 x 32 frames x 192 x 320:  (windows, L, heads)  =  (8192, 30, 4)  (1024, 60, 8)  (128, 120, 16)  (64, 240, 16)
(8, 480, 32).  Mean over 10 back-to-back calls after 3; one JSON line per stage.   python tools/winattn_bench.py [stage]"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import harness  # noqa: E402
from xpretrain_b200 import ops  # noqa: E402

STAGES = [(8192, 30, 4), (1024, 60, 8), (128, 120, 16), (64, 240, 16), (8, 480, 32)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("stage", nargs="?", type=int, default=None, help="time this stage only")
    only = ap.parse_args().stage
    harness.require_gpu()
    dev = torch.device("cuda", 0)
    bf16 = torch.bfloat16
    for si, (n_win, L, heads) in enumerate(STAGES):
        if only is not None and si != only:
            continue
        C = heads * 32
        n = n_win * L
        torch.manual_seed(si)
        idx = torch.randperm(n).view(n_win, L).to(torch.int32).to(dev)
        qkv = (torch.randn(n, 3 * C, device=dev) * 0.5).to(bf16)
        bias = (torch.randn(1, heads, L, L, device=dev) * 0.1).contiguous()
        out = torch.empty(n, C, dtype=bf16, device=dev)
        dout = torch.randn(n, C, device=dev).to(bf16)
        lse = torch.empty(heads, n, device=dev)
        delta = torch.empty(heads, n, device=dev)
        dqkv = torch.empty_like(qkv)
        ds = torch.empty(n_win, heads, L, L, dtype=bf16, device=dev)
        d_f = ops.window_desc(n, heads, 32, 3 * C, C, idx, bias)
        d_b = ops.window_desc(n, heads, 32, 3 * C, C, idx, bias, ds_out=ds)
        t_f = harness.window_ms(lambda: ops.seg_attention_fwd(qkv, out, lse, d_f), 10, 3) * 1e3
        t_b = harness.window_ms(lambda: ops.seg_attention_bwd(qkv, out, dout, lse, delta, dqkv, d_b, 1.0), 10, 3) * 1e3
        fl = 4.0 * n * L * C                                   # QK^T + PV over the real window length
        harness.emit({"stage": si, "windows": n_win, "L": L, "heads": heads,
                      "fwd_us": round(t_f, 1), "fwd_tflops": round(fl / t_f / 1e6, 1),
                      "bwd_us": round(t_b, 1), "bwd_tflops": round(2.5 * fl / t_b / 1e6, 1)})   # bwd: delta + dkv + dq


if __name__ == "__main__":
    main()
