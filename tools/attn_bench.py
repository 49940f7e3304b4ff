"""Time the wgmma attention kernels alone: the staged proxy-token kernels at the BENCH shape (B = 64, 12 heads, 12 frames,
196 + 4 tokens), the streamed proxy-token kernels at ViT-L/14 shapes (L = 256 and 576) and the dense kernels at the
joint space-time TimeSformer shapes (16 clips, 16 heads, N = 392, 1120, 6272).  CUDA events on the launching stream, L2
flushed between iterations, median of `--iters`.  Prints one JSON line per shape.

    python tools/attn_bench.py [B] [--shapes staged,long,dense] [--lib PATH] [--digest]

--lib loads another build of the library (for example the parent commit's, to compare two builds on the same card);
--digest adds a SHA-256 of out, lse and dqkv per shape, computed from seeded inputs, so that two builds can be checked for
bitwise equal results.  FLOPs: 1.474 GFLOP forward per (sample, layer) at the BENCH shape (SURVEY.md §8d), otherwise
4·N·N_keys·64 per head as counted by the kernels' live pairs; backward x2.5."""
import argparse
import hashlib
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import harness  # noqa: E402
from xpretrain_b200 import _lib, ops  # noqa: E402

dev = torch.device("cuda", 0)
bf16 = torch.bfloat16


def inputs(rows, C):
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = torch.randn(rows, 3 * C, generator=g, device=dev).mul_(0.8).to(bf16)
    qkv[:, :C] *= 0.35
    dout = torch.randn(rows, C, generator=g, device=dev).to(bf16)
    return qkv, dout


def digest(*ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.contiguous().view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()


def vip(B, H, T, L, M):
    C, S = 64 * H, M + T * L
    qkv, dout = inputs(B * S, C)
    out = torch.empty(B * S, C, dtype=bf16, device=dev)
    lse = torch.empty(B, H, S, device=dev)
    dqkv = torch.empty(B * S, 3 * C, dtype=bf16, device=dev)
    ws = ops.vip_attention_workspace(B, H, T, M, dev)
    fwd = lambda: ops.vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C)
    bwd = lambda: ops.vip_attention_bwd(qkv, out, dout, lse, dqkv, ws, B, H, T, L, M, C, 0.125)
    # frame queries see M + L keys; global queries see M + T*L keys
    flop = 1.474e9 * B if (B, H, T, L, M) == (B, 12, 12, 196, 4) else 4.0 * 64 * H * B * (T * L * (M + L) + M * S)
    return dict(B=B, H=H, T=T, L=L, M=M), fwd, bwd, flop, (out, lse, dqkv)


def dense(n_seq, H, N):
    C, n = 64 * H, n_seq * N
    qkv, dout = inputs(n, C)
    out = torch.empty(n, C, dtype=bf16, device=dev)
    lse = torch.empty(H, n, device=dev)
    delta = torch.empty(H, n, device=dev)
    dqkv = torch.empty(n, 3 * C, dtype=bf16, device=dev)
    desc = ops.dense_desc(n, H, 3 * C, C, n_seq=n_seq, seq_len=N)
    fwd = lambda: ops.dense_attention_fwd(qkv, out, lse, desc)
    bwd = lambda: ops.dense_attention_bwd(qkv, out, dout, lse, delta, dqkv, desc, 0.125)
    return dict(n_seq=n_seq, H=H, N=N), fwd, bwd, 4.0 * 64 * H * n_seq * N * N, (out, lse, dqkv)


def run(args, flush, name, shape, fwd, bwd, flop, outputs):
    res = {"name": name}
    if args.digest:   # from freshly seeded inputs, before any timing
        fwd(); bwd()
        torch.cuda.synchronize()
        res["digest"] = digest(*outputs)
    res["fwd_ms"] = harness.median_ms(fwd, args.iters, 3, flush)
    res["bwd_ms"] = harness.median_ms(bwd, args.iters, 3, flush)
    res["fwd_tflops"] = flop / res["fwd_ms"] / 1e9
    res["bwd_tflops"] = 2.5 * flop / res["bwd_ms"] / 1e9
    res["shape"] = shape
    harness.emit(res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("B", nargs="?", type=int, default=64, help="batch of the staged shape")
    ap.add_argument("--shapes", default="staged", help="comma-separated subset of staged, long, dense, or all")
    ap.add_argument("--lib", default=None, help="path of the library to load instead of the in-tree build")
    ap.add_argument("--digest", action="store_true", help="print a SHA-256 of out, lse and dqkv per shape")
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    harness.require_gpu()
    if args.lib:
        _lib.LIB_PATH = args.lib
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    shapes = {
        "staged": [("vip_staged_b16", lambda: vip(args.B, 12, 12, 196, 4))],
        "long": [("vip_long_l256", lambda: vip(96, 16, 12, 256, 4)), ("vip_long_l576", lambda: vip(40, 16, 12, 576, 4))],
        "dense": [(f"dense_n{N}", lambda N=N: dense(16, 16, N)) for N in (392, 1120, 6272)],
    }
    for key in (shapes if args.shapes == "all" else args.shapes.split(",")):
        for name, make in shapes[key]:
            run(args, flush, name, *make())
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
