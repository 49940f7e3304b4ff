"""Time the proxy-token attention kernels alone at the BENCH shape (B = 64, 12 heads, 12 frames, 196 + 4 tokens):
TMA + wgmma forward and backward.  CUDA events on the
launching stream, L2 flushed between iterations.  FLOPs: 1.474 GFLOP forward per (sample, layer) (SURVEY.md §8d), x2.5 backward."""
import json
import sys

import torch

sys.path.insert(0, __file__.rsplit("/", 2)[0])
from xpretrain_b200 import ops  # noqa: E402

B, H, T, L, M = int(sys.argv[1]) if len(sys.argv) > 1 else 64, 12, 12, 196, 4
C, S = 64 * H, M + T * L
dev = torch.device("cuda", 0)
bf16 = torch.bfloat16
g = torch.Generator(device="cpu").manual_seed(0)
qkv = (torch.randn(B * S, 3 * C, generator=g) * 0.8).to(dev).to(bf16)
qkv[:, :C] *= 0.35
out = torch.empty(B * S, C, dtype=bf16, device=dev)
dout = torch.randn(B * S, C, generator=g).to(dev).to(bf16)
lse = torch.empty(B, H, S, device=dev)
dqkv = torch.empty(B * S, 3 * C, dtype=bf16, device=dev)
ws = ops.vip_attention_workspace(B, H, T, M, dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


f_fwd = 1.474e9 * B
res = {}
res["fwd_ms"] = timeit(lambda: ops.vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C))
res["bwd_ms"] = timeit(lambda: ops.vip_attention_bwd(qkv, out, dout, lse, dqkv, ws, B, H, T, L, M, C, 0.125))
res["fwd_tflops"] = f_fwd / res["fwd_ms"] / 1e9
res["bwd_tflops"] = 2.5 * f_fwd / res["bwd_ms"] / 1e9
res["shape"] = dict(B=B, H=H, T=T, L=L, M=M)
print(json.dumps(res))
