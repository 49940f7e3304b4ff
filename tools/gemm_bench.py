"""Time the wgmma GEMM on every GEMM shape of a ViP layer at B = 64 (M = 150784): the forward QKV, out-proj,
fc1 + QuickGELU (two outputs) and fc2, their input gradients (dgrad) and their weight gradients (wgrad, split-K fp32
atomics).  CUDA events, L2 flushed between iterations.  XP_GEMM_CASES=a,b keeps the cases whose names contain a or b."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import harness  # noqa: E402
from xpretrain_b200 import _lib, ops  # noqa: E402


def main():
    harness.require_gpu()
    dev = torch.device("cuda", 0)
    bf16 = torch.bfloat16
    M, C, I = 150784, 768, 3072
    g = torch.Generator(device="cpu").manual_seed(0)
    rnd = lambda *s: (torch.randn(*s, generator=g) * 0.05).to(dev).to(bf16)  # noqa: E731
    x, w_qkv, w_o, w1, w2 = rnd(M, C), rnd(3 * C, C), rnd(C, C), rnd(I, C), rnd(C, I)
    b_qkv, b_c, b_i = torch.zeros(3 * C, device=dev), torch.zeros(C, device=dev), torch.zeros(I, device=dev)
    y_qkv, y_c, y_i, pre = (torch.empty(M, 3 * C, dtype=bf16, device=dev), torch.empty(M, C, dtype=bf16, device=dev),
                            torch.empty(M, I, dtype=bf16, device=dev), torch.empty(M, I, dtype=bf16, device=dev))
    f1, g_qkv = rnd(M, I), rnd(M, 3 * C)
    dw_qkv, dw_o, dw1, dw2 = (torch.zeros(3 * C, C, device=dev), torch.zeros(C, C, device=dev),
                              torch.zeros(I, C, device=dev), torch.zeros(C, I, device=dev))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    cases = {
        "qkv (K=768, N=2304, q-scale)": (lambda: ops.linear_fwd(x, w_qkv, b_qkv, y_qkv, scale_cols=C, col_scale=0.125), 2.0 * M * 3 * C * C),
        "out_proj (K=768, N=768)": (lambda: ops.linear_fwd(x, w_o, b_c, y_c), 2.0 * M * C * C),
        "out_proj + residual": (lambda: ops.linear_fwd(x, w_o, b_c, y_c, residual=x, ldr=C), 2.0 * M * C * C),
        "fc1 + QuickGELU, pre stored (K=768, N=3072)": (lambda: ops.linear_fwd(x, w1, b_i, y_i, act=_lib.ACT_QUICK_GELU, aux=pre, ld_aux=I), 2.0 * M * I * C),
        "fc1 plain": (lambda: ops.linear_fwd(x, w1, b_i, y_i), 2.0 * M * I * C),
        "fc2 (K=3072, N=768)": (lambda: ops.linear_fwd(f1, w2, b_c, y_c), 2.0 * M * I * C),
        "dgrad fc2 + dQuickGELU (K=768, N=3072)": (lambda: ops.linear_dgrad(x, w2, y_i, act=_lib.ACT_DQUICK_GELU, aux=pre, ld_aux=I), 2.0 * M * I * C),
        "dgrad fc1 (K=3072, N=768)": (lambda: ops.linear_dgrad(f1, w1, y_c), 2.0 * M * I * C),
        "dgrad out_proj (K=768, N=768)": (lambda: ops.linear_dgrad(x, w_o, y_c), 2.0 * M * C * C),
        "dgrad qkv (K=2304, N=768)": (lambda: ops.linear_dgrad(g_qkv, w_qkv, y_c), 2.0 * M * 3 * C * C),
        "wgrad qkv (split-K, fp32 atomics)": (lambda: ops.linear_wgrad(g_qkv, x, dw_qkv), 2.0 * M * 3 * C * C),
        "wgrad out_proj (split-K, fp32 atomics)": (lambda: ops.linear_wgrad(x, x, dw_o), 2.0 * M * C * C),
        "wgrad fc1 (split-K, fp32 atomics)": (lambda: ops.linear_wgrad(f1, x, dw1), 2.0 * M * I * C),
        "wgrad fc2 (split-K, fp32 atomics)": (lambda: ops.linear_wgrad(x, f1, dw2), 2.0 * M * I * C),
    }
    out = {}
    only = [t for t in os.environ.get("XP_GEMM_CASES", "").split(",") if t]
    for name, (fn, fl) in cases.items():
        if only and not any(t in name for t in only):
            continue
        ms = harness.median_ms(fn, 6, 2, flush)
        out[name] = {"ms": round(ms, 4), "tflops": round(fl / ms / 1e9, 1)}
    harness.emit(out)


if __name__ == "__main__":
    main()
