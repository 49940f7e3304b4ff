"""Float64 reference of the dense attention kernel (dense_attention.cu), and its bf16 arm.

Same conventions as oracle/attention_ref.py, whose `sdpa` it uses: the kernel's own operands (fused token-major qkv with q
pre-scaled by head_dim**-0.5, the output gradient), float64 results, `q_scale` applied to dq.  With `arm="dense"` the
computation rounds to bf16 where the kernel does: P·V with P = hi + lo (fwd_step of attn_wgmma.cuh, shared with the ViP
kernels), P and dS rounded as MMA operands in the backward, delta from the bf16 O and dO, outputs rounded once.

  dense_ref   n_seq sequences of seq_len consecutive rows; every row attends to every row of its own sequence
              ('joint_space_time': one clip of H*W*T tokens, timesformer.py:202-205; 'space_only': one frame)

Pinned on the CPU to the TimeSformer oracle's attention (tests/test_timesformer_variants_cpu.py).  Pure torch; runs on
the CPU or on a GPU.  Heads are computed one at a time, so a 6272-row sequence fits in a few GB of float64."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle.attention_ref import F64, bf, sdpa


def dense_ref(qkv, dout, n_seq: int, seq_len: int, heads: int, q_scale: float = 1.0,
              arm: Optional[str] = None) -> Dict:
    """qkv [n_rows, >= 3C] (C = 64 heads), dout [n_rows, >= C] or None.  Returns out [n_rows, C], lse [heads, n_rows] and,
    with dout, dqkv [n_rows, 3C]; rows past n_seq * seq_len stay zero."""
    assert arm in (None, "dense")
    C, n = 64 * heads, n_seq * seq_len
    n_rows = qkv.shape[0]
    x = qkv[:n].to(F64)
    out = x.new_zeros(n_rows, C)
    lse = x.new_zeros(heads, n_rows)
    dqkv = x.new_zeros(n_rows, 3 * C) if dout is not None else None
    rd = bf if arm is not None else (lambda t: t)
    for h in range(heads):
        cols = slice(h * 64, (h + 1) * 64)
        q, k, v = (x[:, i * C:(i + 1) * C][:, cols].reshape(n_seq, seq_len, 64) for i in range(3))
        g = dout[:n, cols].to(F64).reshape(n_seq, seq_len, 64) if dout is not None else None
        r = sdpa(q, k, v, g, arm="vip" if arm is not None else None, q_scale=q_scale)
        out[:n, cols] = rd(r["out"].reshape(n, 64))
        lse[h, :n] = r["lse"].reshape(n)
        if dout is not None:
            for i, name in enumerate(("dq", "dk", "dv")):
                dqkv[:n, i * C + h * 64:i * C + (h + 1) * 64] = rd(r[name].reshape(n, 64))
        del r
    res = {"out": out, "lse": lse}
    if dout is not None:
        res["dqkv"] = dqkv
    return res
