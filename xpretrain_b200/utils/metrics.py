"""Retrieval evaluation on the H100 (SURVEY.md §8f.3) — drop-in for CLIP-ViP/src/utils/metrics.py as validate() uses it
(run_pretrain.py:173-176, tasks/run_video_retrieval.py:155-172).

    sim = cal_cossim(text_feats, vis_feats)        # CUDA fp32 tensors stay on the device (no .cpu().numpy() per batch)
    t2v = compute_metrics(sim);  v2t = compute_metrics(sim, transpose=True)      # == compute_metrics(sim.T) of the reference
    sim_dsl = dsl(sim)                             # sim * np_softmax(sim * 100, axis=0)

`compute_metrics` returns the reference's tuple (r1, r5, r10, median rank, mean rank) with its tie quirk: the device counts, per
query, the entries strictly larger than / equal to the diagonal (no sort); the O(N) bookkeeping on those counts is host numpy.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops


def _f32(t) -> torch.Tensor:
    """t as contiguous fp32 (numpy input becomes a host tensor, which the kernels refuse: there is no CPU path)."""
    return torch.as_tensor(t).detach().to(torch.float32).contiguous()


def cal_cossim(feats1: torch.Tensor, feats2: torch.Tensor) -> torch.Tensor:
    """metrics.py:3-5: feats1 [N1, d] @ feats2 [N2, d].T -> [N1, N2] fp32 (fp32 FFMA accumulation on the device)."""
    a, b = _f32(feats1), _f32(feats2)
    if a.shape[1] != b.shape[1]:
        raise ValueError("feature widths differ")
    out = torch.empty(a.shape[0], b.shape[0], dtype=torch.float32, device=a.device)
    ops.sim_f32(a, b, out)
    return out


def dsl(sim: torch.Tensor, theta: float = 100.0) -> torch.Tensor:
    """run_video_retrieval.py:169-170: sim * softmax(theta * sim, axis=0) (a new tensor; `sim` is left untouched)."""
    out = _f32(sim).clone()
    scratch = torch.empty(2 * out.shape[1], dtype=torch.float32, device=out.device)
    ops.dsl_reweight(out, theta, scratch)
    return out


def rank_counts(sim: torch.Tensor, transpose: bool = False):
    """(greater, equal) int32 device vectors: entries of row i (column i if transpose) larger than / equal to sim[i, i]."""
    s = _f32(sim)
    if s.shape[0] != s.shape[1]:
        raise ValueError("compute_metrics needs a square similarity matrix (query i pairs with item i)")
    n = s.shape[0]
    greater, equal = (torch.empty(n, dtype=torch.int32, device=s.device) for _ in range(2))
    ops.rank_counts(s, transpose, greater, equal)
    return greater, equal


def compute_metrics(x: torch.Tensor, transpose: bool = False):
    """metrics.py:41-53 on a device similarity matrix; compute_metrics(sim, transpose=True) == reference compute_metrics(sim.T)."""
    greater, equal = rank_counts(x, transpose)
    return metrics_from_counts(greater.cpu().numpy(), equal.cpu().numpy())


def metrics_from_counts(g: np.ndarray, e: np.ndarray):
    """The O(N) host part of compute_metrics: the reference's rank list `ind` (metrics.py:42-47) is, per query,
    g_i, g_i + 1, .., g_i + e_i - 1 (one entry per value tied with the diagonal), then recall@1/5/10, median and mean rank.
    A query whose diagonal is NaN or +-inf has e_i = 0 and drops out of `ind`, as in the reference (its sort(-x) -
    diag(-x) is never 0 there)."""
    g, e = np.asarray(g, dtype=np.int64), np.asarray(e, dtype=np.int64)
    ind = np.repeat(g, e) + (np.arange(int(e.sum())) - np.repeat(np.cumsum(e) - e, e))
    r1 = float(np.sum(ind == 0)) / len(ind)
    r5 = float(np.sum(ind < 5)) / len(ind)
    r10 = float(np.sum(ind < 10)) / len(ind)
    return r1, r5, r10, np.median(ind) + 1, np.mean(ind) + 1
