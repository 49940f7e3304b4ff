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

from .. import _lib
from .._lib import check, lib


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _f32_cuda(t: torch.Tensor, what: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise _lib.XpError(f"xpretrain_b200.utils.metrics: {what} must be a CUDA tensor (there is no CPU path)")
    return t.detach().to(torch.float32).contiguous()


def cal_cossim(feats1: torch.Tensor, feats2: torch.Tensor) -> torch.Tensor:
    """metrics.py:3-5: feats1 [N1, d] @ feats2 [N2, d].T -> [N1, N2] fp32 (fp32 FFMA accumulation on the device)."""
    a, b = _f32_cuda(feats1, "feats1"), _f32_cuda(feats2, "feats2")
    if a.shape[1] != b.shape[1]:
        raise ValueError("feature widths differ")
    out = torch.empty(a.shape[0], b.shape[0], dtype=torch.float32, device=a.device)
    check(lib().xp_sim_f32(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.shape[0], b.shape[0], a.shape[1], out.stride(0),
                           _stream()), "xp_sim_f32")
    return out


def dsl(sim: torch.Tensor, theta: float = 100.0) -> torch.Tensor:
    """run_video_retrieval.py:169-170: sim * softmax(theta * sim, axis=0) (a new tensor; `sim` is left untouched)."""
    out = _f32_cuda(sim, "sim").clone()
    scratch = torch.empty(2 * out.shape[1], dtype=torch.float32, device=out.device)
    check(lib().xp_dsl_reweight(out.data_ptr(), out.shape[0], out.shape[1], out.stride(0), float(theta), scratch.data_ptr(),
                                _stream()), "xp_dsl_reweight")
    return out


def rank_counts(sim: torch.Tensor, transpose: bool = False):
    """(greater, equal) int32 device vectors: entries of row i (column i if transpose) larger than / equal to sim[i, i]."""
    s = _f32_cuda(sim, "sim")
    if s.shape[0] != s.shape[1]:
        raise ValueError("compute_metrics needs a square similarity matrix (query i pairs with item i)")
    n = s.shape[0]
    greater = torch.empty(n, dtype=torch.int32, device=s.device)
    equal = torch.empty(n, dtype=torch.int32, device=s.device)
    check(lib().xp_rank_counts(s.data_ptr(), n, s.stride(0), 1 if transpose else 0, greater.data_ptr(), equal.data_ptr(),
                               _stream()), "xp_rank_counts")
    return greater, equal


def compute_metrics(x: torch.Tensor, transpose: bool = False):
    """metrics.py:41-53 on a device similarity matrix; compute_metrics(sim, transpose=True) == reference compute_metrics(sim.T)."""
    greater, equal = rank_counts(x, transpose)
    return metrics_from_counts(greater.cpu().numpy(), equal.cpu().numpy())


def metrics_from_counts(g: np.ndarray, e: np.ndarray):
    """The O(N) host part of compute_metrics: the reference's rank list `ind` (metrics.py:42-47) is, per query,
    g_i, g_i + 1, .., g_i + e_i - 1 (one entry per value tied with the diagonal), then recall@1/5/10, median and mean rank."""
    g, e = np.asarray(g, dtype=np.int64), np.asarray(e, dtype=np.int64)
    ind = np.repeat(g, e) + (np.arange(int(e.sum())) - np.repeat(np.cumsum(e) - e, e))
    r1 = float(np.sum(ind == 0)) / len(ind)
    r5 = float(np.sum(ind < 5)) / len(ind)
    r10 = float(np.sum(ind < 10)) / len(ind)
    return r1, r5, r10, np.median(ind) + 1, np.mean(ind) + 1
