"""CPU oracle for SURVEY.md §8(f).3: retrieval evaluation (similarity matrix, DSL re-weighting, recall@k / median / mean rank).

TEST INFRASTRUCTURE ONLY — never imported by the product package.

Restates (numpy, like the reference) CLIP-ViP/src/utils/metrics.py:
  cal_cossim       :3-5    sim = feats1 @ feats2.T
  np_softmax       :7-39   softmax(theta * X) along an axis with the max subtracted
  compute_metrics  :41-53  ranks of the diagonal in each row sorted by decreasing similarity.  Tie quirk kept: every
                           position whose sorted value EQUALS the diagonal is counted, so a row with k tied entries contributes k
                           ranks g, g+1, .., g+k-1 (g = number of strictly larger entries) and len(ind) can exceed the row count.
and the DSL step of tasks/run_video_retrieval.py:169-170: sim * softmax(100 * sim, axis=0).
Parity pinned: tests/golden/make_golden_metrics.py imports the reference module itself and compares bit-for-bit.
"""
import numpy as np


def cal_cossim(feats1, feats2):
    return np.dot(feats1, feats2.T)


def np_softmax(x, theta=1.0, axis=0):
    y = np.atleast_2d(x) * float(theta)
    y = y - np.expand_dims(np.max(y, axis=axis), axis)
    y = np.exp(y)
    return y / np.expand_dims(np.sum(y, axis=axis), axis)


def dsl(sim, theta=100.0):
    return sim * np_softmax(sim * theta, axis=0)


def rank_counts(x):
    """(greater[i], equal[i]) = how many entries of row i are strictly larger than / equal to x[i, i].  compute_metrics
    finds the diagonal's positions as the zeros of sort(-x) - diag(-x); with a NaN or +-inf diagonal that difference is NaN
    or inf everywhere, never 0, so such a row has no position in the rank list: equal[i] = 0."""
    d = np.diag(x)[:, None]
    return (x > d).sum(1), ((x == d) & np.isfinite(d)).sum(1)


def ranks_from_counts(greater, equal):
    """The `ind` array of compute_metrics: for every row the positions greater .. greater + equal - 1."""
    return np.concatenate([g + np.arange(e) for g, e in zip(greater, equal)])


def metrics_from_ranks(ind):
    ind = np.asarray(ind)
    return (float(np.sum(ind == 0)) / len(ind), float(np.sum(ind < 5)) / len(ind), float(np.sum(ind < 10)) / len(ind),
            np.median(ind) + 1, np.mean(ind) + 1)


def compute_metrics(x):
    return metrics_from_ranks(ranks_from_counts(*rank_counts(x)))
