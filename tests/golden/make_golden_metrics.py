"""Golden vectors for the retrieval evaluation (SURVEY.md §8(f).3) from the REAL reference.

Needs a checkout of the reference, named by XP_REFERENCE_ROOT:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_metrics.py

Imports CLIP-ViP/src/utils/metrics.py unmodified (pure numpy), evaluates a synthetic text/video feature set the way
validate() does (run_pretrain.py:173-176, tasks/run_video_retrieval.py:155-172: simple and DSL, both directions) — including
duplicated items, which exercise compute_metrics' tie quirk — asserts oracle/metrics_oracle.py agrees bit-for-bit and stores
the features and the metrics (retrieval_metrics_n57.pt).  Then the same for similarity matrices holding special values
(NaN, +-inf and +-0, on and off the diagonal, and few distinct levels): the reference's metric tuples and rank lists `ind`
in both directions (retrieval_metrics_specials.pt).
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ["XP_REFERENCE_ROOT"]     # a checkout of microsoft/XPretrain
sys.dont_write_bytecode = True

from oracle import metrics_oracle as O  # noqa: E402


def reference():
    spec = importlib.util.spec_from_file_location("ref_metrics", os.path.join(REF, "CLIP-ViP/src/utils/metrics.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    return ref


def reference_ind(x):
    """The rank list compute_metrics builds (metrics.py:42-47), restated to store it beside the reference's tuple."""
    with np.errstate(invalid="ignore"):
        return np.where(np.sort(-x, axis=1) - np.diag(-x)[:, None] == 0)[1]


def special_matrices():
    rng = np.random.RandomState(5)
    out = []
    x = rng.randn(6, 6).astype(np.float32)
    x[1, 1], x[2, 2] = np.inf, -np.inf                              # infinite diagonals
    out.append(x)
    n = 40
    x = rng.randn(n, n).astype(np.float32)
    x[0, 0], x[1, 1], x[2, 2] = np.nan, np.inf, -np.inf
    x[3, 3], x[3, 5], x[3, 6], x[3, 7] = 0.0, -0.0, 0.0, np.inf     # a +0 diagonal tied with -0 and +0
    x[4, 4], x[4, 0], x[4, 9] = -0.0, 0.0, np.nan                   # a -0 diagonal
    x[5, 5], x[5, 1], x[5, 2] = np.inf, np.inf, -np.inf             # +inf tied with +inf on the diagonal
    x[6, 6], x[6, 3] = -np.inf, -np.inf
    mask = rng.rand(n, n)
    x[(mask < 0.05) & ~np.eye(n, dtype=bool)] = np.nan
    x[(mask > 0.95) & ~np.eye(n, dtype=bool)] = np.inf
    x[(mask > 0.45) & (mask < 0.5) & ~np.eye(n, dtype=bool)] = -np.inf
    out.append(x)
    out.append((rng.randint(0, 4, (33, 33)) / 4).astype(np.float32))              # few levels: many ties
    z = rng.randint(0, 3, (17, 17))
    out.append(np.where(z == 0, np.float32(0.0), np.where(z == 1, np.float32(-0.0), np.float32(0.25))).astype(np.float32))
    return out


def specials(ref):
    gold = {"sims": [], "tuples": [], "ind": []}
    for x in special_matrices():
        for m in (x, x.T):
            with np.errstate(invalid="ignore"):
                want = ref.compute_metrics(m)
            got = O.compute_metrics(m)
            assert all(np.array_equal(a, b) for a, b in zip(want, got)), (want, got)
            ind = reference_ind(m)
            assert np.array_equal(ind, O.ranks_from_counts(*O.rank_counts(m)))
            gold["tuples"].append(tuple(float(v) for v in want))
            gold["ind"].append(torch.from_numpy(ind.astype(np.int64)))
        gold["sims"].append(torch.from_numpy(x))
    print(gold["tuples"])
    torch.save(gold, os.path.join(HERE, "retrieval_metrics_specials.pt"))


def main():
    ref = reference()
    specials(ref)

    rng = np.random.RandomState(3)
    n, d = 57, 64
    vis = rng.randn(n, d).astype(np.float32)
    txt = (vis + 0.8 * rng.randn(n, d)).astype(np.float32)          # correlated pairs: ranks spread over a few positions
    vis[7], txt[7] = vis[3], txt[3]                                 # an exact duplicate item  -> tied similarities
    vis[20] = vis[11]                                               # a duplicated video only  -> ties in the t2v direction
    vis /= np.linalg.norm(vis, axis=1, keepdims=True)
    txt /= np.linalg.norm(txt, axis=1, keepdims=True)

    sim = ref.cal_cossim(txt, vis)
    assert np.array_equal(sim, O.cal_cossim(txt, vis))
    out = {}
    for kind in ("simple", "DSL"):
        if kind == "DSL":
            sim_ref = sim * ref.np_softmax(sim * 100, axis=0)
            assert np.array_equal(sim_ref, O.dsl(sim, 100.0))
        else:
            sim_ref = sim
        for direction, m in (("t2v", sim_ref), ("v2t", sim_ref.T)):
            want = ref.compute_metrics(m)
            got = O.compute_metrics(m)
            assert all(float(a) == float(b) for a, b in zip(want, got)), (kind, direction, want, got)
            out[f"{kind}_{direction}"] = tuple(float(v) for v in want)
            g, e = O.rank_counts(m)
            out[f"{kind}_{direction}_greater"], out[f"{kind}_{direction}_equal"] = torch.from_numpy(g), torch.from_numpy(e)
    assert int(out["simple_t2v_equal"].max()) >= 2, "the fixture must contain ties"
    print({k: v for k, v in out.items() if isinstance(v, tuple)})
    torch.save({"txt": torch.from_numpy(txt), "vis": torch.from_numpy(vis), "sim": torch.from_numpy(sim), **out},
               os.path.join(HERE, "retrieval_metrics_n57.pt"))


if __name__ == "__main__":
    main()
