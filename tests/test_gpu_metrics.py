"""H100: retrieval evaluation kernels (SURVEY.md §8f.3) vs the reference golden and the numpy oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import metrics_oracle as MO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "these tests need the H100"
    return torch.device("cuda", 0)


def test_metrics_match_reference_golden_including_ties(dev, golden_dir):
    from xpretrain_b200.utils import metrics as M

    gold = torch.load(os.path.join(golden_dir, "retrieval_metrics_n57.pt"), weights_only=False)
    sim = M.cal_cossim(gold["txt"].to(dev), gold["vis"].to(dev))
    assert torch.allclose(sim.cpu(), gold["sim"], rtol=0, atol=1e-6)
    # duplicated items must give bit-identical similarities (every output element uses the same summation order)
    assert torch.equal(sim[:, 7], sim[:, 3]) and torch.equal(sim[7], sim[3]) and torch.equal(sim[:, 20], sim[:, 11])
    for direction, tr in (("t2v", False), ("v2t", True)):
        g, e = M.rank_counts(sim, transpose=tr)
        # integer work: exact against numpy counting on the SAME (device-computed) matrix ...
        x = sim.cpu().numpy()
        wg, we = MO.rank_counts(x.T if tr else x)
        assert np.array_equal(g.cpu().numpy(), wg) and np.array_equal(e.cpu().numpy(), we)
        # ... and the metric tuple equals the reference's (the fixture's similarities are well separated except exact ties)
        got = M.compute_metrics(sim, transpose=tr)
        assert tuple(float(v) for v in got) == gold[f"simple_{direction}"], (direction, got)
    d = M.dsl(sim, 100.0)
    assert np.allclose(d.cpu().numpy(), MO.dsl(sim.cpu().numpy(), 100.0), rtol=2e-5, atol=1e-9)
    for direction, tr in (("t2v", False), ("v2t", True)):
        got = M.compute_metrics(d, transpose=tr)
        assert tuple(float(v) for v in got) == gold[f"DSL_{direction}"], (direction, got)


@pytest.mark.parametrize("n,d", [(1000, 512), (130, 70), (1, 8)])
def test_sim_and_ranks_at_retrieval_sizes(dev, n, d):
    """MSR-VTT-sized evaluation (1k x 1k x 512) and ragged shapes: fp32 similarity and exact rank counts."""
    from xpretrain_b200.utils import metrics as M

    g = torch.Generator().manual_seed(n)
    vis = torch.nn.functional.normalize(torch.randn(n, d, generator=g), dim=-1)
    txt = torch.nn.functional.normalize(vis + 0.7 * torch.randn(n, d, generator=g), dim=-1)
    sim = M.cal_cossim(txt.to(dev), vis.to(dev))
    want = txt.double() @ vis.double().t()
    assert float((sim.cpu().double() - want).abs().max()) < 2e-6
    x = sim.cpu().numpy()
    for tr in (False, True):
        gr, eq = M.rank_counts(sim, transpose=tr)
        wg, we = MO.rank_counts(x.T if tr else x)
        assert np.array_equal(gr.cpu().numpy(), wg) and np.array_equal(eq.cpu().numpy(), we)
        assert tuple(float(v) for v in M.compute_metrics(sim, transpose=tr)) == \
            tuple(float(v) for v in MO.compute_metrics(x.T if tr else x))


def test_no_cpu_path():
    from xpretrain_b200 import _lib
    from xpretrain_b200.utils import metrics as M

    with pytest.raises(_lib.XpError):
        M.cal_cossim(torch.zeros(2, 4), torch.zeros(2, 4))
