"""H100: the retrieval evaluation kernels of retrieval.cu against float64 references of the same operations, with the
rules of contract_harness.py.  The R@1/5/10, MedR and MeanR users report are computed from these, so a subtle error here
misreports results without failing any training run.

  sim_f32      every element: |got - exact| <= gamma_d sum_k |a_k b_k|, gamma_d = d u / (1 - d u), u = 2^-24 (one fp32
               rounding per fmaf, in any order), exact and sum |ab| in float64 from the fp32 inputs; rectangular shapes,
               d = 1 to 1024, 5000 x 5000 x 512; output pitch ld > Nb with guard rows; bitwise repeatable; position
               invariance: duplicated items in other 64-tiles and on both sides of a tile edge give the same bits, and
               any row / column subset gives the same bits as the full matrix; ranks equal the float64 ranks where the
               similarity gaps are 8 x the element bound
  dsl          per 128-column block (one colstats CTA): ||got - exact|| <= 1.5 ||arm - exact|| + 2^-16 ||exact||, exact the
               float64 sim * softmax(theta sim, axis=0) of the same fp32 sim, the arm the reference's own numpy float32
               computation (metrics_oracle.dsl); every element within the derived bound of `dsl_bound`; subnormal weights
               stay distinct and non-zero; duplicated rows / columns across blocks keep identical bits; NaN / inf / signed
               zero patterns of numpy float32; pad columns, guard rows, a NaN-filled scratch, metrics.dsl leaves its input
  rank_counts  exact against metrics_oracle.rank_counts on the same device matrix, both directions, through a pitched view,
               N across the warp and CTA edges; few distinct levels, signed zeros, NaN and inf; compute_metrics tuple for
               tuple; the reference's own rank lists and tuples on special values (a NaN or +-inf diagonal drops its
               query); int32 outputs in guarded buffers
  refusals     every argument refusal of the three entry points and of their ops wrappers: XpError, no launch
"""
import numpy as np
import pytest
import torch

from contract_harness import Guarded, Out, Report, calibrated, same_bits, within
from oracle import metrics_oracle as MO

pytestmark = pytest.mark.gpu

f32, i32 = torch.float32, torch.int32
U = 2.0 ** -24
TINY = 2.0 ** -149                     # the smallest fp32 subnormal
PAD_COLS = 37                          # output pitch ld = width + PAD_COLS
REPORT = Report("retrieval: sim_f32 / dsl worst |err| / bound; dsl worst block ratio err(kernel) / err(numpy float32)",
                width=60)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    REPORT.print()


def _ops():
    from xpretrain_b200 import ops
    return ops


def _metrics():
    from xpretrain_b200.utils import metrics
    return metrics


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def features(n, d, seed, dev, like=None, noise=0.7):
    """n unit-norm fp32 feature rows (correlated with the rows of `like` when given, as text with its video)."""
    g = _gen(seed)
    x = torch.randn(n, d, generator=g)
    if like is not None:
        x = like.cpu()[:n] + noise * x
    return torch.nn.functional.normalize(x, dim=-1).to(dev)


def sim_exact(a, b):
    """float64 A B^T and sum_k |a_k b_k| of the fp32 inputs (float64 products of fp32 values are exact; the float64 sums
    add about d 2^-53 relative, far below the fp32 bound)."""
    a64, b64 = a.double(), b.double()
    return a64 @ b64.t(), a64.abs() @ b64.abs().t()


def sim_bound(d, abs_sum):
    gamma = d * U / (1 - d * U)
    return gamma * abs_sum


def run_sim(dev, a, b, ld=None):
    out = Out(dev, a.shape[0], b.shape[0], f32, ld=ld or b.shape[0] + PAD_COLS)
    _ops().sim_f32(a, b, out.t)
    torch.cuda.synchronize()
    return out


# ============================================================================================================ sim_f32
SIM_SHAPES = [(1, 1, 1), (1, 1000, 16), (63, 65, 15), (64, 64, 17), (65, 63, 70), (130, 64, 512), (64, 130, 768),
              (1000, 130, 1024), (130, 1000, 1), (1000, 1000, 512), (63, 1000, 768), (5000, 5000, 512)]


@pytest.mark.parametrize("Na,Nb,d", SIM_SHAPES, ids=[f"{a}x{b}x{d}" for a, b, d in SIM_SHAPES])
def test_sim_f32_elementwise_coverage_repeatable(dev, Na, Nb, d):
    tag = f"sim {Na}x{Nb}x{d}"
    b = features(Nb, d, Nb * 7 + d, dev)
    a = features(Na, d, Na * 3 + d, dev, like=b if Na <= Nb else None)
    out = run_sim(dev, a, b)
    got = out.check(f"{tag}: coverage")
    exact, ab = sim_exact(a, b)
    within(REPORT, "sim_f32: element |err| / (gamma_d sum |ab|)", got, exact, sim_bound(d, ab))
    again = run_sim(dev, a, b, ld=b.shape[0] + 3)
    assert same_bits(again.check(f"{tag}: second call"), got), f"{tag}: not bitwise repeatable"


def test_sim_f32_position_invariance(dev):
    """Duplicated items in other 64-row / 64-column tiles and on both sides of the tile edges 63/64 and 127/128 give
    identical bits; sim(A[rows], B[cols]) == sim(A, B)[rows][:, cols] bit for bit for arbitrary index subsets."""
    Na, Nb, d = 200, 300, 70
    a = features(Na, d, 1, dev).clone()
    b = features(Nb, d, 2, dev).clone()
    row_dups = [(63, 64), (127, 128), (5, 130), (0, 199), (64, 190)]
    col_dups = [(63, 64), (127, 128), (3, 250), (10, 299), (130, 131)]
    for src, dst in row_dups:
        a[dst] = a[src]
    for src, dst in col_dups:
        b[dst] = b[src]
    full = run_sim(dev, a, b).check("sim duplicates: coverage")
    for src, dst in row_dups:
        assert same_bits(full[dst], full[src]), f"rows {src} and {dst} hold the same item but differ"
    for src, dst in col_dups:
        assert same_bits(full[:, dst], full[:, src]), f"columns {src} and {dst} hold the same item but differ"
    g = _gen(3)
    for n_r, n_c in ((77, 91), (1, 300), (200, 1), (65, 129)):
        rows = torch.randperm(Na, generator=g)[:n_r].to(dev)
        cols = torch.randperm(Nb, generator=g)[:n_c].to(dev)
        sub = run_sim(dev, a[rows].contiguous(), b[cols].contiguous()).check("sim subset: coverage")
        assert same_bits(sub, full[rows][:, cols]), f"sim of a {n_r} x {n_c} subset differs from the full matrix's"


def test_sim_f32_ranks_are_fp32_grade(dev):
    """B_j = c + t_j w: row i's similarities are equally spaced by tau |a_i . w|, and tau is set so that the spacing is
    8 x the worst element bound (about 2e-4: far below bf16's 2^-9 or TF32's 2^-11 resolution of a 0.5 similarity).
    The ranks rank_counts finds in the device matrix must be those of the float64 matrix."""
    N, d = 256, 512
    g = _gen(4)
    w = torch.nn.functional.normalize(torch.randn(d, generator=g, dtype=torch.float64), dim=0)
    c = torch.randn(d, generator=g, dtype=torch.float64)
    c = torch.nn.functional.normalize(c - (c @ w) * w, dim=0)
    a = torch.nn.functional.normalize(torch.randn(N, d, generator=g, dtype=torch.float64) + 20.0 * w, dim=-1).float()
    ab_max = float((a.double().abs() @ (c.abs() + 0.05 * w.abs())).max())      # |b_j| <= |c| + 0.05 |w| below
    tau = 8 * sim_bound(d, ab_max) / float((a.double() @ w).abs().min())
    t = (torch.arange(N, dtype=torch.float64) - N / 2) * tau
    b = (c[None, :] + t[:, None] * w[None, :]).float()
    a, b = a.to(dev), b.to(dev)
    exact, ab = sim_exact(a, b)
    bound = sim_bound(d, ab)
    srt = exact.sort(dim=1).values
    assert float((srt[:, 1:] - srt[:, :-1]).min()) >= 4 * float(bound.max()), "construction: gaps below 4 x the bound"
    out = run_sim(dev, a, b, ld=N + 5)
    got = out.check("sim fp32-grade ranks: coverage")
    within(REPORT, "sim_f32: element |err| / (gamma_d sum |ab|)", got, exact, bound)
    ex = exact.cpu().numpy()
    for tr in (False, True):
        gr, eq = rank_into_guards(dev, out.t, tr)
        wg, we = MO.rank_counts(ex.T if tr else ex)
        assert np.array_equal(gr, wg) and np.array_equal(eq, we), f"transpose={tr}: ranks differ from the float64 ranks"


# ============================================================================================================ DSL
def dsl_exact(sim, theta):
    """float64 sim * softmax(theta sim, axis=0) of the fp32 sim."""
    x = sim.double()
    return x * torch.softmax(theta * x, dim=0)


def dsl_bound(sim, theta):
    """|got - exact| per element of the kernel's
        m = max_r fl(theta v_r);  s = serial fp32 sum_r expf(fl(theta v_r - m));  out = fl(v fl(expf(fl(theta v - m)) / s))
    With E_r = exp(theta v_r - m) and S = sum_r E_r (S >= 1: the maximum's term is 1), the softmax weight is E_r / S for
    any shift m, so m's own rounding is a common shift and cancels.  The argument of expf is off from theta v - m by the
    rounding of theta v and of the subtraction (the two may be fused; either way at most u (|theta v| + |theta v - m|));
    exp turns that absolute error into a relative one of the same size, and CUDA's IEEE expf (no fast math) adds at most
    2 ulp, 4u relative:  e_r = E_r (1 + eta_r),  eta_r = u (|theta v_r| + |theta v_r - m|) + 4u.  The serial fp32 sum over
    `rows` non-negative terms adds gamma_{rows-1} relative, so s = S (1 + sigma) with sigma <= gamma_{rows-1} +
    sum_r (E_r / S) eta_r.  The division and the multiplication round once each (2u).  So
        |got - exact| <= |exact| (eta + sigma + 2u)(1 + 2 (eta + sigma + 2u)) + (3 |v| + 1) 2^-149
    the absolute term for results in the subnormal range: expf's 2 subnormal ulp (over s >= 1, times |v|) and the half ulp
    of the division and of the product.  Columns holding NaN or inf are NaN here: they are held by the specials test."""
    x = sim.double()
    rows = x.shape[0]
    y = theta * x
    t = y - y.max(dim=0, keepdim=True).values
    eta = U * (y.abs() + t.abs()) + 4 * U
    w = torch.softmax(y, dim=0)
    gamma = (rows - 1) * U / (1 - (rows - 1) * U)
    sigma = gamma * (1 + eta.max(dim=0, keepdim=True).values) + (w * eta).sum(0, keepdim=True)
    rel = eta + sigma + 2 * U
    return dsl_exact(sim, theta).abs() * rel * (1 + 2 * rel) + (3 * x.abs() + 1) * TINY


def run_dsl(dev, sim, theta, ld=None, scratch_fill=float("nan")):
    rows, cols = sim.shape
    out = Out(dev, rows, cols, f32, ld=ld or cols + PAD_COLS, init=sim)
    scratch = torch.full((2 * cols,), scratch_fill, dtype=f32, device=dev)
    _ops().dsl_reweight(out.t, theta, scratch)
    torch.cuda.synchronize()
    return out


def block_ids(rows, cols, device):
    """slice index [rows, cols] = col // 128: one dsl_colstats CTA."""
    ids = (torch.arange(cols, device=device) // 128)[None, :].expand(rows, cols)
    return ids, lambda i: f"(columns {128 * i}..{min(128 * i + 127, cols - 1)})"


def retrieval_sim(dev, rows, cols, d, seed):
    """A text x video similarity matrix as evaluation computes it: correlated unit features through sim_f32."""
    vis = features(cols, d, seed, dev)
    txt = features(rows, d, seed + 1, dev, like=vis if rows <= cols else None)
    out = torch.empty(rows, cols, dtype=f32, device=dev)
    _ops().sim_f32(txt, vis, out)
    return out


DSL_SHAPES = [(1000, 127, 100.0), (1000, 128, 1.0), (1000, 129, 200.0), (57, 300, 100.0), (300, 57, 1.0),
              (1, 130, 100.0), (130, 1, 100.0), (2000, 257, 200.0), (5000, 5000, 100.0)]


@pytest.mark.parametrize("rows,cols,theta", DSL_SHAPES, ids=[f"{r}x{c}-theta{t:g}" for r, c, t in DSL_SHAPES])
def test_dsl_calibrated_and_elementwise(dev, rows, cols, theta):
    tag = f"dsl {rows}x{cols} theta {theta:g}"
    sim = retrieval_sim(dev, rows, cols, 256, rows + cols)
    out = run_dsl(dev, sim, theta, ld=cols + (PAD_COLS if cols < 1000 else 8))
    got = out.check(f"{tag}: coverage")
    exact = dsl_exact(sim, theta)
    with np.errstate(under="ignore"):
        arm = torch.from_numpy(MO.dsl(sim.cpu().numpy(), theta)).to(dev)
    assert arm.dtype == f32
    ids, label = block_ids(rows, cols, dev)
    calibrated(REPORT, "dsl: block err / numpy-fp32 err", got, exact, arm, ids, label)
    within(REPORT, "dsl: element |err| / bound", got, exact, dsl_bound(sim, theta))
    again = run_dsl(dev, sim, theta, scratch_fill=0.0)
    assert same_bits(again.check(f"{tag}: zero scratch"), got), f"{tag}: bits depend on the scratch's contents or the call"


@pytest.mark.parametrize("theta", [100.0, 200.0])
def test_dsl_subnormal_weights_stay_distinct(dev, theta):
    """N = 192 columns (a full and a partial colstats block): every column holds its maximum M once (off the diagonal)
    and N - 1 distinct levels with theta (v - M) spread over [-97, -88], so their weights exp(theta (v - M)) / S are fp32
    subnormals and the results about 0.55 of that: 270 subnormal ulps at theta (v - M) = -97, where adjacent levels
    (4.8 % apart) are about 13 ulps apart, against an element bound of a few ulps there.  Each row and each column sees every
    level once (a Latin square), so the float64 ranks have no ties; the kernel's results must be non-zero, within the
    element bound, and rank exactly as the float64 ones.  Then a deeper window, theta (v - M) down to -102 at |v| ~ 1:
    results of 3 to 10^6 subnormal ulps, non-zero and within the bound.  Flushing denormals would zero them all."""
    N = 192
    levels = -88.0 - 9.0 * torch.arange(N, dtype=torch.float64) / (N - 1)
    M = 0.55 + 92.5 / theta
    idx = (torch.arange(N)[:, None] + 5 * torch.arange(N)[None, :]) % N      # gcd(5, 192) = 1: rows and columns permute
    sim = (M + levels[idx] / theta).float()
    sim[(torch.arange(N) + 7) % N, torch.arange(N)] = M                      # one maximum per column and per row
    sim = sim.to(dev)
    out = run_dsl(dev, sim, theta)
    got = out.check(f"dsl subnormal theta {theta:g}: coverage")
    exact = dsl_exact(sim, theta)
    sub = exact.abs() < 2.0 ** -126
    assert int(sub.sum()) == N * (N - 1) and float(exact.abs().min()) > 100 * TINY, "construction"
    assert int((got[sub] == 0).sum()) == 0, f"{int((got[sub] == 0).sum())} subnormal results flushed to zero"
    within(REPORT, "dsl: element |err| / bound", got, exact, dsl_bound(sim, theta))
    ex = exact.cpu().numpy()
    for tr in (False, True):
        gr, eq = rank_into_guards(dev, got, tr)
        wg, we = MO.rank_counts(ex.T if tr else ex)
        assert np.array_equal(gr, wg) and np.array_equal(eq, we), \
            f"theta {theta:g} transpose={tr}: ranks of the re-weighted matrix differ from the float64 ranks"
    # the deep end of the window: 40 rows, column maximum in row 0
    deep = -88.0 - 14.0 * torch.arange(39, dtype=torch.float64) / 38
    M2 = 1.0 + 95.0 / theta
    col = torch.cat([torch.tensor([M2], dtype=torch.float64), M2 + deep / theta])
    sim2 = torch.stack([col, col.flip(0), col.roll(7)], dim=1).float().to(dev)
    got2 = run_dsl(dev, sim2, theta).check(f"dsl deep subnormal theta {theta:g}: coverage")
    exact2 = dsl_exact(sim2, theta)
    assert float(exact2.abs().min()) > TINY, "construction"
    assert int((got2 == 0).sum()) == 0, f"{int((got2 == 0).sum())} results down to theta (v - M) = -102 flushed to zero"
    within(REPORT, "dsl: element |err| / bound", got2, exact2, dsl_bound(sim2, theta))


def test_dsl_ties_survive_across_blocks(dev):
    """Duplicated columns (in other 128-column blocks, and on both sides of the 127/128 edge) and duplicated rows keep
    identical bits after the re-weighting."""
    rows, cols = 700, 300
    sim = retrieval_sim(dev, rows, cols, 128, 11).clone()
    col_dups = [(5, 200), (127, 128), (0, 299), (130, 255)]
    row_dups = [(3, 650), (63, 64), (0, 699)]
    for s, t in col_dups:
        sim[:, t] = sim[:, s]
    for s, t in row_dups:
        sim[t] = sim[s]
    for theta in (1.0, 100.0, 200.0):
        got = run_dsl(dev, sim, theta).check(f"dsl ties theta {theta:g}: coverage")
        for s, t in col_dups:
            assert same_bits(got[:, t], got[:, s]), f"theta {theta:g}: duplicated columns {s} / {t} differ after DSL"
        for s, t in row_dups:
            assert same_bits(got[t], got[s]), f"theta {theta:g}: duplicated rows {s} / {t} differ after DSL"


def _pattern(x):
    """(NaN, +inf, -inf, +0, -0) masks."""
    x = torch.as_tensor(x)
    zero = x == 0
    neg = torch.signbit(x)
    return torch.isnan(x), x == float("inf"), x == float("-inf"), zero & ~neg, zero & neg


def test_dsl_special_values_follow_numpy(dev):
    """NaN anywhere in a column makes the whole column NaN; +inf does too (inf - inf); -inf gives that entry NaN (-inf x 0)
    and weight 0 elsewhere; an all -inf column is NaN; +-0 keep their sign.  Pattern for pattern as numpy float32; the
    columns without specials within the element bound."""
    rows, cols = 300, 260
    sim = 0.5 * retrieval_sim(dev, rows, cols, 64, 21)         # theta |v - max| <= 100: no result near underflow
    sim[17, 3] = float("nan")
    sim[299, 140] = float("nan")
    sim[0, 5] = float("inf")
    sim[250, 129] = float("-inf")
    sim[:, 200] = float("-inf")
    sim[8, 7] = 0.0
    sim[9, 7] = -0.0
    sim[10:20, 131] = -0.0
    sim[20:30, 131] = 0.0
    theta = 100.0
    out = run_dsl(dev, sim, theta)
    got = out.t.clone()
    moved = int((torch.ne(out.buf.view(i32), out.snap.view(i32)))[out.outside].sum())
    assert moved == 0, f"{moved} guard / pad elements overwritten"
    with np.errstate(all="ignore"):
        want = MO.dsl(sim.cpu().numpy(), theta)
    for name, g, w in zip(("NaN", "+inf", "-inf", "+0", "-0"), _pattern(got.cpu()), _pattern(torch.from_numpy(want))):
        assert torch.equal(g, w), f"{name} pattern differs from numpy float32 at {int((g != w).sum())} elements"
    finite_cols = torch.isfinite(sim).all(0)
    assert int(finite_cols.sum()) == cols - 5
    s = sim[:, finite_cols]
    within(REPORT, "dsl: element |err| / bound", got[:, finite_cols], dsl_exact(s, theta), dsl_bound(s, theta))


def test_metrics_dsl_leaves_its_input(dev):
    M = _metrics()
    sim = retrieval_sim(dev, 130, 129, 64, 31)
    snap = sim.clone()
    d = M.dsl(sim, 100.0)
    assert same_bits(sim, snap), "metrics.dsl changed its input"
    assert same_bits(d, run_dsl(dev, sim, 100.0).check("dsl")), "metrics.dsl differs from the kernel on a pitched copy"


# ============================================================================================================ rank_counts
def rank_into_guards(dev, sim, transpose):
    """rank_counts of a (possibly pitched) square device matrix into guarded int32 outputs: every element written, guards
    intact; returns (greater, equal) as numpy."""
    n = sim.shape[0]
    gr, eq = Guarded(dev, (n,), i32), Guarded(dev, (n,), i32)
    _ops().rank_counts(sim, transpose, gr.t, eq.t)
    torch.cuda.synchronize()
    return gr.written("greater").cpu().numpy(), eq.written("equal").cpu().numpy()


def check_ranks(dev, sim, tag):
    """Counts exact against numpy on the same matrix in both directions, and compute_metrics tuple for tuple."""
    M = _metrics()
    x = sim.cpu().numpy()
    for tr in (False, True):
        gr, eq = rank_into_guards(dev, sim, tr)
        wg, we = MO.rank_counts(x.T if tr else x)
        assert np.array_equal(gr, wg), f"{tag} transpose={tr}: greater differs at {np.flatnonzero(gr != wg)[:8]}"
        assert np.array_equal(eq, we), f"{tag} transpose={tr}: equal differs at {np.flatnonzero(eq != we)[:8]}"
        got = tuple(float(v) for v in M.compute_metrics(sim, transpose=tr))
        want = tuple(float(v) for v in MO.compute_metrics(x.T if tr else x))
        assert got == want, f"{tag} transpose={tr}: metrics {got} != {want}"


RANK_N = [1, 2, 31, 32, 33, 127, 128, 129, 1000, 4999]


@pytest.mark.parametrize("N", RANK_N)
def test_rank_counts_exact_pitched(dev, N):
    vis = features(N, 256, N, dev)
    txt = features(N, 256, N + 1, dev, like=vis, noise=1.5)
    out = run_sim(dev, txt, vis, ld=N + 13)
    check_ranks(dev, out.check(f"rank N{N}: sim"), f"rank N{N}")
    check_ranks(dev, out.t, f"rank N{N} pitched")


@pytest.mark.parametrize("N", [33, 129, 1000])
def test_rank_counts_ties_and_specials(dev, N):
    g = _gen(N + 5)
    few = (torch.randint(0, 4, (N, N), generator=g).float() / 4).to(dev)
    check_ranks(dev, few, f"few levels N{N}")
    z = torch.randint(0, 3, (N, N), generator=g).float()
    z = torch.where(z == 0, torch.tensor(0.0), torch.where(z == 1, torch.tensor(-0.0), torch.tensor(0.25)))
    check_ranks(dev, z.to(dev), f"signed zeros N{N}")
    sp = torch.randn(N, N, generator=g)
    sp[torch.rand(N, N, generator=g) < 0.05] = float("nan")
    sp[torch.rand(N, N, generator=g) < 0.05] = float("inf")
    sp[torch.rand(N, N, generator=g) < 0.05] = float("-inf")
    sp[0, 0] = float("nan")                       # NaN and +-inf diagonals drop their query from the rank list
    sp[1, 1] = float("inf")
    sp[2, 2] = float("-inf")
    buf = torch.full((N + 3, N + 9), 7.0)
    buf[:N, :N] = sp
    check_ranks(dev, buf.to(dev)[:N, :N], f"specials N{N} pitched")


def test_metrics_match_reference_on_special_values(dev, golden_dir):
    """The reference's own compute_metrics on matrices holding NaN, +-inf and +-0 on and off the diagonal, and few levels
    (tests/golden/make_golden_metrics.py): the device counts give its rank list and its tuple, in both directions."""
    import os

    M = _metrics()
    gold = torch.load(os.path.join(golden_dir, "retrieval_metrics_specials.pt"), weights_only=False)
    k = 0
    for x in gold["sims"]:
        sim = x.to(dev)
        for tr in (False, True):
            gr, eq = rank_into_guards(dev, sim, tr)
            assert np.array_equal(MO.ranks_from_counts(gr, eq), gold["ind"][k].numpy()), f"matrix {k}: rank list differs"
            got = tuple(float(v) for v in M.compute_metrics(sim, transpose=tr))
            assert got == gold["tuples"][k], f"matrix {k}: metrics {got} != the reference's {gold['tuples'][k]}"
            k += 1


# ============================================================================================================ refusals
def _refused(fn, *args):
    from xpretrain_b200 import _lib
    ops = _ops()
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(_lib.XpError):
        fn(*args)
    assert ops.launch_count() == n0, "a refused call launched a kernel"


def test_refusals_before_any_launch(dev):
    ops = _ops()
    a, b = torch.randn(8, 16, device=dev), torch.randn(12, 16, device=dev)
    out = torch.empty(8, 12, device=dev)
    raw = ops._call
    p = torch.Tensor.data_ptr
    # the library's own refusals, called with valid device pointers
    for Na, Nb, d, ld in ((0, 12, 16, 12), (8, 0, 16, 12), (8, 12, 0, 12), (-1, 12, 16, 12), (8, 12, 16, 11)):
        _refused(raw, "xp_sim_f32", p(a), p(b), p(out), Na, Nb, d, ld)
    scratch = torch.empty(64, device=dev)
    for rows, cols, ld in ((0, 12, 12), (8, 0, 12), (8, -3, 12), (8, 12, 11)):
        _refused(raw, "xp_dsl_reweight", p(out), rows, cols, ld, 100.0, p(scratch))
    sq = torch.randn(12, 12, device=dev)
    gr, eq = torch.empty(12, dtype=i32, device=dev), torch.empty(12, dtype=i32, device=dev)
    for N, ld in ((0, 12), (-2, 12), (12, 11)):
        _refused(raw, "xp_rank_counts", p(sq), N, ld, 0, p(gr), p(eq))
    # through ops: empty operands reach the library's refusals
    _refused(ops.sim_f32, a[:0], b, out[:0])
    _refused(ops.sim_f32, a[:, :0], b[:, :0], out)
    _refused(ops.dsl_reweight, out[:0], 100.0, scratch)
    _refused(ops.rank_counts, sq[:0, :0], False, gr[:0], eq[:0])
    _refused(ops.sim_f32, a, b, torch.empty(12, 16, device=dev).as_strided((8, 12), (11, 1)))     # ld < Nb
    # the wrappers' own checks
    strided = torch.randn(8, 32, device=dev)[:, ::2]                  # read with pitch d it would be the wrong rows
    _refused(ops.sim_f32, strided, b, out)
    _refused(ops.sim_f32, a, torch.randn(16, 12, device=dev).t(), out)
    _refused(ops.sim_f32, a.to(torch.bfloat16), b, out)
    _refused(ops.sim_f32, a, b[:, :8].contiguous(), out)
    _refused(ops.sim_f32, a, b, torch.empty(8, 13, device=dev))
    _refused(ops.sim_f32, a, b, torch.empty(12, 8, device=dev).t())
    _refused(ops.sim_f32, a, b, torch.empty(8, 12, device=dev, dtype=torch.float64))
    _refused(ops.dsl_reweight, out, 100.0, torch.empty(23, device=dev))
    _refused(ops.dsl_reweight, out, 100.0, torch.empty(48, device=dev)[::2])
    _refused(ops.dsl_reweight, out.t(), 100.0, scratch)
    _refused(ops.dsl_reweight, out.double(), 100.0, scratch)
    _refused(ops.rank_counts, out, False, gr[:8], eq[:8])
    _refused(ops.rank_counts, sq, False, gr.long(), eq)
    _refused(ops.rank_counts, sq, True, gr, eq[:11])
    _refused(ops.rank_counts, sq, True, gr, torch.empty(24, dtype=i32, device=dev)[::2])
    _refused(ops.rank_counts, sq.t(), False, gr, eq)
