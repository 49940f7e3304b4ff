"""H100: the LayerNorm and small row kernels of rowops.cu against the float64 references of oracle/gemm_ref.py (pinned to
F.layer_norm and autograd by test_gemm_reference_cpu.py), with the rules of contract_harness.py.

  calibrated   y and dx per logical row: ||got - exact|| <= 1.5 x ||arm - exact|| + 2^-16 x the row's norm, the arm being the
               float64 LayerNorm of the stream value the kernel normalises, rounded once to the output dtype
  statistics   mean / rstd element-wise within 2^-20 relative plus the fp32 summation bound of the row; sum_out exact (one
               fp32 add, or the saturating fp16 round of the fp16 stream)
  reductions   dgamma, dbeta, dres_colsum, colsum: |err| <= (terms + 16) 2^-24 (sum |terms| + |start|), accumulated onto a
               non-zero starting value
  coverage     NaN-filled outputs, guard rows / unmapped rows holding a bit pattern (or zeros) that must survive
  locality     rows no map names are NaN in every input
"""
import pytest
import torch

from contract_harness import DTYPES, GUARD_ROWS, Report, bits, calibrated, same_bits, within
from oracle import gemm_ref as R

pytestmark = pytest.mark.gpu

bf16, f32, f16 = torch.bfloat16, torch.float32, torch.float16
U = 2.0 ** -24
EPS = 1e-5
DT_NAME = {bf16: "bf16", f32: "fp32", f16: "fp16"}
REPORT = Report("row kernels: worst row ratio err(kernel) / err(arm); statistics / reductions: worst |err| / bound")


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


def _gen(seed):
    return torch.Generator().manual_seed(seed)


class Rows:
    """A [total, ld] buffer (GUARD_ROWS extra) whose `rows` (indices into the first `total` rows) are the logical output:
    they start as NaN, every other element holds `fill` (the guard pattern by default) and must keep it."""

    def __init__(self, dev, total, C, dtype, rows=None, ld=None, zero=False):
        ld = ld or C
        self.buf = torch.empty(total + GUARD_ROWS, ld, dtype=dtype, device=dev)
        if zero:
            self.buf.zero_()
        else:
            self.buf.view(DTYPES[dtype][0]).fill_(DTYPES[dtype][1])
        self.rows = torch.arange(total, device=dev) if rows is None else rows
        self.C = C
        self.buf[self.rows, :C] = float("nan")
        self.outside = torch.ones_like(self.buf, dtype=torch.bool)
        self.outside[self.rows, :C] = False
        self.snap = bits(self.buf).clone()

    def check(self, what):
        got = self.buf[self.rows, :self.C]
        bad = int((~torch.isfinite(got.float())).sum())
        assert bad == 0, f"{what}: {bad} of {got.numel()} elements not written (still NaN) or not finite"
        moved = int((bits(self.buf) != self.snap)[self.outside].sum())
        assert moved == 0, f"{what}: {moved} elements outside the output (guard / unmapped rows, pad columns) were overwritten"
        return got


def per_row(tag, name, got, exact, arm):
    """The calibrated rule with one slice per logical row."""
    ids = torch.arange(exact.shape[0], device=exact.device)[:, None].expand(exact.shape)
    calibrated(REPORT, f"{tag}: {name}", got, exact, arm, ids, lambda i: f"row {i}")


def stats_check(tag, mean, rstd, ref, C):
    """mean / rstd within 2^-20 relative, plus the bound of the fp32 row sums (C/32 values per lane, then a tree)."""
    nseq = C / 32 + 16
    s = ref["sum"]
    tol_mean = 2.0 ** -20 * ref["mean"].abs() + nseq * U * s.abs().mean(-1)
    within(REPORT, f"{tag}: mean", mean, ref["mean"], tol_mean + 1e-300)
    rel = 2.0 ** -20 + nseq * U + (tol_mean / ref["std"]) ** 2
    within(REPORT, f"{tag}: rstd", rstd, ref["rstd"], rel * ref["rstd"])


def ln_inputs(dev, rows, C, xdt, seed, with_add):
    g = _gen(seed)
    x = (torch.randn(rows, C, generator=g) * 1.5 + 0.3).to(xdt).to(dev)
    add = (torch.randn(rows, C, generator=g)).to(bf16).to(dev) if with_add else None
    gamma = (1.0 + 0.3 * torch.randn(C, generator=g)).to(dev)
    beta = (0.2 * torch.randn(C, generator=g)).to(dev)
    return x, add, gamma, beta


def ln_fwd(dev, x, add, gamma, beta, rows, C, ydt, tag):
    ops = _ops()
    y = Rows(dev, rows, C, ydt)
    st = Rows(dev, rows, 1, f32)
    rs = Rows(dev, rows, 1, f32)
    so = Rows(dev, rows, C, f16 if x.dtype == f16 else f32) if add is not None else None
    m = ops.rowmap(C)
    ops.layernorm_fwd(x, m, y.buf, m, gamma, beta, st.buf, rs.buf, rows, C, EPS, add=add, addmap=m if add is not None else None,
                      sum_out=None if so is None else so.buf, summap=m if so is not None else None)
    torch.cuda.synchronize()
    return (y.check(f"{tag}: y"), st.check(f"{tag}: mean")[:, 0], rs.check(f"{tag}: rstd")[:, 0],
            None if so is None else so.check(f"{tag}: sum_out"))


NARROW_C = [8, 64, 248, 256, 264, 512, 520, 768, 1024]


@pytest.mark.parametrize("C", NARROW_C)
def test_layernorm_fwd_bwd_calibrated(dev, C):
    """Every x / y dtype pair with and without the fused add at 517 rows, the bf16 pair also at 1, 3 and 4 rows; the
    backward with dres and dres_colsum for every stream dtype, onto non-zero .grad buffers."""
    ops = _ops()
    combos = [(xd, yd, ad, 517) for xd in (bf16, f32, f16) for yd in (bf16, f32, f16) for ad in (False, True)]
    combos += [(bf16, bf16, True, r) for r in (1, 3, 4)]
    for xd, yd, ad, rows in combos:
        tag = f"LN C{C} x {DT_NAME[xd]} y {DT_NAME[yd]}{' +add' if ad else ''} rows{rows}"
        x, add, gamma, beta = ln_inputs(dev, rows, C, xd, C * 7 + rows, ad)
        y, mean, rstd, so = ln_fwd(dev, x, add, gamma, beta, rows, C, yd, tag)
        ex = R.layernorm_ref(x, add, gamma, beta, EPS)
        arm = R.layernorm_ref(x, add, gamma, beta, EPS, y_dtype=yd, arm="kernel")
        per_row(tag, "y", y, ex["y"], arm["y"])
        stats_check(tag, mean, rstd, arm, C)
        if so is not None:
            assert torch.equal(so.double(), arm["sum"]), f"{tag}: sum_out is not the single fp32 add / fp16 round"
    # backward: x as the kernel stores it (the stream sum), the exact statistics rounded to fp32
    for xd in (bf16, f32, f16):
        rows = 517
        tag = f"LN bwd C{C} x {DT_NAME[xd]}"
        g = _gen(C + 11)
        x, _, gamma, _ = ln_inputs(dev, rows, C, xd, C * 3 + 1, False)
        dy = torch.randn(rows, C, generator=g).to(bf16).to(dev)
        dres = torch.randn(rows, C, generator=g).to(bf16).to(dev)
        st = R.layernorm_ref(x, None, gamma, gamma, EPS)
        mean, rstd = st["mean"].float(), st["rstd"].float()
        g0 = [torch.randn(C, generator=g).to(dev) for _ in range(3)]
        dgam, dbet, dcol = (t.clone() for t in g0)
        dx = Rows(dev, rows, C, bf16)
        m = ops.rowmap(C)
        ops.layernorm_bwd(dy, m, x, m, gamma, mean, rstd, dres, m, dx.buf, m, dgam, dbet, rows, C, dres_colsum=dcol)
        torch.cuda.synchronize()
        got = dx.check(f"{tag}: dx")
        ex = R.layernorm_bwd_ref(dy, x, gamma, mean, rstd, dres)
        per_row(tag, "dx", got, ex["dx"], R.bf(ex["dx"]))
        nterm = rows + (rows + 7) // 8 + 16
        for nm, t, s0 in (("dgamma", dgam, g0[0]), ("dbeta", dbet, g0[1]), ("dres_colsum", dcol, g0[2])):
            within(REPORT, f"{tag}: {nm}", t, s0.double() + ex[nm], nterm * U * (ex["abs_" + nm] + s0.double().abs()) + 1e-30)


def test_layernorm_bwd_without_dres(dev):
    ops = _ops()
    for C in (96, 128, 768):                      # Swin-3D's 96 / 128-wide stages run the NVEC = 1 instantiation
        rows = 300
        x, _, gamma, _ = ln_inputs(dev, rows, C, bf16, C, False)
        dy = torch.randn(rows, C, generator=_gen(C)).to(bf16).to(dev)
        st = R.layernorm_ref(x, None, gamma, gamma, EPS)
        mean, rstd = st["mean"].float(), st["rstd"].float()
        g0 = torch.randn(2, C, generator=_gen(C + 1)).to(dev)
        dgam, dbet = g0[0].clone(), g0[1].clone()
        dx = Rows(dev, rows, C, bf16)
        m = ops.rowmap(C)
        ops.layernorm_bwd(dy, m, x, m, gamma, mean, rstd, None, None, dx.buf, m, dgam, dbet, rows, C)
        torch.cuda.synchronize()
        tag = f"LN bwd C{C} no dres"
        ex = R.layernorm_bwd_ref(dy, x, gamma, mean, rstd)
        per_row(tag, "dx", dx.check(tag), ex["dx"], R.bf(ex["dx"]))
        nterm = rows + (rows + 7) // 8 + 16
        within(REPORT, f"{tag}: dgamma", dgam, g0[0].double() + ex["dgamma"],
               nterm * U * (ex["abs_dgamma"] + g0[0].double().abs()))
        within(REPORT, f"{tag}: dbeta", dbet, g0[1].double() + ex["dbeta"], nterm * U * (ex["abs_dbeta"] + g0[1].double().abs()))


def test_layernorm_row_statistics(dev):
    """A row of mean 1e3 and std 1e-2 in the fp32 stream (a one-pass E[x^2] - E[x]^2 would lose the variance entirely),
    and a constant row, whose rstd is eps^-1/2 and whose y is beta."""
    C, rows = 768, 4
    g = _gen(5)
    x = torch.randn(rows, C, generator=g, dtype=torch.float64)
    x[0] = 1e3 + 1e-2 * x[0]
    x[1] = 3.25
    x = x.float().to(dev)
    gamma, beta = (1.0 + 0.3 * torch.randn(C, generator=g)).to(dev), torch.randn(C, generator=g).to(dev)
    for yd in (bf16, f32):
        tag = f"LN statistics y {DT_NAME[yd]}"
        y, mean, rstd, _ = ln_fwd(dev, x, None, gamma, beta, rows, C, yd, tag)
        ex = R.layernorm_ref(x, None, gamma, beta, EPS)
        stats_check(tag, mean, rstd, ex, C)
        assert abs(float(rstd[1]) - EPS ** -0.5) <= 2.0 ** -20 * EPS ** -0.5, float(rstd[1])
        # y element-wise from the statistics' bounds: the fp32 mean of a row at 1e3 is off by O(1e-5), which moves every
        # y of a std-1e-2 row by O(1e-3): what any fp32 kernel gets, not a rounding the bf16 arm models
        nseq = C / 32 + 16
        tol_mean = 2.0 ** -20 * ex["mean"].abs() + nseq * U * x.double().abs().mean(-1)
        rel = 2.0 ** -20 + nseq * U + (tol_mean / ex["std"]) ** 2
        xh = ((x.double() - ex["mean"][:, None]) * ex["rstd"][:, None]).abs()
        e = gamma.double().abs() * ((tol_mean * ex["rstd"])[:, None] + xh * rel[:, None]) + 4 * U * ex["y"].abs()
        if yd == bf16:
            e = e + R.ulp_bf16(ex["y"].abs() + e)
        within(REPORT, f"{tag}: y", y, ex["y"], e + 1e-30)


@pytest.mark.parametrize("xd", [bf16, f32], ids=["x-bf16", "x-fp32"])
def test_layernorm_row_maps(dev, xd):
    """The head's row maps: the CLS row of each sample (group map), the patch rows past the M global rows (grouped map with
    an offset) and the EOS rows (explicit offsets).  Rows no map names are NaN in x; the backward writes dx into a zeros
    buffer through the same map, and every unmapped row must stay zero."""
    ops = _ops()
    Bv, Mg, T, L, C = 3, 4, 2, 49, 768
    S = Mg + T * L
    total = Bv * S
    g = _gen(1)
    gamma, beta = (1.0 + 0.3 * torch.randn(C, generator=g)).to(dev), torch.randn(C, generator=g).to(dev)
    eos = torch.tensor([5, S - 1, 0])
    maps = {
        "CLS": (Bv, ops.rowmap(C, group=1, group_stride=S * C), 0, torch.arange(Bv) * S, None),
        "patch rows": (Bv * T * L, ops.rowmap(C, group=T * L, group_stride=S * C), Mg * C,
                       (torch.arange(Bv)[:, None] * S + Mg + torch.arange(T * L)[None, :]).reshape(-1), None),
        "EOS": (Bv, None, 0, torch.arange(Bv) * S + eos, (torch.arange(Bv) * S + eos) * C),
    }
    for name, (rows, rmap, off, idx, offsets) in maps.items():
        tag = f"LN map {name} x {DT_NAME[xd]}"
        idx = idx.to(dev)
        if offsets is not None:
            off_t = offsets.to(torch.int64).to(dev)
            rmap = ops.rowmap(C, offsets=off_t)
        xb = torch.full((total, C), float("nan"), dtype=xd, device=dev)
        xb[idx] = (torch.randn(rows, C, generator=g) + 0.5).to(xd).to(dev)
        y = Rows(dev, rows, C, bf16)
        st, rs = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
        ops.layernorm_fwd(xb, rmap, y.buf, ops.rowmap(C), gamma, beta, st, rs, rows, C, EPS, x_off=off)
        torch.cuda.synchronize()
        xr = xb[idx]
        ex = R.layernorm_ref(xr, None, gamma, beta, EPS)
        per_row(tag, "y", y.check(f"{tag}: y"), ex["y"], R.layernorm_ref(xr, None, gamma, beta, EPS, arm="kernel")["y"])
        stats_check(tag, st, rs, ex, C)
        dy = torch.randn(rows, C, generator=g).to(bf16).to(dev)
        dx = Rows(dev, total, C, bf16, rows=idx, zero=True)
        dgam, dbet = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
        ops.layernorm_bwd(dy, ops.rowmap(C), xb, rmap, gamma, st, rs, None, None, dx.buf, rmap, dgam, dbet, rows, C,
                          x_off=off, dx_off=off)
        torch.cuda.synchronize()
        b = R.layernorm_bwd_ref(dy, xr, gamma, st, rs)
        per_row(tag, "dx", dx.check(f"{tag}: dx"), b["dx"], R.bf(b["dx"]))
        nterm = rows + 32
        within(REPORT, f"{tag}: dgamma", dgam, b["dgamma"], nterm * U * b["abs_dgamma"] + 1e-30)


@pytest.mark.parametrize("C", [1032, 2048, 2056, 4096])
def test_layernorm_wide(dev, C):
    ops = _ops()
    rows = 37
    tag = f"LN wide C{C}"
    x, _, gamma, beta = ln_inputs(dev, rows, C, bf16, C, False)
    y = Rows(dev, rows, C, bf16)
    mean, rstd = Rows(dev, rows, 1, f32), Rows(dev, rows, 1, f32)
    ops.layernorm_any_fwd(x, y.buf, gamma, beta, mean.buf, rstd.buf, rows, C, EPS)
    torch.cuda.synchronize()
    ex = R.layernorm_ref(x, None, gamma, beta, EPS)
    per_row(tag, "y", y.check(f"{tag}: y"), ex["y"], R.layernorm_ref(x, None, gamma, beta, EPS, arm="kernel")["y"])
    stats_check(tag, mean.check("mean")[:, 0], rstd.check("rstd")[:, 0], ex, C)
    g = _gen(C + 3)
    dy = torch.randn(rows, C, generator=g).to(bf16).to(dev)
    m, r = ex["mean"].float(), ex["rstd"].float()
    g0 = torch.randn(2, C, generator=g).to(dev)
    dgam, dbet = g0[0].clone(), g0[1].clone()
    dx = Rows(dev, rows, C, bf16)
    ops.layernorm_any_bwd(dy, x, gamma, m, r, None, dx.buf, dgam, dbet, rows, C)
    torch.cuda.synchronize()
    b = R.layernorm_bwd_ref(dy, x, gamma, m, r)
    per_row(tag, "dx", dx.check(f"{tag}: dx"), b["dx"], R.bf(b["dx"]))
    nterm = rows + 32
    within(REPORT, f"{tag}: dgamma", dgam, g0[0].double() + b["dgamma"], nterm * U * (b["abs_dgamma"] + g0[0].double().abs()))
    within(REPORT, f"{tag}: dbeta", dbet, g0[1].double() + b["dbeta"], nterm * U * (b["abs_dbeta"] + g0[1].double().abs()))


# ==================================================================================== small row kernels
def test_rowscale_single_rounding(dev):
    """out = residual + scale[r] x with one fp32 operation and one bf16 rounding, scale 0 rows included, out aliasing x."""
    ops = _ops()
    rows, C = 33, 264
    g = _gen(2)
    x = torch.randn(rows, C, generator=g).to(bf16).to(dev)
    res = torch.randn(rows, C, generator=g).to(bf16).to(dev)
    scale = torch.tensor([0.0, 1.0 / 0.9, 2.0] * 11, device=dev)
    for residual in (None, res):
        want = R.bf(R.f32(R.rowscale_ref(x, scale, residual))).to(bf16)
        out = Rows(dev, rows, C, bf16)
        ops.rowscale(x, scale, out.buf[:rows], residual=residual)
        torch.cuda.synchronize()
        assert same_bits(out.check("rowscale"), want), "rowscale is not one fp32 fma rounded once to bf16"
        xa = x.clone()
        ops.rowscale(xa, scale, xa, residual=residual)                 # out aliasing x
        torch.cuda.synchronize()
        assert same_bits(xa, want), "rowscale in place differs"


def test_colsum_strided_scaled_accumulating(dev):
    ops = _ops()
    for rows, C, ld in ((1, 8, 16), (517, 264, 280), (4096, 768, 776)):
        g = _gen(rows)
        buf = torch.randn(rows, ld, generator=g).to(bf16).to(dev)
        buf[:, C:] = float("nan")                                       # pad columns are never read
        x = buf[:, :C]
        c0 = torch.randn(C + 8, generator=g).to(dev)
        c0[C:] = 7.0
        out = c0.clone()
        ops.colsum(x, out[:C], scale=-0.5)
        torch.cuda.synchronize()
        assert torch.equal(out[C:], c0[C:]), "colsum wrote past C"
        ex, ab = R.colsum_ref(x, -0.5)
        within(REPORT, f"colsum rows{rows} C{C} ld{ld}: out", out[:C], c0[:C].double() + ex,
                (rows + 32) * U * (ab + c0[:C].double().abs()) + 1e-30)


def test_gather_scatter_rows_bit_exact(dev):
    ops = _ops()
    C, n_src = 264, 40
    g = _gen(3)
    src = torch.randn(n_src, C, generator=g).to(bf16).to(dev)
    index = torch.tensor([3, -1, 0, 39, 17, -5, 3, 22, 8], dtype=torch.int32, device=dev)
    out = Rows(dev, index.numel(), C, bf16)
    ops.gather_rows(src, index, out.buf[:index.numel()], C)
    torch.cuda.synchronize()
    assert same_bits(out.check("gather"), R.gather_rows_ref(src, index)), "gather_rows is not a bit-exact row copy"
    uniq = torch.tensor([5, -1, 0, 39, 17, -2, 30], dtype=torch.int32, device=dev)
    inp = torch.randn(uniq.numel(), C, generator=g).to(bf16).to(dev)
    hit = uniq[uniq >= 0].long()
    dst = Rows(dev, n_src, C, bf16, rows=hit)
    ops.scatter_rows(inp, uniq, dst.buf, C)
    torch.cuda.synchronize()
    got = dst.check("scatter")                      # untouched destination rows keep their bit pattern
    assert same_bits(got, inp[uniq >= 0]), "scatter_rows is not a bit-exact row copy"


@pytest.mark.parametrize("n", [1, 7, 8, 9, 1003])
def test_cast_bf16_tail(dev, n):
    ops = _ops()
    src = (torch.randn(n, generator=_gen(n)) * 100).to(dev)
    dst = torch.empty(n + 24, dtype=bf16, device=dev)
    dst.view(torch.int16).fill_(DTYPES[bf16][1])
    dst[:n] = float("nan")
    snap = dst.view(torch.int16).clone()
    ops.cast_bf16(src, dst)
    torch.cuda.synchronize()
    assert same_bits(dst[:n], src.to(bf16)), "cast is not round-to-nearest-even"
    assert torch.equal(dst.view(torch.int16)[n:], snap[n:]), "cast wrote past n"


@pytest.mark.parametrize("C", [256, 512, 768])
def test_l2norm_fwd_bwd_elementwise(dev, C):
    ops = _ops()
    rows = 13
    g = _gen(C)
    x = (torch.randn(rows, C, generator=g) * 3).to(dev)
    y, inv = Rows(dev, rows, C, f32), Rows(dev, rows, 1, f32)
    ops.l2norm_fwd(x, y.buf[:rows], inv.buf[:rows, 0])
    torch.cuda.synchronize()
    ref = R.l2norm_ref(x)
    k = (C / 32 + 16) * U
    yk, ik = y.check("l2norm y"), inv.check("l2norm inv_norm")[:, 0]
    within(REPORT, f"l2norm C{C}: y", yk, ref["y"], k * ref["y"].abs() + 1e-30)
    within(REPORT, f"l2norm C{C}: inv_norm", ik, ref["inv_norm"], k * ref["inv_norm"])
    dy = torch.randn(rows, C, generator=g).to(dev)
    dx = Rows(dev, rows, C, bf16)
    ops.l2norm_bwd(dy, yk.contiguous(), ik.contiguous(), dx.buf[:rows], scale=0.5)
    torch.cuda.synchronize()
    ex = R.l2norm_bwd_ref(dy, yk, ik, scale=0.5)
    yd, dyd = yk.double(), dy.double()
    e = 0.5 * ik.double()[:, None] * (yd.abs() * k * (dyd * yd).abs().sum(-1, keepdim=True) + 4 * U * (dyd.abs() + ex.abs()))
    within(REPORT, f"l2norm bwd C{C}: dx", dx.check("l2norm dx"), ex, e + R.ulp_bf16(ex.abs() + e))


# ==================================================================================== alignment
def _refused(fn, *args, **kw):
    from xpretrain_b200 import _lib
    ops = _ops()
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(_lib.XpError, match="16-byte aligned"):
        fn(*args, **kw)
    assert ops.launch_count() == n0, "a refused call launched a kernel"


def _at(dev, n, dtype, off, seed):
    """n random elements starting `off` elements into a fresh allocation (off = 8 bf16 / 4 fp32: 16 bytes in)."""
    buf = torch.randn(n + off, generator=_gen(seed)).to(dtype).to(dev)
    return buf[off:]


def test_aligned_offset_views_run_and_misaligned_views_are_refused(dev):
    """Row operands 16 bytes into their allocations, with a row pitch of C + 8, run and match the references; the same
    operands 2 bytes (one bf16) or 4 bytes (one fp32) off, a row pitch or group stride of C + 4 bf16 (8 bytes off every
    other row), and gamma / beta one element off are refused before any launch."""
    ops = _ops()
    rows, C, ld = 37, 264, 272
    gamma, beta = 1.0 + 0.3 * _at(dev, C, f32, 4, 1), 0.2 * _at(dev, C, f32, 4, 2)
    # LayerNorm forward / backward through pitched maps at an element offset of 8
    xb = _at(dev, rows * ld + 8, bf16, 0, 3)
    x = xb[8:].view(rows, ld)[:, :C]
    y = torch.full((rows * ld + 8,), float("nan"), dtype=bf16, device=dev)
    mean, rstd = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
    m = ops.rowmap(ld)
    ops.layernorm_fwd(xb, m, y, m, gamma, beta, mean, rstd, rows, C, EPS, x_off=8, y_off=8)
    torch.cuda.synchronize()
    yv = y[8:].view(rows, ld)[:, :C]
    ex = R.layernorm_ref(x, None, gamma, beta, EPS)
    per_row("LN offset views", "y", yv, ex["y"], R.layernorm_ref(x, None, gamma, beta, EPS, arm="kernel")["y"])
    assert bool(torch.isnan(y[8:].view(rows, ld)[:, C:].float()).all()) and bool(torch.isnan(y[:8].float()).all()), \
        "LN wrote outside its mapped rows"
    for kw in ({"x_off": 1}, {"y_off": 1}, {"x_off": 8, "y_off": 4}):
        _refused(ops.layernorm_fwd, xb, m, y, m, gamma, beta, mean, rstd, rows, C, EPS, **{"x_off": 8, "y_off": 8, **kw})
    for bad in (ops.rowmap(C + 4), ops.rowmap(C, group=4, group_stride=4 * C + 4)):
        _refused(ops.layernorm_fwd, xb, bad, y, m, gamma, beta, mean, rstd, rows, C, EPS, x_off=8, y_off=8)
        _refused(ops.layernorm_fwd, xb, m, y, bad, gamma, beta, mean, rstd, rows, C, EPS, x_off=8, y_off=8)
    g1, b1 = _at(dev, C, f32, 1, 4), _at(dev, C, f32, 1, 5)
    _refused(ops.layernorm_fwd, xb, m, y, m, g1, beta, mean, rstd, rows, C, EPS, x_off=8, y_off=8)
    _refused(ops.layernorm_fwd, xb, m, y, m, gamma, b1, mean, rstd, rows, C, EPS, x_off=8, y_off=8)
    dyb = _at(dev, rows * ld + 8, bf16, 0, 6)
    dx = torch.full((rows * ld + 8,), float("nan"), dtype=bf16, device=dev)
    dgam, dbet = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    ops.layernorm_bwd(dyb, m, xb, m, gamma, mean, rstd, None, None, dx, m, dgam, dbet, rows, C, dy_off=8, x_off=8, dx_off=8)
    torch.cuda.synchronize()
    b = R.layernorm_bwd_ref(dyb[8:].view(rows, ld)[:, :C], x, gamma, mean, rstd)
    per_row("LN bwd offset views", "dx", dx[8:].view(rows, ld)[:, :C], b["dx"], R.bf(b["dx"]))
    for kw in ({"dy_off": 1}, {"x_off": 1}, {"dx_off": 1}):
        _refused(ops.layernorm_bwd, dyb, m, xb, m, gamma, mean, rstd, None, None, dx, m, dgam, dbet, rows, C,
                 **{"dy_off": 8, "x_off": 8, "dx_off": 8, **kw})
    _refused(ops.layernorm_bwd, dyb, m, xb, m, gamma, mean, rstd, None, None, dx, ops.rowmap(C + 4), dgam, dbet, rows, C,
             dy_off=8, x_off=8, dx_off=8)
    # wide LayerNorm
    Cw, rw = 2048, 5
    xw = _at(dev, rw * Cw, bf16, 8, 7).view(rw, Cw)
    yw = _at(dev, rw * Cw, bf16, 8, 8).view(rw, Cw)
    mw, sw = torch.empty(rw, device=dev), torch.empty(rw, device=dev)
    gw, bw = torch.ones(Cw, device=dev), torch.zeros(Cw, device=dev)
    ops.layernorm_any_fwd(xw, yw, gw, bw, mw, sw, rw, Cw, EPS)
    torch.cuda.synchronize()
    exw = R.layernorm_ref(xw, None, gw, bw, EPS)
    per_row("LN wide offset views", "y", yw, exw["y"], R.layernorm_ref(xw, None, gw, bw, EPS, arm="kernel")["y"])
    _refused(ops.layernorm_any_fwd, _at(dev, rw * Cw, bf16, 1, 9).view(rw, Cw), yw, gw, bw, mw, sw, rw, Cw, EPS)
    _refused(ops.layernorm_any_fwd, xw, _at(dev, rw * Cw, bf16, 1, 9).view(rw, Cw), gw, bw, mw, sw, rw, Cw, EPS)
    # gather / scatter / rowscale / colsum
    n_src = 40
    src = _at(dev, n_src * C, bf16, 8, 10).view(n_src, C)
    index = torch.tensor([3, -1, 0, 39, 17], dtype=torch.int32, device=dev)
    out = _at(dev, index.numel() * C, bf16, 8, 11).view(-1, C)
    ops.gather_rows(src, index, out, C)
    torch.cuda.synchronize()
    assert same_bits(out, R.gather_rows_ref(src, index)), "gather_rows through offset views is not a bit-exact copy"
    _refused(ops.gather_rows, _at(dev, n_src * C, bf16, 1, 12).view(n_src, C), index, out, C)
    _refused(ops.gather_rows, src, index, _at(dev, index.numel() * C, bf16, 1, 13).view(-1, C), C)
    _refused(ops.scatter_rows, _at(dev, index.numel() * C, bf16, 1, 14).view(-1, C), index, src, C)
    _refused(ops.scatter_rows, out, index, _at(dev, n_src * C, bf16, 1, 15).view(n_src, C), C)
    scale = torch.tensor([0.0, 2.0, 1.0 / 0.9] * 13, device=dev)[:rows]
    xr = _at(dev, rows * C, bf16, 8, 16).view(rows, C)
    o = _at(dev, rows * C, bf16, 8, 17).view(rows, C)
    ops.rowscale(xr, scale, o)
    torch.cuda.synchronize()
    assert same_bits(o, R.bf(R.f32(R.rowscale_ref(xr, scale))).to(bf16)), "rowscale through offset views differs"
    _refused(ops.rowscale, _at(dev, rows * C, bf16, 1, 18).view(rows, C), scale, o)
    _refused(ops.rowscale, xr, scale, _at(dev, rows * C, bf16, 1, 19).view(rows, C))
    _refused(ops.rowscale, xr, scale, o, residual=_at(dev, rows * C, bf16, 1, 20).view(rows, C))
    cb = _at(dev, rows * ld, bf16, 0, 21).view(rows, ld)
    cs = torch.zeros(C, device=dev)
    ops.colsum(cb[:, 8:8 + C], cs)
    torch.cuda.synchronize()
    exc, abc = R.colsum_ref(cb[:, 8:8 + C])
    within(REPORT, "colsum offset view: out", cs, exc, (rows + 32) * U * abc + 1e-30)
    _refused(ops.colsum, cb[:, 1:1 + C], cs)
