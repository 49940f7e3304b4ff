"""H100: the kernels at the sizes gradient checkpointing makes reachable (ViT-B/16 layer shapes at B = 128, T = 32: B*S =
803,328 rows), where operands pass 2^31 bytes, 2^32 bytes or 2^31 elements and a 32-bit product, TMA coordinate or cast in
a launch path would misplace rows without making anything non-finite.

  periodic     every large operand repeats a small base block along its rows (period P = 41 x 128 rows, or a few
               samples); no_aliasing asserts that no move by a multiple of 2^31 bytes lands on an element of the same
               residue and column, so a wrapped offset cannot hide behind periodic data
  representative  every output row (sample) has the bits of its representative: the same rows run through the same entry
               point at a small size, which is held to float64 by the rules of the kernel's own contract file (calibrated
               slices, element bounds, exactness)
  reductions   split-K weight gradients, column sums, dgamma / dbeta / dres_colsum and the embedding gradients against the
               float64 reference computed from the base block weighted by its repeat counts, under the same fp32 bounds
  coverage     each large output sits in one allocation with guard bytes on both sides and starts NaN; a chunked scan
               finds every element written and finite and every guard intact
  crossing     each case asserts that its named operands reach past the boundary it claims
Each case allocates at most 16 GiB (checked against mem_get_info first) and frees everything before the next; the report
lists per case the boundaries crossed, the worst ratios of its representatives and its peak max_memory_allocated.
"""
import gc
import time

import pytest
import torch

from contract_harness import (ABS_FLOOR, Big, Guarded, Out, Report, calibrated, crossing, has_power, lse_check,
                              no_aliasing, periodic, same_as_representatives, same_bits, tile_slices, within)
from oracle import attention_ref as A
from oracle import embed_ref as E
from oracle import gemm_ref as R

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
U = 2.0 ** -24
EPS = 1e-5
GIB = 1 << 30
LIMIT = 16 * GIB
QG, DQG = R.ACT_QUICK_GELU, R.ACT_DQUICK_GELU
# ViT-B/16 at B = 128, T = 32: S = 4 + 196 x 32 rows per sample
B_, T_, L_, M_, C_, H_ = 128, 32, 196, 4, 768, 12
S_ = M_ + T_ * L_
ROWS = B_ * S_                # 803,328
F_ = 4 * C_
P = 41 * 128                  # GEMM / row period: whole 128-row tiles, an odd number of them
PS = 3                        # sample period
REPORT = Report("large offsets: boundaries crossed (largest offset / boundary); representatives: worst slice ratio "
                "err(kernel) / err(arm), element |err| / bound; peak max_memory_allocated in GiB", width=96)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    REPORT.print()
    print(f"  file wall time {time.time() - t0:.1f} s")


@pytest.fixture(autouse=True)
def _release():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _ops():
    from xpretrain_b200 import ops
    return ops


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def rnd(g, *shape, scale=1.0, shift=0.0):
    return torch.randn(*shape, generator=g) * scale + shift


def room(dev, case, gib):
    """Skip the case, naming the shortfall, if the card lacks `gib` GiB; start its peak-memory count."""
    need = int(gib * GIB)
    assert need <= LIMIT, f"{case}: sized for {gib} GiB, over the 16 GiB a case may take"
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(dev)
    if free < need:
        pytest.skip(f"{case}: needs {gib:.1f} GiB free, the card has {free / GIB:.1f} GiB ({(need - free) / GIB:.1f} GiB "
                    f"short)")
    torch.cuda.reset_peak_memory_stats(dev)


def peak(dev, case):
    torch.cuda.synchronize()
    p = torch.cuda.max_memory_allocated(dev)
    REPORT.record(f"{case}: peak GiB", p / GIB)
    assert p <= LIMIT, f"{case}: peak {p / GIB:.2f} GiB is over 16 GiB"


def k_split(K, splits):
    kb = (K + 63) // 64
    return min(K, ((kb + splits - 1) // splits) * 64)


# ================================================================================================= GEMM
def _gemm_forms(case, x_base, W, bias, act, aux_base, b_layout, N, K, block_ns, dev):
    """The representative launches: [P, K] rows through ops.gemm at each block_n, held to gemm_ref by the calibrated slice
    rule and the element bound.  Returns {block_n: (out, saved pre-activation or None)}."""
    ops = _ops()
    Bl = W if b_layout == 0 else W.T                     # the logical [N, K] operand
    ex = R.gemm_ref(x_base, Bl, bias=bias, act=act, aux=aux_base)
    arm = R.gemm_ref(x_base, Bl, bias=bias, act=act, aux=aux_base, arm="kernel")
    bound = R.gemm_element_bound(ex, K, 1, act=act, aux=aux_base, bias=bias)
    ids, label = tile_slices(P, N, dev)
    res = {}
    for bn in block_ns:
        tag = f"{case} bn{bn}: representative"
        c = Out(dev, P, N, bf16)
        pre = Out(dev, P, N, bf16) if act == QG else None
        aux = pre.buf if pre is not None else aux_base
        ops.gemm(x_base, W, c.buf, M=P, N=N, K=K, lda=K, ldb=W.shape[1], ldc=N, b_layout=b_layout, bias=bias, act=act,
                 aux=aux, ld_aux=N if aux is not None else 0, block_n=bn)
        torch.cuda.synchronize()
        got = c.check(f"{tag} C")
        within(REPORT, f"{tag} C element", got, ex["exact"], bound)
        calibrated(REPORT, f"{tag} C", got, ex["exact"], arm["out"], ids, label)
        gp = None
        if pre is not None:
            gp = pre.check(f"{tag} pre-activation")
            calibrated(REPORT, f"{tag} pre-activation", gp, ex["pre"], arm["pre"], ids, label)
            pb = R.gemm_element_bound(ex, K, 1, bias=bias)
            within(REPORT, f"{tag} pre-activation element", gp, ex["pre"], pb + R.ulp_bf16(ex["pre"].abs() + pb))
        res[bn] = (got, gp)
    return res


def test_gemm_fc1_quick_gelu_forward(dev):
    """fc1 + bias + QuickGELU with the pre-activation saved, M = 803,328, N = 3072, K = 768: both outputs are past 2^31
    elements and 2^32 bytes.  The dispatcher takes block_n = 128 here (K-major B, 12 k-blocks); 256 is run too."""
    case = "fc1 QuickGELU fwd"
    room(dev, case, 12.5)
    ops, g = _ops(), _gen(1)
    xb = rnd(g, P, C_, scale=C_ ** -0.25).to(bf16).to(dev)
    W = rnd(g, F_, C_, scale=C_ ** -0.25).to(bf16).to(dev)
    bias = rnd(g, F_, scale=0.5).to(dev)
    reps = _gemm_forms(case, xb, W, bias, QG, None, 0, F_, C_, (128, 256), dev)
    no_aliasing(f"{case} x", P, C_, 2, ROWS * C_ * 2)
    no_aliasing(f"{case} C / pre-activation", P, F_, 2, ROWS * F_ * 2)
    x = periodic(xb, ROWS)
    out, pre = Big(dev, (ROWS, F_), bf16), Big(dev, (ROWS, F_), bf16)
    for name, t in (("C", out.t), ("pre-activation", pre.t)):
        crossing(REPORT, case, name, t, "2^31 elements")
        crossing(REPORT, case, name, t, "2^32 bytes")
    for bn, (rc, rp) in reps.items():
        out.t.fill_(float("nan"))
        pre.t.fill_(float("nan"))
        ops.gemm(x, W, out.t, M=ROWS, N=F_, K=C_, lda=C_, ldb=C_, ldc=F_, bias=bias, act=QG, aux=pre.t, ld_aux=F_,
                 block_n=bn)
        torch.cuda.synchronize()
        same_as_representatives(f"{case} bn{bn}: C", out.check(f"{case} bn{bn}: C"), rc)
        same_as_representatives(f"{case} bn{bn}: pre-activation", pre.check(f"{case} bn{bn}: pre-activation"), rp)
    del x, out, pre
    peak(dev, case)


def test_gemm_dgrad_fc2_dquick_gelu(dev):
    """dgrad of fc2 with the dQuickGELU epilogue: dy [M, 768] @ W2 [768, 3072] (MN-major B), times the derivative at the
    saved pre-activation; the aux input and the output are [803,328 x 3072], past 2^31 elements."""
    case = "dgrad fc2 dQuickGELU"
    room(dev, case, 12.5)
    ops, g = _ops(), _gen(2)
    dyb = rnd(g, P, C_, scale=0.5).to(bf16).to(dev)
    W2 = rnd(g, C_, F_, scale=F_ ** -0.25).to(bf16).to(dev)
    auxb = rnd(g, P, F_, scale=2.0).to(bf16).to(dev)
    reps = _gemm_forms(case, dyb, W2, None, DQG, auxb, 1, F_, C_, (128, 256), dev)
    no_aliasing(f"{case} dy", P, C_, 2, ROWS * C_ * 2)
    no_aliasing(f"{case} aux / C", P, F_, 2, ROWS * F_ * 2)
    dy, aux = periodic(dyb, ROWS), periodic(auxb, ROWS)
    out = Big(dev, (ROWS, F_), bf16)
    crossing(REPORT, case, "aux", aux, "2^31 elements")
    crossing(REPORT, case, "C", out.t, "2^31 elements")
    for bn, (rc, _) in reps.items():
        out.t.fill_(float("nan"))
        ops.gemm(dy, W2, out.t, M=ROWS, N=F_, K=C_, lda=C_, ldb=F_, ldc=F_, b_layout=1, act=DQG, aux=aux, ld_aux=F_,
                 block_n=bn)
        torch.cuda.synchronize()
        same_as_representatives(f"{case} bn{bn}: C", out.check(f"{case} bn{bn}: C"), rc)
    del dy, aux, out
    peak(dev, case)


def test_gemm_dgrad_fc1(dev):
    """dgrad of fc1: A = dh [803,328 x 3072] (K = 3072: TMA boxes of an operand past 2^31 elements), B = W1 [3072, 768]
    MN-major.  The dispatcher takes block_n = 256 at this size and 128 at the representative's: both are run at both."""
    case = "dgrad fc1"
    room(dev, case, 7.5)
    ops, g = _ops(), _gen(3)
    dhb = rnd(g, P, F_, scale=F_ ** -0.25).to(bf16).to(dev)
    W1 = rnd(g, F_, C_, scale=F_ ** -0.25).to(bf16).to(dev)
    reps = _gemm_forms(case, dhb, W1, None, R.ACT_NONE, None, 1, C_, F_, (128, 256), dev)
    no_aliasing(f"{case} dh", P, F_, 2, ROWS * F_ * 2)
    no_aliasing(f"{case} C", P, C_, 2, ROWS * C_ * 2)
    dh = periodic(dhb, ROWS)
    out = Big(dev, (ROWS, C_), bf16)
    crossing(REPORT, case, "A (dh)", dh, "2^31 elements")
    crossing(REPORT, case, "A (dh)", dh, "2^32 bytes")
    for bn, (rc, _) in reps.items():
        out.t.fill_(float("nan"))
        ops.gemm(dh, W1, out.t, M=ROWS, N=C_, K=F_, lda=F_, ldb=C_, ldc=C_, b_layout=1, block_n=bn)
        torch.cuda.synchronize()
        same_as_representatives(f"{case} bn{bn}: C", out.check(f"{case} bn{bn}: C"), rc)
    del dh, out
    peak(dev, case)


def _wgrad(dev, case, dy, x, dyb, xb, counts, dropped, seed):
    """ops.linear_wgrad at its wgrad_plan onto a non-zero .grad, against the count-weighted float64 reference and bound;
    `dropped` are the counts of a reduction that stops at the boundary, whose value must fall outside that bound."""
    ops = _ops()
    rows, n_out, n_in = dy.shape[0], dy.shape[1], x.shape[1]
    bn, splits = ops.wgrad_plan(n_out, n_in, rows)
    c0 = rnd(_gen(seed), n_out, n_in).to(dev)
    dw = Out(dev, n_out, n_in, f32, init=c0)
    ops.linear_wgrad(dy, x, dw.t)
    torch.cuda.synchronize()
    got = dw.check(f"{case}: dW")
    ex = R.gemm_ref_counted(dyb.T, xb.T, counts, out_mode=R.OUT_F32_ATOMIC, c0=c0)
    bound = R.gemm_element_bound(ex, k_split(rows, splits), splits, c0=c0, out_mode=R.OUT_F32_ATOMIC)
    tag = f"{case} splits{splits} bn{bn}: dW element"
    has_power(REPORT, f"{tag} (rows past the boundary dropped)", ex["exact"],
              R.gemm_ref_counted(dyb.T, xb.T, dropped, out_mode=R.OUT_F32_ATOMIC, c0=c0)["exact"], bound)
    within(REPORT, tag, got, ex["exact"], bound)


def _dominant(g, rows, cols, dev):
    """bf16 rows of positive column means (0.5 to 1.5) with a 0.25 spread: the sums over many rows dominate the sums of
    their magnitudes, so the fp32 bound of a long reduction is a few percent of its value, not of its noise."""
    mean = 0.5 + torch.rand(cols, generator=g)
    return (mean + 0.25 * rnd(g, rows, cols)).to(bf16).to(dev)


def test_gemm_split_k_wgrad_fc1_fc2(dev):
    """The split-K weight gradients of fc1 (dW1 [3072, 768] += dh^T x) and fc2 (dW2 [768, 3072] += dy^T h) over K = 803,328
    rows, the [rows x 3072] operand past 2^31 elements, fp32 atomics, at the plan ops.wgrad_plan picks.  That operand's
    periods carry their own power of two, so a read from the wrong period changes the sums too."""
    case = "wgrad"
    room(dev, case, 7.0)
    g = _gen(4)
    wb, nb = _dominant(g, P, F_, dev), _dominant(g, P, C_, dev)
    w = R.block_weights((ROWS + P - 1) // P, dev)
    wide, narrow = periodic(wb, ROWS, weights=w), periodic(nb, ROWS)
    crossing(REPORT, case, "[rows x 3072] operand", wide, "2^31 elements")
    counts = R.repeat_counts(ROWS, P, dev, w)
    dropped = R.repeat_counts(-(-(1 << 31) // F_), P, dev, w)        # from the first row past 2^31 elements
    _wgrad(dev, f"{case} fc1", wide, narrow, wb, nb, counts, dropped, 40)
    _wgrad(dev, f"{case} fc2", narrow, wide, nb, wb, counts, dropped, 41)
    del wide, narrow
    peak(dev, case)


def test_colsum_fc1_bias_gradient(dev):
    """xp_colsum_bf16 over [803,328 x 3072] (the fc1 bias gradient): 2.47e9 elements read with grid-split rows, onto a
    non-zero start, against the count-weighted reference under the colsum contract's bound.  Every period carries its own
    power of two and the column sums dominate their magnitudes, so both defects of a 32-bit offset leave the bound in every
    column: the elements past 2^31 never read, or read from 2^32 bytes earlier (inside this 4.94 GB buffer)."""
    case = "colsum fc1 bias"
    room(dev, case, 5.5)
    ops, g = _ops(), _gen(6)
    xb = _dominant(g, P, F_, dev)
    w = R.block_weights((ROWS + P - 1) // P, dev)
    x = periodic(xb, ROWS, weights=w)
    crossing(REPORT, case, "x", x, "2^31 elements")
    c0 = rnd(g, F_).to(dev)
    out = Out(dev, 1, F_, f32, init=c0[None])
    ops.colsum(x, out.t[0], scale=-0.5)
    torch.cuda.synchronize()
    got = out.check(case)[0]
    ex, ab = R.colsum_ref(xb, -0.5, counts=R.repeat_counts(ROWS, P, dev, w))
    exact, bound = c0.double() + ex, (ROWS + 32) * U * (ab + c0.double().abs()) + 1e-30
    dropped, displaced = R.wrapped_column_sums(xb, ROWS, w, 1 << 31)
    has_power(REPORT, f"{case}: out (elements past 2^31 dropped)", exact, c0.double() - 0.5 * dropped, bound)
    has_power(REPORT, f"{case}: out (read 2^32 bytes early)", exact, c0.double() - 0.5 * displaced, bound)
    within(REPORT, f"{case}: out", got, exact, bound)
    del x
    peak(dev, case)


# ======================================================================================= patch embedding
def test_patch_embed_launch_and_wgrad(dev):
    """The patch-embedding GEMM as clip_vip.py issues it, at B = 256, T = 32: grouped output rows (c_group = T*L,
    c_group_stride = S*C, c_offset = M*C) into the [B*S, 768] stream and the periodic position table (r_group, stride 0);
    patches and stream are past 2^31 bytes.  Then its weight gradient over the 1,605,632 patch rows."""
    case = "patch embed"
    room(dev, case, 8.0)
    ops, g = _ops(), _gen(7)
    Bv, Kp = 256, 768
    TL = T_ * L_
    pb = (_dominant(g, PS * TL, Kp, dev).float() * Kp ** -0.25).to(bf16)      # positive: the wgrad's sums dominate
    Wp = rnd(g, C_, Kp, scale=Kp ** -0.25).to(bf16).to(dev)
    table = rnd(g, TL, C_).to(bf16).to(dev)
    # representative: PS samples
    xs = Out(dev, PS * S_, C_, bf16)
    xs.t.view(PS, S_, C_)[:, :M_] = 0.25                   # global rows: not this launch's to write
    xs.outside[:PS * S_].view(PS, S_, C_)[:, :M_] = True
    xs.snap = xs.buf.view(torch.int16).clone()
    ops.gemm(pb, Wp, xs.buf, M=PS * TL, N=C_, K=Kp, lda=Kp, ldb=Kp, ldc=C_, residual=table, ldr=C_, r_group=TL,
             r_group_stride=0, c_group=TL, c_group_stride=S_ * C_, c_offset=M_ * C_)
    torch.cuda.synchronize()
    rep = xs.check(f"{case}: representative")
    got = rep.view(PS, S_, C_)[:, M_:].reshape(PS * TL, C_)
    res = table.repeat(PS, 1)
    ex = R.gemm_ref(pb, Wp, residual=res)
    arm = R.gemm_ref(pb, Wp, residual=res, arm="kernel")
    ids, label = tile_slices(PS * TL, C_, dev)
    calibrated(REPORT, f"{case}: representative x0", got, ex["exact"], arm["out"], ids, label)
    within(REPORT, f"{case}: representative x0 element", got, ex["exact"], R.gemm_element_bound(ex, Kp, 1, residual=res))
    del ex, arm, ids
    no_aliasing(f"{case} patches", PS * TL, Kp, 2, Bv * TL * Kp * 2)
    no_aliasing(f"{case} x0", PS * S_, C_, 2, Bv * S_ * C_ * 2)
    patches = periodic(pb, Bv * TL)
    x0 = Big(dev, (Bv * S_, C_), bf16)
    x0.t.view(Bv, S_, C_)[:, :M_] = 0.25
    crossing(REPORT, case, "patches", patches, "2^31 bytes")
    crossing(REPORT, case, "x0", x0.t, "2^31 bytes")
    ops.gemm(patches, Wp, x0.t, M=Bv * TL, N=C_, K=Kp, lda=Kp, ldb=Kp, ldc=C_, residual=table, ldr=C_, r_group=TL,
             r_group_stride=0, c_group=TL, c_group_stride=S_ * C_, c_offset=M_ * C_)
    torch.cuda.synchronize()
    same_as_representatives(f"{case}: x0 per sample", x0.check(f"{case}: x0").view(Bv, S_ * C_), rep.view(PS, S_ * C_))
    del x0
    # the weight gradient: dW [768, 768] += d_patch^T patches over Bv*T*L rows
    db = _dominant(g, PS * TL, C_, dev)
    w = R.block_weights(-(-Bv // PS), dev)
    d_patch = periodic(db, Bv * TL, weights=w)
    crossing(REPORT, f"{case} wgrad", "d_patch", d_patch, "2^31 bytes")
    _wgrad(dev, f"{case} wgrad", d_patch, patches, db, pb, R.repeat_counts(Bv * TL, PS * TL, dev, w),
           R.repeat_counts(-(-(1 << 31) // (C_ * 2)), PS * TL, dev, w), 70)   # from the first row past 2^31 bytes
    del patches, d_patch
    peak(dev, case)


# ============================================================================================ LayerNorm
def _stats_check(tag, mean, rstd, ref, C):
    """As the row-kernel contract: mean / rstd within 2^-20 relative plus the fp32 row-sum bound."""
    nseq = C / 32 + 16
    tol_mean = 2.0 ** -20 * ref["mean"].abs() + nseq * U * ref["sum"].abs().mean(-1)
    within(REPORT, f"{tag}: mean", mean, ref["mean"], tol_mean + 1e-300)
    rel = 2.0 ** -20 + nseq * U + (tol_mean / ref["std"]) ** 2
    within(REPORT, f"{tag}: rstd", rstd, ref["rstd"], rel * ref["rstd"])


def _per_row(tag, got, exact, arm):
    ids = torch.arange(exact.shape[0], device=exact.device)[:, None].expand(exact.shape)
    calibrated(REPORT, tag, got, exact, arm, ids, lambda i: f"row {i}")


def _patterned(g, rows, cols):
    """Stream rows whose columns keep their sign from row to row: +-(1 to 1.5) per column plus 0.3 noise, so that xhat, and
    with it dgamma = sum dy xhat, does not average out over the rows."""
    sign = torch.where(torch.rand(cols, generator=g) < 0.5, -1.0, 1.0)
    return sign * (1.0 + 0.5 * torch.rand(cols, generator=g)) + 0.3 * rnd(g, rows, cols)


def _ln_power(tag, exc, dropped, g0, nterm, names, got):
    """The column sums of a LayerNorm backward against the count-weighted reference, after the self-check that a pass
    stopping at the boundary row would leave their bound in every column."""
    for i, nm in enumerate(names):
        exact = g0[i].double() + exc[nm]
        bound = nterm * U * (exc["abs_" + nm] + g0[i].double().abs()) + 1e-30
        has_power(REPORT, f"{tag}: {nm} (rows past the boundary dropped)", exact, g0[i].double() + dropped[nm], bound)
        within(REPORT, f"{tag}: {nm}", got[i], exact, bound)


def test_layernorm_fp32_stream_fwd_bwd(dev):
    """The layer's LayerNorms on the fp32 residual stream [803,328 x 768] (2.47 GB): forward with the bf16 branch output
    added and sum_out stored, backward with dres and dres_colsum onto non-zero .grad buffers."""
    case = "LN fp32 stream"
    room(dev, case, 9.0)
    ops, g = _ops(), _gen(8)
    m = ops.rowmap(C_)
    xb = _patterned(g, P, C_).to(dev)
    addb = rnd(g, P, C_, scale=0.25).to(bf16).to(dev)
    gamma, beta = (1.0 + 0.3 * rnd(g, C_)).to(dev), (0.2 * rnd(g, C_)).to(dev)
    # representative
    y, so = Out(dev, P, C_, bf16), Out(dev, P, C_, f32)
    mu, rs = Out(dev, P, 1, f32), Out(dev, P, 1, f32)
    ops.layernorm_fwd(xb, m, y.buf, m, gamma, beta, mu.buf, rs.buf, P, C_, EPS, add=addb, addmap=m, sum_out=so.buf,
                      summap=m)
    torch.cuda.synchronize()
    ry, rso, rmu, rrs = y.check(case), so.check(case), mu.check(case)[:, 0], rs.check(case)[:, 0]
    ex = R.layernorm_ref(xb, addb, gamma, beta, EPS)
    arm = R.layernorm_ref(xb, addb, gamma, beta, EPS, y_dtype=bf16, arm="kernel")
    _per_row(f"{case}: representative y", ry, ex["y"], arm["y"])
    _stats_check(f"{case}: representative", rmu, rrs, arm, C_)
    assert torch.equal(rso.double(), arm["sum"]), f"{case}: representative sum_out is not the single fp32 add"
    del ex, arm
    for nm, es in (("x / sum_out", 4), ("add / y / dy / dres / dx", 2)):
        no_aliasing(f"{case} {nm}", P, C_, es, ROWS * C_ * es)
    x, add = periodic(xb, ROWS), periodic(addb, ROWS)
    bs, byy = Big(dev, (ROWS, C_), f32), Big(dev, (ROWS, C_), bf16)
    bmu, brs = Big(dev, (ROWS,), f32), Big(dev, (ROWS,), f32)
    crossing(REPORT, case, "x", x, "2^31 bytes")
    crossing(REPORT, case, "sum_out", bs.t, "2^31 bytes")
    ops.layernorm_fwd(x, m, byy.t, m, gamma, beta, bmu.t, brs.t, ROWS, C_, EPS, add=add, addmap=m, sum_out=bs.t, summap=m)
    torch.cuda.synchronize()
    for nm, b, r in (("y", byy, ry), ("sum_out", bs, rso), ("mean", bmu, rmu), ("rstd", brs, rrs)):
        same_as_representatives(f"{case} fwd: {nm}", b.check(f"{case} fwd: {nm}"), r)
    del x, add, byy
    # backward: x = the stored stream sum, the kernel's statistics
    dyb, dresb = _dominant(g, P, C_, dev), _dominant(g, P, C_, dev)
    g0 = [rnd(g, C_).to(dev) for _ in range(3)]
    dx = Out(dev, P, C_, bf16)
    dgs = [c.clone() for c in g0]
    ops.layernorm_bwd(dyb, m, rso, m, gamma, rmu, rrs, dresb, m, dx.buf, m, dgs[0], dgs[1], P, C_, dres_colsum=dgs[2])
    torch.cuda.synchronize()
    rdx = dx.check(f"{case} bwd: representative dx")
    exb = R.layernorm_bwd_ref(dyb, rso, gamma, rmu, rrs, dresb)
    _per_row(f"{case} bwd: representative dx", rdx, exb["dx"], R.bf(exb["dx"]))
    dy, dres = periodic(dyb, ROWS), periodic(dresb, ROWS)
    bdx = Big(dev, (ROWS, C_), bf16)
    dgb = [c.clone() for c in g0]
    ops.layernorm_bwd(dy, m, bs.t, m, gamma, bmu.t, brs.t, dres, m, bdx.t, m, dgb[0], dgb[1], ROWS, C_,
                      dres_colsum=dgb[2])
    torch.cuda.synchronize()
    same_as_representatives(f"{case} bwd: dx", bdx.check(f"{case} bwd: dx"), rdx)
    exc = R.layernorm_bwd_ref(dyb, rso, gamma, rmu, rrs, dresb, counts=R.repeat_counts(ROWS, P, dev))
    first = -(-(1 << 31) // (C_ * 4))                                  # the first row of x past 2^31 bytes
    dropped = R.layernorm_bwd_ref(dyb, rso, gamma, rmu, rrs, dresb, counts=R.repeat_counts(first, P, dev))
    _ln_power(f"{case} bwd", exc, dropped, g0, ROWS + (ROWS + 7) // 8 + 16, ("dgamma", "dbeta", "dres_colsum"), dgb)
    del dy, dres, bdx, bs, bmu, brs
    peak(dev, case)


def test_layernorm_grouped_patch_rows(dev):
    """pre_layrnorm as clip_vip.py issues it, at B = 256, T = 32: the bf16 stream x0 (2.47 GB) normalised into the fp32
    stream (4.94 GB) by two launches, the patch rows (x_off = M*C, group T*L, stride S*C) and the global rows (group M),
    then its backward into the compact d_patch / d_global halves."""
    case = "LN grouped"
    room(dev, case, 9.0)
    ops, g = _ops(), _gen(9)
    Bv, TL = 256, T_ * L_
    gamma, beta = (1.0 + 0.3 * rnd(g, C_)).to(dev), (0.2 * rnd(g, C_)).to(dev)
    x0b = _patterned(g, PS * S_, C_).to(bf16).to(dev)
    dyb = _dominant(g, PS * S_, C_, dev)
    pmap, gmap, plain = (ops.rowmap(C_, group=TL, group_stride=S_ * C_), ops.rowmap(C_, group=M_, group_stride=S_ * C_),
                         ops.rowmap(C_))

    def fwd(x0, y, n):
        mp, rp = Big(dev, (n * TL,), f32), Big(dev, (n * TL,), f32)
        mg, rg = Big(dev, (n * M_,), f32), Big(dev, (n * M_,), f32)
        ops.layernorm_fwd(x0, pmap, y, pmap, gamma, beta, mp.t, rp.t, n * TL, C_, EPS, x_off=M_ * C_, y_off=M_ * C_)
        ops.layernorm_fwd(x0, gmap, y, gmap, gamma, beta, mg.t, rg.t, n * M_, C_, EPS)
        torch.cuda.synchronize()
        return [b.check(f"{case}: statistics") for b in (mp, rp, mg, rg)]

    def bwd(dy, x0, st, d_patch, d_glob, n, dg):
        ops.layernorm_bwd(dy, pmap, x0, pmap, gamma, st[0], st[1], None, None, d_patch, plain, dg[0], dg[1], n * TL, C_,
                          dy_off=M_ * C_, x_off=M_ * C_)
        ops.layernorm_bwd(dy, gmap, x0, gmap, gamma, st[2], st[3], None, None, d_glob, plain, dg[0], dg[1], n * M_, C_)
        torch.cuda.synchronize()

    def stream_order(st, n):     # the compact (mean, rstd) of both launches back in stream-row order [n * S]
        return [torch.cat([st[2 + i].view(n, M_), st[i].view(n, TL)], 1).reshape(-1) for i in (0, 1)]

    # representative: PS samples
    ys = Big(dev, (PS * S_, C_), f32)
    st_s = fwd(x0b, ys.t, PS)
    ry = ys.check(f"{case}: representative y")
    ex = R.layernorm_ref(x0b, None, gamma, beta, EPS)
    arm = R.layernorm_ref(x0b, None, gamma, beta, EPS, y_dtype=f32, arm="kernel")
    _per_row(f"{case}: representative y", ry, ex["y"], arm["y"])
    mean_s, rstd_s = stream_order(st_s, PS)
    _stats_check(f"{case}: representative", mean_s, rstd_s, arm, C_)
    dps, dgls = Big(dev, (PS * TL, C_), bf16), Big(dev, (PS * M_, C_), bf16)
    g0 = [rnd(g, C_).to(dev) for _ in range(2)]
    bwd(dyb, x0b, st_s, dps.t, dgls.t, PS, [c.clone() for c in g0])
    rdp, rdg = dps.check(f"{case}: representative d_patch"), dgls.check(f"{case}: representative d_global")
    exb = R.layernorm_bwd_ref(dyb, x0b, gamma, mean_s, rstd_s)
    dxs = exb["dx"].view(PS, S_, C_)
    _per_row(f"{case}: representative d_patch", rdp, dxs[:, M_:].reshape(-1, C_), R.bf(dxs[:, M_:].reshape(-1, C_)))
    _per_row(f"{case}: representative d_global", rdg, dxs[:, :M_].reshape(-1, C_), R.bf(dxs[:, :M_].reshape(-1, C_)))
    del ex, arm, exb, dxs
    # Bv samples
    no_aliasing(f"{case} x0 / dy", PS * S_, C_, 2, Bv * S_ * C_ * 2)
    no_aliasing(f"{case} y", PS * S_, C_, 4, Bv * S_ * C_ * 4)
    no_aliasing(f"{case} d_patch", PS * TL, C_, 2, Bv * TL * C_ * 2)
    x0 = periodic(x0b, Bv * S_)
    y = Big(dev, (Bv * S_, C_), f32)
    crossing(REPORT, case, "x0", x0, "2^31 bytes")
    crossing(REPORT, case, "y (fp32 stream)", y.t, "2^32 bytes")
    st = fwd(x0, y.t, Bv)
    same_as_representatives(f"{case}: y per sample", y.check(f"{case}: y").view(Bv, -1), ry.view(PS, -1))
    for nm, b, r, w in (("patch mean", st[0], st_s[0], TL), ("patch rstd", st[1], st_s[1], TL),
                        ("global mean", st[2], st_s[2], M_), ("global rstd", st[3], st_s[3], M_)):
        same_as_representatives(f"{case}: {nm}", b.view(Bv, w), r.view(PS, w))
    del y
    dy = periodic(dyb, Bv * S_)
    dp, dgl = Big(dev, (Bv * TL, C_), bf16), Big(dev, (Bv * M_, C_), bf16)
    crossing(REPORT, case, "d_patch", dp.t, "2^31 bytes")
    dg = [c.clone() for c in g0]
    bwd(dy, x0, st, dp.t, dgl.t, Bv, dg)
    same_as_representatives(f"{case}: d_patch per sample", dp.check(f"{case}: d_patch").view(Bv, -1), rdp.view(PS, -1))
    same_as_representatives(f"{case}: d_global per sample", dgl.check(f"{case}: d_global").view(Bv, -1),
                            rdg.view(PS, -1))
    rows = Bv * S_
    exc = R.layernorm_bwd_ref(dyb, x0b, gamma, mean_s, rstd_s, counts=R.repeat_counts(rows, PS * S_, dev))
    first = -(-(1 << 31) // (C_ * 2))                                  # the first stream row of x0 past 2^31 bytes
    dropped = R.layernorm_bwd_ref(dyb, x0b, gamma, mean_s, rstd_s, counts=R.repeat_counts(first, PS * S_, dev))
    _ln_power(f"{case} bwd", exc, dropped, g0, rows + (rows + 7) // 8 + 32, ("dgamma", "dbeta"), dg)
    del x0, dy, dp, dgl
    peak(dev, case)


# ============================================================================================ embedding
def test_embed_tables_and_bwd(dev):
    """xp_vip_embed_tables writing the global rows of a [B*S, 768] bf16 stream past 2^31 bytes (B = 256, T = 32,
    temporal_size 12: the interpolated table), and xp_vip_embed_bwd reading d_patch [B*T*L, 768] past 2^31 bytes."""
    case = "embed"
    room(dev, case, 6.0)
    ops, g = _ops(), _gen(10)
    Bv, TL, Tsz = 256, T_ * L_, 12
    pos = rnd(g, 1 + L_, C_).to(dev)
    tmp = rnd(g, Tsz, C_).to(dev)
    cls, added = rnd(g, C_).to(dev), rnd(g, M_ - 1, C_).to(dev)
    # representative: one sample (the tables do not depend on the sample)
    tab_s, x_s = Guarded(dev, (TL, C_), bf16), Guarded(dev, (S_, C_), bf16)
    ops.vip_embed_tables(pos, tmp, cls, added, tab_s.t, x_s.t, 1, T_, L_, M_, C_, Tsz)
    torch.cuda.synchronize()
    rtab = tab_s.written(f"{case}: representative table")
    x_s.guards(f"{case}: representative x0")
    exact, bound, _, want_glob = E.vip_tables_ref(pos, tmp, cls, added, 1, T_, L_, M_, Tsz)
    within(REPORT, f"{case}: representative table", rtab, exact, bound)
    assert same_bits(x_s.t[:M_], want_glob[0]), f"{case}: representative global rows differ from their exact value"
    assert bool(torch.isnan(x_s.t[M_:]).all()), f"{case}: representative wrote into the patch rows"
    no_aliasing(f"{case} x0", S_, C_, 2, Bv * S_ * C_ * 2)
    tab, x0 = Guarded(dev, (TL, C_), bf16), Big(dev, (Bv * S_, C_), bf16)
    crossing(REPORT, case, "x0", x0.t, "2^31 bytes")
    ops.vip_embed_tables(pos, tmp, cls, added, tab.t, x0.t, Bv, T_, L_, M_, C_, Tsz)
    torch.cuda.synchronize()
    assert same_bits(tab.written(f"{case}: table"), rtab), f"{case}: table differs from the representative's"
    x0.guards(f"{case}: x0")
    # global rows written as the representative's, patch rows left NaN (the same bits as the representative's)
    same_as_representatives(f"{case}: x0 per sample", x0.t.view(Bv, S_ * C_), x_s.t.view(1, S_ * C_))
    del x0
    # backward over periodic gradients of PS samples
    dpb = _dominant(g, PS * TL, C_, dev)
    dgb = rnd(g, PS * M_, C_, scale=0.5).to(bf16).to(dev)
    no_aliasing(f"{case} d_patch", PS * TL, C_, 2, Bv * TL * C_ * 2)
    d_patch, d_glob = periodic(dpb, Bv * TL), periodic(dgb, Bv * M_)
    crossing(REPORT, case, "d_patch", d_patch, "2^31 bytes")
    init = {"pos": rnd(g, 1 + L_, C_).to(dev), "temporal": rnd(g, Tsz, C_).to(dev), "cls": rnd(g, C_).to(dev),
            "added": rnd(g, M_ - 1, C_).to(dev)}
    outs = {k: Guarded(dev, tuple(v.shape), f32, init=v) for k, v in init.items()}
    ops.vip_embed_bwd(d_patch, d_glob, outs["pos"].t, outs["temporal"].t, outs["cls"].t, outs["added"].t, Bv, T_, L_,
                      M_, C_, Tsz)
    torch.cuda.synchronize()
    ref = E.vip_bwd_ref(dpb, dgb, init, PS, T_, L_, M_, Tsz, counts=R.repeat_counts(Bv, PS, dev))
    first = -(-(1 << 31) // (TL * C_ * 2))                             # the first sample wholly past 2^31 bytes
    drop = E.vip_bwd_ref(dpb, dgb, init, PS, T_, L_, M_, Tsz, counts=R.repeat_counts(first, PS, dev))
    has_power(REPORT, f"{case} bwd: d_pos patch rows (samples {first}-{Bv - 1} dropped)", ref["pos"][0][1:],
              drop["pos"][0][1:], ref["pos"][1][1:])
    has_power(REPORT, f"{case} bwd: d_temporal (samples {first}-{Bv - 1} dropped)", ref["temporal"][0],
              drop["temporal"][0], ref["temporal"][1])
    for k, o in outs.items():
        within(REPORT, f"{case} bwd: d_{k}", o.written(f"{case} bwd: d_{k}"), *ref[k])
    del d_patch, d_glob
    peak(dev, case)


def test_patchify_fp32_frames(dev):
    """xp_vip_patchify from float32 frames [4096, 3, 224, 224] (a 2.47 GB source), five distinct frames repeated; every
    patch row has the bits of its representative, which are patchify_ref's exactly."""
    case = "patchify fp32"
    room(dev, case, 4.5)
    ops, g = _ops(), _gen(11)
    nf, pf, hw, p = 4096, 5, 224, 16
    base = rnd(g, pf, 3, hw, hw).to(dev)
    rp = (hw // p) ** 2
    small = Big(dev, (pf * rp, 3 * p * p), bf16)
    ops.vip_patchify(base, small.t, p)
    torch.cuda.synchronize()
    rep = small.check(f"{case}: representative")
    assert same_bits(rep, E.patchify_ref(base, p)), f"{case}: representative differs from patchify_ref"
    no_aliasing(f"{case} frames", pf, 3 * hw * hw, 4, nf * 3 * hw * hw * 4)
    frames = periodic(base, nf)
    crossing(REPORT, case, "frames", frames, "2^31 bytes")
    out = Big(dev, (nf * rp, 3 * p * p), bf16)
    ops.vip_patchify(frames, out.t, p)
    torch.cuda.synchronize()
    same_as_representatives(f"{case}: patches", out.check(f"{case}: patches"), rep)
    del frames, out
    peak(dev, case)


# ============================================================================================ attention
def _vip_base(dev, n, H, T, L, M, seed):
    """qkv [n*S, 3C] at the model's logit scale (q pre-scaled), dout [n*S, C]: n distinct samples."""
    g = _gen(seed)
    C, S = 64 * H, M + T * L
    x = rnd(g, n * S, 3 * C)
    x[:, :C] *= 0.125
    return x.to(bf16).to(dev), rnd(g, n * S, C).to(bf16).to(dev)


def _vip_slices(dev, n, H, T, L, M):
    """Slice index [n*S, H] of every (row, head): (b, h, t, 64-row tile) for frame rows, (b, h) for the M global rows."""
    S, nt = M + T * L, (L + 63) // 64
    per = T * nt + 1
    s = torch.arange(S, device=dev)
    f = (s - M).clamp_min(0)
    r = torch.where(s < M, torch.full_like(s, T * nt), (f // L) * nt + (f % L) // 64)
    ids = (torch.arange(n, device=dev)[:, None, None] * H + torch.arange(H, device=dev)[None, None, :]) * per + r[None, :,
                                                                                                                  None]

    def label(i):
        bh, rr = divmod(i, per)
        return f"(b={bh // H}, h={bh % H}, {'global rows' if rr == T * nt else f't={rr // nt}, tile={rr % nt}'})"
    return ids.reshape(n * S, H), label


def _vip_case(dev, case, B, H, T, L, M, seed):
    """Forward and backward of B samples repeating PS distinct ones: out, lse and dqkv of every sample have the bits of a
    PS-sample run, which is held to vip_ref under the calibrated slice rule."""
    ops = _ops()
    C, S = 64 * H, M + T * L
    qs = 64 ** -0.5
    qb, db = _vip_base(dev, PS, H, T, L, M, seed)
    ex = A.vip_ref(qb, db, PS, H, T, L, M, q_scale=qs)
    arm = A.vip_ref(qb, db, PS, H, T, L, M, q_scale=qs, arm="vip")
    ids, label = _vip_slices(dev, PS, H, T, L, M)
    idc = ids.repeat_interleave(64, dim=1)
    o_s, l_s = Out(dev, PS * S, C, bf16), Out(dev, PS * H, S, f32)
    ws = ops.vip_attention_workspace(PS, H, T, M, dev)
    ops.vip_attention_fwd(qb, o_s.t, l_s.t, ws, PS, H, T, L, M, C)
    torch.cuda.synchronize()
    ro, rl = o_s.check(f"{case}: representative out"), l_s.check(f"{case}: representative lse")
    calibrated(REPORT, f"{case}: representative out", ro, ex["out"], arm["out"], idc, label, ABS_FLOOR)
    lse_check(REPORT, f"{case}: representative", rl.view(PS, H, S), ex["lse"])
    out_in, lse_in = ex["out"].to(bf16), ex["lse"].float()        # the backward reads the exact forward, as stored
    dq_s = Out(dev, PS * S, 3 * C, bf16)
    ops.vip_attention_bwd(qb, out_in, db, lse_in.contiguous(), dq_s.t, ws, PS, H, T, L, M, C, qs)
    torch.cuda.synchronize()
    rdq = dq_s.check(f"{case}: representative dqkv")
    for j, nm in enumerate(("dq", "dk", "dv")):
        cs = slice(j * C, (j + 1) * C)
        calibrated(REPORT, f"{case}: representative {nm}", rdq[:, cs], ex["dqkv"][:, cs], arm["dqkv"][:, cs], idc, label,
                   ABS_FLOOR)
    del ex, arm, ids, idc, ws
    no_aliasing(f"{case} qkv / dqkv", PS * S, 3 * C, 2, B * S * 3 * C * 2)
    no_aliasing(f"{case} out / dout", PS * S, C, 2, B * S * C * 2)
    qkv = periodic(qb, B * S)
    out, lse = Big(dev, (B * S, C), bf16), Big(dev, (B, H, S), f32)
    crossing(REPORT, case, "qkv", qkv, "2^31 bytes")
    ws = ops.vip_attention_workspace(B, H, T, M, dev)
    ops.vip_attention_fwd(qkv, out.t, lse.t, ws, B, H, T, L, M, C)
    torch.cuda.synchronize()
    same_as_representatives(f"{case}: out per sample", out.check(f"{case}: out").view(B, -1), ro.view(PS, -1))
    same_as_representatives(f"{case}: lse per sample", lse.check(f"{case}: lse").view(B, -1), rl.view(PS, -1))
    del lse
    periodic(out_in.view(PS, -1), B, out=out.t.view(B, -1))
    dout = periodic(db, B * S)
    lse_b = periodic(lse_in.view(PS, -1), B).view(B, H, S)
    dqkv = Big(dev, (B * S, 3 * C), bf16)
    crossing(REPORT, case, "dqkv", dqkv.t, "2^31 bytes")
    ops.vip_attention_bwd(qkv, out.t, dout, lse_b, dqkv.t, ws, B, H, T, L, M, C, qs)
    torch.cuda.synchronize()
    same_as_representatives(f"{case}: dqkv per sample", dqkv.check(f"{case}: dqkv").view(B, -1), rdq.view(PS, -1))
    del qkv, out, dout, lse_b, dqkv, ws
    peak(dev, case)


def test_vip_attention_staged(dev):
    """vip_attention.cu at B = 128, H = 12, T = 32, L = 196, M = 4: qkv and dqkv [803,328 x 2304] (3.70 GB)."""
    case = "ViP staged B128 T32"
    room(dev, case, 12.0)
    _vip_case(dev, case, B_, H_, T_, L_, M_, 12)


def test_vip_attention_streamed_long_frames(dev):
    """vip_attention_long.cu at L/14-336 widths (C = 1024, H = 16, L = 576, M = 4), B = 40, T = 16: qkv and dqkv
    [368,800 x 3072] (2.27 GB)."""
    case = "ViP streamed L14-336 B40 T16"
    room(dev, case, 9.0)
    _vip_case(dev, case, 40, 16, 16, 576, 4, 13)
