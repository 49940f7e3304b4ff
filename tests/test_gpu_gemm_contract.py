"""H100: xp_gemm against the float64 reference of oracle/gemm_ref.py (pinned to F.linear / the oracle's activations / autograd
by test_gemm_reference_cpu.py), slice by slice and element by element, plus exact checks.

  calibrated   bf16 outputs and the saved pre-activation: per slice, ||got - exact|| <= 1.5 x ||arm - exact|| + 2^-16 x the
               slice's reference norm, where the arm rounds to bf16 exactly where the kernel does.  A slice is one
               consumer's 64-row x 128-column accumulator block: (m_blk, n_blk, mh) of a ping-pong 128 x 128 tile,
               (m_blk, n_blk, cw, h) of a cooperative 128 x 256 tile, i.e. (row // 64, col // 128) under both schedules
  element      every output element: |got - exact| <= the fp32 accumulation bound (K_split + splits) 2^-24 sum|a b| through
               the epilogue, its fp32 roundings and MUFU approximation, and one bf16 ulp (gemm_ref.gemm_element_bound);
               fp32 and split-K atomic outputs get only this rule (their arm error is zero)
  coverage     outputs live in NaN-filled buffers with guard rows, pad columns for ld > N and a bit pattern elsewhere; the
               split-K atomic output starts at a known non-zero value and must end at start + product
  locality     NaN in everything a launch must not read (A / B pad columns up to lda / ldb, rows past M / N, residual /
               aux pad columns, the bias tail): the result is finite and bit-identical to a run with clean padding
  repeatable   non-atomic outputs are bit-identical across calls and across set_sm_limit(1), (7), (0)
"""
import zlib

import pytest
import torch

from contract_harness import Out, Report, calibrated, same_bits, tile_slices, within
from oracle import gemm_ref as R

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
REPORT = Report("GEMM: worst slice ratio err(kernel) / err(bf16 arm); element: worst |err| / bound; tail: worst relative "
                "error", width=78)
NONE, QG, DQG, GE, DGE = R.ACT_NONE, R.ACT_QUICK_GELU, R.ACT_DQUICK_GELU, R.ACT_GELU_ERF, R.ACT_DGELU_ERF
ACT_NAME = {NONE: "none", QG: "QuickGELU", DQG: "dQuickGELU", GE: "GELU", DGE: "dGELU"}


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


def _lib():
    from xpretrain_b200 import _lib
    return _lib


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ============================================================================================ operands
class Operand:
    """A bf16 GEMM operand stored as `layout` says (0: [rows, inner] with pitch ld >= inner; 1: transposed, [inner, rows]
    with pitch ld >= rows), inside an allocation EXTRA rows longer.  `poison()` NaN-fills every element outside the logical
    matrix (pad columns up to ld, rows past the logical ones), `clean()` fills them with finite noise."""
    EXTRA = 5

    def __init__(self, dev, logical, layout, ld, seed):
        self.logical, self.layout, self.ld = logical, layout, ld
        r, c = logical.shape if layout == 0 else logical.T.shape
        assert ld >= c and ld % 8 == 0
        self.buf = torch.zeros(r + self.EXTRA, ld, dtype=bf16, device=dev)
        self.inside = torch.zeros(r + self.EXTRA, ld, dtype=torch.bool, device=dev)
        self.inside[:r, :c] = True
        self.buf[:r, :c] = logical if layout == 0 else logical.T
        self.noise = (torch.randn(self.buf.shape, generator=_gen(seed)) * 4).to(bf16).to(dev)
        self.clean()

    def clean(self):
        self.buf[~self.inside] = self.noise[~self.inside]

    def poison(self):
        self.buf[~self.inside] = float("nan")


def padded(dev, t, ld, fill):
    """t [R, N] inside an [R, ld] buffer whose pad columns hold `fill`; returns the buffer."""
    buf = torch.full((t.shape[0], ld), fill, dtype=t.dtype, device=dev)
    buf[:, :t.shape[1]] = t
    return buf


def rnd(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g) * scale


# ============================================================================================ the harness
def run_gemm(dev, tag, *, M, N, K, block_n, a_layout=0, b_layout=0, lda=None, ldb=None, ldc=None, ldr=None, ld_aux=None,
             act=NONE, out_mode=R.OUT_BF16, bias=False, residual=False, save_pre=False, alpha=1.0, scale_cols=0,
             col_scale=1.0, splits=1, seed=0, a_scale=None, pre_scale=2.0, repeat=True):
    """One launch checked under every rule of the module docstring."""
    ops, lib = _ops(), _lib()
    g = _gen(seed)
    s = K ** -0.25 if a_scale is None else a_scale
    A = rnd(g, M, K, scale=s).to(bf16).to(dev)
    B = rnd(g, N, K, scale=K ** -0.25).to(bf16).to(dev)
    lda = lda or (K if a_layout == 0 else M + (-M) % 8)
    ldb = ldb or (K if b_layout == 0 else N)
    opA, opB = Operand(dev, A, a_layout, lda, seed + 1), Operand(dev, B, b_layout, ldb, seed + 2)
    bias_t = None
    if bias:
        bias_t = torch.full((N + 16,), float("nan"), device=dev)        # the tail beyond N is never read
        bias_t[:N] = rnd(g, N, scale=0.5).to(dev)
    res = rbuf = None
    if residual:
        ldr = ldr or N
        res = rnd(g, M, N).to(bf16).to(dev)
    aux_in = abuf = None
    if act in (DQG, DGE):
        ld_aux = ld_aux or N
        aux_in = rnd(g, M, N, scale=pre_scale).to(bf16).to(dev)
    c0 = None
    if out_mode == R.OUT_F32_ATOMIC:
        c0 = rnd(g, M, N).to(dev)
    ref = R.gemm_ref(A, B, alpha=alpha, bias=None if bias_t is None else bias_t[:N], scale_cols=scale_cols,
                     col_scale=col_scale, act=act, residual=res, aux=aux_in, out_mode=out_mode, c0=c0, arm="kernel")
    ex = R.gemm_ref(A, B, alpha=alpha, bias=None if bias_t is None else bias_t[:N], scale_cols=scale_cols,
                    col_scale=col_scale, act=act, residual=res, aux=aux_in, out_mode=out_mode, c0=c0)
    ldc = ldc or N
    odt = bf16 if out_mode == R.OUT_BF16 else f32

    def launch(pad_fill, sm=0):
        (opA.poison if pad_fill else opA.clean)()
        (opB.poison if pad_fill else opB.clean)()
        fillv = float("nan") if pad_fill else 0.5
        rb = padded(dev, res, ldr, fillv) if res is not None else None
        ab = padded(dev, aux_in, ld_aux, fillv) if aux_in is not None else None
        c = Out(dev, M, N, odt, ldc, init=c0)
        pre = Out(dev, M, N, bf16, ld_aux or N) if save_pre else None
        ops.set_sm_limit(sm)
        try:
            ops.gemm(opA.buf, opB.buf, c.buf, M=M, N=N, K=K, lda=lda, ldb=ldb, ldc=ldc, a_layout=a_layout,
                     b_layout=b_layout, bias=bias_t, residual=rb, ldr=ldr or 0,
                     aux=ab if ab is not None else (pre.buf if pre is not None else None),
                     ld_aux=(ld_aux or N) if (ab is not None or pre is not None) else 0, act=act, out_mode=out_mode,
                     splits=splits, scale_cols=scale_cols, col_scale=col_scale, alpha=alpha, block_n=block_n)
            torch.cuda.synchronize()
        finally:
            ops.set_sm_limit(0)
        return c.check(f"{tag}: C"), (pre.check(f"{tag}: aux (pre-activation)") if pre is not None else None)

    got, pre = launch(True)
    ids, label = tile_slices(M, N, dev)
    kb = (K + 63) // 64
    K_split = min(K, ((kb + splits - 1) // splits) * 64)
    bound = R.gemm_element_bound(ex, K_split, splits, alpha=alpha, col_scale=col_scale, act=act, aux=aux_in, residual=res,
                                 bias=None if bias_t is None else bias_t[:N], c0=c0, out_mode=out_mode)
    within(REPORT, f"{tag}: C element", got, ex["exact"], bound)
    if out_mode == R.OUT_BF16:
        calibrated(REPORT, f"{tag}: C", got, ex["exact"], ref["out"], ids, label)
    if pre is not None:
        calibrated(REPORT, f"{tag}: aux", pre, ex["pre"], ref["pre"], ids, label)
        pb = R.gemm_element_bound(ex, K_split, splits, alpha=alpha, col_scale=col_scale, bias=bias_t[:N] if bias else None)
        pb = pb + R.ulp_bf16(ex["pre"].abs() + pb)
        within(REPORT, f"{tag}: aux element", pre, ex["pre"], pb)
    # locality: clean padding gives the same bits; repeatability across calls and grid sizes (non-atomic outputs)
    if out_mode != R.OUT_F32_ATOMIC:
        got2, pre2 = launch(False)
        assert same_bits(got2, got), f"{tag}: NaN padding of A / B / residual / aux / bias changed C"
        assert pre is None or same_bits(pre2, pre), f"{tag}: NaN padding changed the saved pre-activation"
        if repeat:
            for sm in (1, 7, 0):
                got3, pre3 = launch(True, sm)
                assert same_bits(got3, got), f"{tag}: C not bit-identical with set_sm_limit({sm})"
                assert pre is None or same_bits(pre3, pre), f"{tag}: aux not bit-identical with set_sm_limit({sm})"
    else:
        got2, _ = launch(False)
        within(REPORT, f"{tag}: C (clean padding) element", got2, ex["exact"], bound)
    return got, pre, ex


# ====================================================================== the model's launches at reduced M
MODEL_M = 200      # two 128-row blocks, the second one partial
MODEL = []
for C in (512, 768, 1024):
    for bn in (128, 256):
        MODEL += [
            (f"qkv C{C}", C, bn, dict(N=3 * C, K=C, bias=True, scale_cols=C, col_scale=0.125)),
            (f"out_proj C{C}", C, bn, dict(N=C, K=C, bias=True)),
            (f"out_proj+residual C{C}", C, bn, dict(N=C, K=C, bias=True, residual=True)),
            (f"fc1 QuickGELU C{C}", C, bn, dict(N=4 * C, K=C, bias=True, act=QG, save_pre=True)),
            (f"fc1 GELU C{C}", C, bn, dict(N=4 * C, K=C, bias=True, act=GE, save_pre=True)),
            (f"fc2 C{C}", C, bn, dict(N=C, K=4 * C, bias=True)),
            (f"dgrad fc2 dQuickGELU C{C}", C, bn, dict(N=4 * C, K=C, b_layout=1, act=DQG)),
            (f"dgrad fc2 dGELU C{C}", C, bn, dict(N=4 * C, K=C, b_layout=1, act=DGE)),
            (f"dgrad fc1 C{C}", C, bn, dict(N=C, K=4 * C, b_layout=1)),
        ]


@pytest.mark.parametrize("name,C,bn,kw", MODEL, ids=[f"{m[0].replace(' ', '-')}-bn{m[2]}" for m in MODEL])
def test_gemm_model_launches(dev, name, C, bn, kw):
    run_gemm(dev, f"{name} bn{bn}", M=MODEL_M, block_n=bn, seed=C + bn, **kw)


@pytest.mark.parametrize("C", [512, 768, 1024])
def test_gemm_wgrad_accumulates_into_grad(dev, C):
    """ops.linear_wgrad at the wgrad_plan split: dW [N, K] += dy^T x over `rows` tokens, both operands MN-major, fp32
    atomics into a .grad that already holds a value."""
    ops = _ops()
    rows = 4096
    for n_out, n_in, nm in ((3 * C, C, "qkv"), (4 * C, C, "fc1"), (C, 4 * C, "fc2")):
        tag = f"wgrad {nm} C{C}"
        g = _gen(C + n_out)
        dy = rnd(g, rows, n_out, scale=0.5).to(bf16).to(dev)
        x = rnd(g, rows, n_in).to(bf16).to(dev)
        c0 = rnd(g, n_out, n_in).to(dev)
        bn, splits = ops.wgrad_plan(n_out, n_in, rows)
        dw = Out(dev, n_out, n_in, f32, init=c0)
        ops.linear_wgrad(dy, x, dw.t)
        torch.cuda.synchronize()
        got = dw.check(tag)
        ex = R.gemm_ref(dy.T, x.T, out_mode=R.OUT_F32_ATOMIC, c0=c0)
        kb = (rows + 63) // 64
        K_split = ((kb + splits - 1) // splits) * 64
        within(REPORT, f"{tag} splits{splits} bn{bn}: dW element", got, ex["exact"],
               R.gemm_element_bound(ex, K_split, splits, c0=c0, out_mode=R.OUT_F32_ATOMIC))


# ================================================================================================ edges
EDGES = []
for bn in (128, 256):
    EDGES += [(f"M{m}", bn, dict(M=m, N=264, K=520, bias=True)) for m in (1, 63, 64, 65, 129)]
    EDGES += [(f"N{n}", bn, dict(M=129, N=n, K=520, bias=True)) for n in (8, 120, 136, 248, 264)]
    EDGES += [(f"K{k}", bn, dict(M=129, N=264, K=k, bias=True)) for k in (8, 56, 72, 520)]
    EDGES += [
        ("ldc ldr ld_aux > N", bn, dict(M=129, N=136, K=72, ldc=152, ldr=168, residual=True, bias=True)),
        ("ldc ld_aux > N QuickGELU", bn, dict(M=129, N=136, K=72, ldc=144, ld_aux=160, act=QG, save_pre=True, bias=True)),
        ("ld_aux > N dGELU", bn, dict(M=129, N=136, K=72, ldc=152, ld_aux=176, b_layout=1, act=DGE)),
        ("lda ldb > K", bn, dict(M=129, N=136, K=72, lda=88, ldb=96, bias=True)),
        ("lda ldb > M N (MN-major)", bn, dict(M=129, N=136, K=72, a_layout=1, b_layout=1, lda=152, ldb=160)),
        ("a MN-major b K-major", bn, dict(M=65, N=264, K=520, a_layout=1, b_layout=0, lda=80, ldb=528)),
        ("bias split-K 3", bn, dict(M=129, N=264, K=520, bias=True, out_mode=R.OUT_F32_ATOMIC, splits=3)),
        ("residual OUT_F32", bn, dict(M=129, N=136, K=520, residual=True, ldr=144, out_mode=R.OUT_F32, bias=True)),
        ("alpha -0.37 bf16", bn, dict(M=129, N=264, K=520, alpha=-0.37, bias=True)),
    ]
    EDGES += [(f"scale_cols {sc}", bn, dict(M=129, N=264, K=72, bias=True, scale_cols=sc, col_scale=0.125))
              for sc in (2, 136, 200)]


@pytest.mark.parametrize("name,bn,kw", EDGES, ids=[f"{e[0].replace(' ', '-')}-bn{e[1]}" for e in EDGES])
def test_gemm_edges(dev, name, bn, kw):
    run_gemm(dev, f"edge {name} bn{bn}", block_n=bn, seed=zlib.crc32(name.encode()) % 1000, **kw)


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("a_layout,b_layout", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_gemm_layouts_with_poisoned_padding(dev, a_layout, b_layout, bn):
    """Both layouts of both operands, each with a pitch beyond its logical inner dimension and NaN in every pad element."""
    M, N, K = 129, 264, 136
    run_gemm(dev, f"layouts a{a_layout} b{b_layout} bn{bn}", M=M, N=N, K=K, block_n=bn, a_layout=a_layout,
             b_layout=b_layout, lda=(152 if a_layout == 0 else 144), ldb=(160 if b_layout == 0 else 280), bias=True,
             seed=a_layout * 2 + b_layout)


# ================================================================================== patch embed, NCE head
@pytest.mark.parametrize("patch", [16, 14], ids=["K768", "K588-pitch592"])
def test_gemm_patch_embed_grouped(dev, patch):
    """The patch-embedding launch (clip_vip.py): rows of T*L patches per video written past the M global rows of each
    [S, C] sample (c_group), plus the periodic position + temporal table (r_group, r_group_stride = 0)."""
    ops = _ops()
    Bv, T, L, Mg, C = 2, 3, 49, 4, 768
    S, Kp = Mg + T * L, 3 * patch * patch
    ldp = ops.patch_pitch(patch)
    g = _gen(patch)
    P = rnd(g, Bv * T * L, Kp, scale=Kp ** -0.25).to(bf16).to(dev)
    W = rnd(g, C, Kp, scale=Kp ** -0.25).to(bf16).to(dev)
    table = rnd(g, T * L, C).to(bf16).to(dev)
    opP, opW = Operand(dev, P, 0, ldp, 1), Operand(dev, W, 0, ldp, 2)
    ref_rows = R.gemm_ref(P, W, residual=table.repeat(Bv, 1), arm="kernel")
    ex = R.gemm_ref(P, W, residual=table.repeat(Bv, 1))

    def launch(poison):
        (opP.poison if poison else opP.clean)()
        (opW.poison if poison else opW.clean)()
        x0 = Out(dev, Bv * S, C, bf16)
        glob = torch.zeros(Bv * S, dtype=torch.bool, device=dev)
        glob.view(Bv, S)[:, :Mg] = True
        x0.outside[:Bv * S][glob] = True        # the global rows are not this launch's to write
        x0.buf[:Bv * S][glob] = 0.25
        x0.snap = x0.buf.view(torch.int16).clone()
        x0.t = x0.buf[:Bv * S].view(Bv, S, C)[:, Mg:]
        ops.gemm(opP.buf, opW.buf, x0.buf, M=Bv * T * L, N=C, K=Kp, lda=ldp, ldb=ldp, ldc=C, residual=table, ldr=C,
                 r_group=T * L, r_group_stride=0, c_group=T * L, c_group_stride=S * C, c_offset=Mg * C)
        torch.cuda.synchronize()
        return x0.check(f"patch{patch}").reshape(Bv * T * L, C)
    got = launch(True)
    tag = f"patch-embed K{Kp} ld{ldp}"
    ids, label = tile_slices(Bv * T * L, C, dev)
    calibrated(REPORT, f"{tag}: x0", got, ex["exact"], ref_rows["out"], ids, label)
    within(REPORT, f"{tag}: x0 element", got, ex["exact"], R.gemm_element_bound(ex, Kp, 1, residual=table.repeat(Bv, 1)))
    assert same_bits(launch(False), got), f"{tag}: NaN pad columns / rows changed the output"


def test_gemm_nce_head_launches(dev):
    """The InfoNCE gradient GEMMs of optimization/loss.py: OUT_F32, alpha = scale, A = g [N, Np] with lda = Np > K = N, as a
    row window of a K-major A and as a column window (a_offset) of an MN-major A; and the projection head's OUT_F32."""
    ops = _ops()
    N, Np, d, r0, rows = 40, 48, 256, 8, 24
    g = _gen(9)
    G = rnd(g, N, Np).to(bf16).to(dev)
    G[:, N:] = float("nan")                            # pad columns of g beyond K = N are never read
    T = rnd(g, N, d).to(bf16).to(dev)                  # B stored [K = N, d]: MN-major
    scale = 14.3
    for bn in (128, 256):
        out = Out(dev, rows, d, f32)
        ops.gemm(G, T, out.buf, M=rows, N=d, K=N, lda=Np, ldb=d, ldc=d, b_layout=1, out_mode=R.OUT_F32, alpha=scale,
                 a_offset=r0 * Np, block_n=bn)
        torch.cuda.synchronize()
        got = out.check("nce dX")
        ex = R.gemm_ref(G[r0:r0 + rows, :N], T.T, alpha=scale, out_mode=R.OUT_F32)
        within(REPORT, f"nce dX bn{bn}: dX element", got, ex["exact"],
               R.gemm_element_bound(ex, N, 1, alpha=scale, out_mode=R.OUT_F32))
        # d_txt: A = g^T as an MN-major window: column r0.. of g's rows, K = N rows of pitch Np
        Gm = rnd(g, N, Np).to(bf16).to(dev)
        Gm[:, :r0] = float("nan")
        Gm[:, r0 + rows:] = float("nan")
        out = Out(dev, rows, d, f32)
        ops.gemm(Gm, T, out.buf, M=rows, N=d, K=N, lda=Np, ldb=d, ldc=d, a_layout=1, b_layout=1, out_mode=R.OUT_F32,
                 alpha=scale, a_offset=r0, block_n=bn)
        torch.cuda.synchronize()
        got = out.check("nce dY")
        ex = R.gemm_ref(Gm[:, r0:r0 + rows].T, T.T, alpha=scale, out_mode=R.OUT_F32)
        within(REPORT, f"nce dY a_offset bn{bn}: dY element", got, ex["exact"],
               R.gemm_element_bound(ex, N, 1, alpha=scale, out_mode=R.OUT_F32))
    # projection head: fp32 features of pooled bf16 rows
    run_gemm(dev, "projection OUT_F32", M=5, N=256, K=768, block_n=128, out_mode=R.OUT_F32, seed=3)


# ======================================================================================= epilogue sweep
def _all_finite_bf16(dev):
    """Every finite bf16 value (65 280 of them, both zeros included), padded to 64 x 1024 with zeros."""
    bits = torch.arange(65536, dtype=torch.int32)
    v = (bits.to(torch.int16)).view(bf16)
    v = v[torch.isfinite(v.float())]
    assert v.numel() == 65280
    full = torch.zeros(64 * 1024, dtype=bf16)
    full[:v.numel()] = v
    return full.view(64, 1024).to(dev), v.numel()


@pytest.mark.parametrize("act", [QG, GE, DQG, DGE], ids=[ACT_NAME[a] for a in (QG, GE, DQG, DGE)])
def test_gemm_epilogue_sweep_every_bf16_value(dev, act):
    """The activation isolated from the MMA: A = the 64 x 64 identity (K = 64) and B^T holds every finite bf16 value, so
    the fp32 accumulator is exactly that value (forward GELUs); for the dGELU epilogues B is all ones and aux holds the
    sweep.  Every element against the float64 function, within one bf16 ulp plus the documented approximation error:
    |x| 2^-12 (QuickGELU), (1 + 1.702 |x|) 2^-12 (dQuickGELU), a few fp32 ulps of erff / __expf (GELU)."""
    ops = _ops()
    vals, n = _all_finite_bf16(dev)
    eye = torch.eye(64, dtype=bf16, device=dev)
    Bt = vals.T.contiguous() if act in (QG, GE) else torch.ones(1024, 64, dtype=bf16, device=dev)   # [N, K]
    aux = vals.clone() if act in (DQG, DGE) else torch.empty(64, 1024, dtype=bf16, device=dev)
    for bn in (128, 256):
        c = Out(dev, 64, 1024, bf16)
        ops.gemm(eye, Bt, c.buf, M=64, N=1024, K=64, lda=64, ldb=64, ldc=1024, act=act, aux=aux, ld_aux=1024, block_n=bn)
        torch.cuda.synchronize()
        got = c.check(f"sweep {ACT_NAME[act]}").reshape(-1)[:n].double()
        x = vals.reshape(-1)[:n].double()
        if act in (QG, GE):
            pre, v = aux.reshape(-1)[:n].float(), vals.reshape(-1)[:n].float()
            normal = v.abs() >= 2.0 ** -126                 # fp32 denormals flush to zero (--use_fast_math)
            assert bool((pre == v)[normal].all()), "the stored pre-activation is not the accumulator value"
        big = x.abs() < 3.0e38                      # |x| beyond this: the exact results are +-inf / 0 (see below)
        u = 2.0 ** -24
        if act == QG:
            want, approx = R.quick_gelu(x), x.abs() * 2.0 ** -12
        elif act == GE:
            want, approx = R.gelu(x), 8 * u * (x.abs() + 1.0)
        elif act == DQG:
            want, approx = R.quick_gelu_grad(x), (1.0 + 1.702 * x.abs()) * 2.0 ** -12
        else:
            want, approx = R.gelu_grad(x), 8 * u * (1.0 + x.abs())
        want_c = want.clamp(-3.3e38, 3.3e38)
        assert bool(torch.isfinite(got).all()), f"sweep {ACT_NAME[act]}: non-finite outputs"
        err = (got - want_c).abs()
        # + |want| below 2^-125: fp32 denormal results flush to zero (--use_fast_math)
        bound = approx + R.ulp_bf16(want_c.abs() + approx) + torch.where(want_c.abs() < 2.0 ** -125, want_c.abs(), 0.0)
        bound = bound + 2.0 ** -133
        bad = (err > bound) & big
        w = int((err / bound * big).argmax())
        assert not bool(bad.any()), (f"sweep {ACT_NAME[act]} bn{bn}: {int(bad.sum())} values out of bound, worst x = "
                                     f"{float(x[w]):.6e}: got {float(got[w]):.6e}, want {float(want[w]):.6e}")
        tail = (x >= -10) & (x <= -3)
        rel = (err / want.abs().clamp_min(1e-300))[tail]
        REPORT.record(f"sweep {ACT_NAME[act]}: worst relative error on x in [-10, -3]", float(rel.max()))
        REPORT.record(f"sweep {ACT_NAME[act]}: worst relative error on x in [-5, -3]", float(rel[x[tail] >= -5].max()))
        REPORT.record(f"sweep {ACT_NAME[act]}: worst |err| / |x| on x in [-10, -3]", float((err / x.abs())[tail].max()))
        REPORT.record(f"sweep {ACT_NAME[act]}: worst |err| / bound", float((err / bound)[big].max()))


def test_dquick_gelu_at_the_ends_of_bf16_range(dev):
    """dQuickGELU of a saved pre-activation of +-3.3e38 (finite in bf16): the exact derivative, 1 and 0, not NaN."""
    ops = _ops()
    eye = torch.eye(64, dtype=bf16, device=dev)
    ones = torch.ones(128, 64, dtype=bf16, device=dev)
    aux = torch.zeros(64, 128, dtype=bf16, device=dev)
    aux[:, 0::2], aux[:, 1::2] = 3.3e38, -3.3e38
    c = Out(dev, 64, 128, bf16)
    ops.gemm(eye, ones, c.buf, M=64, N=128, K=64, lda=64, ldb=64, ldc=128, act=DQG, aux=aux, ld_aux=128)
    torch.cuda.synchronize()
    got = c.check("dQuickGELU +-3.3e38").float()
    assert bool((got[:, 0::2] == 1).all()) and bool((got[:, 1::2] == 0).all()), got[0, :4]


# ==================================================================================== contract checks
def test_gemm_rejects_unimplemented_epilogue_combinations(dev):
    """Combinations the epilogue would silently compute differently are refused before launch: a residual with any
    activation (the residual add is an alternative to the activation), aux with grouped rows (aux is addressed row *
    ld_aux), an odd scale_cols (tested once per column pair).  Buffers are sized for the plain addressing, so a launch
    that went ahead would stay in bounds."""
    from xpretrain_b200._lib import XpError
    ops = _ops()
    M, N, K = 64, 128, 64
    a = torch.randn(M, K, device=dev).to(bf16)
    b = torch.randn(N, K, device=dev).to(bf16)
    c = torch.zeros(2 * M, N, dtype=bf16, device=dev)
    r = torch.randn(2 * M, N, device=dev).to(bf16)
    aux = torch.zeros(2 * M, N, dtype=bf16, device=dev)
    for act in (QG, GE):
        with pytest.raises(XpError):
            ops.gemm(a, b, c, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, residual=r, ldr=N, act=act, aux=aux, ld_aux=N)
        with pytest.raises(XpError):
            ops.gemm(a, b, c, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, residual=r, ldr=N, act=act)
    with pytest.raises(XpError):
        ops.gemm(a, b, c, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, act=QG, aux=aux, ld_aux=N, c_group=32, c_group_stride=64 * N)
    for sc in (1, 3, 135):
        with pytest.raises(XpError):
            ops.gemm(a, b, c, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, scale_cols=sc, col_scale=0.5)
    torch.cuda.synchronize()


def test_quick_gelu_realistic_tail_calibrated_against_autocast(dev):
    """fc1 + QuickGELU on realistic pre-activations N(0, sigma), sigma 1 and 3 (a third of them in the MUFU sigmoid's
    negative tail for sigma = 3): per slice, the kernel against the float64 function is held to 1.5 x the error of the
    reference's own bf16 autocast arithmetic (gemm_ref arm 'torch_bf16')."""
    ops = _ops()
    M, C = 256, 768
    N = 4 * C
    for sigma in (1.0, 3.0):
        for bn in (128, 256):
            g = _gen(int(sigma) * 10 + bn)
            A = rnd(g, M, C, scale=C ** -0.25).to(bf16).to(dev)
            B = rnd(g, N, C, scale=sigma * C ** -0.25).to(bf16).to(dev)
            c, pre = Out(dev, M, N, bf16), Out(dev, M, N, bf16)
            ops.gemm(A, B, c.buf, M=M, N=N, K=C, lda=C, ldb=C, ldc=N, act=QG, aux=pre.buf, ld_aux=N, block_n=bn)
            torch.cuda.synchronize()
            got = c.check("fc1 realistic")
            ex = R.gemm_ref(A, B, act=QG)
            arm = R.gemm_ref(A, B, act=QG, arm="torch_bf16")
            ids, label = tile_slices(M, N, dev)
            calibrated(REPORT, f"fc1 QuickGELU N(0,{sigma:g}) bn{bn}: C vs autocast arm", got, ex["exact"], arm["out"], ids,
                       label)
            tail = ex["pre"] < -4.0 / 1.702
            rel = ((got.double() - ex["exact"]).abs() / ex["exact"].abs().clamp_min(1e-300))[tail]
            REPORT.record(f"fc1 QuickGELU N(0,{sigma:g}): worst relative error where 1.702 x < -4", float(rel.max()))
