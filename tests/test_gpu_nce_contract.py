"""H100: the contrastive-loss kernels against the float64 references of oracle/nce_ref.py (pinned to the autograd oracles
and the reference-class goldens by test_nce_reference_cpu.py), slice by slice and element by element, plus exact checks.

  calibrated   one slicing everywhere, (row // 64, col // 128): one warpgroup's half of a fused 128 x 128 tile, one
               64 x 128 tile of nce.cu, one consumer block of the gradient GEMMs.  Per slice,
               ||got - exact|| <= 1.5 x ||arm - exact|| + 2^-16 x ||exact||, on s dL/dZ of every path and on the feature
               gradients of the backward
  element      every element of s dL/dZ within nce_ref's derived bound; loss and d logit_scale within theirs
  coverage     outputs live in NaN-filled buffers with guard rows and bit-patterned pad columns: the fused kernel writes
               exactly the N x N block of g_scaled and all of vis_hi / txt_hi; xp_nce_terms / xp_nce_dsl write zeros in
               columns [n, ceil4(n)) and nothing beyond; the logits' pad columns hold NaN and are never used
  workspace    NaN-filled workspaces give bit-identical results (for the fused kernel, its partials, with the three
               counters zero); the fused kernel's counters read back zero after every call
  repeatable   loss, d logit_scale and s dL/dZ are bit-identical across calls on every path; the exchange (mode 0) on
               every simulated rank is bit-identical to the pre-gathered mode 1 on the same rows
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from contract_harness import Out, Report, calibrated, same_bits, tile_slices, within
from oracle import nce_ref as R

pytestmark = pytest.mark.gpu

bf16, f32, F64 = torch.bfloat16, torch.float32, torch.float64
REPORT = Report("NCE: worst slice ratio err(kernel) / err(bf16 arm); element / scalar: worst |err| / bound")
LOG_SCALES = (0.0, 2.659, 4.6052)      # s = 1, the CLIP initialisation, the drivers' clamp at 100
TABLES = ("NCEContrastiveLoss", "VidImgDivideNCELearnableTempLoss", "NCELearnableTempLoss_vs_vc",
          "NCELearnableTempLoss_vs_vc_fc", "NCELearnableTempLoss_vsc", "NCELearnableTempLoss_vsc_fc")
KINDS = ("seeded", "bf16", "adversarial")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    REPORT.print()


def _lib():
    from xpretrain_b200 import _lib
    return _lib


def _ops():
    from xpretrain_b200 import ops
    return ops


def _loss():
    from xpretrain_b200.optimization import loss
    return loss


def ceil4(n):
    return (n + 3) // 4 * 4


def ceil8(n):
    return (n + 7) // 8 * 8


# ============================================================================================ the rules
def tiled(tag, name, got, exact, arm):
    """The calibrated rule per (row // 64, col // 128) slice."""
    calibrated(REPORT, f"{tag}: {name}", got, exact, arm, *tile_slices(*exact.shape, exact.device))


def scalar(tag, name, got, exact, bound):
    err = abs(float(got) - float(exact))
    REPORT.record(f"{tag}: {name}", err / float(bound))
    assert err <= float(bound), f"{tag}: {name} {float(got):.8g} vs exact {float(exact):.8g}: |err| {err:.3e} > {float(bound):.3e}"


def check_sg(tag, got, ref, k=0, name="s dL/dZ"):
    tiled(tag, name, got, ref["exact"][k], ref["arm"][k])
    within(REPORT, f"{tag}: {name} element", got, ref["exact"][k], ref["bound"][k])


def check_scalars(tag, loss, dscale, ref):
    scalar(tag, "loss", loss, ref["loss"], ref["loss_bound"])
    if dscale is not None:
        scalar(tag, "d logit_scale", dscale, ref["dscale"], ref["dscale_bound"])


# ============================================================================================ features
def features(n, d, kind, seed, base=None):
    """fp32 [n, d] unit-norm rows.  seeded: N(0, 1) rows (correlated with `base` when given); bf16: the same rounded to
    bf16, so that lo = 0; adversarial: seeded, plus a duplicated row (ties), a near-one-hot row (with its near-one-hot
    partner in `base`: at s = 100 every off-diagonal probability of its row and column underflows and G is tiny) and a
    last row equal to the mean of the others."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, d, generator=g)
    if base is not None:
        x = x + 0.5 * base.cpu()
    x = F.normalize(x, dim=-1)
    if kind == "bf16":
        x = x.to(bf16).float()
    elif kind == "adversarial" and n >= 5:
        x[1] = x[0]
        e = torch.zeros(d)
        e[3] = 1.0
        x[2] = F.normalize(e + 1e-3 * torch.randn(d, generator=g), dim=0)
        x[n - 1] = x[:n - 1].mean(0)
    return x


def pair(n, d, kind, seed):
    v = features(n, d, kind, seed)
    t = features(n, d, kind, seed + 1, base=v)
    if kind == "adversarial" and n >= 5:
        t[1] = t[0]
        t[2] = v[2]
        t[n - 1] = t[:n - 1].mean(0)
    return v, t


def scale_ls(dev, ls):
    return torch.tensor([ls], dtype=f32, device=dev)


# ============================================================================================ fused kernel
def fused_ws(dev, N):
    """The fused kernel's workspace and the float offset of its three counters (nce_fused.cu:410-414)."""
    nt = (N + 127) // 128
    return _ops().nce_gather_workspace(N, dev), 4 * nt * nt * 128 + 2 * nt * nt


def poison_ws(ws, off):
    ws[:off] = float("nan")
    ws[off:off + 3].view(torch.int32).zero_()


def counters(ws, off):
    return ws[off:off + 3].view(torch.int32).tolist()


def launch_fused(dev, *, world, b, d, peers, ls, ws, off, ld_g, mode=1, rank=0, epoch=0, vis_local=None, txt_local=None):
    """One xp_nce_gather_fused call into NaN-filled outputs; returns (loss, dscale, g [N, N], vis_hi, txt_hi)."""
    N = world * b
    assert counters(ws, off) == [0, 0, 0], "the counters must be zero before a launch"
    g, vh, th = Out(dev, N, N, bf16, ld_g), Out(dev, N, d, bf16), Out(dev, N, d, bf16)
    loss = torch.full((1,), float("nan"), device=dev)
    dscale = torch.full((1,), float("nan"), device=dev)
    assert g.buf.stride(0) == ld_g
    _ops().nce_gather_fused(vis_local, txt_local, peers, ls, g.buf, vh.buf, th.buf, loss, dscale, ws, rank=rank, world=world,
                            b=b, d=d, epoch=epoch, mode=mode)
    torch.cuda.synchronize()
    assert counters(ws, off) == [0, 0, 0], "the fused kernel left its counters non-zero"
    return (loss.clone(), dscale.clone(), g.check("fused g_scaled"), vh.check("fused vis_hi"), th.check("fused txt_hi"))


def same_outputs(a, b):
    return all(same_bits(x, y) for x, y in zip(a, b))


def check_backward(tag, g, vh, th, V, T, ref, row0=0, nrows=None, scale=1.0):
    """_nce_backward's rows [row0, row0 + nrows) of dV, dT against `scale` x the float64 gradient, per 64-row block."""
    XL = _loss()
    N = V.shape[0]
    nrows = N if nrows is None else nrows
    d_vis, d_txt = XL._nce_backward(g, vh, th, row0, nrows, scale)
    torch.cuda.synchronize()
    ex = R.feature_grads(((0, 1),), ref["exact"], [V, T])
    arm = R.feature_grads(((0, 1),), ref["arm"], [R.bf(V), R.bf(T)])
    rows = slice(row0, row0 + nrows)
    tiled(tag, "dV", d_vis, scale * ex[0][rows], scale * arm[0][rows])
    tiled(tag, "dT", d_txt, scale * ex[1][rows], scale * arm[1][rows])


FUSED = [  # (world, b, d, kind, log-scale)
    (1, 1, 64, "seeded", 0.0), (1, 127, 256, "bf16", 2.659), (1, 128, 512, "adversarial", 4.6052),
    (1, 129, 768, "seeded", 4.6052), (1, 255, 1024, "adversarial", 2.659), (1, 256, 64, "bf16", 4.6052),
    (1, 257, 512, "adversarial", 0.0), (1, 1408, 512, "seeded", 4.6052), (1, 1409, 256, "adversarial", 4.6052),
    (1, 1536, 1024, "bf16", 2.659), (43, 3, 512, "adversarial", 4.6052), (51, 5, 256, "seeded", 2.659),
    (8, 64, 768, "adversarial", 4.6052), (3, 5, 1024, "bf16", 0.0),
]


@pytest.mark.parametrize("world,b,d,kind,ls", FUSED, ids=[f"w{c[0]}-b{c[1]}-d{c[2]}-{c[3]}-ls{c[4]}" for c in FUSED])
def test_fused_kernel_mode1(dev, world, b, d, kind, ls):
    """N = 1 to 1536 (1408: the largest two-stage grid, 11^2 tiles; 1409: the first compact grid), per-rank batches of 3
    and 5 rows, d = 64 to 1024, rows read through the rank-major pointer table."""
    N = world * b
    tag = f"fused N{N} (w{world} b{b}) d{d} {kind} ls{ls}"
    V, T = pair(N, d, kind, seed=N + d)
    Vd, Td = V.to(dev), T.to(dev)
    vis = [Vd[r * b:(r + 1) * b].clone() for r in range(world)]
    txt = [Td[r * b:(r + 1) * b].clone() for r in range(world)]
    peers = torch.tensor([x.data_ptr() for x in vis + txt], dtype=torch.int64, device=dev)
    lsd = scale_ls(dev, ls)
    ws, off = fused_ws(dev, N)
    ld_g = ceil8(N) + (8 if N % 2 else 0)
    kw = dict(world=world, b=b, d=d, peers=peers, ls=lsd, ws=ws, off=off, ld_g=ld_g)
    first = launch_fused(dev, **kw)
    poison_ws(ws, off)
    second = launch_fused(dev, **kw)
    assert same_outputs(first, second), f"{tag}: NaN partials or a second call changed the outputs"
    loss, dscale, g, vh, th = first
    assert same_bits(vh, Vd.to(bf16)) and same_bits(th, Td.to(bf16)), f"{tag}: vis_hi / txt_hi are not bf16 of the rows"
    lg = R.split_logits(Vd, Td)
    ref = R.terms([lg["exact"]], R.INFONCE, R.scale_of(lsd), z_err=[lg["err"]], z_arm=[lg["arm"]],
                  reduce_depth=R.fused_depth(N))
    check_sg(tag, g, ref)
    check_scalars(tag, loss, dscale, ref)
    gfull = torch.zeros(N, ceil8(N), dtype=bf16, device=dev)
    gfull[:, :N] = g
    check_backward(tag, gfull, vh, th, Vd, Td, ref)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("b", [3, 64, 192])
def test_fused_kernel_exchange_mode0_simulated_on_one_gpu(dev, world, b):
    """Mode 0 with the `world` exchange buffers as ordinary allocations on one device.  Before launching as rank r the
    host publishes every other rank's rows in its slot (epoch & 1), raises words k != r of buffer r to the epoch and reads
    them back (every one must be >= the epoch, so the kernel's flag wait returns at once); rank r's own slot and the other
    slot of every buffer hold NaN, so a missing or misplaced publish and a wrong-slot read show.  Epochs 1-3 with fresh
    rows, each as every rank: the outputs are bit-identical on every rank and to mode 1 on the same rows, the kernel
    publishes rank r's rows, and rank r's backward rows match `world` x the global gradient."""
    d = 256
    N = world * b
    tag = f"mode0 w{world} b{b}"
    nbytes = _ops().nce_gather_exchange_bytes(b, d, world)
    slot = 2 * b * d                                       # floats per slot: [vis b x d | txt b x d]
    bufs = [torch.zeros(nbytes // 4, dtype=f32, device=dev) for _ in range(world)]
    table = torch.tensor([x.data_ptr() for x in bufs], dtype=torch.int64, device=dev)
    lsd = scale_ls(dev, 4.6052)
    wss = [fused_ws(dev, N) for _ in range(world)]
    ld_g = ceil8(N)

    def slot_view(k, parity):
        return bufs[k][256 + parity * slot:256 + (parity + 1) * slot]

    for epoch in (1, 2, 3):
        V, T = pair(N, d, "adversarial" if epoch == 2 else "seeded", seed=100 * epoch + N)
        Vd, Td = V.to(dev), T.to(dev)
        vis = [Vd[r * b:(r + 1) * b].clone() for r in range(world)]
        txt = [Td[r * b:(r + 1) * b].clone() for r in range(world)]
        peers = torch.tensor([x.data_ptr() for x in vis + txt], dtype=torch.int64, device=dev)
        ws1, off1 = fused_ws(dev, N)
        want = launch_fused(dev, world=world, b=b, d=d, peers=peers, ls=lsd, ws=ws1, off=off1, ld_g=ld_g)
        par = epoch & 1
        for r in range(world):
            for k in range(world):
                slot_view(k, 1 - par).fill_(float("nan"))
                if k == r:
                    slot_view(k, par).fill_(float("nan"))
                else:
                    slot_view(k, par).copy_(torch.cat([vis[k].reshape(-1), txt[k].reshape(-1)]))
            flags = bufs[r][:256].view(torch.int32)
            for k in range(world):
                if k != r:
                    flags[k] = epoch
            torch.cuda.synchronize()
            raised = flags[:world].tolist()
            assert all(raised[k] >= epoch for k in range(world) if k != r), f"{tag}: flags {raised} below epoch {epoch}"
            ws, off = wss[r]
            poison_ws(ws, off)
            got = launch_fused(dev, world=world, b=b, d=d, peers=table, ls=lsd, ws=ws, off=off, ld_g=ld_g, mode=0,
                               rank=r, epoch=epoch, vis_local=vis[r], txt_local=txt[r])
            assert same_outputs(got, want), f"{tag} epoch {epoch} rank {r}: outputs differ from mode 1 on the same rows"
            mine = torch.cat([vis[r].reshape(-1), txt[r].reshape(-1)])
            assert same_bits(slot_view(r, par), mine), f"{tag} epoch {epoch} rank {r}: its rows were not published"
            assert int(bufs[r][:256].view(torch.int32)[r]) == epoch, f"{tag}: rank {r} did not raise its own flag"
    loss, dscale, g, vh, th = want
    lg = R.split_logits(Vd, Td)
    ref = R.terms([lg["exact"]], R.INFONCE, R.scale_of(lsd), z_err=[lg["err"]], z_arm=[lg["arm"]],
                  reduce_depth=R.fused_depth(N))
    check_sg(tag, g, ref)
    check_scalars(tag, loss, dscale, ref)
    gfull = torch.zeros(N, ld_g, dtype=bf16, device=dev)
    gfull[:, :N] = g
    for r in range(world):
        check_backward(f"{tag} rank {r}", gfull, vh, th, Vd, Td, ref, row0=r * b, nrows=b, scale=float(world))


def test_fused_forward_aligns_a_misaligned_view(dev, monkeypatch):
    """A contiguous view 4 bytes into its allocation: _nce_forward_fused hands the kernel 16-byte aligned rows (checked
    on the host before the launch) and computes the bits of the aligned call."""
    XL, lib = _loss(), _lib()
    N, d = 129, 256
    V, T = pair(N, d, "seeded", seed=5)

    def misaligned(x):
        buf = torch.empty(N * d + 1, dtype=f32, device=dev)
        view = buf[1:].view(N, d)
        view.copy_(x)
        return view
    vm, tm = misaligned(V), misaligned(T)
    assert vm.is_contiguous() and vm.data_ptr() % 16 == 4 and tm.data_ptr() % 16 == 4
    lsd = scale_ls(dev, 2.659)
    h = lib.lib()
    orig = h.xp_nce_gather_fused
    seen = []

    def checked(aref, stream):
        a = aref._obj
        rows = XL._local_ws[(N, dev)][1].cpu().tolist()          # the pointer table the kernel reads (mode 1)
        ptrs = [a.vis_local, a.txt_local] + rows
        assert all(p % 16 == 0 for p in ptrs), f"misaligned operand handed to the kernel: {[p % 16 for p in ptrs]}"
        seen.append(ptrs)
        return orig(aref, stream)
    monkeypatch.setattr(h, "xp_nce_gather_fused", checked)
    got = XL._nce_forward_fused(vm, tm, lsd)
    want = XL._nce_forward_fused(V.to(dev), T.to(dev), lsd)
    torch.cuda.synchronize()
    assert len(seen) == 2
    for x, y in zip(got, want):
        assert same_bits(x, y), "the misaligned view gives different bits"


# ============================================================================================ xp_nce_terms
def logits_matrix(dev, X, Y, ld):
    """fp32 z = X Y^T (rounded once from float64) inside an [n, ld] buffer whose pad columns hold NaN."""
    n = X.shape[0]
    z = torch.full((n, ld), float("nan"), dtype=f32, device=dev)
    z[:, :n] = (X.to(dev, F64) @ Y.to(dev, F64).T).to(f32)
    return z


def run_terms(dev, tag, zs, table, *, ls=None, scale=1.0, dsl=False):
    """xp_nce_terms / xp_nce_dsl on fp32 logits, twice: into a clean and into a NaN-filled workspace."""
    ops, lib = _ops(), _lib()
    ns = [z.shape[0] for z in zs]
    if dsl:
        nbytes = int(lib.lib().xp_nce_dsl_workspace_bytes(ns[0]))
    else:
        a = lib.XpNceTerms()
        a.n_mats = len(zs)
        for m, n in enumerate(ns):
            a.n[m] = n
        nbytes = int(lib.lib().xp_nce_terms_workspace_bytes(ctypes.byref(a)))
    outs = []
    for poisoned in (False, True):
        ws = torch.full(((nbytes + 3) // 4,), float("nan") if poisoned else 0.0, dtype=f32, device=dev)
        gs = [Out(dev, n, ceil4(n), bf16, z.shape[1]) for n, z in zip(ns, zs)]
        loss = torch.full((1,), float("nan"), device=dev)
        dscale = torch.full((1,), float("nan"), device=dev) if (ls is not None) else None
        if dsl:
            ops.nce_dsl(zs[0], ls, gs[0].buf[:ns[0]], loss, dscale, workspace=ws)
        else:
            ops.nce_terms(zs, [g.buf[:n] for g, n in zip(gs, ns)], table, loss, logit_scale=ls, scale=scale,
                          d_logit_scale=dscale, workspace=ws)
        torch.cuda.synchronize()
        g_out = []
        for g, n in zip(gs, ns):
            full = g.check(f"{tag}: g")
            assert bool((full[:, n:] == 0).all()), f"{tag}: columns [n, ceil4(n)) of g are not zero"
            g_out.append(full[:, :n])
        outs.append((loss, dscale, g_out))
    (l1, d1, g1), (l2, d2, g2) = outs
    assert same_bits(l1, l2) and (d1 is None or same_bits(d1, d2)) and all(same_bits(a, b) for a, b in zip(g1, g2)), \
        f"{tag}: a NaN-filled workspace or a second call changed the outputs"
    return l1, d1, g1


TERMS = []
_NS = (1, 2, 63, 64, 65, 127, 128, 129, 200, 257, 1000)
for _i, _name in enumerate(TABLES):
    for _j, _n in enumerate(_NS):
        for _wide in (False, True):
            _m = None
            if _name == "VidImgDivideNCELearnableTempLoss":
                _m = _n
            TERMS.append((_name, _n, _m, _wide, KINDS[(_i + _j) % 3], LOG_SCALES[(_i + _j + _wide) % 3]))
TERMS += [("VidImgDivideNCELearnableTempLoss", n, m, w, "adversarial", 4.6052)
          for (n, m) in ((64, 65), (129, 1), (300, 131), (1000, 7)) for w in (False, True)]


@pytest.mark.parametrize("name,n,m,wide,kind,ls", TERMS,
                         ids=[f"{t[0]}-n{t[1]}" + (f"-m{t[2]}" if t[2] is not None else "") + ("-wide" if t[3] else "")
                              + f"-{t[4]}-ls{t[5]}" for t in TERMS])
def test_nce_terms_tables(dev, name, n, m, wide, kind, ls):
    """Every TERM_TABLES entry (NCEContrastiveLoss at its fixed scale 1/0.05), row pitch ceil8(n) or wider.  The _vsc
    tables exclude diagonals: past n = 64 those cross 64-row tile boundaries inside a 128-column tile (rowx / colx)."""
    pairs, table = _loss().TERM_TABLES[name]
    v, t = pair(n, 96, kind, seed=n)
    i, c = pair(m or n, 96, kind, seed=n + 7) if m is not None else pair(n, 96, kind, seed=n + 7)
    feats = [v, t, i, c]
    zs = [logits_matrix(dev, feats[r], feats[cc], ceil8(feats[r].shape[0]) + (12 if wide else 0)) for r, cc in pairs]
    fixed = name == "NCEContrastiveLoss"
    lsd = None if fixed else scale_ls(dev, ls)
    tag = f"terms {name}"
    loss, dscale, gs = run_terms(dev, f"{tag} n{n}", zs, table, ls=lsd, scale=20.0)
    s = R.scale_of(scale=20.0, device=dev) if fixed else R.scale_of(lsd)
    ref = R.terms([z[:, :z.shape[0]].to(F64) for z in zs], table, s)
    for k, g in enumerate(gs):
        check_sg(tag, g, ref, k, name=f"s dL/dZ[{k}]")
    check_scalars(tag, loss, dscale, ref)


DSL = [(n, ls) for n in (1, 2, 64, 65, 129, 300, 1024, 2048) for ls in LOG_SCALES + (math.log(200.0),)]


@pytest.mark.parametrize("n,ls", DSL, ids=[f"n{c[0]}-ls{c[1]:.4g}" for c in DSL])
def test_nce_dsl(dev, n, ls):
    """NCELearnableTempDSLLoss's chain up to s = 200, where G_Z = Pc (GA (1 + Z) - u_j) + Pr (GB (1 + Z) - w_i) cancels."""
    kind = KINDS[n % 3]
    v, t = pair(n, 128, kind, seed=3 * n)
    z = logits_matrix(dev, v, t, ceil8(n))
    lsd = scale_ls(dev, ls)
    loss, dscale, gs = run_terms(dev, f"dsl n{n}", [z], None, ls=lsd, dsl=True)
    ref = R.dsl(z[:, :n].to(F64), R.scale_of(lsd))
    tag = f"dsl ls{ls:.4g}"
    check_sg(tag, gs[0], ref)
    check_scalars(tag, loss, dscale, ref)


# ============================================================================================ multi-launch path
MULTI = [(1537, 512), (2048, 512), (3000, 512), (20, 96), (300, 96)]


@pytest.mark.parametrize("N,d", MULTI, ids=[f"N{c[0]}-d{c[1]}" for c in MULTI])
def test_multi_launch_infonce(dev, N, d):
    """Global batches beyond the fused kernel, and widths it does not take (d % 64 != 0): G, loss and d logit_scale of
    _nce_forward, then NCELearnableTempLoss forward + backward, twice each (bit-identical)."""
    XL = _loss()
    V, T = pair(N, d, "adversarial", seed=N)
    Vd, Td = V.to(dev), T.to(dev)
    lsd = scale_ls(dev, 4.6052)
    tag = "multi-launch"
    first = XL._nce_forward(Vd, Td, lsd)
    second = XL._nce_forward(Vd, Td, lsd)
    torch.cuda.synchronize()
    for x, y in zip(first, second):                          # G's columns past ceil4(N) are never written
        assert same_bits(x[..., :N], y[..., :N]), f"{tag} N{N}: loss, G or d logit_scale differ between two calls"
    loss, g, vh, th, dscale = first
    lg = R.split_logits(Vd, Td)
    ref = R.terms([lg["exact"]], R.INFONCE, R.scale_of(lsd), z_err=[lg["err"]], z_arm=[lg["arm"]])
    check_sg(tag, g[:, :N], ref)
    check_scalars(tag, loss, dscale, ref)
    grads = []
    for _ in range(2):
        v, t, p = (x.clone().requires_grad_(True) for x in (Vd, Td, lsd.reshape(())))
        out = XL.NCELearnableTempLoss()(v, t, p)
        out.backward()
        grads.append((out.detach(), v.grad, t.grad, p.grad))
    torch.cuda.synchronize()
    assert all(same_bits(a.reshape(-1), b.reshape(-1)) for a, b in zip(*grads)), f"{tag} N{N}: module results differ"
    ex = R.feature_grads(((0, 1),), ref["exact"], [Vd, Td])
    arm = R.feature_grads(((0, 1),), ref["arm"], [R.bf(Vd), R.bf(Td)])
    tiled(f"{tag} module", "dV", grads[0][1], ex[0], arm[0])
    tiled(f"{tag} module", "dT", grads[0][2], ex[1], arm[1])
    check_scalars(f"{tag} module", grads[0][0], grads[0][3], ref)


# ============================================================================================ module API
MODULES = ("NCELearnableTempLoss", "NCEContrastiveLoss", "NCELearnableTempDSLLoss", "VidImgNCELearnableTempLoss") + TABLES[1:]


def _module_ref(dev, name, feats, lsd):
    """(pairs, the features the gradient GEMMs multiply, reference) of a build_loss_func loss on fp32 features."""
    XL = _loss()
    if name in ("NCELearnableTempLoss", "VidImgNCELearnableTempLoss", "NCELearnableTempDSLLoss"):
        if name == "VidImgNCELearnableTempLoss":
            X, Y = torch.cat([feats[0], feats[2]]), torch.cat([feats[1], feats[3]])
        else:
            X, Y = feats[0], feats[1]
        lg = R.split_logits(X, Y)
        if name == "NCELearnableTempDSLLoss":
            ref = R.dsl(lg["exact"], R.scale_of(lsd), z_err=lg["err"], z_arm=lg["arm"])
        else:
            depth = R.fused_depth(X.shape[0]) if X.shape[0] <= XL.FUSED_MAX_N and X.shape[1] % 64 == 0 else None
            ref = R.terms([lg["exact"]], R.INFONCE, R.scale_of(lsd), z_err=[lg["err"]], z_arm=[lg["arm"]],
                          reduce_depth=depth)
        return ((0, 1),), [X, Y], ref
    pairs, table = XL.TERM_TABLES[name]
    lgs = [R.split_logits(feats[r], feats[c]) for r, c in pairs]
    s = R.scale_of(scale=20.0, device=dev) if name == "NCEContrastiveLoss" else R.scale_of(lsd)
    ref = R.terms([x["exact"] for x in lgs], table, s, z_err=[x["err"] for x in lgs], z_arm=[x["arm"] for x in lgs])
    return pairs, feats, ref


@pytest.mark.parametrize("name", MODULES)
def test_module_api_feature_gradients(dev, name):
    """Every build_loss_func name: loss and d logit_scale within their bounds, and each feature gradient per 64-row block
    against the float64 closed form, calibrated by the GEMM arm (bf16 s dL/dZ times the bf16 features), including the
    accumulation of a feature that sits in two matrices (cap in B and D).  Arguments the reference never reads get None
    or zero."""
    from xpretrain_b200.optimization import build_loss_func
    n, d = 200, 256
    m = 131 if name == "VidImgDivideNCELearnableTempLoss" else n
    v, t = pair(n, d, "adversarial", seed=11)
    i, c = pair(m, d, "seeded", seed=12)
    feats = [x.to(dev) for x in (v, t, i, c)]
    lsd = scale_ls(dev, 4.6052)
    fn = build_loss_func({"loss_name": name, "temp": 0.05})
    two = name in ("NCELearnableTempLoss", "NCEContrastiveLoss", "NCELearnableTempDSLLoss")
    args = [f.clone().requires_grad_(True) for f in (feats[:2] if two else feats)]
    p = lsd.reshape(()).clone().requires_grad_(True)
    loss = fn(*args) if name == "NCEContrastiveLoss" else fn(*args, p)
    loss.backward()
    torch.cuda.synchronize()
    pairs, mats, ref = _module_ref(dev, name, feats[:2] if two else feats, lsd)
    ex = R.feature_grads(pairs, ref["exact"], mats)
    arm = R.feature_grads(pairs, ref["arm"], [R.bf(x) for x in mats])
    if name == "VidImgNCELearnableTempLoss":
        ex = {0: ex[0][:n], 1: ex[1][:n], 2: ex[0][n:], 3: ex[1][n:]}
        arm = {0: arm[0][:n], 1: arm[1][:n], 2: arm[0][n:], 3: arm[1][n:]}
    tag = f"module {name}"
    for k, x in enumerate(args):
        if k in ex:
            tiled(tag, f"d feature {k}", x.grad, ex[k], arm[k])
        else:
            assert x.grad is None or float(x.grad.abs().max()) == 0.0, f"{tag}: argument {k} is not read but has a gradient"
    check_scalars(tag, loss.detach(), None if name == "NCEContrastiveLoss" else p.grad, ref)


@pytest.mark.parametrize("grad_scale", [None, 4.0])
def test_gather_nce_loss_single_process(dev, grad_scale):
    """gather_nce_loss without a process group: the fused kernel on the local rows; grad_scale multiplies the feature
    gradients (all_reduce(SUM)-then-slice semantics), not d logit_scale."""
    from xpretrain_b200.optimization.loss import gather_nce_loss
    N, d = 300, 512
    V, T = pair(N, d, "adversarial", seed=21)
    Vd, Td = V.to(dev), T.to(dev)
    lsd = scale_ls(dev, 2.659)
    v, t, p = (x.clone().requires_grad_(True) for x in (Vd, Td, lsd.reshape(())))
    loss = gather_nce_loss(v, t, p, grad_scale=grad_scale)
    loss.backward()
    torch.cuda.synchronize()
    pairs, mats, ref = _module_ref(dev, "NCELearnableTempLoss", [Vd, Td], lsd)
    sc = 1.0 if grad_scale is None else grad_scale
    ex = R.feature_grads(pairs, ref["exact"], mats)
    arm = R.feature_grads(pairs, ref["arm"], [R.bf(x) for x in mats])
    tag = f"gather_nce_loss grad_scale={grad_scale}"
    tiled(tag, "dV", v.grad, sc * ex[0], sc * arm[0])
    tiled(tag, "dT", t.grad, sc * ex[1], sc * arm[1])
    check_scalars(tag, loss.detach(), p.grad, ref)
