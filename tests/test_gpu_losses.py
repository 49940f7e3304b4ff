"""H100: the contrastive-loss family of loss.py (xp_nce_terms / xp_nce_dsl) against the fp32 oracle
(oracle/loss_family_oracle.py, pinned to the reference classes by tests/golden/nce_family_n16.pt)."""
import ctypes
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
FAMILY = ("NCEContrastiveLoss", "NCELearnableTempDSLLoss", "VidImgNCELearnableTempLoss", "VidImgDivideNCELearnableTempLoss",
          "NCELearnableTempLoss_vs_vc", "NCELearnableTempLoss_vs_vc_fc", "NCELearnableTempLoss_vsc",
          "NCELearnableTempLoss_vsc_fc")
TEMP = 0.05


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20))


def _keys(name):
    if name in ("NCEContrastiveLoss", "NCELearnableTempDSLLoss"):
        return ("vis", "txt")
    return ("vis", "txt", "img", "cap")


def _features(name, N, d, M=None, seed=0):
    """Seeded unit-norm features with a positive diagonal; the image / caption pair has M rows for VidImgDivide."""
    if name != "VidImgDivideNCELearnableTempLoss":
        M = None
    g = torch.Generator().manual_seed(seed + N * 7 + d + (M or 0))
    out = []
    for k in _keys(name):
        n = M if (M is not None and k in ("img", "cap")) else N
        if k in ("vis", "img"):
            base = F.normalize(torch.randn(n, d, generator=g), dim=-1)
            out.append(base)
        else:
            out.append(F.normalize(torch.randn(n, d, generator=g) + 0.5 * out[-1 if k == "txt" else 2][:n], dim=-1))
    return out


def _oracle(name, feats, logit_scale):
    from oracle import loss_family_oracle as LF
    xs = [f.clone().requires_grad_(True) for f in feats]
    ls = logit_scale.clone().requires_grad_(True)
    loss = LF.nce_family_loss(name, xs, TEMP if name == "NCEContrastiveLoss" else ls)
    loss.backward()
    return loss.detach(), [x.grad for x in xs], (None if name == "NCEContrastiveLoss" else ls.grad)


def _ours(name, feats, logit_scale, dev, dtype=f32):
    from xpretrain_b200.optimization import build_loss_func
    xs = [f.to(dev, dtype).requires_grad_(True) for f in feats]
    ls = logit_scale.to(dev).requires_grad_(True)
    fn = build_loss_func({"loss_name": name, "temp": TEMP})
    loss = fn(*xs) if name == "NCEContrastiveLoss" else fn(*xs, ls)
    loss.backward()
    return loss.detach(), [x.grad for x in xs], (None if name == "NCEContrastiveLoss" else ls.grad)


def _check(name, got, want):
    (gl, gg, gd), (wl, wg, wd) = got, want
    assert abs(float(gl) - float(wl)) < 2e-4 * max(1.0, abs(float(wl))), (name, float(gl), float(wl))
    for a, b in zip(gg, wg):
        if b is None:                                  # an argument the reference class never reads
            assert a is None or float(a.abs().max()) == 0.0, name
        else:
            assert rel(a.cpu(), b) < 6e-3, (name, rel(a.cpu(), b))
    if wd is not None:
        assert abs(float(gd) - float(wd)) < 2e-3 * max(1.0, abs(float(wd))), (name, float(gd), float(wd))


@pytest.mark.parametrize("name", FAMILY)
def test_loss_family_reference_golden(dev, golden_dir, name):
    """The fixture written from the reference's own classes and autograd (N = 16, d = 128; M = 10 image pairs)."""
    gold = torch.load(os.path.join(golden_dir, "nce_family_n16.pt"), weights_only=False)
    case = gold["cases"][name]
    feats = [gold["feats"][k] for k in case["keys"]]
    want = (case["loss"], [case["grads"].get(k) for k in case["keys"]], case["d_logit_scale"])
    _check(name, _ours(name, feats, gold["logit_scale"], dev), want)


@pytest.mark.parametrize("name", FAMILY)
@pytest.mark.parametrize("N,d,M", [(512, 512, None), (20, 512, None)])
def test_loss_family_against_oracle(dev, name, N, d, M):
    feats = _features(name, N, d, M)
    ls = torch.tensor(4.6)
    _check(name, _ours(name, feats, ls, dev), _oracle(name, feats, ls))


@pytest.mark.parametrize("N,M", [(512, 200), (20, 37)])
def test_vid_img_divide_with_its_own_image_batch(dev, N, M):
    name = "VidImgDivideNCELearnableTempLoss"
    feats = _features(name, N, 512, M)
    assert feats[2].shape[0] == M != N
    ls = torch.tensor(4.6)
    _check(name, _ours(name, feats, ls, dev), _oracle(name, feats, ls))


@pytest.mark.parametrize("N,logit_scale", [(512, math.log(200.0)), (1024, 4.6), (1024, math.log(200.0))])
def test_dsl_at_the_drivers_clamp_and_large_batch(dev, N, logit_scale):
    """DSL's G_Z subtracts u_j and w_i; bf16 storage of s * G_Z still meets the 6e-3 gradient bar at s = 200 (the
    drivers' clamp) and N = 1024."""
    name = "NCELearnableTempDSLLoss"
    feats = _features(name, N, 512)
    ls = torch.tensor(logit_scale)
    _check(name, _ours(name, feats, ls, dev), _oracle(name, feats, ls))


@pytest.mark.parametrize("name", ("NCELearnableTempDSLLoss", "NCELearnableTempLoss_vsc", "VidImgDivideNCELearnableTempLoss",
                                  "NCEContrastiveLoss"))
def test_bf16_features_return_bf16_gradients(dev, name):
    feats = [f.to(bf16).float() for f in _features(name, 64, 256, 48)]
    ls = torch.tensor(4.6)
    got = _ours(name, feats, ls, dev, dtype=bf16)
    assert got[0].dtype == f32
    for gr in got[1]:
        assert gr is None or gr.dtype == bf16
    _check(name, got, _oracle(name, feats, ls))


def _tables():
    from xpretrain_b200.optimization.loss import TERM_TABLES
    return TERM_TABLES


@pytest.mark.parametrize("table", ["NCELearnableTempLoss_vsc_fc", "VidImgDivideNCELearnableTempLoss", "DSL"])
def test_kernel_outputs_are_bit_identical_across_calls_and_match_dl_dz(dev, table):
    """loss, d logit_scale and s * dL/dZ of two calls on the same logits are bit-identical (fixed-order reductions), and
    s * G matches autograd of the oracle loss with respect to the scaled logits (bf16 storage)."""
    from oracle import loss_family_oracle as LF
    from xpretrain_b200 import ops
    g = torch.Generator().manual_seed(5)
    s = 100.0
    sizes = (300, 300, 300) if table != "VidImgDivideNCELearnableTempLoss" else (300, 131)
    if table == "DSL":
        sizes = (300,)
    zs = [torch.randn(n, n, generator=g) * 0.1 + 0.3 * torch.eye(n) for n in sizes]
    ls = torch.tensor([math.log(s)], device=dev)

    def run():
        zd = [torch.zeros(n, (n + 7) // 8 * 8, device=dev) for n in sizes]
        for a, b in zip(zd, zs):
            a[:, :b.shape[0]] = b.to(dev)
        gd = [torch.full_like(a, float("nan"), dtype=bf16) for a in zd]
        loss, dscale = torch.empty(1, device=dev), torch.empty(1, device=dev)
        if table == "DSL":
            ops.nce_dsl(zd[0], ls, gd[0], loss, dscale)
        else:
            ops.nce_terms(zd, gd, _tables()[table][1], loss, logit_scale=ls, d_logit_scale=dscale)
        torch.cuda.synchronize()
        return loss.cpu(), dscale.cpu(), [x[:, :n].cpu() for x, n in zip(gd, sizes)]

    l1, d1, g1 = run()
    l2, d2, g2 = run()
    assert torch.equal(l1, l2) and torch.equal(d1, d2) and all(torch.equal(a, b) for a, b in zip(g1, g2))
    # autograd of the oracle with respect to the scaled logits
    zz = [(z * s).requires_grad_(True) for z in zs]
    if table == "DSL":
        n = sizes[0]
        labels = torch.arange(n)
        a, b = zz[0] * torch.softmax(zz[0], 0), zz[0].t() * torch.softmax(zz[0].t(), 0)
        want = F.cross_entropy(a, labels) + F.cross_entropy(b, labels)
    else:
        names = ("vt", "vc", "ic") if table != "VidImgDivideNCELearnableTempLoss" else ("vt", "ic")
        want = LF.nce_terms_loss(dict(zip(names, zz)), LF.NCE_TERM_TABLES[table])
    want.backward()
    assert abs(float(l1) - float(want)) < 2e-4 * max(1.0, abs(float(want)))
    dl = sum(float((z.grad * z).sum()) for z in zz)
    assert abs(float(d1) - dl) < 2e-3 * max(1.0, abs(dl))
    for a, z in zip(g1, zz):
        assert not torch.isnan(a.float()).any() and rel(a.float(), s * z.grad) < 6e-3


def test_cpu_tensors_raise_xp_error():
    from xpretrain_b200._lib import XpError
    from xpretrain_b200.optimization import build_loss_func
    v = torch.randn(8, 64)
    for name in FAMILY:
        fn = build_loss_func({"loss_name": name, "temp": TEMP})
        with pytest.raises(XpError):
            fn(v, v) if name == "NCEContrastiveLoss" else fn(*([v] * len(_keys(name))), torch.tensor(4.6))


def test_shape_mismatch_raises_value_error(dev):
    from xpretrain_b200.optimization import build_loss_func
    v, c = torch.randn(16, 64, device=dev), torch.randn(12, 64, device=dev)
    p = torch.tensor(4.6, device=dev)
    for name in ("NCELearnableTempLoss_vs_vc", "NCELearnableTempLoss_vs_vc_fc", "NCELearnableTempLoss_vsc",
                 "NCELearnableTempLoss_vsc_fc"):
        with pytest.raises(ValueError):
            build_loss_func({"loss_name": name})(v, v, v, c, p)
    with pytest.raises(ValueError):
        build_loss_func({"loss_name": "VidImgDivideNCELearnableTempLoss"})(v, v, c, v, p)
    with pytest.raises(ValueError):
        build_loss_func({"loss_name": "NCELearnableTempDSLLoss"})(v, c, p)


def test_term_table_validation_at_the_abi(dev):
    """xp_nce_terms refuses a target whose diagonal is excluded, a union of matrices with different n, and n <= 0."""
    from xpretrain_b200 import _lib
    z = [torch.zeros(16, 16, device=dev), torch.zeros(8, 8, device=dev)]
    g = [torch.zeros(16, 16, dtype=bf16, device=dev), torch.zeros(8, 8, dtype=bf16, device=dev)]
    loss, ws = torch.empty(1, device=dev), torch.empty(1 << 16, device=dev)

    def call(n, terms):
        a = _lib.XpNceTerms()
        a.n_mats, a.n_terms = 2, len(terms)
        for m in range(2):
            a.z[m], a.g[m], a.ld[m], a.n[m] = z[m].data_ptr(), g[m].data_ptr(), z[m].stride(0), n[m]
        for t, (axis, members, excl, target) in enumerate(terms):
            a.term[t].axis, a.term[t].members, a.term[t].excl_diag, a.term[t].target = axis, members, excl, target
        a.scale, a.loss, a.workspace = 1.0, loss.data_ptr(), ws.data_ptr()
        stream = torch.cuda.current_stream().cuda_stream
        return _lib.lib().xp_nce_terms(ctypes.byref(a), stream), _lib.lib().xp_last_error().decode()

    assert call((16, 8), [(0, 1, 0, 0), (0, 2, 0, 1)])[0] == 0
    rc, msg = call((16, 8), [(0, 1, 1, 0)])
    assert rc != 0 and "diagonal" in msg
    rc, msg = call((16, 8), [(0, 3, 0, 0)])
    assert rc != 0 and "one n" in msg
    rc, msg = call((0, 8), [(0, 2, 0, 1)])
    assert rc != 0 and "n > 0" in msg
    torch.cuda.synchronize()
