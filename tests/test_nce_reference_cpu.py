"""CPU: the float64 references of the contrastive-loss kernels (oracle/nce_ref.py) against the autograd oracles
(oracle/loss_family_oracle.py, oracle/clipvip_oracle.py) in float64 and against the reference-class goldens; the split
arm against exact logits; and the bf16 arms against the derived element bound."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import clipvip_oracle as O
from oracle import loss_family_oracle as LF
from oracle import nce_ref as R

F64 = torch.float64
TABLES = ("NCEContrastiveLoss", "VidImgDivideNCELearnableTempLoss", "NCELearnableTempLoss_vs_vc",
          "NCELearnableTempLoss_vs_vc_fc", "NCELearnableTempLoss_vsc", "NCELearnableTempLoss_vsc_fc")


def _tables():
    from xpretrain_b200.optimization.loss import TERM_TABLES
    return TERM_TABLES


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _feats(n, d, m=None, seed=0, dtype=F64):
    g = torch.Generator().manual_seed(seed)
    v = F.normalize(torch.randn(n, d, generator=g, dtype=F64), dim=-1)
    out = [v, F.normalize(torch.randn(n, d, generator=g, dtype=F64) + 0.5 * v, dim=-1)]
    i = F.normalize(torch.randn(m or n, d, generator=g, dtype=F64), dim=-1)
    out += [i, F.normalize(torch.randn(m or n, d, generator=g, dtype=F64) + 0.5 * i, dim=-1)]
    return [x.to(dtype) for x in out]


def _scale(name, ls):
    return R.scale_of(scale=20.0) if name == "NCEContrastiveLoss" else R.scale_of(ls)


@pytest.mark.parametrize("name", TABLES)
@pytest.mark.parametrize("ls", [0.0, 2.659, math.log(200.0)])
def test_terms_match_autograd_of_the_oracle(name, ls):
    """loss, s dL/dZ of every matrix, d logit_scale and the feature gradients through feature_grads equal float64 autograd
    of loss_family_oracle.nce_family_loss."""
    pairs, table = _tables()[name]
    feats = [f.requires_grad_(True) for f in _feats(9, 16, 6 if "Divide" in name else None, seed=len(name))]
    lst = torch.tensor(ls, dtype=torch.float32).to(F64).requires_grad_(True)      # the fp32 log-scale the kernels read
    s = _scale(name, torch.tensor(ls, dtype=torch.float32))
    loss = LF.nce_family_loss(name, feats, 0.05 if name == "NCEContrastiveLoss" else lst)
    z = [(feats[r] @ feats[c].T).detach() for r, c in pairs]
    Zs = [(x * s.v).requires_grad_(True) for x in z]
    names = {(0, 1): "vt", (0, 3): "vc", (2, 3): "ic"}
    want_z = LF.nce_terms_loss({names[p]: Z for p, Z in zip(pairs, Zs)}, LF.NCE_TERM_TABLES[name])
    ref = R.terms(z, table, s)
    assert abs(float(ref["loss"]) - float(loss.detach())) < 1e-12 * max(1.0, abs(float(loss.detach())))
    want_z.backward()
    for got, Z in zip(ref["exact"], Zs):
        assert _rel(got, s.v * Z.grad) < 1e-12
    loss.backward()
    fg = R.feature_grads(pairs, ref["exact"], [f.detach() for f in feats])
    for i, f in enumerate(feats):
        if i in fg:
            assert _rel(fg[i], f.grad) < 1e-12, i
        else:
            assert f.grad is None or float(f.grad.abs().max()) == 0.0
    if name != "NCEContrastiveLoss":
        assert abs(float(ref["dscale"]) - float(lst.grad)) < 1e-12 * max(1.0, abs(float(lst.grad)))


@pytest.mark.parametrize("ls", [0.0, 2.659, 4.6052, math.log(200.0)])
def test_infonce_and_dsl_match_the_oracles(ls):
    v, t = [f.requires_grad_(True) for f in _feats(11, 16, seed=3)[:2]]
    lst = torch.tensor(ls, dtype=torch.float32).to(F64).requires_grad_(True)      # the fp32 log-scale the kernels read
    s = R.scale_of(torch.tensor(ls, dtype=torch.float32))
    z = (v @ t.T).detach()
    for which in ("infonce", "dsl"):
        for x in (v, t, lst):
            x.grad = None
        if which == "infonce":
            ref = R.terms([z], R.INFONCE, s)
            loss = O.nce_learnable_temp_loss(v, t, lst)
            cf = O.nce_closed_form_grads(v.detach(), t.detach(), lst.detach())
        else:
            ref = R.dsl(z, s)
            loss = LF.nce_dsl_loss(v, t, lst)
            cf = LF.nce_dsl_closed_form_grads(v.detach(), t.detach(), lst.detach())
        loss.backward()
        assert abs(float(ref["loss"]) - float(loss.detach())) < 1e-12 * max(1.0, abs(float(loss.detach()))), which
        assert abs(float(ref["dscale"]) - float(lst.grad)) < 1e-11 * max(1.0, abs(float(lst.grad))), which
        fg = R.feature_grads(((0, 1),), ref["exact"], [v.detach(), t.detach()])
        assert _rel(fg[0], v.grad) < 1e-11 and _rel(fg[1], t.grad) < 1e-11, which
        assert _rel(fg[0], cf[0]) < 1e-11 and _rel(fg[1], cf[1]) < 1e-11, which


def _golden(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name), weights_only=False)


def test_reference_goldens_infonce_and_vsc_fc(golden_dir):
    """The fixtures written from the reference's own classes and autograd (fp32): nce_loss_w4 (NCELearnableTempLoss over
    a 4-rank gather) and nce_vsc_fc_n24 (NCELearnableTempLoss_vsc_fc)."""
    gold = _golden(golden_dir, "nce_loss_w4.pt")
    V, T = torch.cat(gold["vis_per_rank"]), torch.cat(gold["txt_per_rank"])
    ref = R.terms([V.to(F64) @ T.to(F64).T], R.INFONCE, R.scale_of(gold["logit_scale"]))
    fg = R.feature_grads(((0, 1),), ref["exact"], [V, T])
    assert abs(float(ref["loss"]) - float(gold["loss"])) < 1e-5 * abs(float(gold["loss"]))
    assert _rel(fg[0], gold["d_vis"].to(F64)) < 2e-5 and _rel(fg[1], gold["d_txt"].to(F64)) < 2e-5
    assert abs(float(ref["dscale"]) - float(gold["d_logit_scale"])) < 1e-5 * max(1.0, abs(float(gold["d_logit_scale"])))
    gold = _golden(golden_dir, "nce_vsc_fc_n24.pt")
    feats = [gold[k] for k in ("vis", "txt", "img", "cap")]
    pairs, table = _tables()["NCELearnableTempLoss_vsc_fc"]
    ref = R.terms([feats[r].to(F64) @ feats[c].to(F64).T for r, c in pairs], table, R.scale_of(gold["logit_scale"]))
    fg = R.feature_grads(pairs, ref["exact"], feats)
    assert abs(float(ref["loss"]) - float(gold["loss"])) < 1e-5 * abs(float(gold["loss"]))
    for i, k in enumerate(("d_vis", "d_txt", "d_img", "d_cap")):
        assert _rel(fg[i], gold[k].to(F64)) < 2e-5, k
    assert abs(float(ref["dscale"]) - float(gold["d_logit_scale"])) < 1e-5 * max(1.0, abs(float(gold["d_logit_scale"])))


@pytest.mark.parametrize("name", ("NCELearnableTempDSLLoss", "VidImgNCELearnableTempLoss") + TABLES)
def test_reference_golden_loss_family(golden_dir, name):
    gold = _golden(golden_dir, "nce_family_n16.pt")
    case = gold["cases"][name]
    feats = [gold["feats"][k] for k in case["keys"]]
    s = R.scale_of(scale=1.0 / gold["temp"]) if name == "NCEContrastiveLoss" else R.scale_of(gold["logit_scale"])
    if name == "NCELearnableTempDSLLoss":
        pairs, ref = ((0, 1),), R.dsl(feats[0].to(F64) @ feats[1].to(F64).T, s)
    elif name == "VidImgNCELearnableTempLoss":
        V, T = torch.cat([feats[0], feats[2]]), torch.cat([feats[1], feats[3]])
        pairs, ref = ((0, 1),), R.terms([V.to(F64) @ T.to(F64).T], R.INFONCE, s)
        feats = [V, T]
    else:
        pairs, table = _tables()[name]
        ref = R.terms([feats[r].to(F64) @ feats[c].to(F64).T for r, c in pairs], table, s)
    fg = R.feature_grads(pairs, ref["exact"], feats)
    if name == "VidImgNCELearnableTempLoss":
        n = case["grads"]["vis"].shape[0]
        fg = {0: fg[0][:n], 1: fg[1][:n], 2: fg[0][n:], 3: fg[1][n:]}
    assert abs(float(ref["loss"]) - float(case["loss"])) < 1e-5 * abs(float(case["loss"]))
    for i, k in enumerate(case["keys"]):
        if k in case["grads"]:
            assert _rel(fg[i], case["grads"][k].to(F64)) < 2e-5, k
        else:
            assert i not in fg, k
    if case["d_logit_scale"] is not None:
        assert abs(float(ref["dscale"]) - float(case["d_logit_scale"])) < 1e-5 * max(1.0, abs(float(case["d_logit_scale"])))


def test_split_arm_is_exact_on_bf16_inputs_and_drops_only_lo_lo():
    g = torch.Generator().manual_seed(1)
    V, T = torch.randn(40, 192, generator=g), torch.randn(33, 192, generator=g)
    r = R.split_logits(V.bfloat16().float(), T.bfloat16().float())
    assert torch.equal(r["arm"], r["exact"])                                  # lo = 0
    r = R.split_logits(V, T)
    lolo = (V.double().abs() @ T.double().abs().T) * 2.0 ** -16               # |lo| <= 2^-8 |v| on each side
    assert bool(((r["arm"] - r["exact"]).abs() <= lolo).all())
    assert float((r["arm"] - r["exact"]).abs().max()) > 0
    assert bool((r["err"] >= (r["arm"] - r["exact"]).abs()).all())


def _adversarial(n, d, seed):
    """Seeded unit-norm correlated features with duplicate rows, near-one-hot pairs and a row equal to the mean of the
    others (rows 0-1, 2-3 and n-1)."""
    v, t = _feats(n, d, seed=seed, dtype=torch.float32)[:2]
    v[1], t[1] = v[0], t[0]
    e = torch.zeros(d)
    e[0] = 1.0
    v[2] = t[2] = e
    v[n - 1], t[n - 1] = v[:n - 1].mean(0), t[:n - 1].mean(0)
    return v, t


@pytest.mark.parametrize("ls", [0.0, 4.6052, math.log(200.0)])
def test_a_kernel_that_rounds_only_like_the_arm_meets_the_element_bound(ls):
    """The bf16 arms, which round exactly where the kernels round, lie inside the derived element bound of every path:
    the fused / split-logits InfoNCE, a term table excluding diagonals, and DSL."""
    v, t = _adversarial(150, 64, seed=7)
    s = R.scale_of(torch.tensor(ls))
    lg = R.split_logits(v, t)
    for ref in (R.terms([lg["exact"]], R.INFONCE, s, z_err=[lg["err"]], z_arm=[lg["arm"]]),
                R.terms([lg["exact"], lg["exact"].T.contiguous()], _tables()["NCELearnableTempLoss_vsc"][1], s),
                R.dsl(lg["arm"], s)):
        for ex, arm, b in zip(ref["exact"], ref["arm"], ref["bound"]):
            assert bool(((arm - ex).abs() <= b).all()), float(((arm - ex).abs() / b).max())
        assert float(ref["loss_bound"]) < 1e-3 * max(1.0, abs(float(ref["loss"])))
