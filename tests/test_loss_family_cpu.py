"""CPU: the contrastive-loss family of loss.py — the oracle replays the reference fixture (tests/golden/nce_family_n16.pt,
written by `tests/golden/make_golden_loss_family.py` from the reference's own classes), and build_loss_func exposes the
reference's names, constructors and forward arities."""
import os
import types

import pytest
import torch

from oracle import loss_family_oracle as LF


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


FAMILY = ("NCEContrastiveLoss", "NCELearnableTempDSLLoss", "VidImgNCELearnableTempLoss", "VidImgDivideNCELearnableTempLoss",
          "NCELearnableTempLoss_vs_vc", "NCELearnableTempLoss_vs_vc_fc", "NCELearnableTempLoss_vsc",
          "NCELearnableTempLoss_vsc_fc")
# forward(...) arguments of the reference classes (loss.py:76, 134, 151, 170, 193, 212, 235, 264, 296)
ARITY = {"NCELearnableTempLoss": 3, "NCEContrastiveLoss": 2, "NCELearnableTempDSLLoss": 3, "VidImgNCELearnableTempLoss": 5,
         "VidImgDivideNCELearnableTempLoss": 5, "NCELearnableTempLoss_vs_vc": 5, "NCELearnableTempLoss_vs_vc_fc": 5,
         "NCELearnableTempLoss_vsc": 5, "NCELearnableTempLoss_vsc_fc": 5}
LEGACY = ("TripletContrastiveLoss", "HardNegLoss", "MILNCEContrastiveLoss")


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "nce_family_n16.pt"), weights_only=False)


@pytest.mark.parametrize("name", FAMILY)
def test_loss_family_oracle_replays_reference_golden(gold, name):
    case = gold["cases"][name]
    xs = [gold["feats"][k].clone().requires_grad_(True) for k in case["keys"]]
    ls = gold["logit_scale"].clone().requires_grad_(True)
    loss = LF.nce_family_loss(name, xs, gold["temp"] if name == "NCEContrastiveLoss" else ls)
    loss.backward()
    assert abs(float(loss.detach()) - float(case["loss"])) < 1e-5 * abs(float(case["loss"]))
    for k, x in zip(case["keys"], xs):
        if k in case["grads"]:
            assert _rel(x.grad, case["grads"][k]) < 1e-5, k
        else:                                               # an argument the reference class never reads
            assert x.grad is None, k
    if case["d_logit_scale"] is not None:
        assert abs(float(ls.grad) - float(case["d_logit_scale"])) < 1e-5 * max(1.0, abs(float(case["d_logit_scale"])))


def test_dsl_closed_form_replays_reference_golden(gold):
    case = gold["cases"]["NCELearnableTempDSLLoss"]
    dv, dt, dl = LF.nce_dsl_closed_form_grads(gold["feats"]["vis"], gold["feats"]["txt"], gold["logit_scale"])
    assert _rel(dv, case["grads"]["vis"]) < 1e-5 and _rel(dt, case["grads"]["txt"]) < 1e-5
    assert abs(float(dl) - float(case["d_logit_scale"])) < 1e-5 * max(1.0, abs(float(case["d_logit_scale"])))


def test_product_term_tables_match_the_oracle_tables():
    """The bit-mask tables the kernels run (optimization/loss.py) state the same terms as the oracle's named tables."""
    from xpretrain_b200.optimization.loss import TERM_TABLES

    names = {(0, 1): "vt", (0, 3): "vc", (2, 3): "ic"}
    for name, (pairs, terms) in TERM_TABLES.items():
        mats = [names[p] for p in pairs]
        got = set()
        for axis, members, excl, target in terms:
            got.add(("row" if axis == 0 else "col", tuple(m for k, m in enumerate(mats) if members >> k & 1),
                     tuple(m for k, m in enumerate(mats) if excl >> k & 1), mats[target]))
        want = {(a, tuple(m), tuple(e), t) for a, m, e, t in LF.NCE_TERM_TABLES[name]}
        if name == "VidImgDivideNCELearnableTempLoss":              # its second matrix is I C^T of the image batch
            assert pairs == ((0, 1), (2, 3))
        assert got == want, name


@pytest.mark.parametrize("name", sorted(ARITY))
@pytest.mark.parametrize("as_dict", [True, False])
def test_build_loss_func_builds_every_name_with_the_reference_arity(name, as_dict):
    import inspect

    from xpretrain_b200.optimization.loss import build_loss_func

    cfg = {"loss_name": name, "temp": 0.05}
    mod = build_loss_func(cfg if as_dict else types.SimpleNamespace(**cfg))
    assert type(mod).__name__ == name
    assert len(inspect.signature(mod.forward).parameters) == ARITY[name]
    if name == "NCEContrastiveLoss":
        assert mod.temp == 0.05


@pytest.mark.parametrize("name", LEGACY)
def test_legacy_losses_raise_and_list_the_built_names(name):
    from xpretrain_b200.optimization.loss import build_loss_func

    with pytest.raises(NotImplementedError) as e:
        build_loss_func({"loss_name": name})
    for built in ARITY:
        assert repr(built) in str(e.value)


def test_shape_mismatch_raises_before_any_launch():
    """ValueError on CPU tensors proves the check runs before the first kernel (which would raise XpError)."""
    from xpretrain_b200.optimization.loss import build_loss_func

    v, t, c = torch.randn(8, 16), torch.randn(8, 16), torch.randn(6, 16)
    p = torch.tensor(4.6)
    with pytest.raises(ValueError):
        build_loss_func({"loss_name": "NCELearnableTempLoss_vs_vc"})(v, t, v, c, p)
    with pytest.raises(ValueError):
        build_loss_func({"loss_name": "NCELearnableTempLoss_vsc_fc"})(v, c, v, t, p)
    with pytest.raises(ValueError):
        build_loss_func({"loss_name": "NCELearnableTempDSLLoss"})(v, c, p)
    with pytest.raises(ValueError):
        build_loss_func({"loss_name": "NCEContrastiveLoss", "temp": 0.05})(v, torch.randn(8, 12))
    with pytest.raises(ValueError):
        build_loss_func({"loss_name": "VidImgNCELearnableTempLoss"})(v, t, c, v, p)
