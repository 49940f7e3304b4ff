"""Golden vectors for the contrastive-loss family of CLIP-ViP/src/optimization/loss.py from the REAL reference.

Needs a checkout of the reference, named by XP_REFERENCE_ROOT:

    XP_REFERENCE_ROOT=<path to XPretrain> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_loss_family.py

Imports the reference's own loss classes unmodified, runs them and their autograd on seeded features in fp64 and fp32 on
CPU, asserts that oracle/loss_family_oracle.py reproduces every loss and gradient, and writes nce_family_n16.pt, which
tests/test_loss_family_cpu.py (CPU) and tests/test_gpu_losses.py (GPU) replay without the reference.  No reference source
is copied; only numeric outputs are stored.
"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ["XP_REFERENCE_ROOT"]     # a checkout of microsoft/XPretrain
sys.path.insert(0, os.path.join(REF, "CLIP-ViP"))
sys.dont_write_bytecode = True

from oracle import loss_family_oracle as LF  # noqa: E402


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


NCE_FAMILY = ("NCEContrastiveLoss", "NCELearnableTempDSLLoss", "VidImgNCELearnableTempLoss", "VidImgDivideNCELearnableTempLoss",
              "NCELearnableTempLoss_vs_vc", "NCELearnableTempLoss_vs_vc_fc", "NCELearnableTempLoss_vsc",
              "NCELearnableTempLoss_vsc_fc")


def nce_family_case():
    """Every loss class of loss.py:143-324 plus NCEContrastiveLoss (:67-83) on one set of features: N = 16, d = 128, and an
    image/caption pair with M = 10 rows for VidImgDivideNCELearnableTempLoss.  Per class, the oracle's loss and gradients
    (autograd through oracle.loss_family_oracle.nce_family_loss) and, for the DSL loss, its closed-form gradients must match
    the reference class's autograd in fp64 (<= 1e-12 relative) and in fp32 (<= 1e-5); stores the reference's fp32 loss and
    gradients."""
    import src.optimization.loss as ref

    g = torch.Generator().manual_seed(13)
    N, M, d = 16, 10, 128
    base = torch.nn.functional.normalize(torch.randn(N, d, generator=g), dim=-1)
    feats = {k: torch.nn.functional.normalize(torch.randn(N, d, generator=g) + 0.5 * base, dim=-1)
             for k in ("vis", "txt", "img", "cap")}
    ib = torch.nn.functional.normalize(torch.randn(M, d, generator=g), dim=-1)
    feats["img_m"], feats["cap_m"] = (torch.nn.functional.normalize(torch.randn(M, d, generator=g) + 0.5 * ib, dim=-1)
                                      for _ in range(2))
    temp, logit_scale = 0.05, torch.tensor(4.6)
    gold = {"feats": feats, "logit_scale": logit_scale, "temp": temp, "cases": {}}
    for name in NCE_FAMILY:
        keys = (("vis", "txt") if name in ("NCEContrastiveLoss", "NCELearnableTempDSLLoss") else
                ("vis", "txt", "img_m", "cap_m") if name == "VidImgDivideNCELearnableTempLoss" else ("vis", "txt", "img", "cap"))
        for dt in (torch.float64, torch.float32):
            xs = [feats[k].to(dt).clone().requires_grad_(True) for k in keys]
            ls = logit_scale.to(dt).clone().requires_grad_(True)
            mod = getattr(ref, name)(types.SimpleNamespace(temp=temp))
            args = xs if name == "NCEContrastiveLoss" else xs + [ls]
            loss = mod(*args)
            loss.backward()
            want = [x.grad for x in xs] + ([] if name == "NCEContrastiveLoss" else [ls.grad])
            ys = [feats[k].to(dt).clone().requires_grad_(True) for k in keys]
            ls2 = logit_scale.to(dt).clone().requires_grad_(True)
            lo = LF.nce_family_loss(name, ys, temp if name == "NCEContrastiveLoss" else ls2)
            lo.backward()
            got = [y.grad for y in ys] + ([] if name == "NCEContrastiveLoss" else [ls2.grad])
            tol = 1e-12 if dt == torch.float64 else 1e-5
            assert abs(float(lo.detach()) - float(loss.detach())) <= tol * abs(float(loss.detach())), name
            for a, b in zip(got, want):
                if b is None:                                   # a feature the reference class never reads
                    assert a is None, name
                    continue
                assert rel(a, b) <= tol if b.dim() else abs(float(a) - float(b)) <= tol * max(1.0, abs(float(b))), (name, dt)
            if name == "NCELearnableTempDSLLoss":
                cf = LF.nce_dsl_closed_form_grads(xs[0].detach(), xs[1].detach(), ls.detach())
                for a, b in zip(cf, want):
                    assert (rel(a, b) if b.dim() else abs(float(a) - float(b)) / max(1.0, abs(float(b)))) <= tol, (name, dt)
        gold["cases"][name] = {"keys": keys, "loss": loss.detach(),
                               "grads": {k: x.grad for k, x in zip(keys, xs) if x.grad is not None},
                               "d_logit_scale": None if name == "NCEContrastiveLoss" else ls.grad}
        print(f"[nce_family_n16] {name}: oracle matches the reference's loss and autograd (fp64 and fp32)")
    path = os.path.join(HERE, "nce_family_n16.pt")
    torch.save(gold, path)
    print(f"  wrote {path} ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    nce_family_case()
