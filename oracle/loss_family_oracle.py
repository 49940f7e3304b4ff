"""CPU oracle for the contrastive-loss family of CLIP-ViP/src/optimization/loss.py — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

fp32 / fp64 plain-PyTorch restatements of every loss class the product builds besides NCELearnableTempLoss and
NCELearnableTempLoss_vsc_fc (those are in clipvip_oracle.py): the learnable / fixed temperature InfoNCE variants as a
table of cross-entropy terms, plus the dual-softmax loss and its closed-form gradients.  Pinned by
`tests/golden/make_golden_loss_family.py` against the reference's own classes and their autograd; replayed on any machine
by tests/test_loss_family_cpu.py.  Only tests, tools and the golden generator import it.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from .clipvip_oracle import nce_learnable_temp_loss

Tensor = torch.Tensor

# The contrastive-loss family of loss.py as data.  Matrices (logits, before the scale): "vt" = V T^T, "vc" = V C^T,
# "ic" = I C^T.  A term is (axis, members, members entering without their diagonal, target): for each index i the LSE over
# the union of row / column i of the members minus the target's diagonal entry, averaged over i; the loss is the sum.
NCE_TERM_TABLES = {
    "NCEContrastiveLoss": (("row", ("vt",), (), "vt"), ("col", ("vt",), (), "vt")),                     # loss.py:76-83
    "VidImgDivideNCELearnableTempLoss": (("row", ("vt",), (), "vt"), ("col", ("vt",), (), "vt"),        # :170-183
                                         ("row", ("ic",), (), "ic"), ("col", ("ic",), (), "ic")),
    "NCELearnableTempLoss_vs_vc": (("row", ("vt",), (), "vt"), ("col", ("vt",), (), "vt"),              # :212-225
                                   ("row", ("vc",), (), "vc"), ("col", ("vc",), (), "vc")),
    "NCELearnableTempLoss_vs_vc_fc": (("row", ("vt",), (), "vt"), ("col", ("vt",), (), "vt"),           # :235-254
                                      ("row", ("vc",), (), "vc"), ("col", ("vc",), (), "vc"),
                                      ("row", ("ic",), (), "ic"), ("col", ("ic",), (), "ic")),
    "NCELearnableTempLoss_vsc": (("col", ("vt",), (), "vt"), ("col", ("vc",), (), "vc"),                # :264-286
                                 ("row", ("vt", "vc"), ("vc",), "vt"), ("row", ("vt", "vc"), ("vt",), "vc")),
    "NCELearnableTempLoss_vsc_fc": (("col", ("vt",), (), "vt"), ("col", ("vc",), (), "vc"),             # :296-324
                                    ("row", ("vt", "vc"), ("vc",), "vt"), ("row", ("vt", "vc"), ("vt",), "vc"),
                                    ("col", ("ic",), (), "ic"), ("row", ("ic",), (), "ic")),
}


def nce_terms_loss(mats: Dict[str, Tensor], terms) -> Tensor:
    """Sum over `terms` (see NCE_TERM_TABLES) of mean_i(LSE over the members' row / column i - target_ii); mats are scaled."""
    total = 0.0
    for axis, members, excl, target in terms:
        parts = []
        for m in members:
            x = mats[m] if axis == "row" else mats[m].t()
            if m in excl:
                eye = torch.eye(x.shape[0], dtype=torch.bool, device=x.device)
                x = x.masked_fill(eye, float("-inf"))
            parts.append(x)
        total = total + (torch.logsumexp(torch.cat(parts, 1), 1) - mats[target].diagonal()).mean()
    return total


def nce_dsl_loss(vis: Tensor, txt: Tensor, logit_scale: Tensor) -> Tensor:
    """NCELearnableTempDSLLoss.forward, loss.py:193-202: CE over the rows of A' = Z * softmax(Z, 0) and over the rows of
    Z^T * softmax(Z^T, 0) (= the columns of B' = Z * softmax(Z, 1)); the re-weighting is not detached."""
    z = vis @ txt.t() * logit_scale.exp()
    labels = torch.arange(z.shape[0], device=z.device)
    return F.cross_entropy(z * torch.softmax(z, 0), labels) + F.cross_entropy(z.t() * torch.softmax(z.t(), 0), labels)


def nce_dsl_closed_form_grads(vis: Tensor, txt: Tensor, logit_scale: Tensor):
    """Closed-form gradients of nce_dsl_loss: with Pc / Pr the column / row softmax of Z, A' = Z Pc, B' = Z Pr,
    GA = (softmax_row(A') - I)/N, GB = (softmax_col(B') - I)/N, u_j = sum_i GA Z Pc, w_i = sum_j GB Z Pr:
    G_Z = Pc (GA (1 + Z) - u_j) + Pr (GB (1 + Z) - w_i);  dV = s G_Z T, dT = s G_Z^T V, d logit_scale = sum G_Z Z."""
    s = logit_scale.exp()
    z = vis @ txt.t() * s
    n = z.shape[0]
    eye = torch.eye(n, dtype=z.dtype, device=z.device)
    pc, pr = torch.softmax(z, 0), torch.softmax(z, 1)
    ga = (torch.softmax(z * pc, 1) - eye) / n
    gb = (torch.softmax(z * pr, 0) - eye) / n
    u = (ga * z * pc).sum(0, keepdim=True)
    w = (gb * z * pr).sum(1, keepdim=True)
    g = pc * (ga * (1 + z) - u) + pr * (gb * (1 + z) - w)
    return s * g @ txt, s * g.t() @ vis, (g * z).sum()


def nce_family_loss(name: str, feats, t) -> Tensor:
    """Any built loss of loss.py by class name.  feats: the forward's feature arguments (vis, txt[, img, cap]);
    t: the learnable log-scale tensor, or cfg.temp (a float) for NCEContrastiveLoss."""
    if name == "NCELearnableTempLoss":
        return nce_learnable_temp_loss(feats[0], feats[1], t)
    if name == "NCELearnableTempDSLLoss":
        return nce_dsl_loss(feats[0], feats[1], t)
    if name == "VidImgNCELearnableTempLoss":                              # loss.py:151-160
        return nce_learnable_temp_loss(torch.cat([feats[0], feats[2]]), torch.cat([feats[1], feats[3]]), t)
    s = 1.0 / t if name == "NCEContrastiveLoss" else t.exp()
    mats = {"vt": feats[0] @ feats[1].t() * s}
    if len(feats) > 2:
        mats["vc"] = feats[0] @ feats[3].t() * s if feats[0].shape[0] == feats[3].shape[0] else None
        mats["ic"] = feats[2] @ feats[3].t() * s
    return nce_terms_loss(mats, NCE_TERM_TABLES[name])
