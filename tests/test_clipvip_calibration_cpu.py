"""The bf16 arm of CLIP-ViP (clipvip_arm.py) on the CPU, and negative controls for the rule it defines.

On a tiny CLIP-ViP (width 128, 2 heads of 64, 32 px frames in 8 px patches, T = 3 frames interpolated from a 12-row
temporal table, M = 4 global rows, Lt = 8 tokens, 2 + 2 layers), one deliberate mistake is planted in the arm and the
mistaken arm is taken as "ours"; against the fp32 oracle and the correct arm it must break the rule the GPU module is
held to (every gradient whole and per slice).  Each case also records, without asserting it, whether the checks the
CLIP-ViP golden tests used before that rule would have let the mistake through (old_checks): each gradient's norm within
+-15 % of the oracle's, the cosine of the first 256 elements of each gradient above 0.97, and the worst bias / LayerNorm
vector error of ours against the worst of the arm (x 1.5).  Measured on these inputs:

  mistake                                         +-15 % norms   first-256 cosine   worst vector vs worst vector
  proxies without position row 0                  pass           pass               pass
  align_corners=True temporal interpolation       fail           fail               fail
  global queries see frame 0 only                 fail           fail               fail
  patch grid transposed                           pass           pass               fail
  q bias left unscaled by the q scale             fail           fail               fail
  temporal table reversed                         pass           pass               fail
The proxies' missing position row passes every old check; the rule catches it (first through layer 0's layer_norm1.weight
at 1.7 x the arm's error).
"""
import pytest
import torch

from clipvip_arm import Bf16Arm, features_objective, oracle_run, rule_violations
from oracle import clipvip_oracle as O

TINY = O.ClipVipCfg(vision=O.TowerCfg(128, 2, 2, 512), text=O.TowerCfg(128, 2, 2, 512), image_size=32, patch=8,
                    proj_dim=64, vocab=1000, max_text_pos=16, temporal_size=12, add_cls_num=3)
B, T, LT = 3, 3, 8

# mistake: (+-15 % norms pass, first-256 cosine passes, worst vector vs worst vector passes), as measured (see above)
OLD_CHECKS = {
    "proxy_no_pos0": (True, True, True),
    "align_corners": (False, False, False),
    "global_sees_frame0": (False, False, False),
    "patch_grid_transposed": (True, True, False),
    "q_bias_unscaled": (False, False, False),
    "temporal_reversed": (True, True, False),
}


@pytest.fixture(scope="module")
def runs():
    sd = O.init_state_dict(TINY, seed=3)
    video, ids, mask = O.synthetic_batch(B, T, LT, TINY, seed=4, ragged_text=True)
    obj = features_objective(B, TINY.proj_dim, seed=5)
    want = oracle_run(sd, video, ids, mask, TINY, obj, "fp32")
    arm = oracle_run(sd, video, ids, mask, TINY, obj, "bf16")
    return sd, video, ids, mask, obj, want, arm


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def old_checks(ours, want, arm):
    """(norms within +-15 %, first-256 cosines > 0.97, worst vector <= 1.5 x the arm's worst vector) of the golden tests
    before the rule, over the gradients of the fp32 oracle."""
    norms = cos = True
    vec_ours, vec_arm = [], []
    for n, w in want[2].items():
        g = ours[2][n]
        if float(w.norm()) >= 1e-4:
            norms &= 0.85 < float(g.norm()) / float(w.norm()) < 1.15
        a, b = g.flatten()[:256].double(), w.flatten()[:256].double()
        if float(b.norm()) >= 1e-6:
            cos &= float(torch.nn.functional.cosine_similarity(a, b, dim=0)) > 0.97
        if w.dim() == 1 and "k_proj.bias" not in n and float(w.norm()) > 1e-6:
            vec_ours.append(_rel(g, w))
            vec_arm.append(_rel(arm[2][n], w))
    return norms, cos, max(vec_ours) <= 1.5 * max(vec_arm)


def test_arm_runs_and_passes_its_own_rule(runs):
    """The correct arm, as "ours", passes the rule (ratio 1 everywhere) and stays within bf16 rounding of the oracle."""
    sd, video, ids, mask, obj, want, arm = runs
    bad, worst, _ = rule_violations("cpu arm", arm, want, arm, None, ids)
    assert not bad, bad
    assert abs(worst[0] - 1.0) < 1e-3
    assert set(arm[2]) == set(want[2])
    for n in want[2]:
        if not n.endswith("k_proj.bias"):          # zero exactly: the arm's is all rounding
            assert 0 < _rel(arm[2][n], want[2][n]) < 0.1, n
    assert 0 < _rel(arm[0], want[0]) < 2e-2 and 0 < _rel(arm[1], want[1]) < 2e-2


@pytest.mark.parametrize("stream", ["fp16", "bf16"])
def test_stream_arms_differ_from_the_fp32_stream_arm(runs, stream):
    """The fp16 and bf16 stream arms round the stream: their features move off the fp32-stream arm's, the bf16 one most."""
    sd, video, ids, mask, obj, want, arm = runs
    other = oracle_run(sd, video, ids, mask, TINY, obj, "bf16", stream=stream)
    d = _rel(other[0], arm[0]) + _rel(other[1], arm[1])
    assert d > 0
    if stream == "bf16":
        fp16 = oracle_run(sd, video, ids, mask, TINY, obj, "bf16", stream="fp16")
        assert d > _rel(fp16[0], arm[0]) + _rel(fp16[1], arm[1])


@pytest.mark.parametrize("mistake", list(OLD_CHECKS))
def test_mistake_in_the_arm_breaks_the_rule(runs, mistake):
    sd, video, ids, mask, obj, want, arm = runs
    ours = oracle_run(sd, video, ids, mask, TINY, obj, "bf16", arm=Bf16Arm(mistake=mistake))
    bad, _, _ = rule_violations(f"cpu {mistake}", ours, want, arm, None, ids)
    assert bad, f"{mistake}: the mistake passes the calibrated rule"
    old = old_checks(ours, want, arm)
    print(f"{mistake}: {len(bad)} violations, first: {bad[0]}\n  old checks (norms, first-256 cosine, worst vector): {old}")
    if old != OLD_CHECKS[mistake]:
        print(f"  (recorded {OLD_CHECKS[mistake]})")
