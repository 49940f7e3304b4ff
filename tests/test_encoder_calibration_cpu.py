"""Negative controls for the calibrated rule that test_gpu_encoder_calibration.py holds the encoders to, on the CPU.

On a tiny Swin-3D and a tiny divided TimeSformer, the fp32 oracle is run with one deliberate mistake and taken as "ours";
against the clean fp32 oracle it must break the same rule (whole tensors and slices) that the GPU modules are held to,
with the oracle's own bf16 CPU run as the arm.  Each case also records whether the thresholds the module tests used before
the rule would have let the mistake through (see old_checks): the output check alone (Swin-3D rel-L2 < 2e-2 and cosine >
0.9997, TimeSformer < 1.5e-2 and > 0.9998), and the golden checks, which add cosines > 0.985 (Swin-3D) / 0.99 and dx >
0.995 (TimeSformer) on the few gradients a golden stores.  The test asserts that record; the measured margins were:

  mistake                                                        output alone           golden checks
  Swin-3D relative_position_index transposed                     pass (rel 7e-4)        fail (a bias table, cos -0.07)
  Swin-3D shift mask taken as mask[w // B], not mask[w % nW]     pass (rel 1.7e-3)      fail (a bias table, cos 0.74)
  Swin-3D DropPath factors of two samples swapped (last block)   fail (rel 0.28)        fail
  Swin-3D one window type missing from the bias-table gradient   pass (exact)           fail (a bias table, cos 0.976)
  TimeSformer time table added with its frames reversed          fail (rel 3e-2)        fail
The golden checks catch these only through the bias tables and the time table they happen to store (the released-config
check read six gradients, one bias table among them); the rule needs no such luck: every gradient is checked, whole and
per slice.
"""
import os

import pytest
import torch

from contract_harness import calibrated_model_rows
from encoder_cases import model_rows, swin_oracle, tsf_oracle
from oracle import swin3d_oracle as SO
from oracle import timesformer_oracle as TO

SWIN = SO.Swin3DCfg(patch_size=(1, 4, 4), embed_dim=16, depths=(2, 2), num_heads=(2, 4), stages=(0, 1),
                    downsample_stages=(0,), window_size=((2, 3, 3), (2, 3, 3)))
SWIN_SHAPE = (2, 4, 24, 24)            # B, D, H, W: 4 x 6 x 6 tokens, 8 shifted window types per sample in layer 0
TSF = TO.TimeSformerCfg(depth=2, num_frames=4, H=3, W=4, embed_dim=32, num_heads=2)
TSF_SHAPE = (2, 4, 3, 4)               # B, T, H, W


def _cos(a, b):
    return float(torch.nn.functional.cosine_similarity(a.double().flatten(), b.double().flatten(), dim=0))


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def old_checks(kind, ours, want, golden_dir):
    """The module tests' checks before the rule -> (output alone passes, golden checks pass).  Output: rel-L2 and cosine.
    Golden: the output, dx of the first frame (TimeSformer) and the gradients a golden stores (first 8 rows of each matrix,
    Swin-3D bias tables whole), from swin3d_small_b2 / timesformer_interp_b2 with Swin-3D's layer 2 mapped to the tiny
    model's last layer."""
    gold = "swin3d_small_b2" if kind == "swin" else "timesformer_interp_b2"
    names = torch.load(os.path.join(golden_dir, gold + ".pt"), weights_only=False)["grads"]
    names = [n.replace("layers.2.", "layers.1.") for n in names]
    out_rel, out_cos, dx_cos, g_cos = (2e-2, 0.9997, None, 0.985) if kind == "swin" else (1.5e-2, 0.9998, 0.995, 0.99)
    out_ok = _rel(ours[0], want[0]) < out_rel and _cos(ours[0], want[0]) > out_cos

    def part(n, g):
        return g if g.dim() < 2 or n.endswith("relative_position_bias_table") else g[:8]
    grads_ok = all(_cos(part(n, ours[2][n]), part(n, want[2][n])) > g_cos for n in names)
    dx_ok = dx_cos is None or _cos(ours[1][:, 0], want[1][:, 0]) > dx_cos
    return out_ok, out_ok and dx_ok and grads_ok


def _drop_masks():
    """keep 0.5: factors 0 or 2, samples 0 and 1 different in every block."""
    return [(torch.tensor([2.0, 0.0]), torch.tensor([2.0, 2.0])) for _ in range(sum(SWIN.depths))]


def _swin_mistake(name, monkeypatch, sd, masks):
    """-> (state dict, masks) of the mistaken run, with SO patched where the mistake is in the arithmetic."""
    if name == "index_transposed":
        sd = {k: (v.t().contiguous() if k.endswith("relative_position_index") else v) for k, v in sd.items()}
    elif name == "droppath_swapped":
        masks = list(masks)
        masks[-1] = (masks[-1][0].flip(0), masks[-1][1])
    elif name in ("mask_by_sample", "bias_grad_missing_type"):
        orig = SO.window_attention

        def patched(sd_, p, xw, heads, mask):
            if mask is None:
                return orig(sd_, p, xw, heads, mask)
            nW, w = mask.shape[0], torch.arange(xw.shape[0])
            if name == "mask_by_sample":
                return orig(sd_, p, xw, heads, mask[w // (xw.shape[0] // nW)])
            per_window = mask[w % nW]          # one mask per window: the same arithmetic, windows separable
            frozen = dict(sd_, **{p + "relative_position_bias_table": sd_[p + "relative_position_bias_table"].detach()})
            return torch.where((w % nW == 0)[:, None, None], orig(frozen, p, xw, heads, per_window),
                               orig(sd_, p, xw, heads, per_window))
        monkeypatch.setattr(SO, "window_attention", patched)
    return sd, masks


SWIN_MISTAKES = {  # name: (output alone passes, golden checks pass)
    "index_transposed": (True, False), "mask_by_sample": (True, False), "droppath_swapped": (False, False),
    "bias_grad_missing_type": (True, False)}


@pytest.mark.parametrize("name", list(SWIN_MISTAKES))
def test_swin3d_mistake_breaks_the_calibrated_rule(monkeypatch, golden_dir, name):
    B, D, H, W = SWIN_SHAPE
    sd = SO.init_state_dict(SWIN, seed=1)
    video = SO.synthetic_video(B, D, H, W, SWIN, seed=2)
    masks = _drop_masks() if name == "droppath_swapped" else None
    out_shape = SO.swin3d_forward(sd, video, SWIN).shape
    w_out = torch.randn(out_shape, generator=torch.Generator().manual_seed(3)) / (out_shape[1:].numel()) ** 0.5
    want = swin_oracle(sd, video, w_out, SWIN, masks, "fp32")
    arm = swin_oracle(sd, video, w_out, SWIN, masks, "bf16")
    bad_sd, bad_masks = _swin_mistake(name, monkeypatch, sd, masks)
    ours = swin_oracle(bad_sd, video, w_out, SWIN, bad_masks, "fp32")
    rows, slices = model_rows(ours, want, arm, None)
    bad, _, _ = calibrated_model_rows(f"cpu swin {name}", rows, slices)
    assert bad, f"{name}: the mistake passes the calibrated rule"
    print(f"{name}: {len(bad)} violations, first: {bad[0]}")
    assert old_checks("swin", ours, want, golden_dir) == SWIN_MISTAKES[name]


def test_timesformer_reversed_time_table_breaks_the_calibrated_rule(monkeypatch, golden_dir):
    B, T, H, W = TSF_SHAPE
    sd = TO.init_state_dict(TSF, seed=4)
    x = TO.synthetic_input(B, T, H, W, TSF, seed=5)
    w_out = torch.randn(B, T, TSF.embed_dim, H, W, generator=torch.Generator().manual_seed(6)) / (B * T * H * W) ** 0.5
    want = tsf_oracle(sd, x, w_out, TSF, None, "fp32")
    arm = tsf_oracle(sd, x, w_out, TSF, None, "bf16")
    orig = TO.interpolated_tables
    monkeypatch.setattr(TO, "interpolated_tables", lambda *a: (lambda pos, time: (pos, time.flip(0)))(*orig(*a)))
    ours = tsf_oracle(sd, x, w_out, TSF, None, "fp32")
    rows, slices = model_rows(ours, want, arm, None)
    bad, _, _ = calibrated_model_rows("cpu tsf time_reversed", rows, slices)
    assert bad, "the reversed time table passes the calibrated rule"
    print(f"time_reversed: {len(bad)} violations, first: {bad[0]}")
    assert old_checks("tsf", ours, want, golden_dir) == (False, False)
