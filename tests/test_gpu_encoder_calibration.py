"""H100: the divided-space-time TimeSformer (BASELINE.json config #4) and the Swin-3D video encoder (config #5) under the
calibrated rule of DESIGN.md §2, every gradient whole.

Each case compares three runs with the fp32 oracle on this GPU:
  ours      the module (bf16 kernels and a bf16 token stream)
  arm       the oracle with bf16 weights, input and activations: both modules keep their token stream in bf16, so this is
            the arm that rounds where they do (as for the joint TimeSformer in test_gpu_timesformer_variants.py); its
            attention backward forms delta from the stored bf16 output, as the kernels do (KernelRoundedSoftmaxAV)
  autocast  the oracle under bf16 autocast: its ratio is printed, never asserted
and asserts
  whole     the output, dx (TimeSformer; the Swin-3D function returns no video gradient) and every parameter gradient:
            err(ours) <= 1.5 x err(arm); the parameters that receive a gradient are exactly the oracle's (none for the
            TimeSformer's `norm`, nor for Swin-3D's `norm_local` / `local_feat_proj`)
  slices    contract_harness.calibrated, per slice with its floor of 2^-16 x the slice's norm: the output per
            (sample, frame), every relative_position_bias_table gradient per head column, every qkv weight and bias gradient
            per q / k / v third (the TimeSformer's attn.qkv and temporal_attn.qkv)
The fp32 oracle runs without TF32 (Swin-3D's patch embedding is a conv3d).  `pytest -s` prints each case's worst
whole-tensor and slice ratio and, at the end of the module, the worst of this module's cases.  The runs and the cases
live in encoder_cases.py; the full-width TimeSformer and the released Swin-3D config run the same cases under their
long-standing names in test_gpu_timesformer.py and test_gpu_swin3d.py.
"""
import os

import pytest
import torch

from contract_harness import Report
from encoder_cases import swin3d_case, timesformer_case
from oracle import swin3d_oracle as SO
from oracle import timesformer_oracle as TO

pytestmark = pytest.mark.gpu

REPORT = Report("encoder calibration: worst err / bf16-arm err per case (whole tensor, slice)", width=36,
                fmt=lambda v: f"whole {v[0][0]:.3f} ({v[0][1]})  slice {v[1][0]:.3f} ({v[1][1]})")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    REPORT.print()


TSF_GOLDENS = ["timesformer_interp_b2", "timesformer_native_b2", "timesformer_train_droppath"]
TINY_TSF = dict(depth=2, num_frames=4, H=3, W=4, embed_dim=128, num_heads=2)
TSF_CASES = {  # name: (cfg, B, T, H, W, weight seed, data seed)
    "bench_8x7x7": (dict(depth=2), 4, 8, 7, 7, 5, 6),                    # bench.py's geometry: both tables interpolated
    "t1": (TINY_TSF, 3, 1, 3, 4, 7, 8),                                  # one frame: temporal groups of one token
    "hw1": (TINY_TSF, 3, 4, 1, 1, 9, 10),                                # a 1 x 1 grid: spatial groups of one token
}


@pytest.mark.parametrize("name", TSF_GOLDENS)
def test_timesformer_golden_configs_calibrated(dev, golden_dir, name):
    gold = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    train = gold.get("rate") is not None
    timesformer_case(dev, f"tsf {name}", TO.TimeSformerCfg(**gold["cfg"]), gold["B"], gold["T"], gold["H"], gold["W"],
                     gold["weight_seed"], gold["data_seed"], rate=gold["rate"] if train else None,
                     masks=gold["masks"] if train else None, report=REPORT)


@pytest.mark.parametrize("name", list(TSF_CASES))
def test_timesformer_calibrated(dev, name):
    cfg, B, T, H, W, ws, ds = TSF_CASES[name]
    timesformer_case(dev, f"tsf {name}", TO.TimeSformerCfg(**cfg), B, T, H, W, ws, ds, report=REPORT)


SWIN_GOLDENS = {"swin3d_small_b2": {"colsum"}, "swin3d_padded_b1": {"colsum"}, "swin3d_train_droppath": {"colsum"}}
SMALL = dict(embed_dim=64, depths=(2, 2, 2), num_heads=(2, 4, 8), stages=(0, 1, 2), downsample_stages=(0, 1),
             window_size=((2, 3, 5), (4, 3, 5), (8, 3, 5)))
SWIN_CASES = {  # name: (cfg, B, D, H, W, weight seed, data seed, bias-gradient branches)
    # bench.py's geometry: 28 x 28 tokens, every stage pads its windows, PatchMerging pads 7 -> 4
    "bench_1x32x224x224": ({}, 1, 32, 224, 224, 6, 7, {"colsum"}),
    "small_b3_shifted": (SMALL, 3, 4, 48, 48, 8, 9, {"colsum"}),              # the mask cycle crosses samples
    "temporal_shift_3d": (dict(SMALL, temporal_no_shifting=False), 2, 8, 48, 80, 10, 11, {"colsum"}),   # 27 regions
    "no_patch_norm": (dict(SMALL, patch_norm=False), 2, 4, 48, 80, 12, 13, {"colsum"}),
    "d1": (SMALL, 2, 1, 48, 80, 14, 15, {"colsum", "torch"}),                  # windows clamp to D = 1: L = 15
    "d3": (SMALL, 2, 3, 48, 80, 16, 17, {"colsum", "torch"}),                  # stage 1 clamps to D = 3: L = 45
}


@pytest.mark.parametrize("name", list(SWIN_GOLDENS))
def test_swin3d_golden_configs_calibrated(dev, golden_dir, name):
    gold = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    rate = gold["train_rate"]
    swin3d_case(dev, f"swin {name}", SO.Swin3DCfg(**gold["cfg"]), gold["B"], gold["D"], gold["H"], gold["W"],
                gold["weight_seed"], gold["data_seed"], SWIN_GOLDENS[name], rate=rate,
                masks=gold["masks"] if rate else None, report=REPORT)


@pytest.mark.parametrize("name", list(SWIN_CASES))
def test_swin3d_calibrated(dev, name):
    cfg, B, D, H, W, ws, ds, branches = SWIN_CASES[name]
    swin3d_case(dev, f"swin {name}", SO.Swin3DCfg(**cfg), B, D, H, W, ws, ds, branches, report=REPORT)
