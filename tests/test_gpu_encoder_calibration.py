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
  slices    test_gpu_attention_contract.calibrated, per slice with its floor of 2^-16 x the slice's norm: the output per
            (sample, frame), every relative_position_bias_table gradient per head column, every qkv weight and bias gradient
            per q / k / v third (the TimeSformer's attn.qkv and temporal_attn.qkv)
The fp32 oracle runs without TF32 (Swin-3D's patch embedding is a conv3d).  `pytest -s` prints each case's worst
whole-tensor and slice ratio and, at the end of the module, the worst of this module's cases.  The full-width TimeSformer
and the released Swin-3D config run these same checks (timesformer_case / swin3d_case) under their long-standing names in
test_gpu_timesformer.py and test_gpu_swin3d.py.
"""
import contextlib
import os

import pytest
import torch

from oracle import swin3d_oracle as SO
from oracle import timesformer_oracle as TO
from test_gpu_timesformer_variants import calibrated_model_rows

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
SUMMARY = {}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if SUMMARY:
        print("\nencoder calibration: worst err / bf16-arm err per case (whole tensor, slice)")
        for k in sorted(SUMMARY):
            (w, wn), (s, sn) = SUMMARY[k]
            print(f"  {k:36s} whole {w:.3f} ({wn})  slice {s:.3f} ({sn})")


@contextlib.contextmanager
def _no_tf32():
    """The fp32 oracle is the truth: no TF32 in its matmuls or in Swin-3D's conv3d patch embedding."""
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


# =================================================================================================== shared pieces
def frame_slices(out):
    """Slice ids of an output whose first two dims are (sample, frame)."""
    B, T = out.shape[:2]
    ids = torch.arange(B * T, device=out.device).view(B, T, *[1] * (out.dim() - 2)).expand(out.shape)
    return ids, lambda i: f"(sample {i // T}, frame {i % T})"


def param_slices(grads):
    """Per head column of every relative_position_bias_table gradient, per q / k / v third of every qkv gradient."""
    out = {}
    for n, g in grads.items():
        if n.endswith("relative_position_bias_table"):
            out[n] = (torch.arange(g.shape[1], device=g.device).expand(g.shape), lambda i: f"head {i}")
        elif n.endswith("qkv.weight") or n.endswith("qkv.bias"):
            C = g.shape[0] // 3
            ids = (torch.arange(3 * C, device=g.device) // C).view(-1, *[1] * (g.dim() - 1)).expand(g.shape)
            out[n] = (ids, lambda i: "qkv"[i])
    return out


def model_rows(ours, want, arm, ac):
    """ours / want / arm / ac: (out, dx or None, {name: grad}) -> rows for calibrated_model_rows, and the slice map."""
    assert set(ours[2]) == set(want[2]), f"gradients received differ from the oracle's: {set(ours[2]) ^ set(want[2])}"
    rows = [("out", ours[0], want[0], arm[0], ac and ac[0])]
    if want[1] is not None:
        rows.append(("dx", ours[1], want[1], arm[1], ac and ac[1]))
    rows += [(n, ours[2][n], want[2][n], arm[2][n], ac and ac[2][n]) for n in sorted(want[2])]
    return rows, {"out": frame_slices(want[0]), **param_slices(want[2])}


def check_case(tag, ours, want, arm, ac):
    rows, slices = model_rows(ours, want, arm, ac)
    bad, worst, worst_sl = calibrated_model_rows(tag, rows, slices)
    SUMMARY[tag] = (worst, worst_sl)
    assert not bad, "\n".join(bad)


class KernelRoundedSoftmaxAV(torch.autograd.Function):
    """softmax(s) @ v of the bf16 arm, with the backward the attention kernels use on purpose (seg_attention.cu, as
    oracle/attention_ref.sdpa's arms): delta = rowsum(dO * O) from the stored bf16 output O, not from the probabilities
    (torch's softmax backward).  Exactly, both deltas are equal; in bf16 they differ by the rounding of O, and that
    difference is all that the k part of every qkv bias gradient (zero exactly: a shift of every key leaves each softmax
    row unchanged) and much of a bias-table gradient (a sum of dS) are made of."""

    @staticmethod
    def forward(ctx, s, v):
        p = s.softmax(-1)
        o = p @ v
        ctx.save_for_backward(p, v, o)
        return o

    @staticmethod
    def backward(ctx, do):
        p, v, o = ctx.saved_tensors
        delta = (do.float() * o.float()).sum(-1, keepdim=True)
        ds = (p.float() * ((do @ v.transpose(-1, -2)).float() - delta)).to(p.dtype)
        return ds, p.transpose(-1, -2) @ do


@contextlib.contextmanager
def _arm_core(oracle_module, mode):
    """Within it, the oracle module's attention core is the kernel-rounded one when `mode` is the bf16 arm."""
    orig = oracle_module.softmax_av
    if mode == "bf16":
        oracle_module.softmax_av = KernelRoundedSoftmaxAV.apply
    try:
        yield
    finally:
        oracle_module.softmax_av = orig


def _cast_masks(masks, dt):
    return None if masks is None else [None if m is None else tuple(t.to(dt) for t in m) for m in masks]


# ====================================================================================================== TimeSformer
def tsf_oracle(sd, x, w_out, cfg, masks, mode):
    """mode: 'fp32' (the truth), 'bf16' (bf16 weights, input and activations) or 'autocast'.  -> (out, dx, grads)."""
    dt = bf16 if mode == "bf16" else f32
    sdo = {k: v.detach().to(dt).requires_grad_(True) for k, v in sd.items()}
    xo = x.detach().to(dt).requires_grad_(True)
    with torch.autocast(device_type=x.device.type, dtype=bf16, enabled=mode == "autocast"), _arm_core(TO, mode), \
            _no_tf32():
        out = TO.timesformer_forward(sdo, xo, cfg, drop_masks=_cast_masks(masks, dt) if mode == "bf16" else masks)
        out = out.float()
        (out * w_out).sum().backward()
    return out.detach(), xo.grad, {n: p.grad for n, p in sdo.items() if p.grad is not None}


def timesformer_case(dev, tag, cfg, B, T, H, W, weight_seed, data_seed, rate=None, masks=None):
    """One TimeSformer case under the rule; returns (ours, fp32 oracle), each (out, dx, {name: grad})."""
    from xpretrain_b200.modeling.timesformer import TimeSformer

    sd = TO.init_state_dict(cfg, seed=weight_seed)
    model = TimeSformer(depth=cfg.depth, num_frames=cfg.num_frames, H=cfg.H, W=cfg.W, embed_dim=cfg.embed_dim,
                        num_heads=cfg.num_heads, drop_path_rate=rate or 0.1)
    model.load_state_dict(sd, strict=True)
    model = model.to(dev)
    if masks is not None:
        masks = [None if m is None else tuple(t.to(dev) for t in m) for m in masks]
        model.train()
        model.forced_drop_masks = masks
    else:
        model.eval()
    x = TO.synthetic_input(B, T, H, W, cfg, seed=data_seed).to(dev).requires_grad_(True)
    g = torch.Generator().manual_seed(data_seed + 1)
    w_out = (torch.randn(B, T, cfg.embed_dim, H, W, generator=g) / (B * T * H * W) ** 0.5).to(dev)
    out = model(x)
    (out * w_out).sum().backward()
    ours = (out.detach(), x.grad, {n: p.grad for n, p in model.named_parameters() if p.grad is not None})
    sd = {k: v.to(dev) for k, v in sd.items()}
    runs = [tsf_oracle(sd, x, w_out, cfg, masks, mode) for mode in ("fp32", "bf16", "autocast")]
    check_case(tag, ours, *runs)
    return ours, runs[0]


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
              masks=gold["masks"] if train else None)


@pytest.mark.parametrize("name", list(TSF_CASES))
def test_timesformer_calibrated(dev, name):
    cfg, B, T, H, W, ws, ds = TSF_CASES[name]
    timesformer_case(dev, f"tsf {name}", TO.TimeSformerCfg(**cfg), B, T, H, W, ws, ds)


# ========================================================================================================= Swin-3D
def swin_oracle(sd, video, w_out, cfg, masks, mode):
    """As tsf_oracle; the index buffers stay int64.  -> (out, None, grads)."""
    dt = bf16 if mode == "bf16" else f32
    sdo = {k: (v.detach().to(dt).requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    with torch.autocast(device_type=video.device.type, dtype=bf16, enabled=mode == "autocast"), _arm_core(SO, mode), \
            _no_tf32():
        out = SO.swin3d_forward(sdo, video.to(dt), cfg, drop_masks=_cast_masks(masks, dt) if mode == "bf16" else masks)
        out = out.float()
        (out * w_out).sum().backward()
    return out.detach(), None, {n: p.grad for n, p in sdo.items() if p.is_floating_point() and p.grad is not None}


def bias_grad_branches(model):
    """How the module sums each layer's bias-table gradient (modeling/swin3d.py, _block_bwd): 'colsum' (the column-sum
    kernel, heads * L^2 % 8 == 0) or 'torch' (its fallback for odd windows), over the geometries the last forward built."""
    return {"colsum" if model.num_heads[k[1]] * geo["L"] ** 2 % 8 == 0 else "torch"
            for k, geo in model._tables.items() if k[0] == "layer"}


def swin3d_case(dev, tag, cfg, B, D, H, W, weight_seed, data_seed, branches, rate=None, masks=None):
    """One Swin-3D case under the rule; returns (ours, fp32 oracle), each (out, None, {name: grad})."""
    from xpretrain_b200.modeling.swin3d import SwinTransformer3D

    sd = SO.init_state_dict(cfg, seed=weight_seed)
    model = SwinTransformer3D(patch_size=list(cfg.patch_size), embed_dim=cfg.embed_dim, depths=list(cfg.depths),
                              num_heads=list(cfg.num_heads), stages=list(cfg.stages),
                              downsample_stages=list(cfg.downsample_stages),
                              window_size=[list(w) for w in cfg.window_size], patch_norm=cfg.patch_norm,
                              local_window=cfg.local_window, drop_path_rate=rate or 0.2,
                              temporal_no_shifting=cfg.temporal_no_shifting)
    model.load_state_dict(sd, strict=True)
    model = model.to(dev)
    if masks is not None:
        masks = [None if m is None else tuple(t.to(dev) for t in m) for m in masks]
        model.train()
        model.forced_drop_masks = masks
    else:
        model.eval()
    video = SO.synthetic_video(B, D, H, W, cfg, seed=data_seed).to(dev)
    out, _ = model(video)
    g = torch.Generator().manual_seed(data_seed + 1)
    w_out = (torch.randn(out.shape, generator=g) / out[0].numel() ** 0.5).to(dev)
    (out * w_out).sum().backward()
    assert bias_grad_branches(model) == branches, f"{tag}: bias-table gradient took {bias_grad_branches(model)}"
    ours = (out.detach(), None, {n: p.grad for n, p in model.named_parameters() if p.grad is not None})
    sd = {k: v.to(dev) for k, v in sd.items()}
    runs = [swin_oracle(sd, video, w_out, cfg, masks, mode) for mode in ("fp32", "bf16", "autocast")]
    check_case(tag, ours, *runs)
    return ours, runs[0]


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
               masks=gold["masks"] if rate else None)


@pytest.mark.parametrize("name", list(SWIN_CASES))
def test_swin3d_calibrated(dev, name):
    cfg, B, D, H, W, ws, ds, branches = SWIN_CASES[name]
    swin3d_case(dev, f"swin {name}", SO.Swin3DCfg(**cfg), B, D, H, W, ws, ds, branches)
