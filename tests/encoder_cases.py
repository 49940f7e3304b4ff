"""The divided TimeSformer and the Swin-3D encoder under the calibrated rule (contract_harness.calibrated_model_rows):
the oracle runs that stand on either side of it and one case of each model, shared by test_gpu_encoder_calibration.py,
test_gpu_timesformer.py, test_gpu_swin3d.py and the CPU negative controls of test_encoder_calibration_cpu.py.

  fp32      the oracle, the truth (no TF32)
  bf16      the arm: the oracle with bf16 weights, input and activations (both modules keep their token stream in bf16);
            its attention backward forms delta from the stored bf16 output, as the kernels do (KernelRoundedSoftmaxAV)
  autocast  the oracle under bf16 autocast: its ratio is printed, never asserted
"""
import contextlib

import torch

from contract_harness import calibrated_model_rows, no_tf32
from oracle import swin3d_oracle as SO
from oracle import timesformer_oracle as TO

bf16, f32 = torch.bfloat16, torch.float32


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


def check_case(tag, ours, want, arm, ac, report=None):
    """The rule on one case; its worst whole-tensor and slice ratios go into `report` under `tag`."""
    rows, slices = model_rows(ours, want, arm, ac)
    bad, worst, worst_sl = calibrated_model_rows(tag, rows, slices)
    if report is not None:
        report.record(tag, (worst, worst_sl))
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
            no_tf32():
        out = TO.timesformer_forward(sdo, xo, cfg, drop_masks=_cast_masks(masks, dt) if mode == "bf16" else masks)
        out = out.float()
        (out * w_out).sum().backward()
    return out.detach(), xo.grad, {n: p.grad for n, p in sdo.items() if p.grad is not None}


def timesformer_case(dev, tag, cfg, B, T, H, W, weight_seed, data_seed, rate=None, masks=None, report=None):
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
    check_case(tag, ours, *runs, report=report)
    return ours, runs[0]


# ========================================================================================================= Swin-3D
def swin_oracle(sd, video, w_out, cfg, masks, mode):
    """As tsf_oracle; the index buffers stay int64.  -> (out, None, grads)."""
    dt = bf16 if mode == "bf16" else f32
    sdo = {k: (v.detach().to(dt).requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    with torch.autocast(device_type=video.device.type, dtype=bf16, enabled=mode == "autocast"), _arm_core(SO, mode), \
            no_tf32():
        out = SO.swin3d_forward(sdo, video.to(dt), cfg, drop_masks=_cast_masks(masks, dt) if mode == "bf16" else masks)
        out = out.float()
        (out * w_out).sum().backward()
    return out.detach(), None, {n: p.grad for n, p in sdo.items() if p.is_floating_point() and p.grad is not None}


def bias_grad_branches(model):
    """How the module sums each layer's bias-table gradient (modeling/swin3d.py, _block_bwd): 'colsum' (the column-sum
    kernel, heads * L^2 % 8 == 0) or 'torch' (its fallback for odd windows), over the geometries the last forward built."""
    return {"colsum" if model.num_heads[k[1]] * geo["L"] ** 2 % 8 == 0 else "torch"
            for k, geo in model._tables.items() if k[0] == "layer"}


def swin3d_case(dev, tag, cfg, B, D, H, W, weight_seed, data_seed, branches, rate=None, masks=None, report=None):
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
    check_case(tag, ours, *runs, report=report)
    return ours, runs[0]
