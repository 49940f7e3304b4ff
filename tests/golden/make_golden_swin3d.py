"""Golden vectors for BASELINE.json config #5 (LF-VILA Swin-3D video encoder) from the REAL reference.

Needs a checkout of the reference, named by XP_REFERENCE_ROOT:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_swin3d.py

Imports LF-VILA/src/models/video_encoder.py unmodified behind stub `timm.models.layers` (DropPath, trunc_normal_) and
`mmcv.runner` (load_checkpoint) modules — neither touches the model math — loads the oracle's deterministic weights into the
reference `SwinTransformer3D`, runs forward + backward in fp32 on CPU (eval mode, and one training-mode case with seeded
DropPath), asserts oracle/swin3d_oracle.py agrees to fp32 round-off, and stores small numeric fixtures.
"""
import os
import sys
import types

import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ["XP_REFERENCE_ROOT"]     # a checkout of microsoft/XPretrain
sys.dont_write_bytecode = True

from oracle import swin3d_oracle as O  # noqa: E402


def load_reference():
    class DropPath(nn.Module):                     # timm.models.layers.DropPath (the same algorithm as timesformer.py:98-121)
        def __init__(self, drop_prob=None):
            super().__init__()
            self.drop_prob = drop_prob

        def forward(self, x):
            if self.drop_prob == 0. or not self.training:
                return x
            keep = 1 - self.drop_prob
            shape = (x.shape[0],) + (1,) * (x.ndim - 1)
            rnd = keep + torch.rand(shape, dtype=x.dtype, device=x.device)
            rnd.floor_()
            return x.div(keep) * rnd

    timm, models, layers = types.ModuleType("timm"), types.ModuleType("timm.models"), types.ModuleType("timm.models.layers")
    layers.DropPath, layers.trunc_normal_ = DropPath, nn.init.trunc_normal_
    mmcv, runner = types.ModuleType("mmcv"), types.ModuleType("mmcv.runner")
    runner.load_checkpoint = lambda *a, **k: None
    import importlib.machinery
    for m in (timm, models, layers, mmcv, runner):          # other packages probe sys.modules via importlib.util.find_spec
        m.__spec__ = importlib.machinery.ModuleSpec(m.__name__, None)
    sys.modules.update({"timm": timm, "timm.models": models, "timm.models.layers": layers, "mmcv": mmcv, "mmcv.runner": runner})
    # load the one file by path: `src.models.__init__` pulls in the BERT tower, which needs an old transformers release
    import importlib.util
    src, utils, dist = types.ModuleType("src"), types.ModuleType("src.utils"), types.ModuleType("src.utils.dist")
    dist.master_process = lambda *a, **k: True               # logging helper only (video_encoder.py:13)
    sys.modules.update({"src": src, "src.utils": utils, "src.utils.dist": dist})
    spec = importlib.util.spec_from_file_location("ref_video_encoder", os.path.join(REF, "LF-VILA/src/models/video_encoder.py"))
    ve = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ve)
    return ve


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def run_case(ve, name, cfg, B, D, H, W, weight_seed, data_seed, train_rate=None, torch_seed=0):
    sd = O.init_state_dict(cfg, seed=weight_seed)
    model = ve.SwinTransformer3D(pretrained=None, patch_size=list(cfg.patch_size), embed_dim=cfg.embed_dim,
                                 depths=list(cfg.depths), num_heads=list(cfg.num_heads), stages=list(cfg.stages),
                                 downsample_stages=list(cfg.downsample_stages),
                                 window_size=[list(w) for w in cfg.window_size], patch_norm=cfg.patch_norm,
                                 local_window=cfg.local_window, drop_path_rate=train_rate if train_rate else 0.2)
    missing, unexpected = model.load_state_dict(sd, strict=True)
    if train_rate:
        model.train()
    else:
        model.eval()                       # (the reference's train() override returns None: keep it on its own line)
    video = O.synthetic_video(B, D, H, W, cfg, seed=data_seed)
    if train_rate:
        torch.manual_seed(torch_seed)
    out, out2 = model(video)
    assert out2 is out                     # the (x, x) quirk of :600,:611-613
    g = torch.Generator().manual_seed(data_seed + 1)
    w_out = torch.randn(out.shape, generator=g) / out[0].numel() ** 0.5
    loss = (out * w_out).sum()
    loss.backward()
    ref_grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    no_grad = sorted(n for n, p in model.named_parameters() if p.grad is None)
    assert all(n.startswith(("norm_local", "local_feat_proj")) for n in no_grad), no_grad

    masks = None
    if train_rate:
        torch.manual_seed(torch_seed)
        masks = O.draw_drop_masks(cfg, B, train_rate)
        assert sum(int((m == 0).sum()) for blk in masks if blk is not None for m in blk) > 0
    sdo = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    out_o, stages = O.swin3d_forward(sdo, video, cfg, drop_masks=masks, return_stages=True)
    (out_o * w_out).sum().backward()
    worst = 0.0
    scale0 = float(ref_grads["layers.0.blocks.0.mlp.fc1.weight"].norm())
    for n, gr in ref_grads.items():
        worst = max(worst, float((sdo[n].grad - gr).norm()) / max(float(gr.norm()), 1e-3 * scale0))
    print(f"{name}: out {tuple(out.shape)} rel {rel(out_o, out):.2e}  worst param grad {worst:.2e}")
    assert rel(out_o, out) < 2e-6 and worst < 5e-5
    keep = ["patch_embed.proj.weight", "patch_embed.norm.weight", "layers.0.blocks.0.attn.relative_position_bias_table",
            "layers.0.blocks.1.attn.relative_position_bias_table", "layers.0.blocks.1.attn.qkv.weight",
            "layers.0.blocks.1.attn.qkv.bias", "layers.0.blocks.0.attn.proj.weight", "layers.0.blocks.0.mlp.fc1.weight",
            "layers.0.downsample.reduction.weight", "layers.0.downsample.norm.weight", "norm.weight",
            f"layers.{len(cfg.depths) - 1}.blocks.1.attn.relative_position_bias_table",
            f"layers.{len(cfg.depths) - 1}.blocks.0.mlp.fc2.weight", f"layers.{len(cfg.depths) - 1}.blocks.1.norm1.bias"]
    torch.save({"cfg": vars(cfg), "B": B, "D": D, "H": H, "W": W, "weight_seed": weight_seed, "data_seed": data_seed,
                "train_rate": train_rate, "torch_seed": torch_seed, "masks": masks, "out": out.detach().clone(),
                "loss": loss.detach(), "stage_rows": [s.flatten(0, 3)[:4].detach().clone() for s in stages],
                # first 8 rows of the weight matrices; bias tables (small, and only sparsely touched by clamped windows) and vectors whole
                "grads": {n: (ref_grads[n][:8].clone() if ref_grads[n].dim() >= 2 and "bias_table" not in n
                              else ref_grads[n].clone()) for n in keep},
                "grad_norms": {n: float(ref_grads[n].norm()) for n in keep}},
               os.path.join(HERE, f"{name}.pt"))


def main():
    ve = load_reference()
    small = dict(embed_dim=64, depths=(2, 2, 2), num_heads=(2, 4, 8), stages=(0, 1, 2), downsample_stages=(0, 1),
                 window_size=((2, 3, 5), (4, 3, 5), (8, 3, 5)))
    # 8 x 6 x 10 tokens: shifted windows with a mask in layer 0, clamped windows later, odd-size patch merging (3 x 5 -> 2 x 3),
    # relative_position_index[:N, :N] slicing in the last layer
    run_case(ve, "swin3d_small_b2", O.Swin3DCfg(**small), B=2, D=8, H=48, W=80, weight_seed=0, data_seed=31)
    # 4 x 7 x 7 tokens: every layer zero-pads its windows (the padded tokens' k, v are the qkv bias)
    run_case(ve, "swin3d_padded_b1", O.Swin3DCfg(**small), B=1, D=4, H=56, W=56, weight_seed=1, data_seed=32)
    # training mode with stochastic depth
    run_case(ve, "swin3d_train_droppath", O.Swin3DCfg(**small), B=4, D=4, H=24, W=40, weight_seed=2, data_seed=33,
             train_rate=0.5, torch_seed=91)


if __name__ == "__main__":
    main()
