"""Golden vectors for BASELINE.json config #4 (HD-VILA TimeSformer) from the REAL reference.

Needs a checkout of the reference, named by XP_REFERENCE_ROOT:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_timesformer.py

Loads hd-vila/src/modeling/timesformer.py unmodified (with a `torch._six` shim: the module was written for torch 1.8),
copies the oracle's deterministic weights into the reference `TimeSformer`, runs forward + backward in fp32 on CPU in
eval mode (DropPath inactive), asserts that oracle/timesformer_oracle.py agrees to fp32 round-off — this pins the oracle —
and stores small numeric fixtures (no reference source) for tests/test_oracle_golden.py and tests/test_gpu_timesformer.py.
"""
import collections.abc
import importlib.util
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ["XP_REFERENCE_ROOT"]     # a checkout of microsoft/XPretrain
sys.dont_write_bytecode = True

from oracle import timesformer_oracle as O  # noqa: E402


def load_reference():
    six = types.ModuleType("torch._six")
    six.container_abcs = collections.abc
    sys.modules["torch._six"] = six
    spec = importlib.util.spec_from_file_location("ref_timesformer",
                                                  os.path.join(REF, "hd-vila/src/modeling/timesformer.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def run_case(ref, name, cfg, B, T, H, W, weight_seed, data_seed):
    sd = O.init_state_dict(cfg, seed=weight_seed)
    model = ref.TimeSformer(depth=cfg.depth, num_frames=cfg.num_frames, H=cfg.H, W=cfg.W, embed_dim=cfg.embed_dim,
                            num_heads=cfg.num_heads, drop_path_rate=0.1)
    model.load_state_dict(sd, strict=True)
    model.eval()                                   # DropPath inactive (SURVEY.md §8c)
    x = O.synthetic_input(B, T, H, W, cfg, seed=data_seed).requires_grad_(True)
    g = torch.Generator().manual_seed(data_seed + 1)
    w_out = torch.randn(B, T, cfg.embed_dim, H, W, generator=g) / (B * T * H * W) ** 0.5
    out = model(x)
    loss = (out * w_out).sum()
    loss.backward()
    ref_grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}

    # ---- pin the oracle against the reference
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xo = x.detach().clone().requires_grad_(True)
    out_o, hidden = O.timesformer_forward(sdo, xo, cfg, return_hidden=True)
    loss_o = (out_o * w_out).sum()
    loss_o.backward()
    e_out, e_loss, e_dx = rel(out_o, out), abs(float(loss_o) - float(loss)) / abs(float(loss)), rel(xo.grad, x.grad)
    worst = 0.0
    for n, gr in ref_grads.items():
        scale = max(float(gr.norm()), 1e-3 * float(ref_grads["blocks.0.mlp.fc1.weight"].norm()))
        worst = max(worst, float((sdo[n].grad - gr).norm()) / scale)
    assert "norm.weight" not in ref_grads          # self.norm is constructed but never applied
    print(f"{name}: out {e_out:.2e} loss {e_loss:.2e} dx {e_dx:.2e} worst param grad {worst:.2e}")
    assert e_out < 2e-6 and e_loss < 2e-6 and e_dx < 2e-5 and worst < 5e-5

    keep = ("pos_embed", "time_embed", "blocks.0.temporal_fc.weight", "blocks.0.temporal_attn.qkv.weight",
            "blocks.0.temporal_attn.qkv.bias", "blocks.0.attn.qkv.weight", "blocks.0.attn.proj.bias",
            "blocks.0.temporal_norm1.weight", "blocks.0.norm1.bias", "blocks.0.norm2.weight",
            "blocks.0.mlp.fc1.weight", "blocks.0.mlp.fc1.bias", "blocks.0.mlp.fc2.weight",
            f"blocks.{cfg.depth - 1}.attn.qkv.weight", f"blocks.{cfg.depth - 1}.mlp.fc2.bias",
            f"blocks.{cfg.depth - 1}.temporal_fc.bias")
    gold = {
        "cfg": vars(cfg), "B": B, "T": T, "H": H, "W": W, "weight_seed": weight_seed, "data_seed": data_seed,
        "out": out.detach().clone(), "loss": loss.detach(), "dx_t0": x.grad[:, 0].detach().clone(),
        "dx_norm": float(x.grad.norm()),
        "hidden_rows": torch.stack([h[:, :6].detach() for h in hidden]),
        # first 8 rows of each kept gradient (weights are [out, in]; 1-D parameters are kept whole)
        "grads": {n: (ref_grads[n][:8].clone() if ref_grads[n].dim() == 2 else ref_grads[n].clone()) for n in keep},
        "grad_norms": {n: float(ref_grads[n].norm()) for n in keep},
    }
    torch.save(gold, os.path.join(HERE, f"{name}.pt"))


def run_train_case(ref, name, cfg, B, T, H, W, weight_seed, data_seed, rate, torch_seed):
    """Training mode: stochastic depth active (timesformer.py:98-121).  The oracle draws the DropPath factors from torch's
    global generator in the reference's order, so seeding both identically must give the same forward and gradients."""
    sd = O.init_state_dict(cfg, seed=weight_seed)
    model = ref.TimeSformer(depth=cfg.depth, num_frames=cfg.num_frames, H=cfg.H, W=cfg.W, embed_dim=cfg.embed_dim,
                            num_heads=cfg.num_heads, drop_path_rate=rate)
    model.load_state_dict(sd, strict=True)
    model.train()
    x = O.synthetic_input(B, T, H, W, cfg, seed=data_seed).requires_grad_(True)
    g = torch.Generator().manual_seed(data_seed + 1)
    w_out = torch.randn(B, T, cfg.embed_dim, H, W, generator=g) / (B * T * H * W) ** 0.5
    torch.manual_seed(torch_seed)
    out = model(x)
    loss = (out * w_out).sum()
    loss.backward()
    ref_grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}

    torch.manual_seed(torch_seed)
    masks = O.draw_drop_masks(cfg, B, T, H, W, rate)
    dropped = sum(int((m == 0).sum()) for blk in masks if blk is not None for m in blk)
    assert masks[0] is None and dropped > 0, "the case must actually drop some paths"
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xo = x.detach().clone().requires_grad_(True)
    out_o = O.timesformer_forward(sdo, xo, cfg, drop_masks=masks)
    (out_o * w_out).sum().backward()
    e_out, e_dx = rel(out_o, out), rel(xo.grad, x.grad)
    worst = max(float((sdo[n].grad - gr).norm()) / max(float(gr.norm()), 1e-3 * float(ref_grads["blocks.0.mlp.fc1.weight"].norm()))
                for n, gr in ref_grads.items())
    print(f"{name}: {dropped} dropped paths; out {e_out:.2e} dx {e_dx:.2e} worst param grad {worst:.2e}")
    assert e_out < 2e-6 and e_dx < 2e-5 and worst < 5e-5
    keep = ("blocks.1.temporal_fc.weight", "blocks.1.temporal_attn.proj.weight", "blocks.1.attn.proj.weight",
            "blocks.1.attn.proj.bias", "blocks.1.mlp.fc2.weight", "blocks.1.mlp.fc2.bias", "blocks.2.mlp.fc1.weight",
            "blocks.0.attn.qkv.weight", "time_embed")
    torch.save({"cfg": vars(cfg), "B": B, "T": T, "H": H, "W": W, "weight_seed": weight_seed, "data_seed": data_seed,
                "rate": rate, "torch_seed": torch_seed, "masks": masks, "out": out.detach().clone(), "loss": loss.detach(),
                "dx_t0": x.grad[:, 0].detach().clone(),
                "grads": {n: (ref_grads[n][:8].clone() if ref_grads[n].dim() == 2 else ref_grads[n].clone()) for n in keep},
                "grad_norms": {n: float(ref_grads[n].norm()) for n in keep}},
               os.path.join(HERE, f"{name}.pt"))


def main():
    ref = load_reference()
    # training mode with DropPath: 3 blocks (rates 0, 0.25, 0.5), B = 4 so that sample-level drops occur
    run_train_case(ref, "timesformer_train_droppath", O.TimeSformerCfg(depth=3, num_frames=4, H=3, W=4, embed_dim=128, num_heads=2),
                   B=4, T=4, H=3, W=4, weight_seed=2, data_seed=13, rate=0.5, torch_seed=77)
    # head_dim 64 (the kernels' head size); both interpolation paths: grid 4x6 -> 3x5, frames 4 -> 3
    run_case(ref, "timesformer_interp_b2", O.TimeSformerCfg(depth=2, num_frames=4, H=4, W=6, embed_dim=128, num_heads=2),
             B=2, T=3, H=3, W=5, weight_seed=0, data_seed=11)
    # native grid / frame count, more tokens than one 64-row attention block, ragged tails (HW = 70, T = 7)
    run_case(ref, "timesformer_native_b2", O.TimeSformerCfg(depth=2, num_frames=7, H=7, W=10, embed_dim=128, num_heads=2),
             B=2, T=7, H=7, W=10, weight_seed=1, data_seed=12)


if __name__ == "__main__":
    main()
