"""Golden vectors for HD-VILA's TimeSformer with attention_type 'joint_space_time' and 'space_only', from the REAL reference.

Needs a checkout of the reference, named by XP_REFERENCE_ROOT:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_timesformer_variants.py

Loads hd-vila/src/modeling/timesformer.py unmodified (through make_golden_timesformer.py's `torch._six` shim), builds its
`TimeSformer` with each attention type, copies oracle/timesformer_variants_oracle.py's deterministic weights into it
(strict: the parameter trees must match), runs forward + backward in fp32 on the CPU, asserts that the oracle agrees —
to the bit in eval mode, to fp32 round-off in train mode with DropPath — and stores small numeric fixtures (no reference
source) for tests/test_timesformer_variants_cpu.py and tests/test_gpu_timesformer_variants.py.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.dont_write_bytecode = True

from make_golden_timesformer import load_reference, rel  # noqa: E402
from oracle import timesformer_oracle as TO  # noqa: E402
from oracle import timesformer_variants_oracle as V  # noqa: E402


def run_case(ref, name, kind, cfg, B, T, H, W, weight_seed, data_seed, train_rate=None, torch_seed=None):
    sd = V.init_state_dict(cfg, kind, seed=weight_seed)
    model = ref.TimeSformer(depth=cfg.depth, num_frames=cfg.num_frames, H=cfg.H, W=cfg.W, embed_dim=cfg.embed_dim,
                            num_heads=cfg.num_heads, drop_path_rate=0.1 if train_rate is None else train_rate,
                            attention_type=kind)
    ref_keys = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert ref_keys == V.param_shapes(cfg, kind), "oracle parameter tree differs from the reference's"
    model.load_state_dict(sd, strict=True)
    model.train() if train_rate is not None else model.eval()
    x = TO.synthetic_input(B, T, H, W, cfg, seed=data_seed).requires_grad_(True)
    g = torch.Generator().manual_seed(data_seed + 1)
    w_out = torch.randn(B, T, cfg.embed_dim, H, W, generator=g) / (B * T * H * W) ** 0.5
    if torch_seed is not None:
        torch.manual_seed(torch_seed)
    out = model(x)
    loss = (out * w_out).sum()
    loss.backward()
    ref_grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    assert "norm.weight" not in ref_grads          # self.norm is constructed but never applied

    masks = None
    if train_rate is not None:
        torch.manual_seed(torch_seed)
        masks = V.draw_drop_masks(cfg, kind, B, T, train_rate)
        dropped = sum(int((m == 0).sum()) for blk in masks if blk is not None for m in blk)
        assert masks[0] is None and dropped > 0, "the case must actually drop some paths"
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xo = x.detach().clone().requires_grad_(True)
    out_o = V.timesformer_forward(sdo, xo, cfg, kind, drop_masks=masks)
    (out_o * w_out).sum().backward()
    worst = max(float((sdo[n].grad - gr).norm()) / max(float(gr.norm()), 1e-3 * float(ref_grads["blocks.0.mlp.fc1.weight"].norm()))
                for n, gr in ref_grads.items())
    e_out, e_dx = rel(out_o, out), rel(xo.grad, x.grad)
    exact = torch.equal(out_o, out)
    print(f"{name}: out {'bit-exact' if exact else f'{e_out:.2e}'} dx {e_dx:.2e} worst param grad {worst:.2e}")
    if train_rate is None:
        assert exact, "eval-mode forward must match the reference bit for bit"
    assert e_out < 2e-6 and e_dx < 2e-5 and worst < 5e-5

    keep = [n for n in ("pos_embed", "time_embed", "blocks.0.attn.qkv.weight", "blocks.0.attn.qkv.bias",
                        "blocks.0.attn.proj.weight", "blocks.0.norm1.weight", "blocks.0.norm2.bias",
                        "blocks.0.mlp.fc1.weight", f"blocks.{cfg.depth - 1}.attn.qkv.weight",
                        f"blocks.{cfg.depth - 1}.mlp.fc2.bias") if n in ref_grads]
    gold = {
        "cfg": vars(cfg), "attention_type": kind, "B": B, "T": T, "H": H, "W": W, "weight_seed": weight_seed,
        "data_seed": data_seed, "rate": train_rate, "torch_seed": torch_seed, "masks": masks,
        "state_dict_shapes": ref_keys,
        "out": out.detach().clone(), "loss": loss.detach(), "dx_t0": x.grad[:, 0].detach().clone(),
        "dx_norm": float(x.grad.norm()),
        # first 8 rows of each kept gradient (weights are [out, in]; 1-D parameters are kept whole)
        "grads": {n: (ref_grads[n][:8].clone() if ref_grads[n].dim() == 2 else ref_grads[n].clone()) for n in keep},
        "grad_norms": {n: float(g_.norm()) for n, g_ in ref_grads.items()},
    }
    path = os.path.join(HERE, f"{name}.pt")
    torch.save(gold, path)
    size = os.path.getsize(path)
    assert size < 1 << 20, f"{name}.pt is {size} bytes"


def main():
    ref = load_reference()
    # joint over 8 x 7 x 7 = 392 tokens per clip (ragged against 64-row tiles), both table interpolations:
    # grid 4 x 6 -> 7 x 7, frames 4 -> 8
    run_case(ref, "timesformer_joint_interp_b2", "joint_space_time",
             TO.TimeSformerCfg(depth=2, num_frames=4, H=4, W=6, embed_dim=128, num_heads=2),
             B=2, T=8, H=7, W=7, weight_seed=20, data_seed=21)
    # joint at the reference's native grid, 7 x 10 x 16 = 1120 tokens per clip, training mode with DropPath
    # (rates 0, 0.25, 0.5; one clip, so a drop removes a whole branch)
    run_case(ref, "timesformer_joint_native_train", "joint_space_time",
             TO.TimeSformerCfg(depth=3, num_frames=7, H=10, W=16, embed_dim=128, num_heads=2),
             B=1, T=7, H=10, W=16, weight_seed=22, data_seed=23, train_rate=0.5, torch_seed=7)
    # space_only at T = 1 (the only frame count its output path runs at): 7 x 10 = 70 tokens per frame
    run_case(ref, "timesformer_space_only_t1", "space_only",
             TO.TimeSformerCfg(depth=2, num_frames=7, H=7, W=10, embed_dim=128, num_heads=2),
             B=3, T=1, H=7, W=10, weight_seed=24, data_seed=25)


if __name__ == "__main__":
    main()
