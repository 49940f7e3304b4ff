"""CPU oracle for the other two attention types of HD-VILA's TimeSformer: 'joint_space_time' and 'space_only'.

TEST INFRASTRUCTURE ONLY — imported by tests/, tests/golden/make_golden_timesformer_variants.py and tools/; the product
package never imports it.  It builds on oracle/timesformer_oracle.py (the divided model, unchanged): same config, same
seeded synthetic weights and inputs, same attention / table helpers.  Parity pinned:
tests/golden/make_golden_timesformer_variants.py loads these weights into the reference's own `TimeSformer` built with
the matching `attention_type` and asserts agreement (eval mode to the bit, train mode to fp32 round-off).

Reference lines followed (hd-vila/src/modeling/timesformer.py):
  Block.__init__        :181-199   no temporal_norm1 / temporal_attn / temporal_fc unless divided (:187-191)
  Block.forward         :202-205   x + drop_path(attn(norm1(x))); x + drop_path(mlp(norm2(x)))
  TimeSformer.__init__  :438-466   no time_embed for space_only (:440); temporal_fc zero-init only when divided (:458-466)
  TimeSformer.forward   :481-525   joint: blocks on 'b (h w t) m' (dense attention over every token of a clip);
                                   space_only: no time table (:501), blocks on '(b t) (h w) m', frame mean and
                                   reshape(B, T, H, W, C) (:519-522), which only runs at T = 1
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle import timesformer_oracle as TO

TYPES = ("joint_space_time", "space_only")


def param_shapes(cfg: TO.TimeSformerCfg, attention_type: str) -> Dict[str, tuple]:
    """state_dict names / shapes of the reference module built with `attention_type`."""
    assert attention_type in TYPES
    shapes = {}
    for n, shp in TO.param_shapes(cfg).items():
        if ".temporal_" in n or (n == "time_embed" and attention_type == "space_only"):
            continue
        shapes[n] = shp
    return shapes


def init_state_dict(cfg: TO.TimeSformerCfg, attention_type: str, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic synthetic weights with the statistics of TO.init_state_dict (non-trivial biases, LayerNorm affine
    parameters and time table), drawn in this type's parameter order."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for n, shp in param_shapes(cfg, attention_type).items():
        if n.endswith("norm1.weight") or n.endswith("norm2.weight") or n == "norm.weight":
            sd[n] = 1.0 + 0.1 * torch.randn(shp, generator=g)
        else:
            sd[n] = 0.02 * torch.randn(shp, generator=g)
    return sd


def draw_drop_masks(cfg: TO.TimeSformerCfg, attention_type: str, B: int, T: int, drop_path_rate: float, device=None,
                    dtype=torch.float32):
    """Training-mode DropPath factors (timesformer.py:98-113) from torch's global generator in the reference's order: block
    i (rate linspace(0, drop_path_rate, depth)[i], :445) calls drop_path twice (:203-204), each time on the blocks' batch
    of B clips (joint) or B*T frames (space_only).  Returns a list of (m_attn, m_mlp) or None for blocks with rate 0."""
    n = B if attention_type == "joint_space_time" else B * T
    out = []
    for r in [v.item() for v in torch.linspace(0, drop_path_rate, cfg.depth)]:
        if r == 0.0:
            out.append(None)
            continue
        keep = 1 - r
        out.append(tuple(((keep + torch.rand((n, 1, 1), dtype=dtype, device=device)).floor_() / keep).reshape(n)
                         for _ in range(2)))
    return out


def block_forward(sd, i: int, x, cfg: TO.TimeSformerCfg, drop=None):
    """timesformer.py:202-205.  x: [G, N, C], attention over all N tokens of each of the G sequences.  drop: (m_attn,
    m_mlp) factors per sequence or None (eval mode / rate 0)."""
    p = f"blocks.{i}."
    C = cfg.embed_dim
    ln = lambda t, n: F.layer_norm(t, (C,), sd[p + n + ".weight"], sd[p + n + ".bias"], cfg.eps)  # noqa: E731
    r = TO.attention(ln(x, "norm1"), sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"], sd[p + "attn.proj.weight"],
                     sd[p + "attn.proj.bias"], cfg.num_heads)
    if drop is not None:
        r = r * drop[0][:, None, None]
    x = x + r
    h = F.linear(ln(x, "norm2"), sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])
    h = F.linear(F.gelu(h), sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    if drop is not None:
        h = h * drop[1][:, None, None]
    return x + h


def embed(sd, x, cfg: TO.TimeSformerCfg):
    """timesformer.py:481-509: tokens [B, H*W*T, C] in (h w t) order, + pos, + time unless space_only (no time_embed)."""
    B, T, C, H, W = x.shape
    pos = sd["pos_embed"]
    if H != cfg.H or W != cfg.W:
        grid = pos[0].unsqueeze(0).transpose(1, 2).reshape(1, C, cfg.H, cfg.W)
        pos = F.interpolate(grid, size=(H, W), mode="bilinear").flatten(2).transpose(1, 2)
    tok = x.flatten(3).permute(0, 3, 1, 2) + pos[0][None, :, None, :]       # [B, HW, T, C]
    if "time_embed" in sd:
        time = sd["time_embed"]
        if T != time.shape[1]:
            time = F.interpolate(time.transpose(1, 2), size=T, mode="linear").transpose(1, 2)
        tok = tok + time[0][None, None, :, :]
    return tok.reshape(B, H * W * T, C)


def timesformer_forward(sd, x, cfg: TO.TimeSformerCfg, attention_type: str, return_hidden: bool = False,
                        drop_masks=None):
    """timesformer.py:481-525 for 'joint_space_time' / 'space_only'.  Returns [B, T, C, H, W]."""
    assert attention_type in TYPES
    B, T, C, H, W = x.shape
    if attention_type == "space_only" and T != 1:
        # :519-522: the frame mean is followed by reshape(B, T, H, W, C), which fails for T > 1
        raise RuntimeError("space_only: the reference's output reshape fails for T > 1 (timesformer.py:521)")
    tok = embed(sd, x, cfg)       # space_only at T = 1: the '(b t) (h w)' frames are the '(h w t)' rows of each sample
    hidden = [tok]
    for i in range(cfg.depth):
        tok = block_forward(sd, i, tok, cfg, None if drop_masks is None else drop_masks[i])
        hidden.append(tok)
    if attention_type == "space_only":
        tok = tok.reshape(B, T, H * W, C).mean(1)                            # :520
    out = tok.reshape(B, H, W, T, C).permute(0, 3, 4, 1, 2)
    return (out, hidden) if return_hidden else out


def autocast_forward(sd, x, cfg: TO.TimeSformerCfg, attention_type: str, drop_masks=None):
    """The same forward under bf16 autocast on x's device: the calibration arm of DESIGN.md §2."""
    with torch.autocast(device_type=x.device.type, dtype=torch.bfloat16):
        return timesformer_forward(sd, x, cfg, attention_type, drop_masks=drop_masks).float()


def flops_per_sample(cfg: TO.TimeSformerCfg, T: int, H: int, W: int, attention_type: str) -> float:
    """Forward FLOPs (2 per MAC) of one sample: qkv + proj + MLP per block, and the dense attention (4C per query-key
    pair) over n = H*W*T tokens (joint) or over each frame's H*W tokens (space_only)."""
    C, I, n = cfg.embed_dim, cfg.hidden, H * W * T
    lin = 2 * n * C * (3 * C + C + 2 * I)
    att = 4 * C * n * (n if attention_type == "joint_space_time" else H * W)
    return float(cfg.depth * (lin + att))
