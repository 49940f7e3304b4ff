"""CPU oracle for BASELINE.json config #4: HD-VILA's TimeSformer (divided space-time attention).

TEST INFRASTRUCTURE ONLY — imported by tests/, tests/golden/make_golden_timesformer.py and tools/ (baseline timing);
the product package never imports it.

A functional fp32 PyTorch restatement of the reference's `hd-vila/src/modeling/timesformer.py` (eval mode / DropPath
inactive: SURVEY.md §8c).  Parity pinned: tests/golden/make_golden_timesformer.py loads these seeded weights into the
reference's own `TimeSformer`, asserts agreement to fp32 round-off (forward and every parameter gradient) and writes
tests/golden/timesformer_*.pt.

Reference lines followed:
  TimeSformer.forward   timesformer.py:481-525  (+pos, bilinear-interpolated if the grid differs :487-494; +time,
                        linearly interpolated if T differs :504-508; token order (h w t); self.norm never applied)
  Block.forward         timesformer.py:201-226  (temporal attn -> temporal_fc -> residual; spatial attn -> residual; MLP)
  Attention.forward     timesformer.py:156-173  (fused qkv Linear, softmax(q k^T * head_dim**-0.5) v, proj)
  Mlp.forward           timesformer.py:132-138  (fc1, exact-erf GELU, fc2)
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict

import torch
import torch.nn.functional as F


@dataclass
class TimeSformerCfg:
    depth: int = 4            # e2e_model.py:53 (config.timesformer_depth), pretrain_stage1.json
    num_frames: int = 7       # e2e_model.py:53
    H: int = 10
    W: int = 16
    embed_dim: int = 1024
    num_heads: int = 16
    mlp_ratio: float = 4.0
    eps: float = 1e-6         # timesformer.py:424 norm_layer=partial(nn.LayerNorm, eps=1e-6)

    @property
    def hidden(self) -> int:
        return int(self.embed_dim * self.mlp_ratio)


def param_shapes(cfg: TimeSformerCfg) -> Dict[str, tuple]:
    """state_dict names/shapes of the reference module (timesformer.py:421-455)."""
    C, I = cfg.embed_dim, cfg.hidden
    shapes = {"pos_embed": (1, cfg.H * cfg.W, C), "time_embed": (1, cfg.num_frames, C)}
    for i in range(cfg.depth):
        p = f"blocks.{i}."
        for n in ("norm1", "temporal_norm1", "norm2"):
            shapes[p + n + ".weight"] = (C,)
            shapes[p + n + ".bias"] = (C,)
        for a in ("attn", "temporal_attn"):
            shapes[p + a + ".qkv.weight"] = (3 * C, C)
            shapes[p + a + ".qkv.bias"] = (3 * C,)
            shapes[p + a + ".proj.weight"] = (C, C)
            shapes[p + a + ".proj.bias"] = (C,)
        shapes[p + "temporal_fc.weight"] = (C, C)
        shapes[p + "temporal_fc.bias"] = (C,)
        shapes[p + "mlp.fc1.weight"] = (I, C)
        shapes[p + "mlp.fc1.bias"] = (I,)
        shapes[p + "mlp.fc2.weight"] = (C, I)
        shapes[p + "mlp.fc2.bias"] = (C,)
    shapes["norm.weight"] = (C,)   # constructed (timesformer.py:451) but never applied in forward
    shapes["norm.bias"] = (C,)
    return shapes


def init_state_dict(cfg: TimeSformerCfg, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic synthetic weights.  Statistics follow the reference init (weights ~ N(0, 0.02), timesformer.py:466-473)
    except that biases, LayerNorm affine parameters, time_embed and every temporal_fc are made non-trivial (the reference
    zero-initialises them, which would hide those terms from a parity test)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for n, shp in param_shapes(cfg).items():
        if n.endswith("norm1.weight") or n.endswith("norm2.weight") or n == "norm.weight":
            sd[n] = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif n.endswith(".bias"):
            sd[n] = 0.02 * torch.randn(shp, generator=g)
        else:
            sd[n] = 0.02 * torch.randn(shp, generator=g)
    return sd


def synthetic_input(B: int, T: int, H: int, W: int, cfg: TimeSformerCfg, seed: int = 1234) -> torch.Tensor:
    """[B, T, C, H, W] feature maps (the ResNet stage-3 output of e2e_model.py:124-135 is out of scope: N(0,1))."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, T, cfg.embed_dim, H, W, generator=g)


def interpolated_tables(sd, cfg: TimeSformerCfg, T: int, H: int, W: int):
    """pos [H*W, C] and time [T, C] tables as the forward adds them (timesformer.py:487-494, 504-508)."""
    C = cfg.embed_dim
    pos = sd["pos_embed"]
    if H != cfg.H or W != cfg.W:
        grid = pos[0].unsqueeze(0).transpose(1, 2).reshape(1, C, cfg.H, cfg.W)
        pos = F.interpolate(grid, size=(H, W), mode="bilinear").flatten(2).transpose(1, 2)
    time = sd["time_embed"]
    if T != time.shape[1]:
        time = F.interpolate(time.transpose(1, 2), size=T, mode="linear").transpose(1, 2)
    return pos[0], time[0]


def softmax_av(logits, v):
    """softmax(logits) @ v: the attention core, kept in one function so that a calibration arm can give it the backward
    of the attention kernels (tests/encoder_cases.py)."""
    return logits.softmax(dim=-1) @ v


def attention(x, w_qkv, b_qkv, w_proj, b_proj, heads: int):
    """timesformer.py:156-173.  x: [G, N, C] (G independent groups)."""
    G, N, C = x.shape
    qkv = F.linear(x, w_qkv, b_qkv).reshape(G, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    attn = (q @ k.transpose(-2, -1)) * (C // heads) ** -0.5
    out = softmax_av(attn, v).transpose(1, 2).reshape(G, N, C)
    return F.linear(out, w_proj, b_proj)


def draw_drop_masks(cfg: TimeSformerCfg, B: int, T: int, H: int, W: int, drop_path_rate: float, device=None,
                    dtype=torch.float32):
    """Training-mode DropPath factors (timesformer.py:98-113) for every block, drawn from torch's global generator in the
    reference's own order and shapes — block i with rate linspace(0, drop_path_rate, depth)[i] (:445) calls drop_path on
    the temporal residual [(b h w), t, m] (:212), the spatial one [(b t), (h w), m] (:218) and the MLP one [b, n, m] (:225):
    factor = floor(keep + U[0,1)) / keep per leading index.  Seeding torch identically therefore reproduces the reference's
    masks exactly.  Returns a list of (m_t [B*H*W], m_s [B*T], m_m [B]) or None for blocks with rate 0."""
    rates = [r.item() for r in torch.linspace(0, drop_path_rate, cfg.depth)]
    out = []
    for r in rates:
        if r == 0.0:
            out.append(None)
            continue
        keep = 1 - r
        ms = []
        for n in (B * H * W, B * T, B):
            rnd = keep + torch.rand((n, 1, 1), dtype=dtype, device=device)
            ms.append((rnd.floor_() / keep).reshape(n))
        out.append(tuple(ms))
    return out


def block_forward(sd, i: int, x, B: int, T: int, H: int, W: int, cfg: TimeSformerCfg, drop=None):
    """timesformer.py:207-226 (divided_space_time).  x: [B, H*W*T, C], token order (h w t).  `drop` = (m_t, m_s, m_m)
    DropPath factors of this block (see draw_drop_masks) or None (eval mode / rate 0)."""
    p = f"blocks.{i}."
    C, HW = cfg.embed_dim, H * W
    ln = lambda t, n: F.layer_norm(t, (C,), sd[p + n + ".weight"], sd[p + n + ".bias"], cfg.eps)  # noqa: E731
    # temporal: groups (b h w), T tokens each
    xt = x.reshape(B * HW, T, C)
    rt = attention(ln(xt, "temporal_norm1"), sd[p + "temporal_attn.qkv.weight"], sd[p + "temporal_attn.qkv.bias"],
                   sd[p + "temporal_attn.proj.weight"], sd[p + "temporal_attn.proj.bias"], cfg.num_heads)
    if drop is not None:
        rt = rt * drop[0][:, None, None]
    rt = F.linear(rt.reshape(B, HW * T, C), sd[p + "temporal_fc.weight"], sd[p + "temporal_fc.bias"])
    xt = x + rt
    # spatial: groups (b t), H*W tokens each
    xs = xt.reshape(B, HW, T, C).permute(0, 2, 1, 3).reshape(B * T, HW, C)
    rs = attention(ln(xs, "norm1"), sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"], sd[p + "attn.proj.weight"],
                   sd[p + "attn.proj.bias"], cfg.num_heads)
    if drop is not None:
        rs = rs * drop[1][:, None, None]
    rs = rs.reshape(B, T, HW, C).permute(0, 2, 1, 3).reshape(B, HW * T, C)
    x = xt + rs
    # MLP
    h = F.linear(ln(x, "norm2"), sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])
    h = F.gelu(h)
    h = F.linear(h, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    if drop is not None:
        h = h * drop[2][:, None, None]
    return x + h


def embed(sd, x, cfg: TimeSformerCfg):
    """timesformer.py:481-509: [B,T,C,H,W] -> tokens [B, H*W*T, C] in (h w t) order with pos/time tables added."""
    B, T, C, H, W = x.shape
    pos, time = interpolated_tables(sd, cfg, T, H, W)
    tok = x.flatten(3).permute(0, 3, 1, 2)              # [B, HW, T, C]
    tok = tok + pos[None, :, None, :] + time[None, None, :, :]
    return tok.reshape(B, H * W * T, C)


def timesformer_forward(sd, x, cfg: TimeSformerCfg, return_hidden: bool = False, drop_masks=None):
    """timesformer.py:481-525.  Returns [B, T, C, H, W] (the reference's permuted view).  drop_masks: per-block DropPath
    factors from draw_drop_masks (training mode) or None (eval)."""
    B, T, C, H, W = x.shape
    tok = embed(sd, x, cfg)
    hidden = [tok]
    for i in range(cfg.depth):
        tok = block_forward(sd, i, tok, B, T, H, W, cfg, None if drop_masks is None else drop_masks[i])
        hidden.append(tok)
    out = tok.reshape(B, H, W, T, C).permute(0, 3, 4, 1, 2)
    return (out, hidden) if return_hidden else out


def flops_per_sample(cfg: TimeSformerCfg, T: int, H: int, W: int) -> float:
    """Forward FLOPs (2 per MAC) of one sample: per block 2 qkv + 3 C x C linears + MLP + the two attentions."""
    C, I, n = cfg.embed_dim, cfg.hidden, H * W * T
    lin = 2 * n * C * (2 * 3 * C + 3 * C + 2 * I)
    att = 4 * C * n * (T + H * W)                       # QK^T and PV: 2*2*hd*heads = 4C per query-key pair
    return float(cfg.depth * (lin + att))
