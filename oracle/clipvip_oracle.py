"""CPU oracle for the CLIP-ViP hot path — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A functional, plain-PyTorch restatement (fp32 or fp64, no autocast, no custom
kernels) of the reference algorithm for the path named in BASELINE.json:
video tower with video-proxy tokens + CLIP text tower + in-batch InfoNCE.
Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` legs may import this module; the product path under
`xpretrain_b200/` never does.

Parity pinned: `tests/golden/make_golden.py` (run against a checkout of the
reference named by XP_REFERENCE_ROOT) checks every function here against the
reference's own modules (CLIP-ViP/src/modeling/CLIP_ViP.py,
CLIP-ViP/src/optimization/loss.py) to fp32 round-off and writes the golden
vectors that `tests/test_oracle_golden.py` replays on any machine.

All parameters are read from a flat dict keyed exactly like the reference's
`CLIPModel.state_dict()` (SURVEY.md §8b), so the same checkpoint drives the
reference, this oracle and the CUDA path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


@dataclass
class TowerCfg:
    width: int
    heads: int
    layers: int
    mlp: int


@dataclass
class ClipVipCfg:
    """Hyper-parameters of openai/clip-vit-base-patch16 + the ViP additions
    (reference: VidCLIP.py:11-27, configs/pretrain/pretrain_vip_base_16.json:50-56)."""

    vision: TowerCfg = field(default_factory=lambda: TowerCfg(768, 12, 12, 3072))
    text: TowerCfg = field(default_factory=lambda: TowerCfg(512, 8, 12, 2048))
    image_size: int = 224
    patch: int = 16
    proj_dim: int = 512
    vocab: int = 49408
    max_text_pos: int = 77
    temporal_size: int = 12
    add_cls_num: int = 3
    ln_eps: float = 1e-5
    logit_scale_init: float = 4.60

    @property
    def grid(self) -> int:
        return self.image_size // self.patch

    @property
    def patches(self) -> int:
        return self.grid * self.grid


def quick_gelu(x: Tensor) -> Tensor:
    # transformers QuickGELUActivation, selected by hidden_act="quick_gelu" (CLIP_ViP.py:389)
    return x * torch.sigmoid(1.702 * x)


# The arithmetic points below (layer_norm, linear, residual_add, the attention cores and the embedding sums) are module-level
# functions looked up at call time, so that a test can swap in a variant that rounds where a reduced-precision
# implementation rounds (tests/clipvip_arm.py).  The defaults are the fp32 / fp64 reference arithmetic.
def layer_norm(x: Tensor, sd: Dict[str, Tensor], prefix: str, eps: float) -> Tensor:
    return F.layer_norm(x, (x.shape[-1],), sd[prefix + ".weight"], sd[prefix + ".bias"], eps)


def linear(x: Tensor, sd: Dict[str, Tensor], prefix: str) -> Tensor:
    return F.linear(x, sd[prefix + ".weight"], sd.get(prefix + ".bias"))


def residual_add(x: Tensor, h: Tensor) -> Tensor:
    """The residual stream plus a block branch (CLIP_ViP.py:452,458)."""
    return x + h


# --------------------------------------------------------------------------- vision
def temporal_table(sd: Dict[str, Tensor], T: int, pre: str) -> Tensor:
    """CLIP_ViP.py:170-176: [1,temporal_size,C] table, linearly interpolated along time when T differs."""
    table = sd[pre + "temporal_embedding"]
    if T != table.shape[1]:
        table = F.interpolate(table.transpose(1, 2), size=T, mode="linear").transpose(1, 2)
    return table


def vip_embeddings(sd: Dict[str, Tensor], video: Tensor, cfg: ClipVipCfg,
                   pre: str = "vision_model.embeddings.") -> Tuple[Tensor, Tuple[int, int, int]]:
    """CLIP_ViP.py:168-197.  video [B,T,3,H,W] -> ([B, M + T*L, C], (M, T, L)).

    Sequence order: [cls, proxy_0..proxy_{M-2}, frame0 patch0..L-1, frame1 ...]; patch order is
    row-major over the (H/p, W/p) grid (`flatten(2)` at :179).  Every global token gets position 0.
    """
    B, T, C, H, W = video.shape
    w = sd[pre + "patch_embedding.weight"]
    p = cfg.patch
    # stride == kernel, no bias: the conv is an im2col GEMM (CLIP_ViP.py:157-159,178)
    x = video.reshape(B * T, C, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5).reshape(B * T, -1, C * p * p)
    patches = x @ w.reshape(w.shape[0], -1).t()                       # [B*T, L, width]
    L = patches.shape[1]
    patches = patches.reshape(B, T, L, -1)
    pos = sd[pre + "position_embedding.weight"]
    if pre + "temporal_embedding" in sd:    # if_use_temporal_embed = 0 builds no table (CLIP_ViP.py:165-166,183)
        patches = patches + temporal_table(sd, T, pre).unsqueeze(2)
    patches = patches + pos[1:].unsqueeze(0).unsqueeze(0)
    cls = (sd[pre + "class_embedding"] + pos[0]).expand(B, 1, -1)
    proxies = (sd[pre + "added_cls"] + pos[0]).unsqueeze(0).expand(B, -1, -1)
    M = 1 + sd[pre + "added_cls"].shape[0]
    return torch.cat([cls, proxies, patches.reshape(B, T * L, -1)], dim=1), (M, T, L)


def split_heads(x: Tensor, heads: int) -> Tensor:
    B, S, C = x.shape
    return x.reshape(B, S, heads, C // heads).transpose(1, 2)        # [B,H,S,d]


def vip_attention(sd: Dict[str, Tensor], x: Tensor, pre: str, heads: int, size: Tuple[int, int, int]) -> Tensor:
    """CLIPAttention.forward2, CLIP_ViP.py:332-381.

    Patch queries of frame t attend to [M global keys ; L keys of frame t]; the M global
    queries attend to all M + T*L keys.  q is scaled by head_dim**-0.5 AFTER the bias (:341).
    Equivalent to dense attention under the block mask
        allow[i, j] = global(i) or global(j) or frame(i) == frame(j).
    """
    M, T, L = size
    B, S, C = x.shape
    d = C // heads
    q = split_heads(linear(x, sd, pre + "q_proj") * d ** -0.5, heads)
    k = split_heads(linear(x, sd, pre + "k_proj"), heads)
    v = split_heads(linear(x, sd, pre + "v_proj"), heads)
    o = vip_core(q, k, v, size)
    o = o.transpose(1, 2).reshape(B, S, C)
    return linear(o, sd, pre + "out_proj")


def vip_core(q: Tensor, k: Tensor, v: Tensor, size: Tuple[int, int, int]) -> Tensor:
    """Both softmaxes of vip_attention: q (already scaled), k, v [B,H,S,d] -> o [B,H,S,d]."""
    M, T, L = size
    B, heads, S, d = q.shape
    qf = q[:, :, M:].reshape(B, heads, T, L, d)
    kg = k[:, :, :M].unsqueeze(2).expand(B, heads, T, M, d)
    vg = v[:, :, :M].unsqueeze(2).expand(B, heads, T, M, d)
    kf = torch.cat([kg, k[:, :, M:].reshape(B, heads, T, L, d)], dim=3)
    vf = torch.cat([vg, v[:, :, M:].reshape(B, heads, T, L, d)], dim=3)
    of = torch.softmax(qf @ kf.transpose(-1, -2), dim=-1) @ vf      # [B,H,T,L,d]
    og = torch.softmax(q[:, :, :M] @ k.transpose(-1, -2), dim=-1) @ v  # [B,H,M,d]
    return torch.cat([og, of.reshape(B, heads, T * L, d)], dim=2)


def dense_attention(sd: Dict[str, Tensor], x: Tensor, pre: str, heads: int, add_mask: Optional[Tensor]) -> Tensor:
    """CLIPAttention.forward, CLIP_ViP.py:266-330 (text tower).  add_mask is [B,1,S,S] additive."""
    B, S, C = x.shape
    d = C // heads
    q = split_heads(linear(x, sd, pre + "q_proj") * d ** -0.5, heads)
    k = split_heads(linear(x, sd, pre + "k_proj"), heads)
    v = split_heads(linear(x, sd, pre + "v_proj"), heads)
    o = dense_core(q, k, v, add_mask)
    return linear(o.transpose(1, 2).reshape(B, S, C), sd, pre + "out_proj")


def dense_core(q: Tensor, k: Tensor, v: Tensor, add_mask: Optional[Tensor]) -> Tensor:
    """softmax(q k^T + add_mask) v over [B,H,S,d] (q already scaled)."""
    s = q @ k.transpose(-1, -2)
    if add_mask is not None:
        s = s + add_mask
    return torch.softmax(s, dim=-1) @ v


def encoder_layer(sd: Dict[str, Tensor], x: Tensor, pre: str, heads: int, eps: float,
                  size: Optional[Tuple[int, int, int]], add_mask: Optional[Tensor]) -> Tensor:
    """Pre-LN residual block, CLIP_ViP.py:445-460."""
    h = layer_norm(x, sd, pre + "layer_norm1", eps)
    if size is not None:
        h = vip_attention(sd, h, pre + "self_attn.", heads, size)
    else:
        h = dense_attention(sd, h, pre + "self_attn.", heads, add_mask)
    x = residual_add(x, h)
    h = layer_norm(x, sd, pre + "layer_norm2", eps)
    h = linear(quick_gelu(linear(h, sd, pre + "mlp.fc1")), sd, pre + "mlp.fc2")
    return residual_add(x, h)


def vision_tower(sd: Dict[str, Tensor], video: Tensor, cfg: ClipVipCfg, return_hidden: bool = False):
    """CLIPVisionTransformer.forward, CLIP_ViP.py:861-903 (note the reference's `pre_layrnorm` spelling)."""
    x, size = vip_embeddings(sd, video, cfg)
    x = layer_norm(x, sd, "vision_model.pre_layrnorm", cfg.ln_eps)
    hidden = [x]
    for i in range(cfg.vision.layers):
        x = encoder_layer(sd, x, f"vision_model.encoder.layers.{i}.", cfg.vision.heads, cfg.ln_eps, size, None)
        hidden.append(x)
    pooled = layer_norm(x[:, 0], sd, "vision_model.post_layernorm", cfg.ln_eps)
    return (pooled, hidden) if return_hidden else pooled


# ----------------------------------------------------------------------------- text
def text_additive_mask(attention_mask: Tensor, dtype: torch.dtype) -> Tensor:
    """Causal (-inf above the diagonal, CLIP_ViP.py:788-797) + padding (finfo.min on masked keys, :50-61,760)."""
    B, S = attention_mask.shape
    causal = torch.full((S, S), float("-inf"), dtype=dtype, device=attention_mask.device).triu(1)
    inv = 1.0 - attention_mask[:, None, None, :].to(dtype)
    pad = inv.masked_fill(inv.bool(), torch.finfo(dtype).min).expand(B, 1, S, S)
    return causal[None, None] + pad


def text_embeddings(sd: Dict[str, Tensor], input_ids: Tensor) -> Tensor:
    """CLIPTextEmbeddings.forward, CLIP_ViP.py:210-227: token rows plus position rows 0..S-1."""
    pre = "text_model.embeddings."
    return sd[pre + "token_embedding.weight"][input_ids] + sd[pre + "position_embedding.weight"][:input_ids.shape[1]]


def text_tower(sd: Dict[str, Tensor], input_ids: Tensor, attention_mask: Tensor, cfg: ClipVipCfg,
               return_hidden: bool = False):
    """CLIPTextTransformer.forward, CLIP_ViP.py:726-786."""
    B, S = input_ids.shape
    x = text_embeddings(sd, input_ids)
    mask = text_additive_mask(attention_mask, x.dtype)
    hidden = [x]
    for i in range(cfg.text.layers):
        x = encoder_layer(sd, x, f"text_model.encoder.layers.{i}.", cfg.text.heads, cfg.ln_eps, None, mask)
        hidden.append(x)
    x = layer_norm(x, sd, "text_model.final_layer_norm", cfg.ln_eps)
    # EOS pooling: FIRST index of the maximum token id (CLIP_ViP.py:776; pad id == eos id 49407)
    pooled = x[torch.arange(B, device=x.device), input_ids.argmax(dim=-1)]
    return (pooled, hidden) if return_hidden else pooled


# ------------------------------------------------------------------- heads and loss
def l2_normalize(x: Tensor) -> Tensor:
    return x / x.norm(dim=-1, keepdim=True)          # CLIP_ViP.py:1148-1149 (no epsilon)


def clip_vip_forward(sd: Dict[str, Tensor], video: Tensor, input_ids: Tensor, attention_mask: Tensor,
                     cfg: ClipVipCfg) -> Dict[str, Tensor]:
    """VidCLIP.forward (VidCLIP.py:32-53) -> CLIPModel.forward (CLIP_ViP.py:1089-1172)."""
    vis = l2_normalize(linear(vision_tower(sd, video, cfg), sd, "visual_projection"))
    txt = l2_normalize(linear(text_tower(sd, input_ids, attention_mask, cfg), sd, "text_projection"))
    return {"vis_features": vis, "text_features": txt}


def nce_learnable_temp_loss(vis: Tensor, txt: Tensor, logit_scale: Tensor) -> Tensor:
    """NCELearnableTempLoss.forward, loss.py:134-141: CE(rows) + CE(cols), SUM of the two (no 1/2)."""
    z = vis @ txt.t() * logit_scale.exp()
    labels = torch.arange(z.shape[0], device=z.device)
    return F.cross_entropy(z, labels) + F.cross_entropy(z.t(), labels)


def nce_closed_form_grads(vis: Tensor, txt: Tensor, logit_scale: Tensor):
    """Closed-form gradients of the loss above (SURVEY.md §8e): G = (P_row + P_col - 2I)/N."""
    s = logit_scale.exp()
    z = vis @ txt.t() * s
    n = z.shape[0]
    g = (torch.softmax(z, 1) + torch.softmax(z, 0) - 2 * torch.eye(n, dtype=z.dtype)) / n
    return s * g @ txt, s * g.t() @ vis, (g * z).sum()


def nce_vsc_fc_loss(vis: Tensor, txt: Tensor, img: Tensor, cap: Tensor, logit_scale: Tensor) -> Tensor:
    """NCELearnableTempLoss_vsc_fc.forward, loss.py:288-324 (the released pre-training default, pretrain_vip_base_16.json:74-77):
    six cross-entropies over A = s V T^T (video x subtitle), B = s V C^T (video x caption), D = s I C^T (frame x caption):
      columns of A, columns of B                                    (t2v, t2v_2:  :296-301, :316)
      row i over [A_ii | A_i,j!=i | B_i,j!=i] and [B_ii | A_i,j!=i | B_i,j!=i] with label 0   (:303-310, :317)
      columns and rows of D                                         (:312-318)
    each a mean over the N rows, summed."""
    s = logit_scale.exp()
    a, b, d = vis @ txt.t() * s, vis @ cap.t() * s, img @ cap.t() * s
    n = a.shape[0]
    eye = torch.eye(n, dtype=torch.bool, device=a.device)
    ninf = torch.full_like(a, float("-inf"))
    row3 = torch.logsumexp(torch.cat([a, torch.where(eye, ninf, b)], 1), 1)      # A row (all) + B row without its diagonal
    row4 = torch.logsumexp(torch.cat([torch.where(eye, ninf, a), b], 1), 1)      # A row without its diagonal + B row (all)
    da, db, dd = a.diagonal(), b.diagonal(), d.diagonal()
    terms = (torch.logsumexp(a, 0) - da, torch.logsumexp(b, 0) - db, row3 - da, row4 - db,
             torch.logsumexp(d, 0) - dd, torch.logsumexp(d, 1) - dd)
    return sum(t.mean() for t in terms)


def run_reduced_precision(sd: Dict[str, Tensor], video: Tensor, input_ids: Tensor, attention_mask: Tensor, cfg: "ClipVipCfg",
                          device, mode: str):
    """Calibration arm of the parity tests: THIS restatement of the reference algorithm run in reduced precision on `device`.
    mode 'autocast' = fp32 weights under torch.autocast(bf16) — the only way the reference itself runs in bf16 (its `.to(bf16)`
    crashes in the mask code, SURVEY.md §8c); mode 'pure' = every floating tensor in bf16 (what apex amp O2 does in fp16,
    run_pretrain.py:234-236).  Returns (vis, txt, loss, {name: grad}) as fp32 CPU values."""
    dt = torch.bfloat16 if mode == "pure" else torch.float32
    dev = torch.device(device)
    sdg = {k: (v.detach().to(dev, dt, copy=True).requires_grad_(True) if v.is_floating_point() else v.to(dev))
           for k, v in sd.items()}
    with torch.autocast(dev.type, dtype=torch.bfloat16, enabled=(mode == "autocast")):
        o = clip_vip_forward(sdg, video.to(dev, dt), input_ids.to(dev), attention_mask.to(dev), cfg)
        loss = nce_learnable_temp_loss(o["vis_features"].float(), o["text_features"].float(), sdg["logit_scale"].float())
    loss.backward()
    grads = {k: t.grad.detach().float().cpu() for k, t in sdg.items() if t.is_floating_point() and t.grad is not None}
    return o["vis_features"].detach().float().cpu(), o["text_features"].detach().float().cpu(), float(loss.detach()), grads


def gather_rank_major(per_rank: list) -> Tensor:
    """hvd.allgather (run_pretrain.py:344-345) / SyncFunction.forward (LF-VILA/src/utils/dist.py:21-33):
    rank-major concatenation along dim 0."""
    return torch.cat(list(per_rank), dim=0)


# ------------------------------------------------------------------ synthetic setup
def init_state_dict(cfg: ClipVipCfg, seed: int = 0, dtype=torch.float32) -> Dict[str, Tensor]:
    """Random weights with the reference's init statistics (CLIPPreTrainedModel._init_weights,
    CLIP_ViP.py:481-522; added_cls ~ N(0,1) :153).  temporal_embedding is zero in the reference (:166);
    here it is N(0, 0.02) so that the temporal add is exercised (SURVEY.md §8d).  LayerNorm
    weights/biases and Linear biases are perturbed as well so that no term is trivially 1 or 0."""
    g = torch.Generator().manual_seed(seed)

    def n(*shape, std=1.0):
        return torch.randn(*shape, generator=g, dtype=dtype) * std

    sd: Dict[str, Tensor] = {"logit_scale": torch.tensor(cfg.logit_scale_init, dtype=dtype)}

    def tower(prefix: str, tc: TowerCfg):
        in_std = tc.width ** -0.5 * (2 * tc.layers) ** -0.5
        for i in range(tc.layers):
            p = f"{prefix}.encoder.layers.{i}."
            for name in ("q_proj", "k_proj", "v_proj"):
                sd[p + f"self_attn.{name}.weight"] = n(tc.width, tc.width, std=in_std)
                sd[p + f"self_attn.{name}.bias"] = n(tc.width, std=0.02)
            sd[p + "self_attn.out_proj.weight"] = n(tc.width, tc.width, std=tc.width ** -0.5)
            sd[p + "self_attn.out_proj.bias"] = n(tc.width, std=0.02)
            for ln in ("layer_norm1", "layer_norm2"):
                sd[p + ln + ".weight"] = 1.0 + n(tc.width, std=0.05)
                sd[p + ln + ".bias"] = n(tc.width, std=0.05)
            sd[p + "mlp.fc1.weight"] = n(tc.mlp, tc.width, std=(2 * tc.width) ** -0.5)
            sd[p + "mlp.fc1.bias"] = n(tc.mlp, std=0.02)
            sd[p + "mlp.fc2.weight"] = n(tc.width, tc.mlp, std=in_std)
            sd[p + "mlp.fc2.bias"] = n(tc.width, std=0.02)

    v = "vision_model.embeddings."
    sd[v + "class_embedding"] = n(cfg.vision.width, std=cfg.vision.width ** -0.5)
    sd[v + "added_cls"] = n(cfg.add_cls_num, cfg.vision.width)
    sd[v + "patch_embedding.weight"] = n(cfg.vision.width, 3, cfg.patch, cfg.patch, std=0.02)
    sd[v + "position_embedding.weight"] = n(cfg.patches + 1, cfg.vision.width, std=0.02)
    sd[v + "temporal_embedding"] = n(1, cfg.temporal_size, cfg.vision.width, std=0.02)
    sd[v + "position_ids"] = torch.arange(cfg.patches + 1).unsqueeze(0)
    for ln in ("pre_layrnorm", "post_layernorm"):
        sd[f"vision_model.{ln}.weight"] = 1.0 + n(cfg.vision.width, std=0.05)
        sd[f"vision_model.{ln}.bias"] = n(cfg.vision.width, std=0.05)
    tower("vision_model", cfg.vision)
    t = "text_model.embeddings."
    sd[t + "token_embedding.weight"] = n(cfg.vocab, cfg.text.width, std=0.02)
    sd[t + "position_embedding.weight"] = n(cfg.max_text_pos, cfg.text.width, std=0.02)
    sd[t + "position_ids"] = torch.arange(cfg.max_text_pos).unsqueeze(0)
    sd["text_model.final_layer_norm.weight"] = 1.0 + n(cfg.text.width, std=0.05)
    sd["text_model.final_layer_norm.bias"] = n(cfg.text.width, std=0.05)
    tower("text_model", cfg.text)
    sd["visual_projection.weight"] = n(cfg.proj_dim, cfg.vision.width, std=cfg.vision.width ** -0.5)
    sd["text_projection.weight"] = n(cfg.proj_dim, cfg.text.width, std=cfg.text.width ** -0.5)
    return sd


def synthetic_batch(B: int, T: int, Lt: int, cfg: ClipVipCfg, seed: int = 1234, ragged_text: bool = False):
    """SURVEY.md §8d inputs: N(0,1) video, ids in [1, 49406) with EOS (49407) last.  With
    ragged_text the EOS sits at a random position followed by pad=49407 / mask=0, which exercises
    first-max pooling and the padding mask."""
    g = torch.Generator().manual_seed(seed)
    video = torch.randn(B, T, 3, cfg.image_size, cfg.image_size, generator=g)
    ids = torch.randint(1, cfg.vocab - 2, (B, Lt), generator=g)
    mask = torch.ones(B, Lt, dtype=torch.long)
    if ragged_text:
        eos = torch.randint(2, Lt, (B,), generator=g)
        for b in range(B):
            ids[b, eos[b]:] = cfg.vocab - 1
            mask[b, eos[b] + 1:] = 0
    else:
        ids[:, -1] = cfg.vocab - 1
    return video, ids, mask


def flops_per_pair(cfg: ClipVipCfg, T: int, Lt: int) -> Dict[str, float]:
    """Algorithmic FLOPs (2 per MAC) per video-text pair; reproduces BASELINE.md §2 (423.12 G fwd at T=12, Lt=32)."""
    C, mlp, L, M = cfg.vision.width, cfg.vision.mlp, cfg.patches, 1 + cfg.add_cls_num
    S = M + T * L
    d = C // cfg.vision.heads
    qkv = 2 * S * C * 3 * C
    attn = cfg.vision.heads * (2 * 2 * T * L * (M + L) * d + 2 * 2 * M * S * d)
    outp = 2 * S * C * C
    mlpf = 2 * 2 * S * C * mlp
    block = qkv + attn + outp + mlpf
    patch = 2 * T * L * (3 * cfg.patch * cfg.patch) * C
    vproj = 2 * C * cfg.proj_dim
    Ct, mt = cfg.text.width, cfg.text.mlp
    tblock = 2 * Lt * Ct * 3 * Ct + cfg.text.heads * 2 * 2 * Lt * Lt * (Ct // cfg.text.heads) + 2 * Lt * Ct * Ct \
        + 2 * 2 * Lt * Ct * mt
    tproj = 2 * Ct * cfg.proj_dim
    fwd = patch + cfg.vision.layers * block + vproj + cfg.text.layers * tblock + tproj
    # backward = dgrad + wgrad of every GEMM except: patch-embed has no dgrad (input needs no grad)
    bwd = 2 * fwd - patch
    return {"fwd": float(fwd), "train": float(fwd + bwd), "vip_block_fwd": float(block)}
