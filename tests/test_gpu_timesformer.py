"""H100: BASELINE.json config #4 (HD-VILA TimeSformer) — kernels and module against the oracle and the reference goldens."""
import math
import os

import pytest
import torch

from encoder_cases import timesformer_case
from oracle import timesformer_oracle as TO

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


def _cos(a, b):
    return float(torch.nn.functional.cosine_similarity(a.float().flatten(), b.float().flatten(), dim=0))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "these tests need the H100"
    return torch.device("cuda", 0)


# ------------------------------------------------------------------------------ attention kernels
def _ref_attention(qkv, groups, heads):
    """fp32 reference: qkv [rows, 3C] (q pre-scaled); groups = list of LongTensors of row indices."""
    rows, C3 = qkv.shape
    C = C3 // 3
    out = torch.zeros(rows, C, dtype=torch.float32, device=qkv.device)
    lse = torch.zeros(heads, rows, dtype=torch.float32, device=qkv.device)
    x = qkv.float()
    for idx in groups:
        q = x[idx, :C].view(-1, heads, 64).transpose(0, 1)
        k = x[idx, C:2 * C].view(-1, heads, 64).transpose(0, 1)
        v = x[idx, 2 * C:].view(-1, heads, 64).transpose(0, 1)
        s = q @ k.transpose(1, 2)
        lse[:, idx] = torch.logsumexp(s, dim=-1)
        out[idx] = (s.softmax(-1) @ v).transpose(0, 1).reshape(-1, C)
    return out, lse


def _groups(kind, B, T, HW, dev):
    rows = B * HW * T
    r = torch.arange(rows, device=dev)
    if kind == "temporal":
        return list(r.view(B * HW, T))
    return list(r.view(B, HW, T).permute(0, 2, 1).reshape(B * T, HW))


@pytest.mark.parametrize("kind,B,T,HW,heads", [
    ("temporal", 2, 7, 10, 2),        # ragged: 140 rows, 63-row tiles
    ("temporal", 3, 8, 49, 2),        # T = 8: full 64-row tiles, 1176 rows
    ("temporal", 1, 3, 5, 1),         # tiny (interp golden shape)
    ("spatial", 2, 7, 70, 2),         # two key blocks, ragged second
    ("spatial", 2, 3, 15, 1),         # less than one block
    ("spatial", 1, 2, 784, 2),        # 28x28 stress grid: 13 key blocks
    ("spatial", 2, 7, 160, 16),       # reference-native grid, 16 heads
])
def test_seg_attention_fwd_bwd(dev, kind, B, T, HW, heads):
    from xpretrain_b200 import ops

    torch.manual_seed(5)
    C = heads * 64
    rows = B * HW * T
    qkv = torch.randn(rows, 3 * C, device=dev)
    qkv[:, :C] *= 0.125 * 2.0         # pre-scaled q, logits with a spread of a few units
    qkv = qkv.to(bf16)
    groups = _groups(kind, B, T, HW, dev)
    desc = (ops.temporal_desc(rows, T, heads, 3 * C, C) if kind == "temporal"
            else ops.spatial_desc(B, T, HW, heads, 3 * C, C))
    out = torch.full((rows, C), float("nan"), dtype=bf16, device=dev)
    lse = torch.full((heads, rows), float("nan"), device=dev)
    ops.seg_attention_fwd(qkv, out, lse, desc)
    torch.cuda.synchronize()

    q32 = qkv.float().requires_grad_(True)
    ref_out, ref_lse = _ref_attention(q32, groups, heads)
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    assert _rel(out, ref_out.detach()) < 6e-3
    assert float((lse - ref_lse.detach()).abs().max()) < 2e-3

    dout = torch.randn(rows, C, device=dev).to(bf16)
    (ref_out * dout.float()).sum().backward()
    dqkv = torch.full((rows, 3 * C), float("nan"), dtype=bf16, device=dev)
    delta = torch.empty(heads, rows, device=dev)
    ops.seg_attention_bwd(qkv, out, dout, lse, delta, dqkv, desc, 1.0)
    torch.cuda.synchronize()
    assert torch.isfinite(dqkv.float()).all()
    g = q32.grad
    for name, sl in (("dq", slice(0, C)), ("dk", slice(C, 2 * C)), ("dv", slice(2 * C, 3 * C))):
        assert _rel(dqkv[:, sl], g[:, sl]) < 1.2e-2, name


def test_tokenize_round_trip_and_tables(dev):
    from xpretrain_b200 import ops

    torch.manual_seed(2)
    B, T, C, H, W = 2, 3, 128, 5, 7
    x = torch.randn(B, T, C, H, W, device=dev)
    pos = torch.randn(H * W, C, device=dev)
    time = torch.randn(T, C, device=dev)
    tok = torch.empty(B * H * W * T, C, dtype=bf16, device=dev)
    ops.tsf_embed_fwd(x, pos, time, tok, B, T, C, H * W)
    want = (x.flatten(3).permute(0, 3, 1, 2) + pos[None, :, None, :] + time[None, None]).reshape(-1, C)
    assert torch.equal(tok, want.to(bf16))                      # same fp32 adds, one rounding
    ops.tsf_embed_fwd(x.to(bf16), None, None, tok, B, T, C, H * W)
    back = torch.empty(B, T, C, H, W, dtype=bf16, device=dev)
    ops.tsf_untokenize(tok, back, B, T, C, H * W)
    assert torch.equal(back, x.to(bf16))                        # pure layout change: bit exact


# ------------------------------------------------------------------------------------ module
def _build(cfg, sd, dev):
    from xpretrain_b200.modeling.timesformer import TimeSformer

    m = TimeSformer(depth=cfg.depth, num_frames=cfg.num_frames, H=cfg.H, W=cfg.W, embed_dim=cfg.embed_dim,
                    num_heads=cfg.num_heads, drop_path_rate=0.1)
    missing, unexpected = m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


@pytest.mark.parametrize("name", ["timesformer_interp_b2", "timesformer_native_b2"])
def test_module_matches_reference_golden(dev, golden_dir, name):
    gold = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    cfg = TO.TimeSformerCfg(**gold["cfg"])
    sd = TO.init_state_dict(cfg, seed=gold["weight_seed"])
    model = _build(cfg, sd, dev)
    B, T, H, W = gold["B"], gold["T"], gold["H"], gold["W"]
    x = TO.synthetic_input(B, T, H, W, cfg, seed=gold["data_seed"]).to(dev).requires_grad_(True)
    g = torch.Generator().manual_seed(gold["data_seed"] + 1)
    w_out = (torch.randn(gold["out"].shape, generator=g) / (B * T * H * W) ** 0.5).to(dev)
    out = model(x)
    assert out.shape == gold["out"].shape and out.dtype == x.dtype
    e_out = _rel(out.detach().cpu(), gold["out"])
    loss = (out * w_out).sum()
    loss.backward()
    print(f"{name}: out rel-L2 {e_out:.2e}  loss {float(loss):.5f} vs {float(gold['loss']):.5f}")
    assert e_out < 1.5e-2                    # bf16 activations through 2 blocks (cf. BASELINE.md §3 calibration)
    assert _cos(out.detach().cpu(), gold["out"]) > 0.9998
    assert abs(float(loss) - float(gold["loss"])) < 2e-2 * max(1.0, float(gold["out"].norm()) / 50)
    assert _cos(x.grad[:, 0].cpu(), gold["dx_t0"]) > 0.995
    grads = dict(model.named_parameters())
    for n, ref in gold["grads"].items():
        got = grads[n].grad
        assert got is not None, n
        got = (got[:8] if ref.dim() == 2 else got).cpu()
        c = _cos(got, ref)
        print(f"  grad {n}: cos {c:.5f}")
        assert c > 0.99, (n, c)
    assert model.norm.weight.grad is None    # never applied in forward (timesformer.py:451)


def test_full_width_block_against_fp32_oracle_on_gpu(dev):
    """dim 1024 / 16 heads / native 10x16 grid, 7 frames (the reference shape), depth 2: the output, dx and every
    parameter gradient within 1.5 x the bf16 oracle's error of the fp32 oracle, whole and per slice
    (encoder_cases.timesformer_case); and the earlier fixed thresholds on top."""
    (out, dx, grads), (ref, ref_dx, ref_grads) = timesformer_case(dev, "tsf full_width_7x10x16", TO.TimeSformerCfg(depth=2),
                                                                   2, 7, 10, 16, weight_seed=3, data_seed=4)
    assert _rel(out, ref) < 1.5e-2
    assert _cos(dx, ref_dx) > 0.995
    for n in ("blocks.0.temporal_attn.qkv.weight", "blocks.0.attn.qkv.weight", "blocks.1.mlp.fc1.weight",
              "blocks.0.temporal_fc.weight", "blocks.1.norm2.weight", "pos_embed", "time_embed"):
        assert _cos(grads[n], ref_grads[n]) > 0.99, n


def test_training_mode_drop_path_matches_reference_golden(dev, golden_dir):
    """Training mode with stochastic depth: the reference's own train() forward/backward (seeded) vs ours with the same
    dropped paths (the golden stores the factors the reference drew)."""
    gold = torch.load(os.path.join(golden_dir, "timesformer_train_droppath.pt"), weights_only=False)
    cfg = TO.TimeSformerCfg(**gold["cfg"])
    from xpretrain_b200.modeling.timesformer import TimeSformer

    model = TimeSformer(depth=cfg.depth, num_frames=cfg.num_frames, H=cfg.H, W=cfg.W, embed_dim=cfg.embed_dim,
                        num_heads=cfg.num_heads, drop_path_rate=gold["rate"])
    model.load_state_dict(TO.init_state_dict(cfg, seed=gold["weight_seed"]), strict=True)
    model = model.to(dev).train()
    model.forced_drop_masks = [None if m is None else tuple(t.to(dev) for t in m) for m in gold["masks"]]
    B, T, H, W = gold["B"], gold["T"], gold["H"], gold["W"]
    x = TO.synthetic_input(B, T, H, W, cfg, seed=gold["data_seed"]).to(dev).requires_grad_(True)
    g = torch.Generator().manual_seed(gold["data_seed"] + 1)
    w_out = (torch.randn(gold["out"].shape, generator=g) / (B * T * H * W) ** 0.5).to(dev)
    out = model(x)
    (out * w_out).sum().backward()
    assert _rel(out.detach().cpu(), gold["out"]) < 1.5e-2
    assert _cos(x.grad[:, 0].cpu(), gold["dx_t0"]) > 0.995
    grads = dict(model.named_parameters())
    for n, ref in gold["grads"].items():
        got = grads[n].grad
        got = (got[:8] if ref.dim() == 2 else got).cpu()
        assert _cos(got, ref) > 0.99, (n, _cos(got, ref))
    # the same masks in eval mode are ignored (no path is dropped): the output must differ from the training one
    with torch.no_grad():
        out_eval = model.eval()(x)
    assert _rel(out_eval, out.detach()) > 1e-2


def test_training_mode_draws_the_references_rng_stream(dev):
    """Fresh draws: same torch.rand calls / shapes / order as drop_path (timesformer.py:98-113), so seeding torch the same
    way on the same device gives the factors the oracle's restatement draws."""
    from xpretrain_b200.modeling.timesformer import TimeSformer

    cfg = TO.TimeSformerCfg(depth=3, num_frames=4, H=3, W=4, embed_dim=128, num_heads=2)
    model = TimeSformer(depth=3, num_frames=4, H=3, W=4, embed_dim=128, num_heads=2, drop_path_rate=0.5).to(dev)
    torch.manual_seed(5)
    ours = model.draw_drop_masks(4, 4, 3, 4, dev, torch.float32)
    torch.manual_seed(5)
    want = TO.draw_drop_masks(cfg, 4, 4, 3, 4, 0.5, device=dev)
    assert ours[0] is None and want[0] is None
    for a, b in zip(ours[1:], want[1:]):
        for u, v in zip(a, b):
            assert torch.equal(u, v)
