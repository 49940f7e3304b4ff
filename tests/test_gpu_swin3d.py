"""H100: BASELINE.json config #5 (LF-VILA Swin-3D video encoder) — kernels and module against the oracle and the reference goldens."""
import os

import pytest
import torch

from encoder_cases import swin3d_case
from oracle import swin3d_oracle as SO

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


# ------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("n_win,L,heads,nW,n_pad", [
    (6, 30, 2, 1, 0),        # layer-0 window, no mask
    (8, 30, 4, 4, 5),        # shifted: 4 window types with a -100 mask, a few zero-padded positions
    (3, 120, 2, 1, 0),       # two key blocks
    (2, 480, 4, 1, 0),       # the last stage's 32 x 3 x 5 window: 8 key blocks
    (5, 48, 8, 1, 7),        # clamped window (8 x 2 x 3)
])
def test_window_attention_fwd_bwd(dev, n_win, L, heads, nW, n_pad):
    """Indexed window attention (head_dim 32) with an additive bias slab: forward, dq/dk/dv and dL/dlogits vs fp32 torch."""
    from xpretrain_b200 import ops

    torch.manual_seed(L + heads)
    C = heads * 32
    n_tok = n_win * L - n_pad            # real tokens; padded positions get their own extra rows
    n_ext = n_tok + n_pad
    perm = torch.randperm(n_ext)         # windows pick arbitrary rows (roll + partition is a permutation)
    idx = perm.view(n_win, L).to(torch.int32).to(dev)
    qkv = torch.randn(n_ext, 3 * C, device=dev)
    qkv[:, :C] *= 32 ** -0.5 * 3.0
    qkv = qkv.to(bf16)
    bias = torch.randn(nW, heads, L, L, device=dev) * 0.5
    if nW > 1:
        bias = bias + torch.where(torch.rand(nW, 1, L, L, device=dev) < 0.3, -100.0, 0.0)
        bias[:, :, torch.arange(L), torch.arange(L)] = bias[:, :, torch.arange(L), torch.arange(L)].clamp_min(-5)   # keep the diagonal alive
    bias = bias.contiguous()
    out = torch.zeros(n_ext, C, dtype=bf16, device=dev)
    lse = torch.zeros(heads, n_ext, device=dev)
    ops.seg_attention_fwd(qkv, out, lse, ops.window_desc(n_ext, heads, 32, 3 * C, C, idx, bias))
    torch.cuda.synchronize()

    x = qkv.float().requires_grad_(True)
    b32 = bias.clone().requires_grad_(True)
    ref = torch.zeros(n_ext, C, device=dev)
    for w in range(n_win):
        rows = idx[w].long()
        q = x[rows, :C].view(L, heads, 32).transpose(0, 1)
        k = x[rows, C:2 * C].view(L, heads, 32).transpose(0, 1)
        v = x[rows, 2 * C:].view(L, heads, 32).transpose(0, 1)
        p = (q @ k.transpose(1, 2) + b32[w % nW]).softmax(-1)
        ref = ref.index_put((rows,), (p @ v).transpose(0, 1).reshape(L, C))
    assert torch.isfinite(out.float()).all()
    assert _rel(out, ref.detach()) < 8e-3

    dout = torch.randn(n_ext, C, device=dev).to(bf16)
    (ref * dout.float()).sum().backward()
    dqkv = torch.zeros(n_ext, 3 * C, dtype=bf16, device=dev)
    delta = torch.empty(heads, n_ext, device=dev)
    ds = torch.full((n_win, heads, L, L), float("nan"), dtype=bf16, device=dev)
    ops.seg_attention_bwd(qkv, out, dout, lse, delta, dqkv, ops.window_desc(n_ext, heads, 32, 3 * C, C, idx, bias, ds_out=ds), 1.0)
    torch.cuda.synchronize()
    assert torch.isfinite(dqkv.float()).all() and torch.isfinite(ds.float()).all()
    for name, sl in (("dq", slice(0, C)), ("dk", slice(C, 2 * C)), ("dv", slice(2 * C, 3 * C))):
        assert _rel(dqkv[:, sl], x.grad[:, sl]) < 1.5e-2, name
    # bias gradient = sum over the windows of a type of dL/dlogits
    dbias = torch.zeros_like(bias)
    dbias.index_add_(0, torch.arange(n_win, device=dev) % nW, ds.float())
    assert _rel(dbias, b32.grad) < 1.5e-2


def test_wide_layernorm_and_row_gather(dev):
    from xpretrain_b200 import ops

    torch.manual_seed(1)
    rows, C = 300, 2048
    x = torch.randn(rows, C, device=dev).to(bf16)
    gamma, beta = torch.randn(C, device=dev) * 0.1 + 1, torch.randn(C, device=dev) * 0.1
    y = torch.empty_like(x)
    mean, rstd = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
    ops.layernorm_any_fwd(x, y, gamma, beta, mean, rstd, rows, C, 1e-5)
    xr = x.float().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(xr, (C,), gr, br, 1e-5)
    assert _rel(y, ref.detach()) < 4e-3
    dy = torch.randn(rows, C, device=dev).to(bf16)
    ref.backward(dy.float())
    dx = torch.empty_like(x)
    dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    ops.layernorm_any_bwd(dy, x, gamma, mean, rstd, None, dx, dg, db, rows, C)
    assert _rel(dx, xr.grad) < 6e-3 and _rel(dg, gr.grad) < 2e-3 and _rel(db, br.grad) < 2e-3
    # gather (with -1 -> zeros) and its inverse
    src = torch.randn(50, 64, device=dev).to(bf16)
    index = torch.tensor([3, -1, 49, 0, 7, 7 + 1, -1, 20], dtype=torch.int32, device=dev)
    out = torch.full((2, 4 * 64), 9.0, dtype=bf16, device=dev)
    ops.gather_rows(src, index, out, 64)
    want = torch.where(index[:, None] >= 0, src[index.clamp_min(0).long()], torch.zeros((), dtype=bf16, device=dev))
    assert torch.equal(out.view(8, 64), want)
    dst = torch.zeros(50, 64, dtype=bf16, device=dev)
    ops.scatter_rows(out, index, dst, 64)
    live = index[index >= 0].long()
    assert torch.equal(dst[live], src[live]) and float(dst.float().abs().sum()) == float(src[live.unique()].float().abs().sum())


# -------------------------------------------------------------------------------------- module
def _build(cfg, sd, dev, rate=0.2):
    from xpretrain_b200.modeling.swin3d import SwinTransformer3D

    m = SwinTransformer3D(patch_size=list(cfg.patch_size), embed_dim=cfg.embed_dim, depths=list(cfg.depths),
                          num_heads=list(cfg.num_heads), stages=list(cfg.stages), downsample_stages=list(cfg.downsample_stages),
                          window_size=[list(w) for w in cfg.window_size], patch_norm=cfg.patch_norm, local_window=cfg.local_window,
                          drop_path_rate=rate)
    m.load_state_dict(sd, strict=True)
    return m.to(dev)


@pytest.mark.parametrize("name", ["swin3d_small_b2", "swin3d_padded_b1", "swin3d_train_droppath"])
def test_module_matches_reference_golden(dev, golden_dir, name):
    gold = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    cfg = SO.Swin3DCfg(**gold["cfg"])
    model = _build(cfg, SO.init_state_dict(cfg, seed=gold["weight_seed"]), dev, rate=gold["train_rate"] or 0.2)
    if gold["train_rate"]:
        model.train()
        model.forced_drop_masks = [None if m is None else tuple(t.to(dev) for t in m) for m in gold["masks"]]
    else:
        model.eval()
    video = SO.synthetic_video(gold["B"], gold["D"], gold["H"], gold["W"], cfg, seed=gold["data_seed"]).to(dev)
    out, out2 = model(video)
    assert out2 is out and out.shape == gold["out"].shape
    e = _rel(out.detach().cpu(), gold["out"])
    print(f"{name}: out rel-L2 {e:.2e}, cos {_cos(out.detach().cpu(), gold['out']):.6f}")
    assert e < 2e-2 and _cos(out.detach().cpu(), gold["out"]) > 0.9997
    g = torch.Generator().manual_seed(gold["data_seed"] + 1)
    w_out = (torch.randn(out.shape, generator=g) / out[0].numel() ** 0.5).to(dev)
    (out * w_out).sum().backward()
    params = dict(model.named_parameters())
    for n, ref in gold["grads"].items():
        got = params[n].grad
        assert got is not None, n
        got = (got if ref.shape == got.shape else got[:8]).cpu()
        c = _cos(got, ref)
        print(f"  grad {n}: cos {c:.5f}")
        assert c > 0.985, (n, c)
    assert params["norm_local.weight"].grad is None and params["local_feat_proj.reduction.weight"].grad is None


def test_training_mode_draws_the_references_rng_stream(dev):
    cfg = SO.Swin3DCfg(embed_dim=64, depths=(2, 2, 2), num_heads=(2, 4, 8), stages=(0, 1, 2), downsample_stages=(0, 1),
                       window_size=((2, 3, 5), (4, 3, 5), (8, 3, 5)))
    model = _build(cfg, SO.init_state_dict(cfg, seed=0), dev, rate=0.5)
    torch.manual_seed(9)
    ours = model.draw_drop_masks(4, dev, torch.float32)
    torch.manual_seed(9)
    want = SO.draw_drop_masks(cfg, 4, 0.5, device=dev)
    for a, b in zip(ours, want):
        assert (a is None) == (b is None)
        if a is not None:
            assert all(torch.equal(u, v) for u, v in zip(a, b))


def test_released_config_one_sample_against_fp32_oracle_on_gpu(dev):
    """The released VideoEncoder config (6 stages, dims 128..1024, windows up to 32 x 3 x 5), 1 x 32 frames x 96 x 160:
    the output and every parameter gradient within 1.5 x the bf16 oracle's error of the fp32 oracle, whole and per slice
    (encoder_cases.swin3d_case); and the earlier fixed thresholds on top."""
    (out, _, grads), (ref, _, ref_grads) = swin3d_case(dev, "swin released_1x32x96x160", SO.Swin3DCfg(), 1, 32, 96, 160,
                                                       weight_seed=4, data_seed=5, branches={"colsum"})
    assert _rel(out, ref) < 3e-2
    for n in ("layers.2.blocks.5.attn.qkv.weight", "layers.2.blocks.6.attn.relative_position_bias_table",
              "layers.0.blocks.1.mlp.fc1.weight", "layers.4.downsample.reduction.weight", "layers.5.blocks.1.attn.proj.weight",
              "patch_embed.proj.weight"):
        assert _cos(grads[n], ref_grads[n]) > 0.98, n
