"""H100: every C-ABI kernel against a plain fp32 PyTorch statement of the same op on the same (bf16-rounded) inputs."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20))


# ---------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (300, 776, 200), (2356, 2304, 768), (64, 512, 768)])
def test_gemm_forward_epilogues(dev, M, N, K):
    from xpretrain_b200 import _lib, ops
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g).to(dev).to(bf16)
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dev).to(bf16)
    b = torch.randn(N, generator=g).to(dev)
    res = torch.randn(M, N, generator=g).to(dev).to(bf16)
    ref = x.float() @ w.float().t() + b
    out = torch.empty(M, N, dtype=bf16, device=dev)
    ops.linear_fwd(x, w, b, out)
    assert rel(out, ref) < 4e-3
    # q-scale on the first third (scale multiplies the bias too) + residual
    sc = (N // 3) // 8 * 8
    ref2 = ref.clone()
    ref2[:, :sc] *= 0.125
    ops.linear_fwd(x, w, b, out, scale_cols=sc, col_scale=0.125, residual=res, ldr=N)
    assert rel(out, ref2 + res.float()) < 4e-3
    # QuickGELU with the pre-activation saved
    pre = torch.empty(M, N, dtype=bf16, device=dev)
    ops.linear_fwd(x, w, b, out, act=_lib.ACT_QUICK_GELU, aux=pre, ld_aux=N)
    assert rel(pre, ref) < 4e-3
    assert rel(out, ref * torch.sigmoid(1.702 * ref)) < 6e-3
    # fp32 output
    outf = torch.empty(M, N, dtype=f32, device=dev)
    ops.linear_fwd(x, w, None, outf, out_mode=_lib.OUT_F32)
    assert rel(outf, x.float() @ w.float().t()) < 1e-5


@pytest.mark.parametrize("rows,N,K", [(256, 128, 64), (2356 * 2, 768, 3072), (4712, 2304, 768), (64, 512, 768), (1000, 320, 776)])
def test_gemm_dgrad_wgrad(dev, rows, N, K):
    """dx = dy W (MN-major B) with the dQuickGELU epilogue; dW += dy^T x (MN-major A and B, split-K atomics)."""
    from xpretrain_b200 import _lib, ops
    g = torch.Generator(device="cpu").manual_seed(rows + N)
    dy = torch.randn(rows, N, generator=g).to(dev).to(bf16)
    w = (torch.randn(N, K, generator=g) / math.sqrt(N)).to(dev).to(bf16)
    x = torch.randn(rows, K, generator=g).to(dev).to(bf16)
    pre = torch.randn(rows, K, generator=g).to(dev).to(bf16)
    dx = torch.empty(rows, K, dtype=bf16, device=dev)
    ops.linear_dgrad(dy, w, dx)
    ref = dy.float() @ w.float()
    assert rel(dx, ref) < 4e-3
    ops.linear_dgrad(dy, w, dx, act=_lib.ACT_DQUICK_GELU, aux=pre, ld_aux=K)
    s = torch.sigmoid(1.702 * pre.float())
    assert rel(dx, ref * (s * (1 + 1.702 * pre.float() * (1 - s)))) < 6e-3
    dw = torch.zeros(N, K, dtype=f32, device=dev)
    ops.linear_wgrad(dy, x, dw)
    ops.linear_wgrad(dy, x, dw)  # accumulates
    assert rel(dw, 2 * (dy.float().t() @ x.float())) < 1e-4


def test_gemm_grouped_rows_patch_embed_layout(dev):
    """C rows written past M global tokens per video and a periodic residual table (the patch-embedding GEMM)."""
    from xpretrain_b200 import ops
    B, TL, Mg, C, K = 3, 40, 4, 256, 128
    S = Mg + TL
    g = torch.Generator(device="cpu").manual_seed(5)
    a = torch.randn(B * TL, K, generator=g).to(dev).to(bf16)
    w = (torch.randn(C, K, generator=g) / math.sqrt(K)).to(dev).to(bf16)
    table = torch.randn(TL, C, generator=g).to(dev).to(bf16)
    x = torch.full((B * S, C), 7.0, dtype=bf16, device=dev)
    ops.gemm(a, w, x, M=B * TL, N=C, K=K, lda=K, ldb=K, ldc=C, residual=table, ldr=C, r_group=TL, r_group_stride=0,
             c_group=TL, c_group_stride=S * C, c_offset=Mg * C)
    ref = (a.float() @ w.float().t()).view(B, TL, C) + table.float()
    xv = x.view(B, S, C)
    assert rel(xv[:, Mg:], ref) < 4e-3
    assert torch.all(xv[:, :Mg] == 7.0)


# ---------------------------------------------------------------------------------------- row kernels
@pytest.mark.parametrize("C", [512, 768, 1024])
def test_layernorm_fwd_bwd(dev, C):
    from xpretrain_b200 import ops
    rows = 1000
    g = torch.Generator(device="cpu").manual_seed(C)
    x = (torch.randn(rows, C, generator=g) * 2 + 0.5).to(dev).to(bf16)
    gamma = (1 + 0.1 * torch.randn(C, generator=g)).to(dev)
    beta = (0.1 * torch.randn(C, generator=g)).to(dev)
    dy = torch.randn(rows, C, generator=g).to(dev).to(bf16)
    dres = torch.randn(rows, C, generator=g).to(dev).to(bf16)
    y = torch.empty_like(x); mean = torch.empty(rows, device=dev); rstd = torch.empty(rows, device=dev)
    plain = ops.rowmap(C)
    ops.layernorm_fwd(x, plain, y, plain, gamma, beta, mean, rstd, rows, C, 1e-5)
    xf = x.float().requires_grad_(True)
    gf, bf_ = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    ref = F.layer_norm(xf, (C,), gf, bf_, 1e-5)
    assert rel(y, ref.detach()) < 4e-3
    assert rel(mean, xf.detach().mean(-1)) < 1e-5
    ref.backward(dy.float())
    dx = torch.empty_like(x); dg = torch.zeros(C, device=dev); db = torch.zeros(C, device=dev)
    ops.layernorm_bwd(dy, plain, x, plain, gamma, mean, rstd, dres, plain, dx, plain, dg, db, rows, C)
    assert rel(dx, xf.grad + dres.float()) < 5e-3
    assert rel(dg, gf.grad) < 1e-4 and rel(db, bf_.grad) < 1e-4


def test_layernorm_row_maps(dev):
    """CLS-row pooling (group=1) and explicit offsets (EOS pooling)."""
    from xpretrain_b200 import ops
    B, S, C = 5, 37, 512
    g = torch.Generator(device="cpu").manual_seed(1)
    x = torch.randn(B * S, C, generator=g).to(dev).to(bf16)
    gamma, beta = torch.ones(C, device=dev), torch.zeros(C, device=dev)
    y = torch.empty(B, C, dtype=bf16, device=dev)
    mean = torch.empty(B, device=dev); rstd = torch.empty(B, device=dev)
    ops.layernorm_fwd(x, ops.rowmap(C, group=1, group_stride=S * C), y, ops.rowmap(C), gamma, beta, mean, rstd, B, C, 1e-5)
    assert rel(y, F.layer_norm(x.view(B, S, C)[:, 0].float(), (C,))) < 4e-3
    ids = torch.randint(1, 100, (B, S), generator=g)
    ids[:, 9] = 1000; ids[2, 4] = 1000      # ties: first maximum wins
    ids = ids.to(dev)
    off = torch.empty(B, dtype=torch.int64, device=dev)
    idx = torch.empty(B, dtype=torch.int32, device=dev)
    ops.eos_offsets(ids, off, idx, C)
    assert torch.equal(idx.long(), ids.argmax(-1))
    ops.layernorm_fwd(x, ops.rowmap(C, offsets=off), y, ops.rowmap(C), gamma, beta, mean, rstd, B, C, 1e-5)
    assert rel(y, F.layer_norm(x.view(B, S, C)[torch.arange(B), ids.argmax(-1)].float(), (C,))) < 4e-3


def test_l2norm_colsum_cast(dev):
    from xpretrain_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(2)
    x = torch.randn(64, 512, generator=g).to(dev)
    y = torch.empty_like(x); inv = torch.empty(64, device=dev)
    ops.l2norm_fwd(x, y, inv)
    xr = x.clone().requires_grad_(True)
    ref = xr / xr.norm(dim=-1, keepdim=True)
    assert rel(y, ref.detach()) < 1e-6
    dy = torch.randn(64, 512, generator=g).to(dev)
    ref.backward(dy)
    dx = torch.empty(64, 512, dtype=bf16, device=dev)
    ops.l2norm_bwd(dy, y, inv, dx)
    assert rel(dx, xr.grad) < 4e-3
    m = torch.randn(3000, 776, generator=g).to(dev).to(bf16)
    out = torch.zeros(776, device=dev)
    ops.colsum(m, out)
    assert rel(out, m.float().sum(0)) < 1e-4
    src = torch.randn(1003, generator=g).to(dev)
    dst = torch.empty(1003 + 5, dtype=bf16, device=dev)
    ops.cast_bf16(src, dst)
    assert torch.equal(dst[:1003], src.to(bf16))


# ------------------------------------------------------------------------------------------ embeddings
def test_uint8_frames_preprocessing_bit_exact_vs_reference_transform(dev):
    """SURVEY.md §8f.4: decoder frames uint8 [B, T, H, W, 3] -> the reference's `.permute(0,3,1,2).float() / 255.`
    (dataset_pretrain_stage1_all_source.py:182) + torchvision Normalize(mean, std) (dataloader.py:209-233; Resize / CenterCrop to
    the same 224 x 224 are the identity) -> im2col.  Integer input, IEEE fp32 arithmetic, one rounding: bit-exact."""
    from xpretrain_b200 import ops
    B, T, H, W = 2, 3, 224, 224
    g = torch.Generator().manual_seed(12)
    frames = torch.randint(0, 256, (B, T, H, W, 3), dtype=torch.uint8, generator=g)
    frames[0, 0, :2] = 255
    frames[0, 0, 2:4] = 0
    mean = torch.tensor(ops.CLIP_MEAN, dtype=torch.float32)
    std = torch.tensor(ops.CLIP_STD, dtype=torch.float32)
    img = frames.reshape(B * T, H, W, 3).permute(0, 3, 1, 2).float() / 255.                   # reference line 182
    img = img.clone().sub_(mean[:, None, None]).div_(std[:, None, None])                      # torchvision F.normalize
    ref_p = img.reshape(B * T, 3, 14, 16, 14, 16).permute(0, 2, 4, 1, 3, 5).reshape(B * T * 196, 768).to(bf16)
    patches = torch.empty(B * T * 196, 768, dtype=bf16, device=dev)
    ops.vip_patchify_u8(frames.to(dev), patches, 16)
    assert torch.equal(patches.cpu(), ref_p)
    # and the model accepts the raw frames: same features as feeding the reference-transformed float video
    from clipvip_cases import b16, vidclip
    model = vidclip(b16(1, 1), seed=0, dev=dev)
    with torch.no_grad():
        a = model.forward_video(frames.to(dev))
        b = model.forward_video(img.reshape(B, T, 3, H, W).to(dev))
    assert torch.equal(a, b)


@pytest.mark.parametrize("C", [768, 512])
@pytest.mark.parametrize("x_f32", [True, False])
def test_layernorm_with_fp32_residual_add_and_bias_colsum(dev, C, x_f32):
    """`hidden = residual + branch; hidden = layer_norm(hidden)` (CLIP_ViP.py:445-460) in one kernel with the sum kept in fp32,
    and its backward with an fp32 saved input + the residual-branch column sum (the closing Linear's bias gradient)."""
    from xpretrain_b200 import ops
    rows, eps = 517, 1e-5
    g = torch.Generator().manual_seed(C)
    x = (torch.randn(rows, C, generator=g) * 2).to(dev)
    x = x if x_f32 else x.to(bf16)
    add = torch.randn(rows, C, generator=g).to(dev).to(bf16)
    gamma, beta = (1 + 0.1 * torch.randn(C, generator=g)).to(dev), (0.1 * torch.randn(C, generator=g)).to(dev)
    y = torch.empty(rows, C, dtype=bf16, device=dev)
    s_out = torch.empty(rows, C, device=dev)
    mean, rstd = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
    m = ops.rowmap(C)
    ops.layernorm_fwd(x, m, y, m, gamma, beta, mean, rstd, rows, C, eps, add=add, addmap=m, sum_out=s_out, summap=m)
    want_s = x.float() + add.float()
    assert torch.equal(s_out, want_s)                                               # one fp32 add: exact
    sr = want_s.clone().requires_grad_(True)
    want_y = F.layer_norm(sr, (C,), gamma, beta, eps)
    assert rel(y, want_y.detach()) < 4e-3
    y32 = torch.empty(rows, C, device=dev)                                          # fp32 output (pre_layrnorm -> stream)
    ops.layernorm_fwd(x, m, y32, m, gamma, beta, None, None, rows, C, eps)
    assert rel(y32, F.layer_norm(x.float(), (C,), gamma, beta, eps)) < 1e-5
    dy = torch.randn(rows, C, generator=g).to(dev).to(bf16)
    dres = torch.randn(rows, C, generator=g).to(dev).to(bf16)
    want_y.backward(dy.float())
    dx = torch.empty(rows, C, dtype=bf16, device=dev)
    dg, db, dsum = torch.zeros(C, device=dev), torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    ops.layernorm_bwd(dy, m, s_out, m, gamma, mean, rstd, dres, m, dx, m, dg, db, rows, C, dres_colsum=dsum)
    assert rel(dx, sr.grad + dres.float()) < 4e-3
    assert rel(dsum, dres.float().sum(0)) < 1e-5
    assert rel(db, dy.float().sum(0)) < 1e-5 and rel(dg, (dy.float() * ((want_s - want_s.mean(-1, keepdim=True)) * rstd[:, None])).sum(0)) < 1e-4


def test_layernorm_with_fp16_residual_stream(dev):
    """`residual_dtype="fp16"` (the reference's own training precision under apex O2): x fp16 + bf16 branch -> fp32 sum inside the
    kernel, stored as saturating fp16; the normalisation uses exactly the stored values; backward reads the fp16 input."""
    from xpretrain_b200 import ops
    rows, C, eps = 333, 768, 1e-5
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(rows, C, generator=g) * 3).to(dev).half()
    x[0, 0] = 65000.0                                                               # x + add would overflow fp16: must saturate
    add = torch.randn(rows, C, generator=g).to(dev).to(bf16)
    add[0, 0] = 2000.0
    gamma, beta = (1 + 0.1 * torch.randn(C, generator=g)).to(dev), (0.1 * torch.randn(C, generator=g)).to(dev)
    y = torch.empty(rows, C, dtype=bf16, device=dev)
    s_out = torch.empty(rows, C, dtype=torch.float16, device=dev)
    mean, rstd = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
    m = ops.rowmap(C)
    ops.layernorm_fwd(x, m, y, m, gamma, beta, mean, rstd, rows, C, eps, add=add, addmap=m, sum_out=s_out, summap=m)
    want_s = (x.float() + add.float()).clamp(-65504, 65504).half()
    assert torch.equal(s_out, want_s) and float(s_out[0, 0]) == 65504.0
    sr = want_s.float().requires_grad_(True)
    want_y = F.layer_norm(sr, (C,), gamma, beta, eps)
    assert rel(y[1:], want_y.detach()[1:]) < 4e-3
    dy = torch.randn(rows, C, generator=g).to(dev).to(bf16)
    want_y.backward(dy.float())
    dx = torch.empty(rows, C, dtype=bf16, device=dev)
    dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    ops.layernorm_bwd(dy, m, s_out, m, gamma, mean, rstd, None, None, dx, m, dg, db, rows, C)
    assert rel(dx[1:], sr.grad[1:]) < 4e-3
    yh = torch.empty(rows, C, dtype=torch.float16, device=dev)                      # fp16 output (pre_layrnorm -> stream)
    ops.layernorm_fwd(y, m, yh, m, gamma, beta, None, None, rows, C, eps)
    assert rel(yh, F.layer_norm(y.float(), (C,), gamma, beta, eps)) < 1e-3


def test_patchify_and_embed_tables(dev):
    from oracle import clipvip_oracle as O
    from xpretrain_b200 import ops
    cfg = O.ClipVipCfg()
    B, T = 2, 5                                 # T != temporal_size -> linear interpolation of the table
    sd = O.init_state_dict(O.ClipVipCfg(vision=O.TowerCfg(768, 12, 1, 3072), text=O.TowerCfg(512, 8, 1, 2048)), seed=3)
    video = torch.randn(B, T, 3, 224, 224, generator=torch.Generator().manual_seed(4))
    want, (M, _, L) = O.vip_embeddings(sd, video, cfg)
    C, Kp, S = 768, 768, M + T * L
    vd = video.to(dev)
    patches = torch.empty(B * T * L, Kp, dtype=bf16, device=dev)
    ops.vip_patchify(vd, patches, 16)
    ref_p = video.reshape(B * T, 3, 14, 16, 14, 16).permute(0, 2, 4, 1, 3, 5).reshape(B * T * L, Kp)
    assert torch.equal(patches.cpu(), ref_p.to(bf16))        # pure indexing: bit-exact
    pre = "vision_model.embeddings."
    table = torch.empty(T * L, C, dtype=bf16, device=dev)
    x0 = torch.zeros(B * S, C, dtype=bf16, device=dev)
    ops.vip_embed_tables(sd[pre + "position_embedding.weight"].to(dev), sd[pre + "temporal_embedding"].to(dev),
                         sd[pre + "class_embedding"].to(dev), sd[pre + "added_cls"].to(dev), table, x0, B, T, L, M, C, 12)
    w = sd[pre + "patch_embedding.weight"].reshape(C, Kp).to(dev).to(bf16)
    ops.gemm(patches, w, x0, M=B * T * L, N=C, K=Kp, lda=Kp, ldb=Kp, ldc=C, residual=table, ldr=C, r_group=T * L,
             c_group=T * L, c_group_stride=S * C, c_offset=M * C)
    assert rel(x0.view(B, S, C).cpu(), want) < 6e-3
    assert rel(x0.view(B, S, C)[:, :M].cpu(), want[:, :M]) < 3e-3


def test_embed_backward(dev):
    from xpretrain_b200 import ops
    B, T, L, M, C, Tsz = 3, 5, 7, 4, 64, 12
    g = torch.Generator(device="cpu").manual_seed(8)
    dpatch = torch.randn(B, T * L, C, generator=g).to(bf16)
    dglob = torch.randn(B, M, C, generator=g).to(bf16)
    pos = torch.zeros(L + 1, C, requires_grad=True); temporal = torch.zeros(1, Tsz, C, requires_grad=True)
    cls = torch.zeros(C, requires_grad=True); added = torch.zeros(M - 1, C, requires_grad=True)
    tt = F.interpolate(temporal.transpose(1, 2), size=T, mode="linear").transpose(1, 2)
    emb_p = (tt.unsqueeze(2) + pos[1:].unsqueeze(0).unsqueeze(0)).expand(B, T, L, C).reshape(B, T * L, C)
    emb_g = torch.cat([(cls + pos[0]).expand(B, 1, C), (added + pos[0]).unsqueeze(0).expand(B, M - 1, C)], 1)
    ((emb_p * dpatch.float()).sum() + (emb_g * dglob.float()).sum()).backward()
    d_pos = torch.zeros(L + 1, C, device=dev); d_t = torch.zeros(Tsz, C, device=dev)
    d_cls = torch.zeros(C, device=dev); d_add = torch.zeros(M - 1, C, device=dev)
    ops.vip_embed_bwd(dpatch.to(dev), dglob.to(dev), d_pos, d_t, d_cls, d_add, B, T, L, M, C, Tsz)
    assert rel(d_pos.cpu(), pos.grad) < 1e-5 and rel(d_t.cpu(), temporal.grad[0]) < 1e-5
    assert rel(d_cls.cpu(), cls.grad) < 1e-5 and rel(d_add.cpu(), added.grad) < 1e-5


def test_text_embeddings(dev):
    from xpretrain_b200 import ops
    V, C, B, Lt = 1000, 512, 4, 32
    g = torch.Generator(device="cpu").manual_seed(9)
    tok = torch.randn(V, C, generator=g).to(dev); pos = torch.randn(77, C, generator=g).to(dev)
    ids = torch.randint(0, V, (B, Lt), generator=g).to(dev)
    x = torch.empty(B * Lt, C, dtype=bf16, device=dev); err = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.text_embed_fwd(ids, tok, pos, x, Lt, err)
    assert torch.equal(x.view(B, Lt, C), (tok[ids] + pos[:Lt]).to(bf16)) and int(err) == 0
    dx = torch.randn(B * Lt, C, generator=g).to(dev).to(bf16)
    d_tok = torch.zeros(V, C, device=dev); d_pos = torch.zeros(77, C, device=dev)
    ops.text_embed_bwd(ids, dx, d_tok, d_pos, Lt, C, V)
    ref = torch.zeros(V, C, device=dev).index_add_(0, ids.reshape(-1), dx.float())
    assert rel(d_tok, ref) < 1e-5 and rel(d_pos[:Lt], dx.float().view(B, Lt, C).sum(0)) < 1e-5
    bad = ids.clone(); bad[0, 0] = V + 3
    ops.text_embed_fwd(bad, tok, pos, x, Lt, err)
    assert int(err) == 1


# ------------------------------------------------------------------------------------------- attention
def _vip_ref(qkv, B, H, T, L, M, C):
    """Block-masked dense attention in fp32 (== CLIPAttention.forward2, SURVEY Appendix A)."""
    S = M + T * L
    q, k, v = [t.reshape(B, S, H, 64).transpose(1, 2) for t in qkv.float().reshape(B, S, 3, C).unbind(2)]
    frame = torch.cat([torch.full((M,), -1), torch.arange(T).repeat_interleave(L)]).to(qkv.device)
    allow = (frame[:, None] < 0) | (frame[None, :] < 0) | (frame[:, None] == frame[None, :])
    s = (q @ k.transpose(-1, -2)).masked_fill(~allow, float("-inf"))
    o = torch.softmax(s, -1) @ v
    return o.transpose(1, 2).reshape(B * S, C), torch.logsumexp(s, -1)


@pytest.mark.parametrize("B,H,T,L,M", [(2, 2, 3, 196, 4), (1, 12, 2, 196, 4), (2, 1, 4, 20, 2), (1, 2, 1, 196, 4),
                                       (3, 12, 12, 196, 4),      # 432 items: every persistent CTA pipelines across several items
                                       (2, 3, 5, 130, 1), (2, 2, 3, 128, 8), (2, 2, 2, 100, 3)])
def test_vip_attention_fwd_bwd(dev, B, H, T, L, M):
    from xpretrain_b200 import ops
    C, S = 64 * H, M + T * L
    g = torch.Generator(device="cpu").manual_seed(B * 100 + T)
    qkv = (torch.randn(B * S, 3 * C, generator=g) * 0.8).to(dev).to(bf16)
    qkv[:, :C] *= 0.35                                # q is pre-scaled in the real pipeline
    out = torch.empty(B * S, C, dtype=bf16, device=dev)
    lse = torch.empty(B, H, S, device=dev)
    ws = ops.vip_attention_workspace(B, H, T, M, dev)
    ops.vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C)
    qr = qkv.float().requires_grad_(True)
    ref, ref_lse = _vip_ref(qr, B, H, T, L, M, C)
    assert rel(out, ref.detach()) < 6e-3
    assert float((lse - ref_lse.detach()).abs().max()) < 2e-2
    dout = torch.randn(B * S, C, generator=g).to(dev).to(bf16)
    ref.backward(dout.float())
    dqkv = torch.empty(B * S, 3 * C, dtype=bf16, device=dev)
    ops.vip_attention_bwd(qkv, out, dout, lse, dqkv, ws, B, H, T, L, M, C, 1.0)
    for name, sl in (("dq", slice(0, C)), ("dk", slice(C, 2 * C)), ("dv", slice(2 * C, 3 * C))):
        assert rel(dqkv[:, sl], qr.grad[:, sl]) < 2e-2, name
        assert rel(dqkv.view(B, S, 3 * C)[:, :M, sl], qr.grad.view(B, S, 3 * C)[:, :M, sl]) < 2e-2, (name, "global rows")


def test_vip_attention_forward_rescales_when_later_keys_dominate(dev):
    """Softmax range stress: keys whose logits grow along the sequence by far more than e^8 per 16-key chunk (the row maximum
    sits in the last chunk, so the online softmax has to rescale at every key block), for frame and for global queries."""
    from xpretrain_b200 import ops
    B, H, T, L, M = 1, 2, 2, 196, 4
    C, S = 64 * H, M + T * L
    g = torch.Generator(device="cpu").manual_seed(17)
    qkv = torch.randn(B * S, 3 * C, generator=g) * 0.5
    ramp = torch.cat([torch.linspace(4.0, 6.0, M), torch.linspace(0.2, 12.0, L).repeat(T)])     # per key row
    base = torch.randn(1, C, generator=g).sign()                                              # a common direction: q.k grows with the ramp
    qkv[:, :C] = 0.35 * (base + 0.1 * torch.randn(B * S, C, generator=g))
    qkv[:, C:2 * C] = ramp[:, None] * (base + 0.05 * torch.randn(B * S, C, generator=g))
    qkv = qkv.to(dev).to(bf16)
    ref, ref_lse = _vip_ref(qkv.float(), B, H, T, L, M, C)
    s_ref = (qkv.float()[:, :C].reshape(B, S, H, 64).transpose(1, 2) @ qkv.float()[:, C:2 * C].reshape(B, S, H, 64).transpose(1, 2).transpose(-1, -2))
    assert float(s_ref.max() - s_ref.min()) > 100                                              # the logits really span > e^8 many times
    out = torch.zeros(B * S, C, dtype=bf16, device=dev)
    lse = torch.zeros(B, H, S, device=dev)
    ws = ops.vip_attention_workspace(B, H, T, M, dev)
    ops.vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C)
    assert rel(out, ref) < 8e-3
    assert float(((lse - ref_lse).abs() / ref_lse.abs().clamp_min(1.0)).max()) < 1e-3


@pytest.mark.parametrize("Lt", [32, 77, 5])
def test_text_attention_fwd_bwd(dev, Lt):
    from oracle import clipvip_oracle as O
    from xpretrain_b200 import ops
    B, H = 3, 8
    C = 64 * H
    g = torch.Generator(device="cpu").manual_seed(Lt)
    qkv = (torch.randn(B * Lt, 3 * C, generator=g) * 0.7).to(dev).to(bf16)
    qkv[:, :C] *= 0.35
    mask = torch.ones(B, Lt, dtype=torch.int64)
    mask[1, Lt // 2:] = 0
    mask[2, 0] = 0                                    # even the first key padded: rows become uniform over causal keys
    mask = mask.to(dev)
    out = torch.empty(B * Lt, C, dtype=bf16, device=dev)
    probs = torch.empty(B, H, Lt, Lt, device=dev)
    ops.text_attention_fwd(qkv, mask, out, probs, B, H, Lt, C)
    qr = qkv.float().requires_grad_(True)
    q, k, v = [t.reshape(B, Lt, H, 64).transpose(1, 2) for t in qr.reshape(B, Lt, 3, C).unbind(2)]
    add = O.text_additive_mask(mask.cpu(), torch.float32).to(dev)
    p = torch.softmax(q @ k.transpose(-1, -2) + add, -1)
    ref = (p @ v).transpose(1, 2).reshape(B * Lt, C)
    assert rel(probs, p.detach()) < 1e-4
    assert rel(out, ref.detach()) < 5e-3
    dout = torch.randn(B * Lt, C, generator=g).to(dev).to(bf16)
    ref.backward(dout.float())
    dqkv = torch.empty(B * Lt, 3 * C, dtype=bf16, device=dev)
    ops.text_attention_bwd(qkv, dout, probs, dqkv, B, H, Lt, C, 1.0)
    assert rel(dqkv, qr.grad) < 6e-3


# ------------------------------------------------------------------------------------------------ NCE
@pytest.mark.parametrize("world,b", [(4, 8), (8, 64), (3, 50), (8, 192), (2, 3)])
def test_fused_gather_nce_kernel_rank_major_rows_and_unfused_path(dev, world, b, golden_dir):
    """csrc/nce_fused.cu in pre-gathered mode on one GPU: `world` per-rank [b, d] blocks living in separate allocations are
    read through the pointer table in rank-major order (hvd.allgather's concat order, run_pretrain.py:344-345).  Checked
    against the reference-class golden (world 4 x 8), the oracle, and the unfused multi-launch path on the same rows."""
    from oracle import clipvip_oracle as O
    from xpretrain_b200 import ops
    from xpretrain_b200.optimization import loss as XL
    d, N = 512, world * b
    if (world, b) == (4, 8):
        gold = torch.load(os.path.join(golden_dir, "nce_loss_w4.pt"), weights_only=False)
        vis, txt, temp = gold["vis_per_rank"], gold["txt_per_rank"], gold["logit_scale"]
    else:
        g = torch.Generator(device="cpu").manual_seed(N)
        vis = [F.normalize(torch.randn(b, d, generator=g), dim=-1) for _ in range(world)]
        txt = [F.normalize(torch.randn(b, d, generator=g) + 0.5 * v, dim=-1) for v in vis]
        temp = torch.tensor(4.6)
    V, T = O.gather_rank_major(vis), O.gather_rank_major(txt)
    dv, dt, dl = O.nce_closed_form_grads(V, T, temp)
    want = float(O.nce_learnable_temp_loss(V, T, temp))
    if (world, b) == (4, 8):
        assert abs(want - float(gold["loss"])) < 1e-6 and rel(dv, gold["d_vis"]) < 1e-5
    dvis = [x.to(dev) for x in vis]
    dtxt = [x.to(dev) for x in txt]
    ptrs = torch.tensor([x.data_ptr() for x in dvis] + [x.data_ptr() for x in dtxt], dtype=torch.int64, device=dev)
    Np = (N + 7) // 8 * 8
    gmat = torch.zeros(N, Np, dtype=bf16, device=dev)
    vh, th = torch.empty(N, d, dtype=bf16, device=dev), torch.empty(N, d, dtype=bf16, device=dev)
    loss, dscale = torch.empty(1, device=dev), torch.empty(1, device=dev)
    ws = ops.nce_gather_workspace(N, dev)
    tdev = temp.reshape(1).to(dev)
    for _ in range(2):           # twice: the kernel must leave its barrier counters reset
        ops.nce_gather_fused(None, None, ptrs, tdev, gmat, vh, th, loss, dscale, ws, rank=0, world=world, b=b, d=d, epoch=0,
                             mode=1)
    torch.cuda.synchronize()
    s = float(temp.exp())
    P = torch.softmax(s * V @ T.t(), 1) + torch.softmax(s * V @ T.t(), 0) - 2 * torch.eye(N)
    assert abs(float(loss) - want) < 2e-5 * max(1.0, abs(want))                     # fp32-grade logits (hi/lo split)
    assert abs(float(dscale) - float(dl)) < 1e-3 * max(1.0, abs(float(dl)))
    assert rel(gmat[:, :N].float().cpu(), s * P / N) < 5e-3                          # bf16 storage of G
    assert torch.equal(vh.cpu(), V.to(bf16)) and torch.equal(th.cpu(), T.to(bf16))   # rank-major rows, bit-exact
    # the unfused path on the same gathered rows
    l2, g2, _, _, ds2 = XL._nce_forward_unfused(V.to(dev), T.to(dev), temp.to(dev))
    assert abs(float(l2) - float(loss)) < 2e-5 * max(1.0, abs(want)) and rel(g2[:, :N].float(), gmat[:, :N].float()) < 5e-3
    d_vis, d_txt = XL._nce_backward(gmat, vh, th, 0, N, 1.0)
    assert rel(d_vis.cpu(), dv) < 6e-3 and rel(d_txt.cpu(), dt) < 6e-3


@pytest.mark.parametrize("N", [8, 64, 512, 6])
def test_nce_loss_and_grads(dev, N):
    from oracle import clipvip_oracle as O
    from xpretrain_b200.optimization.loss import NCELearnableTempLoss
    g = torch.Generator(device="cpu").manual_seed(N)
    v = F.normalize(torch.randn(N, 512, generator=g), dim=-1)
    t = F.normalize(torch.randn(N, 512, generator=g) + 0.5 * v, dim=-1)
    temp = torch.tensor(4.6)
    vr, tr, pr = v.clone().requires_grad_(True), t.clone().requires_grad_(True), temp.clone().requires_grad_(True)
    want = O.nce_learnable_temp_loss(vr, tr, pr)
    want.backward()
    vd, td, pd = (x.to(dev).requires_grad_(True) for x in (v, t, temp))
    got = NCELearnableTempLoss(None)(vd, td, pd)
    got.backward()
    assert abs(float(got) - float(want)) < 2e-4 * max(1.0, abs(float(want)))
    assert rel(vd.grad.cpu(), vr.grad) < 6e-3 and rel(td.grad.cpu(), tr.grad) < 6e-3
    assert abs(float(pd.grad) - float(pr.grad)) < 2e-3 * max(1.0, abs(float(pr.grad)))


@pytest.mark.parametrize("N", [24, 512, 20])
def test_nce_vsc_fc_loss_and_grads(dev, N, golden_dir):
    """The released pre-training default loss (loss.py:288-324): six-term video/subtitle/caption/frame InfoNCE."""
    import os

    from oracle import clipvip_oracle as O
    from xpretrain_b200.optimization import build_loss_func
    if N == 24:      # the fixture written from the reference's own class and autograd
        gold = torch.load(os.path.join(golden_dir, "nce_vsc_fc_n24.pt"), weights_only=False)
        feats, temp = [gold[k] for k in ("vis", "txt", "img", "cap")], gold["logit_scale"]
        want_loss, want_grads = gold["loss"], [gold[k] for k in ("d_vis", "d_txt", "d_img", "d_cap")]
        want_dscale = gold["d_logit_scale"]
    else:
        g = torch.Generator(device="cpu").manual_seed(N)
        base = F.normalize(torch.randn(N, 512, generator=g), dim=-1)
        feats = [F.normalize(torch.randn(N, 512, generator=g) + 0.5 * base, dim=-1) for _ in range(4)]
        temp = torch.tensor(4.6)
        fr = [f.clone().requires_grad_(True) for f in feats]
        pr = temp.clone().requires_grad_(True)
        want_loss = O.nce_vsc_fc_loss(*fr, pr)
        want_loss.backward()
        want_grads, want_dscale = [f.grad for f in fr], pr.grad
    fd = [f.to(dev).requires_grad_(True) for f in feats]
    pd = temp.to(dev).requires_grad_(True)
    loss_fn = build_loss_func({"loss_name": "NCELearnableTempLoss_vsc_fc"})
    got = loss_fn(*fd, pd)
    got.backward()
    assert abs(float(got) - float(want_loss)) < 2e-4 * max(1.0, abs(float(want_loss)))
    for a, b in zip(fd, want_grads):
        assert rel(a.grad.cpu(), b) < 6e-3
    assert abs(float(pd.grad) - float(want_dscale)) < 2e-3 * max(1.0, abs(float(want_dscale)))
