"""H100: the kernels behind ViT-L/14 towers.  Proxy-token attention for frames of M + L > 208 rows (the streamed kernels)
against a block-masked fp32 reference, and the patch extraction for patch sizes that are not multiples of 8."""
import pytest
import torch

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20))


def _vip_ref(qkv, B, H, T, L, M, C):
    """Block-masked dense attention in fp32 (CLIPAttention.forward2): patch queries of frame t see the M global keys and
    the L keys of frame t; the M global queries see every key."""
    S = M + T * L
    q, k, v = [t.reshape(B, S, H, 64).transpose(1, 2) for t in qkv.float().reshape(B, S, 3, C).unbind(2)]
    frame = torch.cat([torch.full((M,), -1), torch.arange(T).repeat_interleave(L)]).to(qkv.device)
    allow = (frame[:, None] < 0) | (frame[None, :] < 0) | (frame[:, None] == frame[None, :])
    s = (q @ k.transpose(-1, -2)).masked_fill(~allow, float("-inf"))
    o = torch.softmax(s, -1) @ v
    return o.transpose(1, 2).reshape(B * S, C), torch.logsumexp(s, -1)


def _inputs(B, H, T, L, M, seed, dev):
    C, S = 64 * H, M + T * L
    g = torch.Generator(device="cpu").manual_seed(seed)
    qkv = (torch.randn(B * S, 3 * C, generator=g) * 0.8)
    qkv[:, :C] *= 0.35                                # q is pre-scaled in the real pipeline
    dout = torch.randn(B * S, C, generator=g)
    return qkv.to(dev).to(bf16), dout.to(dev).to(bf16)


def _run(qkv, dout, B, H, T, L, M):
    from xpretrain_b200 import ops
    C, S = 64 * H, M + T * L
    dev = qkv.device
    out = torch.empty(B * S, C, dtype=bf16, device=dev)
    lse = torch.empty(B, H, S, device=dev)
    ws = ops.vip_attention_workspace(B, H, T, M, dev)
    ops.vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C)
    dqkv = torch.empty(B * S, 3 * C, dtype=bf16, device=dev)
    ops.vip_attention_bwd(qkv, out, dout, lse, dqkv, ws, B, H, T, L, M, C, 1.0)
    return out, lse, dqkv


@pytest.mark.parametrize("B,H,T,L,M", [
    (2, 2, 3, 205, 4),        # M + L = 209: the first size past the staged kernel
    (2, 2, 2, 201, 8),        # M + L = 209 with the most global tokens
    (2, 3, 3, 300, 3),        # ragged last key block
    (2, 16, 2, 256, 4),       # ViT-L/14 at 224 px, 16 heads
    (3, 2, 1, 576, 4),        # ViT-L/14 at 336 px, image branch (T = 1)
    (1, 2, 2, 1024, 1),       # ViT-L/14 at 448 px
    (4, 16, 12, 256, 4),      # a full-size grid
])
def test_long_frame_attention_fwd_bwd(dev, B, H, T, L, M):
    C, S = 64 * H, M + T * L
    qkv, dout = _inputs(B, H, T, L, M, B * 1000 + L + M, dev)
    out, lse, dqkv = _run(qkv, dout, B, H, T, L, M)
    qr = qkv.float().requires_grad_(True)
    ref, ref_lse = _vip_ref(qr, B, H, T, L, M, C)
    assert rel(out, ref.detach()) < 6e-3
    assert rel(out.view(B, S, C)[:, :M], ref.detach().view(B, S, C)[:, :M]) < 6e-3, "global rows"
    assert float((lse - ref_lse.detach()).abs().max()) < 2e-2
    ref.backward(dout.float())
    for name, sl in (("dq", slice(0, C)), ("dk", slice(C, 2 * C)), ("dv", slice(2 * C, 3 * C))):
        assert rel(dqkv[:, sl], qr.grad[:, sl]) < 2e-2, name
        assert rel(dqkv.view(B, S, 3 * C)[:, :M, sl], qr.grad.view(B, S, 3 * C)[:, :M, sl]) < 2e-2, (name, "global rows")


def test_long_frame_attention_is_deterministic(dev):
    """No float atomics and one writer per partial: two calls give bitwise-equal out, lse and dqkv."""
    B, H, T, L, M = 3, 4, 5, 256, 4
    qkv, dout = _inputs(B, H, T, L, M, 77, dev)
    a = _run(qkv, dout, B, H, T, L, M)
    b = _run(qkv, dout, B, H, T, L, M)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_long_frame_attention_rescales_when_later_keys_dominate(dev):
    """Logits growing along the frame by far more than e^8 per key block: the online softmax rescales at every streamed
    block, for frame and for global queries."""
    from xpretrain_b200 import ops
    B, H, T, L, M = 1, 2, 2, 576, 4
    C, S = 64 * H, M + T * L
    g = torch.Generator(device="cpu").manual_seed(17)
    qkv = torch.randn(B * S, 3 * C, generator=g) * 0.5
    ramp = torch.cat([torch.linspace(4.0, 6.0, M), torch.linspace(0.2, 12.0, L).repeat(T)])
    base = torch.randn(1, C, generator=g).sign()
    qkv[:, :C] = 0.35 * (base + 0.1 * torch.randn(B * S, C, generator=g))
    qkv[:, C:2 * C] = ramp[:, None] * (base + 0.05 * torch.randn(B * S, C, generator=g))
    qkv = qkv.to(dev).to(bf16)
    ref, ref_lse = _vip_ref(qkv.float(), B, H, T, L, M, C)
    out = torch.zeros(B * S, C, dtype=bf16, device=dev)
    lse = torch.zeros(B, H, S, device=dev)
    ws = ops.vip_attention_workspace(B, H, T, M, dev)
    ops.vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C)
    assert rel(out, ref) < 8e-3
    assert float(((lse - ref_lse).abs() / ref_lse.abs().clamp_min(1.0)).max()) < 1e-3


# ------------------------------------------------------------------------------------------- patch extraction
def _unfold_ref(video, p):
    """[F, 3, H, W] -> [F * (H/p) * (W/p), 3 p^2] in Conv2d weight order (c, kh, kw)."""
    Fr, _, H, W = video.shape
    x = video.reshape(Fr, 3, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5)
    return x.reshape(Fr * (H // p) * (W // p), 3 * p * p)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("size", [224, 336])
def test_patchify_patch14_bit_exact(dev, dtype, size):
    from xpretrain_b200 import ops
    p, B, T = 14, 2, 3
    ld = ops.patch_pitch(p)
    assert ld == 592
    video = torch.randn(B, T, 3, size, size, generator=torch.Generator().manual_seed(size)).to(dtype)
    n = B * T * (size // p) ** 2
    patches = torch.full((n, ld), float("nan"), dtype=bf16, device=dev)
    ops.vip_patchify(video.to(dev), patches, p)
    got = patches.cpu()
    assert torch.equal(got[:, :588], _unfold_ref(video.reshape(B * T, 3, size, size), p).float().to(bf16))
    assert torch.equal(got[:, 588:], torch.zeros(n, ld - 588, dtype=bf16))


def test_patchify_u8_patch14_bit_exact_vs_reference_transform(dev):
    from xpretrain_b200 import ops
    p, B, T, H, W = 14, 2, 2, 224, 224
    g = torch.Generator().manual_seed(12)
    frames = torch.randint(0, 256, (B, T, H, W, 3), dtype=torch.uint8, generator=g)
    frames[0, 0, :2] = 255
    frames[0, 0, 2:4] = 0
    mean = torch.tensor(ops.CLIP_MEAN, dtype=torch.float32)
    std = torch.tensor(ops.CLIP_STD, dtype=torch.float32)
    img = frames.reshape(B * T, H, W, 3).permute(0, 3, 1, 2).float() / 255.
    img = img.clone().sub_(mean[:, None, None]).div_(std[:, None, None])
    n = B * T * (H // p) ** 2
    patches = torch.full((n, 592), float("nan"), dtype=bf16, device=dev)
    ops.vip_patchify_u8(frames.to(dev), patches, p)
    got = patches.cpu()
    assert torch.equal(got[:, :588], _unfold_ref(img, p).to(bf16))
    assert torch.equal(got[:, 588:], torch.zeros(n, 4, dtype=bf16))
