"""H100: the persistent GEMM's results do not depend on how its tiles are spread over CTAs and consumer warpgroups.

Every output mode, layout pair and epilogue runs at a ragged shape (M not a multiple of 128, N a multiple of 8 but not
of 128, more k-blocks than ring stages) under several grid caps, so that CTAs run odd and even numbers of tiles and
both consumer warpgroups of a CTA own several of them.  Non-atomic outputs must be bit-identical across grid sizes."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
SM_LIMITS = (1, 2, 3, 7, 0)  # 0: one CTA per SM


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20))


def _per_sm_limit(run):
    """run() under every grid cap of SM_LIMITS; the cap is restored afterwards."""
    from xpretrain_b200 import ops
    outs = []
    try:
        for n in SM_LIMITS:
            ops.set_sm_limit(n)
            outs.append(run())
            torch.cuda.synchronize()
    finally:
        ops.set_sm_limit(0)
    return outs


M, N, K = 1000, 392, 520   # 8 x 4 tiles of 128 x 128, 9 k-blocks of 64


def _operands(dev, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(dev).to(bf16)
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dev).to(bf16)
    b = torch.randn(N, generator=g).to(dev)
    x = torch.randn(M, N, generator=g).to(dev).to(bf16)   # residual or saved pre-activation
    return a, w, b, x


def _gemm(a, w, out, a_layout, b_layout, **kw):
    """out = epilogue(a @ w^T) with a [M, K] and w [N, K] handed to the kernel K-major (layout 0) or MN-major (1)."""
    from xpretrain_b200 import ops
    A = a if a_layout == 0 else a.t().contiguous()
    B = w if b_layout == 0 else w.t().contiguous()
    ops.gemm(A, B, out, M=M, N=N, K=K, lda=A.stride(0), ldb=B.stride(0), ldc=out.stride(0), a_layout=a_layout,
             b_layout=b_layout, **kw)


EPILOGUES = ["plain", "bias_qscale_residual", "quick_gelu", "gelu_erf", "dquick_gelu", "dgelu_erf", "f32", "grouped"]


@pytest.mark.parametrize("block_n", [128, 256])   # ping-pong 128 x 128 tiles, cooperative 128 x 256 tiles
@pytest.mark.parametrize("a_layout,b_layout", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("epi", EPILOGUES)
def test_gemm_bit_identical_across_grid_sizes(dev, epi, a_layout, b_layout, block_n):
    from xpretrain_b200 import _lib
    a, w, b, x = _operands(dev, 7 + EPILOGUES.index(epi))
    ref = a.float() @ w.float().t()
    sc = 128   # q-scale columns
    kw, want, tol = {"block_n": block_n}, None, 4e-3
    if epi == "plain":
        want = ref
    elif epi == "bias_qscale_residual":
        kw.update(bias=b, scale_cols=sc, col_scale=0.125, residual=x, ldr=N)
        want = ref + b
        want[:, :sc] *= 0.125
        want = want + x.float()
    elif epi in ("quick_gelu", "gelu_erf"):
        kw.update(bias=b, act=_lib.ACT_QUICK_GELU if epi == "quick_gelu" else _lib.ACT_GELU_ERF)
        pre_ref = ref + b
        want = (pre_ref * torch.sigmoid(1.702 * pre_ref) if epi == "quick_gelu"
                else torch.nn.functional.gelu(pre_ref))
        tol = 6e-3
    elif epi in ("dquick_gelu", "dgelu_erf"):
        kw.update(aux=x, ld_aux=N, act=_lib.ACT_DQUICK_GELU if epi == "dquick_gelu" else _lib.ACT_DGELU_ERF)
        p = x.float()
        if epi == "dquick_gelu":
            s = torch.sigmoid(1.702 * p)
            want = ref * (s * (1 + 1.702 * p * (1 - s)))
        else:
            want = ref * (0.5 * (1 + torch.erf(p / math.sqrt(2))) + p * torch.exp(-0.5 * p * p) / math.sqrt(2 * math.pi))
        tol = 6e-3
    elif epi == "f32":
        kw.update(bias=b, out_mode=_lib.OUT_F32)
        want, tol = ref + b, 1e-5
    if epi == "grouped":
        # rows scattered in groups of 100 with a 3-row gap, plus a periodic residual table of 100 rows
        G, gap = 100, 3
        table = x[:G].contiguous()
        kw.update(residual=table, ldr=N, r_group=G, r_group_stride=0, c_group=G, c_group_stride=(G + gap) * N)
        full = (ref.view(M // G, G, N) + table.float()).view(M, N)

        def run():
            out = torch.full(((M // G) * (G + gap), N), 7.0, dtype=bf16, device=dev)
            _gemm(a, w, out, a_layout, b_layout, **kw)
            return out
    else:
        def run():
            out = torch.empty(M, N, dtype=f32 if epi == "f32" else bf16, device=dev)
            aux = torch.empty(M, N, dtype=bf16, device=dev) if epi in ("quick_gelu", "gelu_erf") else None
            extra = dict(aux=aux, ld_aux=N) if aux is not None else {}
            _gemm(a, w, out, a_layout, b_layout, **kw, **extra)
            return (out, aux) if aux is not None else out

    outs = _per_sm_limit(run)
    for o in outs[1:]:
        if isinstance(o, tuple):
            assert all(torch.equal(u, v) for u, v in zip(o, outs[0]))
        else:
            assert torch.equal(o, outs[0])
    got = outs[0]
    if epi == "grouped":
        v = got.view(M // G, G + gap, N)
        assert rel(v[:, :G].reshape(M, N), full) < tol
        assert torch.all(v[:, G:] == 7.0)
    elif isinstance(got, tuple):
        out, pre = got
        assert rel(pre, ref + b) < 4e-3
        assert rel(out, want) < tol
    else:
        assert rel(got, want) < tol


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("a_layout,b_layout", [(0, 0), (1, 1)])
def test_gemm_split_k_atomic_across_grid_sizes(dev, a_layout, b_layout, block_n):
    from xpretrain_b200 import _lib
    a, w, _, _ = _operands(dev, 3)
    ref = a.float() @ w.float().t()

    def run():
        out = torch.zeros(M, N, dtype=f32, device=dev)
        _gemm(a, w, out, a_layout, b_layout, out_mode=_lib.OUT_F32_ATOMIC, splits=3, block_n=block_n)
        return out

    for got in _per_sm_limit(run):
        assert rel(got, ref) < 1e-5


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("a_layout,b_layout", [(0, 0), (1, 1)])
def test_gemm_split_k_with_empty_trailing_split(dev, a_layout, b_layout, block_n):
    """K = 9 k-blocks in 4 splits of 3: the last split has no k-blocks and its tiles add nothing."""
    from xpretrain_b200 import _lib, ops
    g = torch.Generator(device="cpu").manual_seed(11)
    m, n, k = 256, 264, 9 * 64
    a = torch.randn(m, k, generator=g).to(dev).to(bf16)
    w = torch.randn(n, k, generator=g).to(dev).to(bf16)
    ref = a.float() @ w.float().t()
    A = a if a_layout == 0 else a.t().contiguous()
    B = w if b_layout == 0 else w.t().contiguous()

    def run():
        out = torch.zeros(m, n, dtype=f32, device=dev)
        ops.gemm(A, B, out, M=m, N=n, K=k, lda=A.stride(0), ldb=B.stride(0), ldc=n, a_layout=a_layout,
                 b_layout=b_layout, out_mode=_lib.OUT_F32_ATOMIC, splits=4, block_n=block_n)
        return out

    for got in _per_sm_limit(run):
        assert rel(got, ref) < 1e-5


def test_gemm_rejects_group_strides_that_break_16_byte_rows(dev):
    """The bf16 epilogue moves 16-byte blocks of 8 columns, so grouped row strides must be multiples of 8 elements."""
    from xpretrain_b200 import _lib, ops
    a = torch.zeros(64, 64, dtype=bf16, device=dev)
    w = torch.zeros(64, 64, dtype=bf16, device=dev)
    out = torch.zeros(4096, dtype=bf16, device=dev)
    with pytest.raises(_lib.XpError, match="group_stride"):
        ops.gemm(a, w, out, M=64, N=64, K=64, lda=64, ldb=64, ldc=64, c_group=16, c_group_stride=16 * 64 + 4)
    with pytest.raises(_lib.XpError, match="group_stride"):
        ops.gemm(a, w, out, M=64, N=64, K=64, lda=64, ldb=64, ldc=64, residual=a, ldr=64, r_group=16,
                 r_group_stride=12)
