"""CPU: the float64 GEMM-epilogue and row-kernel references of oracle/gemm_ref.py against torch's own modules.

The GPU contract tests (test_gpu_gemm_contract.py, test_gpu_rowops_contract.py) measure every kernel against these
references, so they are pinned here in float64 to F.linear plus the oracle's quick_gelu, F.gelu, F.layer_norm, and to
autograd through each of them for the gradient epilogues and the LayerNorm backward."""
import torch
import torch.nn.functional as F

from oracle import clipvip_oracle as O
from oracle import gemm_ref as R

F64 = torch.float64


def _close(a, b, tol=1e-12):
    err = float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))
    assert err < tol, err


def _bf16_operands(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = (torch.randn(M, K, generator=g) * K ** -0.25).to(torch.bfloat16)
    b = (torch.randn(N, K, generator=g) * K ** -0.25).to(torch.bfloat16)
    bias = torch.randn(N, generator=g) * 0.5
    res = torch.randn(M, N, generator=g).to(torch.bfloat16)
    return a, b, bias, res


def test_gemm_ref_matches_linear_and_the_header_order():
    a, b, bias, res = _bf16_operands(37, 48, 40, 0)
    A, B = a.double(), b.double()
    lin = F.linear(A, B, bias.double())
    _close(R.gemm_ref(a, b, bias=bias)["exact"], lin)
    _close(R.gemm_ref(a, b, bias=bias, residual=res)["exact"], lin + res.double())
    # alpha scales the product only; q-scale applies after the bias (CLIP_ViP.py:341) to the first scale_cols columns
    r = R.gemm_ref(a, b, alpha=-0.37, bias=bias, scale_cols=16, col_scale=0.125)["exact"]
    want = F.linear(A, B) * -0.37 + bias.double()
    want[:, :16] *= 0.125
    _close(r, want)
    _close(R.gemm_ref(a, b)["absprod"], A.abs() @ B.abs().T)
    c0 = torch.randn(37, 48, dtype=torch.float32)
    _close(R.gemm_ref(a, b, c0=c0, out_mode=R.OUT_F32_ATOMIC)["exact"], F.linear(A, B) + c0.double())


def test_gemm_ref_activations_match_oracle_and_torch():
    a, b, bias, _ = _bf16_operands(29, 64, 72, 1)
    lin = F.linear(a.double(), b.double(), bias.double())
    q = R.gemm_ref(a, b, bias=bias, act=R.ACT_QUICK_GELU)
    _close(q["exact"], O.quick_gelu(lin))
    _close(q["pre"], lin)
    _close(R.gemm_ref(a, b, bias=bias, act=R.ACT_GELU_ERF)["exact"], F.gelu(lin, approximate="none"))
    arm = R.gemm_ref(a, b, bias=bias, act=R.ACT_QUICK_GELU, arm="kernel")
    assert torch.equal(arm["pre"], lin.to(torch.bfloat16).double())
    assert torch.equal(arm["out"], O.quick_gelu(lin).to(torch.bfloat16).double())
    # the reference's autocast arithmetic on a bf16 fc1 output
    t = lin.to(torch.bfloat16)
    want = (t * torch.sigmoid(1.702 * t)).double()
    assert torch.equal(R.gemm_ref(a, b, bias=bias, act=R.ACT_QUICK_GELU, arm="torch_bf16")["out"], want)


def test_dgelu_epilogues_match_autograd():
    """dgrad of fc2 with the activation's derivative fused: dpre = (dy W) * f'(pre), pinned to autograd through the
    oracle's quick_gelu and F.gelu at the bf16 pre-activation."""
    g = torch.Generator().manual_seed(2)
    M, N, K = 33, 56, 24
    dy = (torch.randn(M, K, generator=g)).to(torch.bfloat16)
    w = (torch.randn(K, N, generator=g) * 0.2).to(torch.bfloat16)          # B stored [K, N]: b_layout = 1
    pre = (torch.randn(M, N, generator=g) * 3).to(torch.bfloat16)
    for act, fn in ((R.ACT_DQUICK_GELU, O.quick_gelu), (R.ACT_DGELU_ERF, lambda x: F.gelu(x, approximate="none"))):
        x = pre.double().requires_grad_(True)
        h = fn(x)
        gout = dy.double() @ w.double()
        h.backward(gout)
        got = R.gemm_ref(dy, w.T, act=act, aux=pre)["exact"]
        _close(got, x.grad, 1e-11)
    # the derivative at the bf16 range's ends: 1 and 0, as torch's bf16 autograd gives
    big = torch.tensor([3.3e38, -3.3e38], dtype=torch.bfloat16).double()
    assert torch.equal(R.quick_gelu_grad(big), torch.tensor([1.0, 0.0], dtype=F64))


def test_layernorm_ref_matches_layer_norm_and_autograd():
    g = torch.Generator().manual_seed(3)
    R_, C = 9, 40
    gamma, beta = torch.randn(C, generator=g, dtype=F64), torch.randn(C, generator=g, dtype=F64)
    x = torch.randn(R_, C, generator=g, dtype=F64) * 2 + 0.5
    add = torch.randn(R_, C, generator=g).to(torch.bfloat16)
    xs = (x + add.double()).requires_grad_(True)
    y = F.layer_norm(xs, (C,), gamma.clone().requires_grad_(True), beta, 1e-5)
    r = R.layernorm_ref(x, add, gamma, beta, 1e-5)
    _close(r["y"], y.detach())
    _close(r["mean"], xs.detach().mean(-1))
    _close(r["rstd"], (xs.detach().var(-1, unbiased=False) + 1e-5) ** -0.5)
    dy = torch.randn(R_, C, generator=g).to(torch.bfloat16)
    dres = torch.randn(R_, C, generator=g).to(torch.bfloat16)
    gm = gamma.clone().requires_grad_(True)
    bt = beta.clone().requires_grad_(True)
    xs2 = xs.detach().clone().requires_grad_(True)
    F.layer_norm(xs2, (C,), gm, bt, 1e-5).backward(dy.double())
    b = R.layernorm_bwd_ref(dy, xs.detach(), gamma, r["mean"], r["rstd"], dres)
    _close(b["dx"], xs2.grad + dres.double(), 1e-11)
    _close(b["dgamma"], gm.grad, 1e-11)
    _close(b["dbeta"], bt.grad)
    _close(b["dres_colsum"], dres.double().sum(0))


def test_layernorm_ref_fp16_stream():
    """The fp16 residual stream: the kernel normalises the saturating fp16 round of x + add; the reference's autograd
    through that stored value gives the same LayerNorm gradients."""
    g = torch.Generator().manual_seed(4)
    C = 32
    x = (torch.randn(4, C, generator=g) * 3e4).to(torch.float16)
    add = (torch.randn(4, C, generator=g) * 3e4).to(torch.bfloat16)
    s = R.stream_sum(x, add)
    want = (x.float() + add.float()).clamp(-65504, 65504).half().double()
    assert torch.equal(s, want) and float(s.abs().max()) <= 65504
    gamma, beta = torch.randn(C, generator=g, dtype=F64), torch.randn(C, generator=g, dtype=F64)
    r = R.layernorm_ref(x, add, gamma, beta, 1e-5, arm="kernel")
    assert torch.equal(r["sum"], want)
    xs = want.clone().requires_grad_(True)
    F.layer_norm(xs, (C,), gamma, beta, 1e-5).backward(torch.ones(4, C, dtype=F64))
    b = R.layernorm_bwd_ref(torch.ones(4, C, dtype=torch.bfloat16), want, gamma, r["mean"], r["rstd"])
    _close(b["dx"], xs.grad, 1e-10)


def test_small_row_references():
    g = torch.Generator().manual_seed(5)
    x = torch.randn(6, 24, generator=g, dtype=F64)
    r = R.l2norm_ref(x)
    _close(r["y"], x / x.norm(dim=-1, keepdim=True))
    xg = x.clone().requires_grad_(True)
    dy = torch.randn(6, 24, generator=g, dtype=F64)
    (xg / xg.norm(dim=-1, keepdim=True)).backward(dy)
    _close(R.l2norm_bwd_ref(dy, r["y"], r["inv_norm"], scale=2.0), 2.0 * xg.grad, 1e-11)
    _close(R.colsum_ref(x, 0.5)[0], 0.5 * x.sum(0))
    idx = torch.tensor([2, -1, 0, 5], dtype=torch.int32)
    out = R.gather_rows_ref(x, idx)
    assert torch.equal(out[1], torch.zeros(24, dtype=F64)) and torch.equal(out[0], x[2])
    dst = torch.zeros(6, 24, dtype=F64)
    sc = R.scatter_rows_ref(out, idx, dst)
    assert torch.equal(sc[5], x[5]) and torch.equal(sc[1], torch.zeros(24, dtype=F64))
    s = torch.tensor([0.0, 2.0, 1.0, 0.5, 3.0, 1.0], dtype=F64)
    _close(R.rowscale_ref(x, s, x), x + s[:, None] * x)


# ---------------------------------------------------------- count-weighted references of periodic operands
def _repeated(base, rows):
    P = base.shape[0]
    return base.repeat((rows + P - 1) // P, *([1] * (base.dim() - 1)))[:rows]


def test_repeat_counts():
    c = R.repeat_counts(1000, 7)
    assert torch.equal(c, torch.bincount(torch.arange(1000) % 7).double())


def test_counted_gemm_equals_the_repeated_reduction_and_its_bound():
    g = torch.Generator().manual_seed(3)
    P, rows, n_out, n_in = 7, 100, 16, 24
    dyb = torch.randn(P, n_out, generator=g).to(torch.bfloat16)
    xb = torch.randn(P, n_in, generator=g).to(torch.bfloat16)
    c0 = torch.randn(n_out, n_in, generator=g)
    got = R.gemm_ref_counted(dyb.T, xb.T, R.repeat_counts(rows, P), out_mode=R.OUT_F32_ATOMIC, c0=c0)
    want = R.gemm_ref(_repeated(dyb, rows).T, _repeated(xb, rows).T, out_mode=R.OUT_F32_ATOMIC, c0=c0)
    for k in ("exact", "pre", "absprod"):
        _close(got[k], want[k])
    bg = R.gemm_element_bound(got, 64, 2, c0=c0, out_mode=R.OUT_F32_ATOMIC)
    bw = R.gemm_element_bound(want, 64, 2, c0=c0, out_mode=R.OUT_F32_ATOMIC)
    _close(bg, bw)


def test_counted_layernorm_bwd_and_colsum_equal_the_repeated_sums():
    g = torch.Generator().manual_seed(4)
    P, rows, C = 5, 37, 24
    x, dy, dres = (torch.randn(P, C, generator=g) for _ in range(3))
    gamma = torch.randn(C, generator=g)
    st = R.layernorm_ref(x, None, gamma, gamma, 1e-5)
    got = R.layernorm_bwd_ref(dy, x, gamma, st["mean"], st["rstd"], dres, counts=R.repeat_counts(rows, P))
    rep = [_repeated(t, rows) for t in (dy, x, st["mean"], st["rstd"], dres)]
    want = R.layernorm_bwd_ref(rep[0], rep[1], gamma, rep[2], rep[3], rep[4])
    for k in ("dgamma", "dbeta", "dres_colsum", "abs_dgamma", "abs_dbeta", "abs_dres_colsum"):
        _close(got[k], want[k])
    _close(got["dx"], want["dx"][:P])                      # dx stays per row
    for a, b in zip(R.colsum_ref(dy, -0.5, counts=R.repeat_counts(rows, P)), R.colsum_ref(_repeated(dy, rows), -0.5)):
        _close(a, b)


def test_counted_embedding_bwd_equals_the_repeated_batch():
    from oracle import embed_ref as E
    g = torch.Generator().manual_seed(5)
    P, B, T, L, M, C, Tsz = 3, 8, 4, 5, 4, 16, 3
    dp = torch.randn(P * T * L, C, generator=g).to(torch.bfloat16)
    dg = torch.randn(P * M, C, generator=g).to(torch.bfloat16)
    init = {"pos": torch.randn(1 + L, C, generator=g), "temporal": torch.randn(Tsz, C, generator=g),
            "cls": torch.randn(C, generator=g), "added": torch.randn(M - 1, C, generator=g)}
    got = E.vip_bwd_ref(dp, dg, init, P, T, L, M, Tsz, counts=R.repeat_counts(B, P))
    want = E.vip_bwd_ref(_repeated(dp.view(P, -1), B).reshape(-1, C), _repeated(dg.view(P, -1), B).reshape(-1, C), init,
                         B, T, L, M, Tsz)
    assert set(got) == set(want)
    for k in got:
        _close(got[k][0], want[k][0])
        _close(got[k][1], want[k][1])


def test_block_weights_grow_along_the_rows_in_powers_of_two():
    w = R.block_weights(10)
    assert torch.equal(w, torch.tensor([1.0, 1, 1, 2, 2, 4, 4, 4, 8, 8], dtype=F64))


def test_weighted_counts_over_a_row_range_equal_the_explicit_rows():
    P, rows = 7, 100
    w = R.block_weights((rows + P - 1) // P)
    row_w = w[torch.arange(rows) // P]
    for start, stop in ((0, rows), (0, 37), (20, 93)):
        want = torch.zeros(P, dtype=F64).index_add_(0, torch.arange(start, stop) % P, row_w[start:stop])
        assert torch.equal(R.repeat_counts(stop, P, weights=w, start=start), want)


def test_wrapped_column_sums_equal_dropped_and_displaced_reads_of_the_explicit_operand():
    """Against the flat [rows x W] operand built row by row: elements at flat offset >= wrap set to zero (never read) or
    taken from wrap elements earlier, for a wrap inside a row and one on a row boundary."""
    g = torch.Generator().manual_seed(6)
    P, W, rows = 7, 24, 101
    xb = torch.randn(P, W, generator=g, dtype=F64)
    w = R.block_weights((rows + P - 1) // P)
    flat = torch.stack([xb[r % P] * w[r // P] for r in range(rows)]).reshape(-1)
    for wrap in (1000, 48 * W):
        dropped, displaced = R.wrapped_column_sums(xb, rows, w, wrap)
        d = flat.clone()
        d[wrap:] = 0
        _close(dropped, d.view(rows, W).sum(0))
        d[wrap:] = flat[:flat.numel() - wrap]
        _close(displaced, d.view(rows, W).sum(0))
    _close(R.repeat_counts(rows, P, weights=w) @ xb, flat.view(rows, W).sum(0))
