"""CPU: the float64 attention references of oracle/attention_ref.py against the pinned oracles' attention modules.

The GPU attention tests (test_gpu_attention_contract.py) measure every kernel against these references, so they are pinned
here on small shapes to the same semantics the goldens pin: the test applies the oracle's q/k/v projections itself, calls
the reference, applies out_proj, and compares outputs and input gradients (autograd through the oracle) in float64."""
import torch

from oracle import attention_ref as R
from oracle import clipvip_oracle as O
from oracle import swin3d_oracle as SO
from oracle import timesformer_oracle as TO

F64 = torch.float64


def _close(a, b, tol=1e-10):
    err = float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))
    assert err < tol, err


def _proj_sd(pre, C, gen):
    sd = {}
    for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
        sd[f"{pre}{n}.weight"] = torch.randn(C, C, generator=gen, dtype=F64) * C ** -0.5
        sd[f"{pre}{n}.bias"] = torch.randn(C, generator=gen, dtype=F64) * 0.1
    return sd


def _qkv_of(sd, pre, x, d):
    """The kernels' fused qkv rows: [q * d^-0.5 | k | v] of the oracle's own projections."""
    q = O.linear(x, sd, pre + "q_proj") * d ** -0.5
    return torch.cat([q, O.linear(x, sd, pre + "k_proj"), O.linear(x, sd, pre + "v_proj")], dim=-1)


def _dx_from(sd, pre, dqkv, C):
    return sum(dqkv[:, i * C:(i + 1) * C] @ sd[pre + n + ".weight"] for i, n in enumerate(("q_proj", "k_proj", "v_proj")))


def test_vip_ref_matches_clipvip_oracle_forward2():
    gen = torch.Generator().manual_seed(0)
    B, H, T, L, M, d = 2, 2, 3, 5, 2, 64
    C, S, pre = H * d, M + T * L, "attn."
    sd = _proj_sd(pre, C, gen)
    x = torch.randn(B, S, C, generator=gen, dtype=F64, requires_grad=True)
    gy = torch.randn(B, S, C, generator=gen, dtype=F64)
    want = O.vip_attention(sd, x, pre, H, (M, T, L))
    (want * gy).sum().backward()

    qkv = _qkv_of(sd, pre, x.detach(), d).reshape(B * S, 3 * C)
    dout = gy.reshape(B * S, C) @ sd[pre + "out_proj.weight"]
    r = R.vip_ref(qkv, dout, B, H, T, L, M, q_scale=d ** -0.5)
    got = O.linear(r["out"].reshape(B, S, C), sd, pre + "out_proj")
    _close(got, want.detach())
    _close(_dx_from(sd, pre, r["dqkv"], C), x.grad.reshape(B * S, C))
    # the lse is that of the dense block-masked softmax
    q, k, _ = (R._heads(qkv[:, i * C:(i + 1) * C], B, S, H) for i in range(3))
    frame = torch.cat([torch.full((M,), -1), torch.arange(T).repeat_interleave(L)])
    allow = (frame[:, None] < 0) | (frame[None, :] < 0) | (frame[:, None] == frame[None, :])
    s = (q @ k.transpose(-1, -2)).masked_fill(~allow, float("-inf"))
    _close(r["lse"], torch.logsumexp(s, -1))


def test_vip_ref_arm_rounds_only_the_outputs_in_the_forward():
    gen = torch.Generator().manual_seed(1)
    B, H, T, L, M = 1, 1, 2, 7, 3
    qkv = torch.randn(B * (M + T * L), 3 * 64, generator=gen, dtype=F64)
    dout = torch.randn(B * (M + T * L), 64, generator=gen, dtype=F64)
    ex = R.vip_ref(qkv, dout, B, H, T, L, M)
    arm = R.vip_ref(qkv, dout, B, H, T, L, M, arm="vip")
    assert torch.equal(arm["out"], R.bf(ex["out"]))
    assert torch.equal(arm["dqkv"], R.bf(arm["dqkv"]))
    assert not torch.equal(arm["dqkv"], R.bf(ex["dqkv"]))     # P and dS are rounded before the products


def test_text_ref_matches_clipvip_oracle_dense_attention():
    gen = torch.Generator().manual_seed(2)
    B, H, Lt, d = 4, 2, 9, 64
    C, pre = H * d, "attn."
    sd = _proj_sd(pre, C, gen)
    mask = torch.ones(B, Lt, dtype=torch.int64)
    mask[1, 6:] = 0          # ragged
    mask[2, 0] = 0           # first key padded
    mask[3, :] = 0           # fully padded sample
    x = torch.randn(B, Lt, C, generator=gen, dtype=F64, requires_grad=True)
    gy = torch.randn(B, Lt, C, generator=gen, dtype=F64)
    want = O.dense_attention(sd, x, pre, H, O.text_additive_mask(mask, F64))
    (want * gy).sum().backward()

    qkv = _qkv_of(sd, pre, x.detach(), d).reshape(B * Lt, 3 * C)
    dout = gy.reshape(B * Lt, C) @ sd[pre + "out_proj.weight"]
    r = R.text_ref(qkv, mask, dout, B, H, Lt, q_scale=d ** -0.5)
    _close(O.linear(r["out"].reshape(B, Lt, C), sd, pre + "out_proj"), want.detach())
    _close(_dx_from(sd, pre, r["dqkv"], C), x.grad.reshape(B * Lt, C))
    assert (r["probs"][..., torch.ones(Lt, Lt, dtype=torch.bool).triu(1)] == 0).all()
    # a fully padded sample attends uniformly over its causal prefix (every logit is finfo.min)
    _close(r["probs"][3, 0], torch.tril(torch.ones(Lt, Lt, dtype=F64)) / torch.arange(1, Lt + 1, dtype=F64)[:, None])


def _tsf_weights(C, gen):
    return (torch.randn(3 * C, C, generator=gen, dtype=F64) * C ** -0.5, torch.randn(3 * C, generator=gen, dtype=F64) * 0.1,
            torch.randn(C, C, generator=gen, dtype=F64) * C ** -0.5, torch.randn(C, generator=gen, dtype=F64) * 0.1)


def test_seg_ref_matches_timesformer_oracle_temporal_and_spatial():
    gen = torch.Generator().manual_seed(3)
    B, T, HW, heads, d = 2, 3, 4, 2, 64
    C, n = heads * d, B * HW * T
    w_qkv, b_qkv, w_proj, b_proj = _tsf_weights(C, gen)
    x = torch.randn(n, C, generator=gen, dtype=F64)            # token order (b, h w, t)
    gy = torch.randn(n, C, generator=gen, dtype=F64)
    for rows in (R.temporal_rows(n, T), R.spatial_rows(B, T, HW)):
        xg = x[rows].clone().requires_grad_(True)              # [groups, len, C]
        want = TO.attention(xg, w_qkv, b_qkv, w_proj, b_proj, heads)
        (want * gy[rows]).sum().backward()
        qkv = torch.nn.functional.linear(x, w_qkv, b_qkv)
        qkv[:, :C] *= d ** -0.5
        r = R.seg_ref(qkv, gy @ w_proj, rows, heads, q_scale=d ** -0.5)
        _close(torch.nn.functional.linear(r["out"], w_proj, b_proj)[rows], want.detach())
        dx = torch.zeros(n, C, dtype=F64)
        dx[rows.reshape(-1)] = xg.grad.reshape(-1, C)
        _close(r["dqkv"] @ w_qkv, dx)


def test_seg_ref_matches_swin3d_oracle_window_attention_with_bias():
    gen = torch.Generator().manual_seed(4)
    ws, heads, d, nW, n_win = (2, 2, 3), 2, 32, 2, 4
    N, C, p = 12, heads * d, "blk."
    rpi = SO.rel_pos_index(ws)
    n_rel = int(rpi.max()) + 1
    sd = {p + "qkv.weight": torch.randn(3 * C, C, generator=gen, dtype=F64) * C ** -0.5,
          p + "qkv.bias": torch.randn(3 * C, generator=gen, dtype=F64) * 0.1,
          p + "proj.weight": torch.randn(C, C, generator=gen, dtype=F64) * C ** -0.5,
          p + "proj.bias": torch.randn(C, generator=gen, dtype=F64) * 0.1,
          p + "relative_position_bias_table": torch.randn(n_rel, heads, generator=gen, dtype=F64),
          p + "relative_position_index": rpi}
    mask = torch.where(torch.rand(nW, N, N, generator=gen) < 0.3, -100.0, 0.0).to(F64)
    xw = torch.randn(n_win, N, C, generator=gen, dtype=F64, requires_grad=True)
    gy = torch.randn(n_win, N, C, generator=gen, dtype=F64)
    want = SO.window_attention(sd, p, xw, heads, mask)
    (want * gy).sum().backward()

    rows = torch.arange(n_win * N).view(n_win, N)
    x = xw.detach().reshape(-1, C)
    qkv = torch.nn.functional.linear(x, sd[p + "qkv.weight"], sd[p + "qkv.bias"])
    qkv[:, :C] *= d ** -0.5
    rel = sd[p + "relative_position_bias_table"][rpi[:N, :N].reshape(-1)].reshape(N, N, heads).permute(2, 0, 1)
    bias = rel[None] + mask[:, None]
    r = R.seg_ref(qkv, gy.reshape(-1, C) @ sd[p + "proj.weight"], rows, heads, d, bias=bias, q_scale=d ** -0.5)
    _close(torch.nn.functional.linear(r["out"], sd[p + "proj.weight"], sd[p + "proj.bias"]), want.detach().reshape(-1, C))
    _close(r["dqkv"] @ sd[p + "qkv.weight"], xw.grad.reshape(-1, C))
    # ds = dL/dlogits: its sums over the windows of a type and over heads give the bias-table and mask gradients
    s_rel = torch.zeros_like(sd[p + "relative_position_bias_table"])
    s_rel.index_add_(0, rpi[:N, :N].reshape(-1), r["ds"].sum(0).permute(1, 2, 0).reshape(N * N, heads))
    tab = sd[p + "relative_position_bias_table"].clone().requires_grad_(True)
    sd2 = dict(sd, **{p + "relative_position_bias_table": tab})
    (SO.window_attention(sd2, p, xw.detach(), heads, mask) * gy).sum().backward()
    _close(s_rel, tab.grad)
