"""H100: every attention kernel against the float64 references of oracle/attention_ref.py (pinned to the oracles by
test_attention_reference_cpu.py), with the project's calibrated rule (contract_harness.py) applied slice by slice, plus
exact checks.

  calibrated   per slice, err(kernel) <= 1.5 x err(bf16 arm) + a floor of 2^-16 x the slice's reference norm, where the arm
               rounds to bf16 exactly where the kernel does; a 64-row tile, frame, head or window cannot hide in the norm
               of the whole tensor.  LSE: per row, |err| <= 1e-4 x max(1, |lse|) (fp32 from fp32 scores).
  q_scale      every backward runs with the model's scale (0.125 for head_dim 64, 32^-0.5 for 32), and the dq of the ViP
               global rows (the combine kernel's scaling) is asserted on its own
  coverage     outputs live in NaN-filled buffers with guard rows (and pad columns, for ld > width) holding a bit
               pattern: every logical element must be written and finite, and nothing else touched
  repeatable   two calls into fresh buffers give the same bits (no attention kernel uses float atomics)
  locality     inputs a slice does not depend on are perturbed with large finite values; the slice must keep every bit
"""
import pytest
import torch

from contract_harness import ABS_FLOOR, Out, Report, calibrated, lse_check, same_bits
from oracle import attention_ref as R

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
PROBS_TOL = 1e-4       # text probabilities are an fp32 output: relative norm per (b, h) against the exact ones
QS64, QS32 = 64 ** -0.5, 32 ** -0.5
REPORT = Report("worst slice ratio err(kernel) / err(bf16 arm), LSE and probs: worst relative error")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    REPORT.print()


def _ops():
    from xpretrain_b200 import ops
    return ops


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ================================================================================ ViP (staged and streamed)
def vip_inputs(dev, B, H, T, L, M, seed, regime="diffuse"):
    """qkv [B*S, 3C] with q pre-scaled, dout [B*S, C].  'diffuse': logits of std ~0.16 and V centred over each frame's
    keys, so that attention outputs are small against V and rounding P (not O) would dominate their error; 'model': the
    model's own scale (logits of std ~1)."""
    g = _gen(seed)
    C, S = 64 * H, M + T * L
    x = torch.randn(B, S, 3 * C, generator=g)
    if regime == "diffuse":
        x[..., :C] *= 0.02
        fr = x[:, M:, 2 * C:].reshape(B, T, L, C)
        x[:, M:, 2 * C:] = (fr - fr.mean(2, keepdim=True)).reshape(B, T * L, C)
        x[:, :M, 2 * C:] *= 0.05
    else:
        x[..., :C] *= 0.125
    dout = torch.randn(B * S, C, generator=g)
    return x.reshape(B * S, 3 * C).to(bf16).to(dev), dout.to(bf16).to(dev)


def vip_fwd(dev, qkv, B, H, T, L, M):
    ops, C, S = _ops(), 64 * H, M + T * L
    out, lse = Out(dev, B * S, C, bf16), Out(dev, B * H, S, f32)
    ws = ops.vip_attention_workspace(B, H, T, M, dev)
    ops.vip_attention_fwd(qkv, out.t, lse.t, ws, B, H, T, L, M, C)
    torch.cuda.synchronize()
    return out.check("vip out"), lse.check("vip lse").view(B, H, S)


def vip_bwd(dev, qkv, out, dout, lse, B, H, T, L, M, q_scale):
    ops, C, S = _ops(), 64 * H, M + T * L
    dqkv = Out(dev, B * S, 3 * C, bf16)
    ws = ops.vip_attention_workspace(B, H, T, M, dev)
    ops.vip_attention_bwd(qkv, out, dout, lse.contiguous(), dqkv.t, ws, B, H, T, L, M, C, q_scale)
    torch.cuda.synchronize()
    return dqkv.check("vip dqkv")


def vip_slices(dev, B, H, T, L, M):
    """Slice index [B*S, H] of every (row, head): (b, h, t, 64-row tile) for frame rows, (b, h) for the M global rows."""
    S, nt = M + T * L, (L + 63) // 64
    per = T * nt + 1
    s = torch.arange(S, device=dev)
    f = (s - M).clamp_min(0)
    r = torch.where(s < M, torch.full_like(s, T * nt), (f // L) * nt + (f % L) // 64)
    b = torch.arange(B, device=dev)[:, None, None]
    h = torch.arange(H, device=dev)[None, None, :]
    ids = (b * H + h) * per + r[None, :, None]                                    # [B, S, H]

    def label(i):
        bh, rr = divmod(i, per)
        bb, hh = divmod(bh, H)
        return f"(b={bb}, h={hh}, global rows)" if rr == T * nt else f"(b={bb}, h={hh}, t={rr // nt}, tile={rr % nt})"
    return ids.reshape(B * S, H), label


VIP_STAGED = [  # M + L <= 208 runs vip_attention.cu (VIP_STAGED_MAX_ROWS, vip_attention.h)
    (1, 2, 2, 200, 8, "diffuse"), (1, 2, 2, 207, 1, "diffuse"), (1, 2, 2, 204, 4, "diffuse"),
    (2, 2, 2, 1, 4, "diffuse"), (2, 2, 3, 63, 4, "diffuse"), (2, 2, 3, 64, 4, "diffuse"), (2, 2, 3, 65, 4, "diffuse"),
    (1, 2, 2, 192, 4, "diffuse"), (1, 2, 2, 193, 4, "diffuse"),
    (2, 2, 1, 100, 4, "diffuse"),           # T = 1
    (2, 1, 3, 50, 4, "diffuse"),            # H = 1
    (2, 4, 12, 196, 4, "model"),            # B/16 frames at the model's logit scale
]
VIP_STREAMED = [  # M + L > 208: vip_attention_long.cu
    (1, 2, 2, 208, 1, "diffuse"),           # the first streamed size
    (1, 2, 2, 320, 4, "diffuse"),           # 5 + 1 tiles: an even count, no half-empty last CTA
    (1, 2, 3, 256, 8, "diffuse"),
    (16, 16, 2, 212, 4, "model"),           # B*H = 256 CTAs along z
]


@pytest.mark.parametrize("B,H,T,L,M,regime", VIP_STAGED + VIP_STREAMED,
                         ids=[f"B{c[0]}H{c[1]}T{c[2]}L{c[3]}M{c[4]}-{c[5]}" for c in VIP_STAGED + VIP_STREAMED])
def test_vip_attention_calibrated(dev, B, H, T, L, M, regime):
    tag = f"vip {'staged' if M + L <= 208 else 'streamed'} B{B} H{H} T{T} L{L} M{M} {regime}"
    C = 64 * H
    qkv, dout = vip_inputs(dev, B, H, T, L, M, seed=B * 1000 + L * 10 + M, regime=regime)
    ex = R.vip_ref(qkv, dout, B, H, T, L, M, q_scale=QS64)
    arm = R.vip_ref(qkv, dout, B, H, T, L, M, q_scale=QS64, arm="vip")
    ids, label = vip_slices(dev, B, H, T, L, M)
    idc = ids.repeat_interleave(64, dim=1)

    out, lse = vip_fwd(dev, qkv, B, H, T, L, M)
    out2, lse2 = vip_fwd(dev, qkv, B, H, T, L, M)
    assert same_bits(out, out2) and same_bits(lse, lse2), f"{tag}: forward not bitwise repeatable"
    calibrated(REPORT, f"{tag}: out", out, ex["out"], arm["out"], idc, label, ABS_FLOOR)
    lse_check(REPORT, tag, lse, ex["lse"])

    # the backward reads the exact forward, rounded as the kernels store it
    out_in, lse_in = ex["out"].to(bf16), ex["lse"].float()
    dqkv = vip_bwd(dev, qkv, out_in, dout, lse_in, B, H, T, L, M, QS64)
    dqkv2 = vip_bwd(dev, qkv, out_in, dout, lse_in, B, H, T, L, M, QS64)
    assert same_bits(dqkv, dqkv2), f"{tag}: backward not bitwise repeatable"
    for j, nm in enumerate(("dq", "dk", "dv")):
        cs = slice(j * C, (j + 1) * C)
        calibrated(REPORT, f"{tag}: {nm}", dqkv[:, cs], ex["dqkv"][:, cs], arm["dqkv"][:, cs], idc, label, ABS_FLOOR)
    # the global rows' dq on its own: summed over frames and scaled by q_scale in the combine kernel
    g = (torch.arange(B * (M + T * L), device=dev) % (M + T * L)) < M
    calibrated(REPORT, f"{tag}: dq global rows", dqkv[g, :C], ex["dqkv"][g, :C], arm["dqkv"][g, :C], idc[g], label,
               ABS_FLOOR)


def _perturb(x, rows, cols, seed, scale):
    g = _gen(seed)
    y = x.clone()
    blk = y[rows][:, cols]
    y[rows.unsqueeze(1), cols.unsqueeze(0)] = (torch.randn(blk.shape, generator=g) * scale).to(x.dtype).to(x.device)
    return y


@pytest.mark.parametrize("L", [100, 230], ids=["staged", "streamed"])
def test_vip_attention_locality_is_exact(dev, L):
    """Frame t's patch rows read only frame t and the global rows: perturbing another frame's q/k/v (forward) or dout
    (backward), another sample, or another head's columns leaves them bitwise unchanged.  L = 230 streams 64-row tiles
    whose last one reads 26 rows of the next frame (or sample) and masks them."""
    B, H, T, M = 2, 2, 3, 4
    C, S = 64 * H, M + T * L
    qkv, dout = vip_inputs(dev, B, H, T, L, M, seed=7 + L)
    ex = R.vip_ref(qkv, None, B, H, T, L, M)
    out_in, lse_in = ex["out"].to(bf16), ex["lse"].float()
    out0, lse0 = vip_fwd(dev, qkv, B, H, T, L, M)
    d0 = vip_bwd(dev, qkv, out_in, dout, lse_in, B, H, T, L, M, QS64)
    s = torch.arange(B * S, device=dev)
    b_of, t_of = s // S, torch.where(s % S < M, -1, (s % S - M) // L)
    allc3, allc = torch.arange(3 * C, device=dev), torch.arange(C, device=dev)
    for tp in (1, T - 1):
        frame = s[t_of == tp]
        keep = (t_of >= 0) & (t_of != tp)
        for scale in (1.0, 30.0):
            out1, lse1 = vip_fwd(dev, _perturb(qkv, frame, allc3, tp, scale), B, H, T, L, M)
            assert same_bits(out1[keep], out0[keep]), f"L={L}: q/k/v of frame {tp} (x{scale}) changed other frames' out"
            lk = keep.view(B, S)[:, None, :].expand(B, H, S)
            assert same_bits(lse1[lk], lse0[lk]), f"L={L}: q/k/v of frame {tp} (x{scale}) changed other frames' lse"
            d1 = vip_bwd(dev, qkv, out_in, _perturb(dout, frame, allc, tp, scale), lse_in, B, H, T, L, M, QS64)
            assert same_bits(d1[keep], d0[keep]), f"L={L}: dout of frame {tp} (x{scale}) changed other frames' dqkv"
    # another sample / another head: the backward reads each call's own forward (out, lse stay consistent with qkv)
    dk0 = vip_bwd(dev, qkv, out0, dout, lse0, B, H, T, L, M, QS64)
    rows1 = s[b_of == 1]
    q1, g1 = _perturb(qkv, rows1, allc3, 11, 8.0), _perturb(dout, rows1, allc, 12, 8.0)
    o1, l1 = vip_fwd(dev, q1, B, H, T, L, M)
    k0 = b_of == 0
    assert same_bits(o1[k0], out0[k0]) and same_bits(l1[0], lse0[0]), f"L={L}: sample 1's inputs changed sample 0's forward"
    d1 = vip_bwd(dev, q1, o1, g1, l1, B, H, T, L, M, QS64)
    assert same_bits(d1[k0], dk0[k0]), f"L={L}: sample 1's inputs changed sample 0's dqkv"
    hc = torch.arange(64, 128, device=dev)
    q1 = _perturb(qkv, s, torch.cat([hc, hc + C, hc + 2 * C]), 14, 8.0)
    o1, l1 = vip_fwd(dev, q1, B, H, T, L, M)
    assert same_bits(o1[:, :64], out0[:, :64]) and same_bits(l1[:, 0], lse0[:, 0]), \
        f"L={L}: head 1's inputs changed head 0's forward"
    d1 = vip_bwd(dev, q1, o1, _perturb(dout, s, hc, 16, 8.0), l1, B, H, T, L, M, QS64)
    h0 = torch.cat([torch.arange(64), torch.arange(64) + C, torch.arange(64) + 2 * C]).to(dev)
    assert same_bits(d1[:, h0], dk0[:, h0]), f"L={L}: head 1's inputs changed head 0's dqkv"


def test_vip_attention_rejects_bad_shapes(dev):
    from xpretrain_b200._lib import XpError
    ops = _ops()
    qkv = torch.zeros(4096, 3 * 128, dtype=bf16, device=dev)
    out, lse = torch.zeros(4096, 128, dtype=bf16, device=dev), torch.zeros(8192, device=dev)
    ws = torch.zeros(1 << 16, device=dev)
    for (B, H, T, L, M, C) in ((1, 2, 2, 50, 0, 128), (1, 2, 2, 50, 9, 128), (1, 2, 2, 0, 4, 128), (1, 2, 2, 50, 4, 96)):
        with pytest.raises(XpError):
            ops.vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C)
        with pytest.raises(XpError):
            ops.vip_attention_bwd(qkv, out, out, lse, qkv, ws, B, H, T, L, M, C, QS64)


# ========================================================================================= text
def text_masks(Lt):
    """Four samples: no padding, ragged (trailing padding), first key padded, fully padded."""
    m = torch.ones(4, Lt, dtype=torch.int64)
    m[1, Lt // 2 + 1:] = 0
    m[2, 0] = 0
    m[3, :] = 0
    return m


def text_inputs(dev, B, H, Lt, seed):
    g = _gen(seed)
    C = 64 * H
    x = torch.randn(B * Lt, 3 * C, generator=g)
    x[:, :C] *= 0.125
    return x.to(bf16).to(dev), torch.randn(B * Lt, C, generator=g).to(bf16).to(dev)


def text_fwd(dev, qkv, mask, B, H, Lt):
    ops, C = _ops(), 64 * H
    out, probs = Out(dev, B * Lt, C, bf16), Out(dev, B * H * Lt, Lt, f32)
    ops.text_attention_fwd(qkv, mask, out.t, probs.t, B, H, Lt, C)
    torch.cuda.synchronize()
    return out.check("text out"), probs.check("text probs").view(B, H, Lt, Lt)


def text_bwd(dev, qkv, dout, probs, B, H, Lt, q_scale):
    ops, C = _ops(), 64 * H
    dqkv = Out(dev, B * Lt, 3 * C, bf16)
    ops.text_attention_bwd(qkv, dout, probs.contiguous(), dqkv.t, B, H, Lt, C, q_scale)
    torch.cuda.synchronize()
    return dqkv.check("text dqkv")


TEXT = [(Lt, H) for Lt in (1, 2, 31, 32, 33, 63, 64, 65, 77) for H in (8, 12)]


@pytest.mark.parametrize("Lt,H", TEXT, ids=[f"Lt{a}H{b}" for a, b in TEXT])
def test_text_attention_calibrated(dev, Lt, H):
    B, C = 4, 64 * H
    qkv, dout = text_inputs(dev, B, H, Lt, seed=Lt * 100 + H)
    b_of = torch.arange(B * Lt, device=dev) // Lt
    ids = (b_of[:, None] * H + torch.arange(H, device=dev)[None, :]).repeat_interleave(64, dim=1)

    def label(i):
        return f"(b={i // H}, h={i % H})"
    for mk in (None, text_masks(Lt)):
        tag = f"text Lt{Lt} H{H} {'no mask' if mk is None else 'padded'}"
        mdev = None if mk is None else mk.to(dev)
        ex = R.text_ref(qkv, mdev, dout, B, H, Lt, q_scale=QS64)
        arm = R.text_ref(qkv, mdev, dout, B, H, Lt, q_scale=QS64, arm="text")
        out, probs = text_fwd(dev, qkv, mdev, B, H, Lt)
        out2, probs2 = text_fwd(dev, qkv, mdev, B, H, Lt)
        assert same_bits(out, out2) and same_bits(probs, probs2), f"{tag}: forward not bitwise repeatable"
        calibrated(REPORT, f"{tag}: out", out, ex["out"], arm["out"], ids, label, ABS_FLOOR)
        zero = ex["probs"] == 0
        assert bool((probs[zero] == 0).all()), f"{tag}: probabilities of masked keys are not exactly 0"
        pe = ((probs.double() - ex["probs"]).flatten(2).norm(dim=2) / ex["probs"].flatten(2).norm(dim=2))
        REPORT.record(f"{tag}: probs", float(pe.max()))
        assert float(pe.max()) <= PROBS_TOL, f"{tag}: probs: worst (b, h) = {divmod(int(pe.argmax()), H)}: {float(pe.max()):.2e}"
        pin = ex["probs"].float()
        dqkv = text_bwd(dev, qkv, dout, pin, B, H, Lt, QS64)
        assert same_bits(dqkv, text_bwd(dev, qkv, dout, pin, B, H, Lt, QS64)), f"{tag}: backward not bitwise repeatable"
        for j, nm in enumerate(("dq", "dk", "dv")):
            cs = slice(j * C, (j + 1) * C)
            calibrated(REPORT, f"{tag}: {nm}", dqkv[:, cs], ex["dqkv"][:, cs], arm["dqkv"][:, cs], ids, label, ABS_FLOOR)


def test_text_attention_locality_is_exact(dev):
    """Causality and padding exactly: k/v of token j never reach rows i < j; dout of row i reaches only dq of row i and
    dk/dv of keys <= i; k/v of a trailing padded key reach nothing (its logit is -FLT_MAX, its probability exactly 0)."""
    B, H, Lt, j = 4, 2, 33, 20
    C = 64 * H
    mask = text_masks(Lt).to(dev)
    qkv, dout = text_inputs(dev, B, H, Lt, seed=5)
    out0, probs0 = text_fwd(dev, qkv, mask, B, H, Lt)
    d0 = text_bwd(dev, qkv, dout, probs0, B, H, Lt, QS64)
    pos = torch.arange(B * Lt, device=dev) % Lt
    kv = torch.arange(C, 3 * C, device=dev)
    for scale in (1.0, 30.0):
        q1 = _perturb(qkv, (pos == j).nonzero().squeeze(1), kv, 1, scale)
        out1, probs1 = text_fwd(dev, q1, mask, B, H, Lt)
        assert same_bits(out1[pos < j], out0[pos < j]), f"k/v of token {j} (x{scale}) changed earlier rows' out"
        assert same_bits(probs1[:, :, :j], probs0[:, :, :j]), f"k/v of token {j} (x{scale}) changed earlier rows' probs"
        i = 10
        d1 = text_bwd(dev, qkv, _perturb(dout, (pos == i).nonzero().squeeze(1), torch.arange(C, device=dev), 2, scale),
                      probs0, B, H, Lt, QS64)
        assert same_bits(d1[pos != i, :C], d0[pos != i, :C]), f"dout of row {i} (x{scale}) changed other rows' dq"
        assert same_bits(d1[pos > i, C:], d0[pos > i, C:]), f"dout of row {i} (x{scale}) changed dk/dv of later keys"
        # sample 1 keeps Lt // 2 + 1 keys: its last key is padded and every row sees a live key
        row = torch.tensor([2 * Lt - 1], device=dev)
        q2 = _perturb(qkv, row, kv, 3, scale)
        out2, probs2 = text_fwd(dev, q2, mask, B, H, Lt)
        d2 = text_bwd(dev, q2, dout, probs2, B, H, Lt, QS64)
        assert same_bits(out2, out0) and same_bits(probs2, probs0), f"k/v of a padded key (x{scale}) changed the forward"
        assert same_bits(d2, d0), f"k/v of a padded key (x{scale}) changed the backward"


# ============================================================================ seg: temporal, spatial, window
def seg_slices(dev, rows, n_rows, H, tile):
    """Slice index [n_rows, H]: (sequence, head, 64-row tile of the sequence), or (sequence, head) with tile=None."""
    n_seq, n = rows.shape
    nt = 1 if tile is None else (n + tile - 1) // tile
    seq = torch.zeros(n_rows, dtype=torch.long)
    pos = torch.zeros(n_rows, dtype=torch.long)
    seq[rows.reshape(-1)] = torch.arange(n_seq).repeat_interleave(n)
    pos[rows.reshape(-1)] = torch.arange(n).repeat(n_seq)
    part = pos // tile if tile is not None else torch.zeros_like(pos)
    ids = ((seq[:, None] * H + torch.arange(H)[None, :]) * nt + part[:, None]).to(dev)

    def label(i):
        sh, tt = divmod(i, nt)
        return f"(sequence={sh // H}, head={sh % H}" + (f", tile={tt})" if tile is not None else ")")
    return ids, label


class Seg:
    """One seg_attention configuration: rows [n_seq, len] of the reference, the kernel descriptor, inputs in buffers of
    pitch ld_qkv / ld_out."""

    def __init__(self, dev, kind, rows, n_rows, H, hd, ld_qkv, ld_out, seed, bias=None):
        self.dev, self.kind, self.rows, self.n_rows, self.H, self.hd = dev, kind, rows, n_rows, H, hd
        self.C = H * hd
        self.ld_qkv, self.ld_out, self.bias = ld_qkv, ld_out, bias
        self.q_scale = hd ** -0.5
        g = _gen(seed)
        x = torch.randn(n_rows, ld_qkv, generator=g)
        x[:, :self.C] *= 0.125 if hd == 64 else QS32 * 3.0
        self.qkv_buf = x.to(bf16).to(dev)
        self.dout_buf = torch.randn(n_rows, ld_out, generator=g).to(bf16).to(dev)

    def qkv(self):
        return self.qkv_buf[:, :3 * self.C]

    def dout(self):
        return self.dout_buf[:, :self.C]

    def desc(self, ds=None):
        ops = _ops()
        if self.kind == "window":
            idx = self.rows.to(torch.int32).to(self.dev).contiguous()
            return ops.window_desc(self.n_rows, self.H, self.hd, self.ld_qkv, self.ld_out, idx, self.bias, ds_out=ds)
        if self.kind == "temporal":
            return ops.temporal_desc(self.n_rows, self.rows.shape[1], self.H, self.ld_qkv, self.ld_out)
        B, T, HW = self.BTHW
        return ops.spatial_desc(B, T, HW, self.H, self.ld_qkv, self.ld_out)

    def ref(self, arm=None, qkv=None, dout=None):
        return R.seg_ref(self.qkv() if qkv is None else qkv[:, :3 * self.C], self.dout() if dout is None else dout[:, :self.C],
                         self.rows.to(self.dev), self.H, self.hd, bias=self.bias, q_scale=self.q_scale, arm=arm)

    def fwd(self, qkv_buf=None):
        out, lse = Out(self.dev, self.n_rows, self.C, bf16, self.ld_out), Out(self.dev, self.H, self.n_rows, f32)
        _ops().seg_attention_fwd(self.qkv_buf if qkv_buf is None else qkv_buf, out.t, lse.t, self.desc())
        torch.cuda.synchronize()
        return out.check(f"{self.kind} out"), lse.check(f"{self.kind} lse")

    def bwd(self, out_in, lse_in, dout_buf=None):
        n_win, L = self.rows.shape
        dqkv = Out(self.dev, self.n_rows, 3 * self.C, bf16, self.ld_qkv)
        delta = Out(self.dev, self.H, self.n_rows, f32)
        ds = Out(self.dev, n_win * self.H * L, L, bf16) if self.kind == "window" else None
        ob = torch.zeros(self.n_rows, self.ld_out, dtype=bf16, device=self.dev)
        ob[:, :self.C] = out_in
        _ops().seg_attention_bwd(self.qkv_buf, ob, self.dout_buf if dout_buf is None else dout_buf, lse_in.contiguous(),
                                 delta.t, dqkv.t, self.desc(None if ds is None else ds.t.view(n_win, self.H, L, L)),
                                 self.q_scale)
        torch.cuda.synchronize()
        delta.check(f"{self.kind} delta")
        return dqkv.check(f"{self.kind} dqkv"), (None if ds is None else ds.check(f"{self.kind} ds_out").view(n_win, self.H, L, L))


def make_temporal(dev, T, H=2, B=2, HW=7, wide=False, seed=0):
    n = B * HW * T
    return Seg(dev, "temporal", R.temporal_rows(n, T), n, H, 64, 3 * 64 * H + (64 if wide else 0),
               64 * H + (32 if wide else 0), seed=seed + T)


def make_spatial(dev, HW, H=2, B=2, T=3, wide=False, seed=0):
    s = Seg(dev, "spatial", R.spatial_rows(B, T, HW), B * HW * T, H, 64, 3 * 64 * H + (64 if wide else 0),
            64 * H + (32 if wide else 0), seed=seed + HW)
    s.BTHW = (B, T, HW)
    return s


def make_window(dev, L, n_win=7, nW=3, H=2, seed=0):
    g = _gen(seed + L)
    n = n_win * L
    rows = torch.randperm(n, generator=g).view(n_win, L)              # roll + window partition is a permutation of rows
    bias = torch.randn(nW, H, L, L, generator=g) * 0.5
    bias = bias + torch.where(torch.rand(nW, 1, L, L, generator=g) < 0.3, -100.0, 0.0)   # shift-mask entries
    bias[:, :, torch.arange(L), torch.arange(L)] = bias[:, :, torch.arange(L), torch.arange(L)].clamp_min(-5.0)
    return Seg(dev, "window", rows, n, H, 32, 3 * 32 * H, 32 * H, seed=seed + L + 1, bias=bias.contiguous().to(dev))


SEG_CASES = ([("temporal", T, False) for T in (1, 2, 5, 12, 16, 64, 65)] + [("temporal", 5, True)] +
             [("spatial", HW, False) for HW in (63, 64, 65, 196)] + [("spatial", 65, True)] +
             [("window", L, False) for L in (30, 64, 65, 480)])


@pytest.mark.parametrize("kind,size,wide", SEG_CASES,
                         ids=[f"{k}{s}{'-wide' if w else ''}" for k, s, w in SEG_CASES])
def test_seg_attention_calibrated(dev, kind, size, wide):
    seg = (make_temporal(dev, size, wide=wide) if kind == "temporal" else
           make_spatial(dev, size, wide=wide) if kind == "spatial" else make_window(dev, size))
    tag = f"{kind} {size}{' ld_qkv>3C ld_out>C' if wide else ''}"
    C = seg.C
    ex, arm = seg.ref(), seg.ref(arm="seg")
    ids, label = seg_slices(dev, seg.rows, seg.n_rows, seg.H, None if kind == "window" else 64)
    idc = ids.repeat_interleave(seg.hd, dim=1)
    out, lse = seg.fwd()
    out2, lse2 = seg.fwd()
    assert same_bits(out, out2) and same_bits(lse, lse2), f"{tag}: forward not bitwise repeatable"
    calibrated(REPORT, f"{tag}: out", out, ex["out"], arm["out"], idc, label, ABS_FLOOR)
    lse_check(REPORT, tag, lse, ex["lse"])

    out_in, lse_in = ex["out"].to(bf16), ex["lse"].float()
    dqkv, ds = seg.bwd(out_in, lse_in)
    dqkv2, ds2 = seg.bwd(out_in, lse_in)
    assert same_bits(dqkv, dqkv2) and (ds is None or same_bits(ds, ds2)), f"{tag}: backward not bitwise repeatable"
    for j, nm in enumerate(("dq", "dk", "dv")):
        cs = slice(j * C, (j + 1) * C)
        calibrated(REPORT, f"{tag}: {nm}", dqkv[:, cs], ex["dqkv"][:, cs], arm["dqkv"][:, cs], idc, label, ABS_FLOOR)
    if ds is not None:
        n_win, L = seg.rows.shape
        dids = (torch.arange(n_win * seg.H, device=dev)[:, None].expand(-1, L * L)).reshape(n_win, seg.H, L, L)
        calibrated(REPORT, f"{tag}: ds_out", ds, ex["ds"], arm["ds"], dids,
                   lambda i: f"(window={i // seg.H}, head={i % seg.H})", ABS_FLOOR)


@pytest.mark.parametrize("kind", ["temporal", "spatial", "window"])
def test_seg_attention_locality_is_exact(dev, kind):
    """One group (temporal: including the groups packed into the same 64-row tile), frame or window perturbed in q/k/v
    (forward) or dout (backward): every other group keeps every bit of its outputs."""
    seg = make_temporal(dev, 5) if kind == "temporal" else make_spatial(dev, 65) if kind == "spatial" else make_window(dev, 65)
    ex = seg.ref()
    out_in, lse_in = ex["out"].to(bf16), ex["lse"].float()
    out0, lse0 = seg.fwd()
    d0, ds0 = seg.bwd(out_in, lse_in)
    grp = 3 if kind != "spatial" else 1
    rows = seg.rows[grp].to(dev)
    other = torch.ones(seg.n_rows, dtype=torch.bool, device=dev)
    other[rows] = False
    for scale in (1.0, 30.0):
        q1 = _perturb(seg.qkv_buf, rows, torch.arange(3 * seg.C, device=dev), 1, scale)
        out1, lse1 = seg.fwd(q1)
        assert same_bits(out1[other], out0[other]) and same_bits(lse1[:, other], lse0[:, other]), \
            f"{kind}: q/k/v of group {grp} (x{scale}) changed other groups' forward"
        d1, ds1 = seg.bwd(out_in, lse_in, _perturb(seg.dout_buf, rows, torch.arange(seg.C, device=dev), 2, scale))
        assert same_bits(d1[other], d0[other]), f"{kind}: dout of group {grp} (x{scale}) changed other groups' dqkv"
        if ds0 is not None:
            w = torch.arange(ds0.shape[0], device=dev) != grp
            assert same_bits(ds1[w], ds0[w]), f"{kind}: dout of window {grp} (x{scale}) changed other windows' ds_out"


def test_seg_attention_rejects_bad_descriptors(dev):
    from xpretrain_b200._lib import XpError
    ops = _ops()
    H, n = 2, 640
    qkv, out = torch.zeros(n, 3 * 128, dtype=bf16, device=dev), torch.zeros(n, 128, dtype=bf16, device=dev)
    lse = torch.zeros(H, n, device=dev)
    bad = []
    d = ops.temporal_desc(n, 8, H, 3 * 128, 128)
    d.head_dim = 48
    bad.append(d)
    bad.append(ops.temporal_desc(n, 8, H, 3 * 128 - 8, 128))              # ld_qkv < 3C
    bad.append(ops.temporal_desc(n, 8, H, 3 * 128, 120))                  # ld_out < C
    d = ops.temporal_desc(n, 8, H, 3 * 128, 128)
    d.n_seq = 65536                                                       # one grid dimension holds 65535 sequences
    bad.append(d)
    for d in bad:
        with pytest.raises(XpError):
            ops.seg_attention_fwd(qkv, out, lse, d)
        with pytest.raises(XpError):
            ops.seg_attention_bwd(qkv, out, out, lse, lse, qkv, d, QS64)
