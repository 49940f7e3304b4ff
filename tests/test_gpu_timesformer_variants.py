"""H100: TimeSformer with attention_type 'joint_space_time' and 'space_only', and the dense attention kernel under them.

  goldens     the three reference goldens of make_golden_timesformer_variants.py, calibrated: for the output, the input
              gradient and every parameter gradient, err(ours) <= 1.5 x err(the oracle run in bf16 on this GPU), both
              against the fp32 oracle (itself pinned to the goldens on the CPU).  The module keeps its token stream and
              output in bf16, as the divided path does, so the arm is the oracle with bf16 weights and activations; the
              bf16-autocast oracle (fp32 residual stream and output) is printed beside it: 11-28x closer on the
              goldens' worst tensor, 1.7x at 8 x 28 x 28 (measured on an H100 80GB HBM3 at 700 W)
  contract    xp_dense_attention_* in the style of test_gpu_attention_contract.py: seq_len 1 to 6272 at 16 heads,
              calibrated per (sequence, head, 64-row tile) against the float64 dense_ref and its bf16 arm, exact sequence
              locality (NaN in neighbouring sequences and past the last one), full write coverage, bitwise repeats
  stress      joint attention at 8 x 28 x 28 (6272 tokens per clip) at width 1024, fwd + bwd against the fp32 oracle
"""
import os

import pytest
import torch

from contract_harness import ABS_FLOOR, Out, Report, calibrated, calibrated_model_rows, lse_check, same_bits
from oracle import timesformer_oracle as TO
from oracle import timesformer_variants_oracle as V
from oracle.dense_attention_ref import dense_ref

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
QS64 = 0.125
GOLDENS = ["timesformer_joint_interp_b2", "timesformer_joint_native_train", "timesformer_space_only_t1"]
REPORT = Report("dense attention: worst slice ratio err(kernel) / err(bf16 arm), LSE: worst relative error")


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


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


# ============================================================================================ module
def _model(cfg, kind, sd, dev, rate=0.1):
    from xpretrain_b200.modeling.timesformer import TimeSformer

    m = TimeSformer(depth=cfg.depth, num_frames=cfg.num_frames, H=cfg.H, W=cfg.W, embed_dim=cfg.embed_dim,
                    num_heads=cfg.num_heads, drop_path_rate=rate, attention_type=kind)
    m.load_state_dict(sd, strict=True)
    return m.to(dev)


def _oracle_run(sd, x, w_out, cfg, kind, masks, mode):
    """mode: 'fp32' (the truth), 'autocast' (bf16 autocast) or 'bf16' (bf16 weights, input and activations)."""
    dt = bf16 if mode == "bf16" else f32
    sdo = {k: v.detach().to(dt).requires_grad_(True) for k, v in sd.items()}
    xo = x.detach().to(dt).requires_grad_(True)
    if mode == "autocast":
        out = V.autocast_forward(sdo, xo, cfg, kind, drop_masks=masks)
    else:
        m = None if masks is None else [None if b is None else tuple(t.to(dt) for t in b) for b in masks]
        out = V.timesformer_forward(sdo, xo, cfg, kind, drop_masks=m).float()
    (out * w_out).sum().backward()
    return out.detach(), xo.grad, {n: p.grad for n, p in sdo.items() if p.grad is not None}


def _calibrated_model_check(tag, model, x, w_out, cfg, kind, sd, masks):
    """Output, dx and every parameter gradient: err(ours) <= 1.5 x err(bf16 oracle) against the fp32 oracle."""
    out = model(x)
    (out * w_out).sum().backward()
    want, want_dx, want_g = _oracle_run(sd, x, w_out, cfg, kind, masks, "fp32")
    arm, arm_dx, arm_g = _oracle_run(sd, x, w_out, cfg, kind, masks, "bf16")
    ac, ac_dx, ac_g = _oracle_run(sd, x, w_out, cfg, kind, masks, "autocast")
    ours_g = {n: p.grad for n, p in model.named_parameters() if p.grad is not None}
    assert set(ours_g) == set(want_g), set(ours_g) ^ set(want_g)
    rows = [("out", out.detach(), want, arm, ac), ("dx", x.grad, want_dx, arm_dx, ac_dx)]
    rows += [(n, ours_g[n], want_g[n], arm_g[n], ac_g[n]) for n in sorted(want_g)]
    bad, _, _ = calibrated_model_rows(tag, rows)
    assert not bad, "\n".join(bad)
    return out


@pytest.mark.parametrize("name", GOLDENS)
def test_module_matches_reference_golden_calibrated(dev, golden_dir, name):
    gold = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    kind, cfg = gold["attention_type"], TO.TimeSformerCfg(**gold["cfg"])
    B, T, H, W = gold["B"], gold["T"], gold["H"], gold["W"]
    sd = V.init_state_dict(cfg, kind, seed=gold["weight_seed"])
    train = gold["rate"] is not None
    model = _model(cfg, kind, sd, dev, rate=gold["rate"] if train else 0.1)
    masks = None
    if train:
        model.train()
        masks = [None if m is None else tuple(t.to(dev) for t in m) for m in gold["masks"]]
        model.forced_drop_masks = masks
    else:
        model.eval()
    x = TO.synthetic_input(B, T, H, W, cfg, seed=gold["data_seed"]).to(dev).requires_grad_(True)
    g = torch.Generator().manual_seed(gold["data_seed"] + 1)
    w_out = (torch.randn(gold["out"].shape, generator=g) / (B * T * H * W) ** 0.5).to(dev)
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    out = _calibrated_model_check(name, model, x, w_out, cfg, kind, sd_dev, masks)
    # and against the reference's own numbers
    assert out.shape == gold["out"].shape and out.dtype == x.dtype
    assert _rel(out.detach().cpu(), gold["out"]) < 1.5e-2
    assert model.norm.weight.grad is None
    if train:       # the same factors in eval mode are ignored
        with torch.no_grad():
            assert _rel(model.eval()(x), out.detach()) > 1e-2


def test_joint_training_draws_the_references_rng_stream(dev):
    from xpretrain_b200.modeling.timesformer import TimeSformer

    cfg = TO.TimeSformerCfg(depth=3, num_frames=2, H=2, W=3, embed_dim=128, num_heads=2)
    m = TimeSformer(depth=3, num_frames=2, H=2, W=3, embed_dim=128, num_heads=2, drop_path_rate=0.5,
                    attention_type='joint_space_time').to(dev)
    torch.manual_seed(11)
    ours = m.draw_drop_masks(4, 2, 2, 3, dev, torch.float32)
    torch.manual_seed(11)
    want = V.draw_drop_masks(cfg, 'joint_space_time', 4, 2, 0.5, device=dev)
    for a, b in zip(ours[1:], want[1:]):
        for u, v in zip(a, b):
            assert torch.equal(u, v)


def test_joint_stress_grid_full_width_against_fp32_oracle(dev):
    """8 x 28 x 28 = 6272 tokens per clip (BASELINE's stress grid) at width 1024 / 16 heads, one block, two clips."""
    cfg = TO.TimeSformerCfg(depth=1, num_frames=8, H=28, W=28)
    kind = 'joint_space_time'
    sd = V.init_state_dict(cfg, kind, seed=31)
    model = _model(cfg, kind, sd, dev).eval()
    x = TO.synthetic_input(2, 8, 28, 28, cfg, seed=32).to(dev).requires_grad_(True)
    w_out = torch.randn(x.shape, generator=torch.Generator().manual_seed(33)).to(dev) / x[0, :, 0].numel() ** 0.5
    _calibrated_model_check("joint 8x28x28", model, x, w_out, cfg, kind, {k: v.to(dev) for k, v in sd.items()}, None)


# ========================================================================================== kernel
def dense_inputs(dev, n_seq, L, H, seed, extra_rows=0, ld_pad=0):
    """qkv [n_seq*L + extra, 3C + ld_pad] with q pre-scaled (logits of std ~1), dout [n_seq*L + extra, C + ld_pad // 3];
    the extra rows past the last sequence and the pad columns hold NaN."""
    g = torch.Generator().manual_seed(seed)
    C, n = 64 * H, n_seq * L
    x = torch.randn(n, 3 * C, generator=g)
    x[:, :C] *= 0.125
    qkv = torch.full((n + extra_rows, 3 * C + ld_pad), float("nan"), dtype=bf16)
    qkv[:n, :3 * C] = x.to(bf16)
    dout = torch.full((n + extra_rows, C + ld_pad // 3), float("nan"), dtype=bf16)
    dout[:n, :C] = torch.randn(n, C, generator=g).to(bf16)
    return qkv.to(dev), dout.to(dev)


def dense_fwd(dev, qkv, n_seq, L, H, ld_out=None):
    ops, C, n = _ops(), 64 * H, n_seq * L
    out, lse = Out(dev, n, C, bf16, ld=ld_out), Out(dev, H, n, f32)
    ops.dense_attention_fwd(qkv, out.t, lse.t, ops.dense_desc(n, H, qkv.stride(0), out.buf.stride(0), n_seq=n_seq,
                                                              seq_len=L))
    torch.cuda.synchronize()
    return out.check("dense out"), lse.check("dense lse")


def dense_bwd(dev, qkv, out, dout, lse, n_seq, L, H):
    ops, C, n = _ops(), 64 * H, n_seq * L
    dqkv = Out(dev, n, 3 * C, bf16, ld=qkv.stride(0))
    o = torch.full((out.shape[0], dout.stride(0)), float("nan"), dtype=bf16, device=dev)   # out at dout's pitch
    o[:, :C] = out
    delta = torch.full((H, n), float("nan"), device=dev)
    ops.dense_attention_bwd(qkv, o, dout, lse.contiguous(), delta, dqkv.t,
                            ops.dense_desc(n, H, qkv.stride(0), dout.stride(0), n_seq=n_seq, seq_len=L), QS64)
    torch.cuda.synchronize()
    return dqkv.check("dense dqkv")


def dense_slices(dev, n_seq, L, H):
    """Slice index [n, H] of every (row, head): (sequence, head, 64-row tile)."""
    nt = (L + 63) // 64
    r = torch.arange(n_seq * L, device=dev)
    s, t = r // L, (r % L) // 64
    ids = (s[:, None] * H + torch.arange(H, device=dev)[None, :]) * nt + t[:, None]

    def label(i):
        sh, tt = divmod(i, nt)
        return f"(seq={sh // H}, head={sh % H}, tile={tt})"
    return ids, label


DENSE = [  # (n_seq, seq_len, heads, extra rows past the last sequence, qkv pitch pad)
    (3, 1, 16, 2, 0), (3, 63, 16, 2, 0), (3, 64, 16, 2, 0), (3, 65, 16, 2, 0), (2, 392, 16, 3, 0),
    (2, 1120, 16, 0, 0), (1, 6272, 16, 5, 0),
    (3, 130, 2, 7, 24),       # ld_qkv = 3C + 24, ld_out = C + 8
    (5, 200, 4, 0, 48),
]


@pytest.mark.parametrize("n_seq,L,H,extra,pad", DENSE, ids=[f"S{c[0]}L{c[1]}H{c[2]}x{c[3]}p{c[4]}" for c in DENSE])
def test_dense_attention_calibrated(dev, n_seq, L, H, extra, pad):
    tag = f"dense S{n_seq} L{L} H{H}"
    C, n = 64 * H, n_seq * L
    qkv, dout = dense_inputs(dev, n_seq, L, H, seed=L * 10 + n_seq, extra_rows=extra, ld_pad=pad)
    ex = dense_ref(qkv, dout, n_seq, L, H, q_scale=QS64)
    arm = dense_ref(qkv, dout, n_seq, L, H, q_scale=QS64, arm="dense")
    ids, label = dense_slices(dev, n_seq, L, H)
    idc = ids.repeat_interleave(64, dim=1)
    ld_out = C + pad // 3 if pad else None
    out, lse = dense_fwd(dev, qkv, n_seq, L, H, ld_out)
    out2, lse2 = dense_fwd(dev, qkv, n_seq, L, H, ld_out)
    assert same_bits(out, out2) and same_bits(lse, lse2), f"{tag}: forward not bitwise repeatable"
    calibrated(REPORT, f"{tag}: out", out, ex["out"][:n], arm["out"][:n], idc, label, ABS_FLOOR)
    lse_check(REPORT, tag, lse, ex["lse"][:, :n])
    # the backward reads the exact forward, rounded as the kernel stores it
    out_in, lse_in = ex["out"][:n].to(bf16), ex["lse"][:, :n].float()
    dqkv = dense_bwd(dev, qkv, out_in, dout, lse_in, n_seq, L, H)
    dqkv2 = dense_bwd(dev, qkv, out_in, dout, lse_in, n_seq, L, H)
    assert same_bits(dqkv, dqkv2), f"{tag}: backward not bitwise repeatable"
    for j, nm in enumerate(("dq", "dk", "dv")):
        cs = slice(j * C, (j + 1) * C)
        calibrated(REPORT, f"{tag}: {nm}", dqkv[:, cs], ex["dqkv"][:n, cs], arm["dqkv"][:n, cs], idc, label, ABS_FLOOR)


@pytest.mark.parametrize("L", [63, 65, 392])
def test_dense_attention_sequence_locality_is_exact(dev, L):
    """NaN in every other sequence (q, k, v and dout) leaves the remaining sequences' out, lse and dqkv bitwise unchanged:
    the ragged last tile of a sequence reads the next one's rows and must not let them in."""
    n_seq, H = 4, 2
    C, n = 64 * H, n_seq * L
    qkv, dout = dense_inputs(dev, n_seq, L, H, seed=L, extra_rows=3)
    out0, lse0 = dense_fwd(dev, qkv, n_seq, L, H)
    d0 = dense_bwd(dev, qkv, out0, dout, lse0, n_seq, L, H)
    seq = torch.arange(n, device=dev) // L
    for poisoned in ((1, 3), (0, 2)):
        bad = (seq == poisoned[0]) | (seq == poisoned[1])
        q1, g1 = qkv.clone(), dout.clone()
        q1[:n][bad] = float("nan")
        g1[:n][bad] = float("nan")
        ops = _ops()
        out1, lse1 = Out(dev, n, C, bf16), Out(dev, H, n, f32)
        ops.dense_attention_fwd(q1, out1.t, lse1.t, ops.dense_desc(n, H, 3 * C, C, n_seq=n_seq, seq_len=L))
        torch.cuda.synchronize()
        keep = ~bad
        assert same_bits(out1.t[keep], out0[keep]), f"L={L}: NaN in sequences {poisoned} reached another sequence's out"
        assert same_bits(lse1.t[:, keep], lse0[:, keep]), f"L={L}: NaN in sequences {poisoned} reached another's lse"
        o1 = out0.clone()
        o1[bad] = float("nan")
        dq1 = Out(dev, n, 3 * C, bf16)
        ops.dense_attention_bwd(q1, o1, g1, lse0.contiguous(), torch.empty(H, n, device=dev), dq1.t,
                                ops.dense_desc(n, H, 3 * C, C, n_seq=n_seq, seq_len=L), QS64)
        torch.cuda.synchronize()
        assert same_bits(dq1.t[keep], d0[keep]), f"L={L}: NaN in sequences {poisoned} reached another sequence's dqkv"


def test_dense_attention_rejects_bad_descriptors(dev):
    from xpretrain_b200._lib import XpError
    ops = _ops()
    qkv = torch.zeros(1024, 3 * 128, dtype=bf16, device=dev)
    out, lse = torch.zeros(1024, 128, dtype=bf16, device=dev), torch.zeros(2, 1024, device=dev)
    for kw in (dict(n_seq=0, seq_len=4), dict(n_seq=2, seq_len=0), dict(n_seq=3, seq_len=400), dict(n_seq=70000, seq_len=1)):
        with pytest.raises(XpError):
            ops.dense_attention_fwd(qkv, out, lse, ops.dense_desc(1024, 2, 3 * 128, 128, **kw))
    with pytest.raises(XpError):                                    # ld_qkv < 3C
        ops.dense_attention_fwd(qkv, out, lse, ops.dense_desc(1024, 2, 3 * 128 - 8, 128, n_seq=1, seq_len=8))
    with pytest.raises(XpError):                                    # ld not a multiple of 8
        ops.dense_attention_fwd(qkv, out, lse, ops.dense_desc(1024, 2, 3 * 128, 130, n_seq=1, seq_len=8))
