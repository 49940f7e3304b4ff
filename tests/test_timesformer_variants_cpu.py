"""CPU: TimeSformer with attention_type 'joint_space_time' and 'space_only' — the oracle replays the reference goldens of
tests/golden/make_golden_timesformer_variants.py, the module builds the reference's parameter tree for every type, the
float64 dense-attention reference is pinned to the oracle's attention, and space_only at T > 1 fails before any launch."""
import os

import pytest
import torch

from oracle import timesformer_oracle as TO
from oracle import timesformer_variants_oracle as V
from oracle.dense_attention_ref import dense_ref

GOLDENS = ["timesformer_joint_interp_b2", "timesformer_joint_native_train", "timesformer_space_only_t1"]


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)


@pytest.mark.parametrize("name", GOLDENS)
def test_variant_oracle_replays_reference_golden(golden_dir, name):
    gold = _load(golden_dir, name)
    kind = gold["attention_type"]
    cfg = TO.TimeSformerCfg(**gold["cfg"])
    B, T, H, W = gold["B"], gold["T"], gold["H"], gold["W"]
    sd = {k: v.requires_grad_(True) for k, v in V.init_state_dict(cfg, kind, seed=gold["weight_seed"]).items()}
    x = TO.synthetic_input(B, T, H, W, cfg, seed=gold["data_seed"]).requires_grad_(True)
    g = torch.Generator().manual_seed(gold["data_seed"] + 1)
    w_out = torch.randn(B, T, cfg.embed_dim, H, W, generator=g) / (B * T * H * W) ** 0.5
    out = V.timesformer_forward(sd, x, cfg, kind, drop_masks=gold["masks"])
    loss = (out * w_out).sum()
    loss.backward()
    assert out.shape == gold["out"].shape
    assert _rel(out.detach(), gold["out"]) < 1e-6
    assert abs(float(loss.detach()) - float(gold["loss"])) <= 1e-5 * max(1.0, abs(float(gold["loss"])))
    assert _rel(x.grad[:, 0], gold["dx_t0"]) < 1e-5
    for n, ref in gold["grads"].items():
        got = sd[n].grad[:8] if ref.dim() == 2 else sd[n].grad
        assert _rel(got, ref) < 1e-5, n
    for n, nrm in gold["grad_norms"].items():
        assert abs(float(sd[n].grad.norm()) - nrm) <= 1e-5 * nrm + 1e-12, n
    assert sd["norm.weight"].grad is None            # constructed, never applied (timesformer.py:451)
    if gold["masks"] is not None:                     # the training case drops at least one branch
        assert any(m is not None and any(bool((t == 0).any()) for t in m) for m in gold["masks"])


@pytest.mark.parametrize("name", GOLDENS)
def test_module_state_dict_matches_reference_tree(golden_dir, name):
    from xpretrain_b200.modeling.timesformer import TimeSformer

    gold = _load(golden_dir, name)
    cfg = TO.TimeSformerCfg(**gold["cfg"])
    m = TimeSformer(depth=cfg.depth, num_frames=cfg.num_frames, H=cfg.H, W=cfg.W, embed_dim=cfg.embed_dim,
                    num_heads=cfg.num_heads, attention_type=gold["attention_type"])
    ours = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert ours == gold["state_dict_shapes"]
    assert list(ours) == list(gold["state_dict_shapes"])          # same order as the reference's module tree
    m.load_state_dict(V.init_state_dict(cfg, gold["attention_type"], seed=0), strict=True)
    assert not any(".temporal_" in k for k in ours)
    assert ("time_embed" in ours) == (gold["attention_type"] == "joint_space_time")


def test_joint_init_has_no_temporal_fc_zeroing_and_divided_is_unchanged():
    from xpretrain_b200.modeling.timesformer import TimeSformer

    torch.manual_seed(0)
    joint = TimeSformer(depth=2, num_frames=2, H=2, W=2, embed_dim=128, num_heads=2, attention_type='joint_space_time')
    assert float(joint.blocks[1].attn.proj.weight.std()) > 0.01
    assert joint.no_weight_decay() == {'pos_embed', 'time_embed'}
    div = TimeSformer(depth=2, num_frames=2, H=2, W=2, embed_dim=128, num_heads=2)
    assert float(div.blocks[1].temporal_fc.weight.abs().max()) == 0.0     # timesformer.py:458-466
    with pytest.raises(ValueError):
        TimeSformer(depth=1, embed_dim=128, num_heads=2, attention_type='spatial')


def test_space_only_beyond_one_frame_raises_before_any_launch():
    """The reference cannot run space_only at T > 1 (its reshape after the frame mean fails, timesformer.py:519-522).  The
    module raises RuntimeError before touching the kernels: with CPU tensors any launch would raise XpError instead."""
    from xpretrain_b200._lib import XpError
    from xpretrain_b200.modeling.timesformer import TimeSformer

    m = TimeSformer(depth=1, num_frames=2, H=2, W=3, embed_dim=128, num_heads=2, attention_type='space_only')
    with pytest.raises(RuntimeError) as e:
        m(torch.randn(1, 2, 128, 2, 3))
    assert not isinstance(e.value, XpError)
    cfg = TO.TimeSformerCfg(depth=1, num_frames=2, H=2, W=3, embed_dim=128, num_heads=2)
    with pytest.raises(RuntimeError):
        V.timesformer_forward(V.init_state_dict(cfg, 'space_only'), torch.randn(1, 2, 128, 2, 3), cfg, 'space_only')
    # at T = 1 the module goes on to the kernels: on CPU tensors that is the no-CPU-path error
    with pytest.raises(XpError):
        m(torch.randn(1, 1, 128, 2, 3))


def test_drop_masks_follow_the_reference_draw_order():
    """Two draws per block on the blocks' batch (B clips for joint, B*T frames for space_only), none in block 0."""
    from xpretrain_b200.modeling.timesformer import TimeSformer

    for kind, n in (("joint_space_time", 3), ("space_only", 3)):
        cfg = TO.TimeSformerCfg(depth=3, num_frames=1, H=2, W=2, embed_dim=128, num_heads=2)
        m = TimeSformer(depth=3, num_frames=1, H=2, W=2, embed_dim=128, num_heads=2, drop_path_rate=0.5,
                        attention_type=kind)
        torch.manual_seed(3)
        ours = m.draw_drop_masks(3, 1, 2, 2, None, torch.float32)
        torch.manual_seed(3)
        want = V.draw_drop_masks(cfg, kind, 3, 1, 0.5)
        assert ours[0] is None and want[0] is None
        for a, b in zip(ours[1:], want[1:]):
            assert len(a) == len(b) == 2
            for u, v in zip(a, b):
                assert u.shape == (n,) and torch.equal(u, v)


@pytest.mark.parametrize("n_seq", [1, 2])
def test_dense_ref_matches_oracle_attention(n_seq):
    """dense_ref on the kernels' operands (q pre-scaled) equals the oracle's Attention core in float64, forward and
    backward.  One-hot tokens through the oracle's qkv Linear make the qkv rows free parameters: qkv[i] = W[:, i] + b."""
    heads, C = 2, 128
    seq_len = C
    g = torch.Generator().manual_seed(9)
    qkv_rows, douts, grads, outs = [], [], [], []
    for _ in range(n_seq):
        w = (torch.randn(3 * C, C, generator=g, dtype=torch.float64) * 2.0).requires_grad_(True)
        b = torch.zeros(3 * C, dtype=torch.float64)
        eye = torch.eye(C, dtype=torch.float64)[None]
        out = TO.attention(eye, w, b, torch.eye(C, dtype=torch.float64), torch.zeros(C, dtype=torch.float64), heads)[0]
        dout = torch.randn(seq_len, C, generator=g, dtype=torch.float64)
        (out * dout).sum().backward()
        qkv = w.detach().t().clone()
        qkv[:, :C] *= 0.125
        qkv_rows.append(qkv)
        douts.append(dout)
        grads.append(w.grad.t())
        outs.append(out.detach())
    qkv = torch.cat(qkv_rows)
    ref = dense_ref(qkv, torch.cat(douts), n_seq, seq_len, heads, q_scale=0.125)
    assert _rel(ref["out"], torch.cat(outs)) < 1e-12
    assert _rel(ref["dqkv"], torch.cat(grads)) < 1e-12
    s = (qkv[:seq_len, :64] @ qkv[:seq_len, C:C + 64].t())
    assert torch.allclose(ref["lse"][0, :seq_len], torch.logsumexp(s, -1), rtol=0, atol=1e-12)
    # the bf16 arm differs by rounding only
    arm = dense_ref(qkv, torch.cat(douts), n_seq, seq_len, heads, q_scale=0.125, arm="dense")
    assert 0 < _rel(arm["out"], ref["out"]) < 1e-2 and 0 < _rel(arm["dqkv"], ref["dqkv"]) < 3e-2
