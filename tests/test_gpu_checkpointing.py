"""H100: gradient checkpointing of the CLIP-ViP encoders, ViT-B and ViT-L/14, and of the per-frame CLIP model
(`CLIPModel.gradient_checkpointing_enable()`).

A checkpointed tower keeps only each block's input and rebuilds the block's saved tensors in the backward by rerunning the
same kernels.  The recompute must reproduce the forward bit for bit, so loss and features must be equal with the switch on and
off, and gradients may differ only by the reordering of the split-K fp32 atomics of the weight-gradient GEMMs
(contract_harness.reordering_violations).
"""
import gc

import pytest
import torch

from clipvip_cases import b16, l14, ragged_batch, small_golden_case, train_step, vidclip
from contract_harness import GRAD_REL, reordering_violations

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


def _model(dev, cfg):
    return vidclip(cfg, seed=0, temporal_init=True, dev=dev)


def _assert_same(off, on):
    bad, worst = reordering_violations({"loss": off[0], "vis": off[1], "txt": off[2]},
                                       {"loss": on[0], "vis": on[1], "txt": on[2]}, off[3], on[3])
    print(f"  worst gradient difference {worst[0]:.2e} (relative to max |g|) at {worst[1]}")
    assert not bad, "\n".join(bad)


def _off_on(model, video, ids, mask):
    cm = model.clipmodel
    cm.gradient_checkpointing_disable()
    off = train_step(model, video, ids, mask)
    cm.gradient_checkpointing_enable()
    assert cm.is_gradient_checkpointing
    on = train_step(model, video, ids, mask)
    cm.gradient_checkpointing_disable()
    return off, on


# The ViP model at B = 4, T = 12 with its temporal table redrawn; the per-frame model (its tower reruns per frame) and
# ViT-L/14 (the streamed attention) at B = 3, T = 3 with their construction-time weights.
VIP = {"cfg": b16(2, 2), "per_frame": False, "temporal_init": True, "B": 4, "T": 12}
FRAME = {"cfg": b16(2, 2), "per_frame": True, "temporal_init": False, "B": 3, "T": 3}
L14 = {"cfg": l14(224, 2, 2), "per_frame": False, "temporal_init": False, "B": 3, "T": 3}
SWEEP = {
    "fp32": {},
    "fp16_stream": {"stream": "fp16"},
    "bf16_stream": {"stream": "bf16"},
    "uint8_video": {"u8": True},
    "t4_interp": {"T": 4},
    "frozen_text": {"frozen": True},
    "vit_b32": {"cfg": b16(2, 2, patch=32)},
    "sm_reserve8": {"reserve": 8},
    "frame_clip_fp32": FRAME,
    "frame_clip_fp16_stream": {**FRAME, "stream": "fp16"},
    "frame_clip_bf16_stream": {**FRAME, "stream": "bf16"},
    "frame_clip_uint8_video": {**FRAME, "u8": True},
    "vit_l14_fp32": L14,
    "vit_l14_fp16_stream": {**L14, "stream": "fp16"},
    "vit_l14_bf16_stream": {**L14, "stream": "bf16"},
    "vit_l14_uint8_video": {**L14, "u8": True},
}


@pytest.mark.parametrize("case", list(SWEEP))
def test_checkpointing_reproduces_results_depth2(dev, case):
    c = {**VIP, **SWEEP[case]}
    model = vidclip(c["cfg"], stream=c.get("stream", "fp32"), per_frame=c["per_frame"], seed=0,
                    temporal_init=c["temporal_init"], dev=dev)
    if c.get("frozen"):
        model.freeze_text_encoder(freeze_text_proj=True)
    model.clipmodel.nccl_sm_reserve = c.get("reserve", 0)
    video, ids, mask = ragged_batch(c["B"], c["T"], 24, u8=c.get("u8", False), dev=dev)
    off, on = _off_on(model, video, ids, mask)
    assert off[1].shape == (c["B"], c["cfg"].proj_dim)
    if c.get("frozen"):
        assert all(g is None for n, g in on[3].items() if n.startswith("clipmodel.text_model."))
    _assert_same(off, on)


def test_checkpointing_reproduces_results_full_depth(dev):
    model = _model(dev, b16(12, 12))
    video, ids, mask = ragged_batch(4, 12, 32, dev=dev)
    off, on = _off_on(model, video, ids, mask)
    _assert_same(off, on)


def test_checkpointing_depth2_ragged_against_reference_golden(dev, golden_dir):
    small_golden_case(dev, golden_dir, "depth2_b3_t12_ragged", checkpointing=True)


def _kept_by_forward(model, video, ids, mask):
    """Bytes the forward leaves allocated (the tensors saved for the backward, plus the two feature matrices).  Before each
    reading, gc.collect() frees unreachable tensors of earlier steps and empty_cache() completes the frees that wait on another
    stream (record_stream), so that neither reading counts them."""
    def settle():
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    model.zero_grad(set_to_none=True)
    settle()
    before = torch.cuda.memory_allocated()
    out = model(video=video, text_input_ids=ids, text_input_mask=mask)
    settle()
    kept = torch.cuda.memory_allocated() - before
    del out
    torch.cuda.synchronize()
    return kept


def _predicted_kept_bytes(cfg, B, T, Lt):
    """Checkpointed forward, fp32 stream: one [rows, C] fp32 boundary per block, plus what both modes keep outside the
    blocks: the patch matrix, the embedding output x0 and the pre_layrnorm statistics, the last block's stream and branch
    output, and the attention workspace (text: the stream and branch of the last block)."""
    C, L, M, H = cfg.vision.hidden_size, cfg.num_patches, 1 + cfg.add_cls_num, cfg.vision.num_attention_heads
    rows = B * (M + T * L)
    Kp = 3 * cfg.patch_size ** 2
    vis = cfg.vision.num_hidden_layers * rows * C * 4
    vis += B * T * L * Kp * 2 + rows * C * 2 + 2 * rows * 4
    vis += rows * C * (4 + 2) + B * H * T * M * 3 * 64 * 4
    Ct, rows_t = cfg.text.hidden_size, B * Lt
    txt = cfg.text.num_hidden_layers * rows_t * Ct * 4 + rows_t * Ct * (4 + 2)
    return vis + txt


def test_checkpointing_forward_keeps_only_boundaries(dev):
    model = _model(dev, b16(12, 12))
    B, T, Lt = 4, 12, 32
    video, ids, mask = ragged_batch(B, T, Lt, dev=dev)
    model.clipmodel.gradient_checkpointing_enable()
    train_step(model, video, ids, mask)                      # weight copies and streams exist before the measurement
    kept = _kept_by_forward(model, video, ids, mask)
    want = _predicted_kept_bytes(model.clipmodel.config, B, T, Lt)
    print(f"  checkpointed forward keeps {kept / 2**20:.1f} MiB, predicted {want / 2**20:.1f} MiB")
    assert abs(kept - want) <= 0.05 * want, (kept, want)


def _step_peak(model, video, ids, mask):
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    train_step(model, video, ids, mask)
    return torch.cuda.max_memory_allocated() - base


def test_checkpointing_halves_peak_memory(dev):
    model = _model(dev, b16(12, 12))
    video, ids, mask = ragged_batch(4, 12, 32, dev=dev)
    train_step(model, video, ids, mask)
    peak_off = _step_peak(model, video, ids, mask)
    model.clipmodel.gradient_checkpointing_enable()
    peak_on = _step_peak(model, video, ids, mask)
    print(f"  peak over forward + backward: {peak_off / 2**20:.0f} MiB off, {peak_on / 2**20:.0f} MiB on "
          f"({peak_on / peak_off:.2f})")
    assert peak_on <= 0.5 * peak_off, (peak_on, peak_off)


def test_checkpointing_is_ignored_in_eval_mode(dev):
    model = _model(dev, b16(2, 2))
    video, ids, mask = ragged_batch(4, 12, 24, dev=dev)
    model.eval()
    train_step(model, video, ids, mask)
    kept_off = _kept_by_forward(model, video, ids, mask)
    off = train_step(model, video, ids, mask)
    model.clipmodel.gradient_checkpointing_enable()
    kept_on = _kept_by_forward(model, video, ids, mask)
    out = model(video=video, text_input_ids=ids, text_input_mask=mask)
    ctx = out["vis_features"].grad_fn                  # the autograd node holds both towers' saved state
    for sv in (ctx.vis, ctx.txt):
        assert sv.recompute is None and all(isinstance(s, tuple) for s in sv.layers)
    del out, ctx, sv
    on = train_step(model, video, ids, mask)
    # the same tensors are saved (checked above); two readings of the same code path are not exact to the byte (they have
    # differed by 0.2 MiB), which is far below one block's saved state (about 260 MiB here)
    assert abs(kept_on - kept_off) <= 2**20, (kept_on, kept_off)
    _assert_same(off, on)
    model.train()
    assert _kept_by_forward(model, video, ids, mask) < kept_off - 2**28      # the same flag takes effect in training mode


def test_checkpointing_hands_over_the_same_gradient_buffers(dev):
    model = _model(dev, b16(2, 2))
    video, ids, mask = ragged_batch(4, 12, 24, dev=dev)
    cm = model.clipmodel
    seen = {}
    for mode in ("off", "on"):
        (cm.gradient_checkpointing_enable if mode == "on" else cm.gradient_checkpointing_disable)()
        rec = seen[mode] = []
        cm.grad_ready_hook = lambda flat: rec.append(flat.detach().clone())
        train_step(model, video, ids, mask)
    cm.grad_ready_hook = None
    assert [t.numel() for t in seen["on"]] == [t.numel() for t in seen["off"]]
    assert len(seen["off"]) == 2 * 2 + 2                  # one per layer, then the rest of each tower
    for a, b in zip(seen["off"], seen["on"]):      # flat buffers: the q/k/v bias gradient is one fused vector in them
        assert float((a - b).abs().max()) <= GRAD_REL * float(a.abs().max())
