"""H100: gradient checkpointing of the CLIP-ViP encoders (`CLIPModel.gradient_checkpointing_enable()`).

A checkpointed tower keeps only each block's input and rebuilds the block's saved tensors in the backward by rerunning the
same kernels.  The recompute must reproduce the forward bit for bit, so loss and features must be equal with the switch on and
off, and gradients may differ only by the reordering of the split-K fp32 atomics of the weight-gradient GEMMs
(contract_harness.reordering_violations).
"""
import gc
import os
from types import SimpleNamespace

import pytest
import torch

from contract_harness import GRAD_REL, reordering_violations

pytestmark = pytest.mark.gpu

# the bars of test_gpu_parity.py's small-golden case (set there from the reference's own bf16 deviation)
EMB_REL_L2 = 1.2e-2
ROW_COSINE = 1.0 - 1e-3
LOSS_REL = 1e-2
GRAD_COSINE = 0.97


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


def _model(dev, v_layers, t_layers, patch=16, stream="fp32", seed=0):
    from xpretrain_b200.modeling import VidCLIP
    from xpretrain_b200.modeling.clip_vip import ClipVipConfig, TowerConfig
    add = SimpleNamespace(type="ViP", temporal_size=12, if_use_temporal_embed=1, logit_scale_init_value=4.6, add_cls_num=3)
    mc = ClipVipConfig(vision=TowerConfig(768, 12, v_layers, 3072), text=TowerConfig(512, 8, t_layers, 2048),
                       patch_size=patch, residual_fp32=(stream != "bf16"), residual_dtype=("fp16" if stream == "fp16" else "fp32"))
    torch.manual_seed(seed)
    model = VidCLIP(SimpleNamespace(clip_config=mc, clip_weights="", clip_vision_additional_config=add))
    with torch.no_grad():
        model.clipmodel.vision_model.embeddings.temporal_embedding.normal_(0, 0.02)
    return model.to(dev)


def _inputs(dev, B, T, Lt, u8=False, seed=1):
    g = torch.Generator().manual_seed(seed)
    if u8:
        video = torch.randint(0, 256, (B, T, 224, 224, 3), generator=g, dtype=torch.uint8)
    else:
        video = torch.randn(B, T, 3, 224, 224, generator=g)
    ids = torch.randint(1, 49406, (B, Lt), generator=g)
    mask = torch.ones(B, Lt, dtype=torch.long)
    eos = torch.randint(2, Lt, (B,), generator=g)          # ragged: EOS, then padding with mask 0
    for b in range(B):
        ids[b, eos[b]:] = 49407
        mask[b, eos[b] + 1:] = 0
    return video.to(dev), ids.to(dev), mask.to(dev)


def _step(model, video, ids, mask):
    from xpretrain_b200.optimization.loss import NCELearnableTempLoss
    model.zero_grad(set_to_none=True)
    out = model(video=video, text_input_ids=ids, text_input_mask=mask)
    loss = NCELearnableTempLoss()(out["vis_features"], out["text_features"], model.clipmodel.logit_scale)
    loss.backward()
    torch.cuda.synchronize()
    grads = {n: (p.grad.detach().clone() if p.grad is not None else None) for n, p in model.named_parameters()}
    return loss.detach(), out["vis_features"].detach(), out["text_features"].detach(), grads


def _assert_same(off, on):
    bad, worst = reordering_violations({"loss": off[0], "vis": off[1], "txt": off[2]},
                                       {"loss": on[0], "vis": on[1], "txt": on[2]}, off[3], on[3])
    print(f"  worst gradient difference {worst[0]:.2e} (relative to max |g|) at {worst[1]}")
    assert not bad, "\n".join(bad)


def _off_on(model, video, ids, mask):
    cm = model.clipmodel
    cm.gradient_checkpointing_disable()
    off = _step(model, video, ids, mask)
    cm.gradient_checkpointing_enable()
    assert cm.is_gradient_checkpointing
    on = _step(model, video, ids, mask)
    cm.gradient_checkpointing_disable()
    return off, on


SWEEP = {
    "fp32": {},
    "fp16_stream": {"stream": "fp16"},
    "bf16_stream": {"stream": "bf16"},
    "uint8_video": {"u8": True},
    "t4_interp": {"T": 4},
    "frozen_text": {"frozen": True},
    "vit_b32": {"patch": 32},
    "sm_reserve8": {"reserve": 8},
}


@pytest.mark.parametrize("case", list(SWEEP))
def test_checkpointing_reproduces_results_depth2(dev, case):
    c = SWEEP[case]
    model = _model(dev, 2, 2, patch=c.get("patch", 16), stream=c.get("stream", "fp32"))
    if c.get("frozen"):
        model.freeze_text_encoder(freeze_text_proj=True)
    model.clipmodel.nccl_sm_reserve = c.get("reserve", 0)
    video, ids, mask = _inputs(dev, 4, c.get("T", 12), 24, u8=c.get("u8", False))
    off, on = _off_on(model, video, ids, mask)
    if c.get("frozen"):
        assert all(g is None for n, g in on[3].items() if n.startswith("clipmodel.text_model."))
    _assert_same(off, on)


def test_checkpointing_reproduces_results_full_depth(dev):
    model = _model(dev, 12, 12)
    video, ids, mask = _inputs(dev, 4, 12, 32)
    off, on = _off_on(model, video, ids, mask)
    _assert_same(off, on)


def test_checkpointing_depth2_ragged_against_reference_golden(dev, golden_dir):
    from oracle import clipvip_oracle as O
    from xpretrain_b200.modeling import VidCLIP
    from xpretrain_b200.modeling.clip_vip import ClipVipConfig, TowerConfig
    from xpretrain_b200.optimization.loss import build_loss_func
    gold = torch.load(os.path.join(golden_dir, "depth2_b3_t12_ragged.pt"), weights_only=False)
    meta = gold["meta"]
    cfg = O.ClipVipCfg(vision=O.TowerCfg(768, 12, meta["vision_layers"], 3072), text=O.TowerCfg(512, 8, meta["text_layers"], 2048))
    sd = O.init_state_dict(cfg, seed=meta["weight_seed"])
    video, ids, mask = O.synthetic_batch(meta["B"], meta["T"], meta["Lt"], cfg, seed=meta["data_seed"], ragged_text=meta["ragged"])
    assert torch.equal(ids, gold["input_ids"])
    add = SimpleNamespace(type="ViP", temporal_size=cfg.temporal_size, if_use_temporal_embed=1,
                          logit_scale_init_value=cfg.logit_scale_init, add_cls_num=cfg.add_cls_num)
    mc = ClipVipConfig(vision=TowerConfig(768, 12, cfg.vision.layers, 3072), text=TowerConfig(512, 8, cfg.text.layers, 2048))
    model = VidCLIP(SimpleNamespace(clip_config=mc, clip_weights="", clip_vision_additional_config=add))
    missing, unexpected = model.clipmodel.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    model = model.to(dev)
    model.clipmodel.gradient_checkpointing_enable()
    out = model(video=video.to(dev), text_input_ids=ids.to(dev), text_input_mask=mask.to(dev))
    loss = build_loss_func({"loss_name": "NCELearnableTempLoss"})(out["vis_features"], out["text_features"],
                                                                    model.clipmodel.logit_scale)
    vis, txt = out["vis_features"].detach().cpu(), out["text_features"].detach().cpu()
    rel = lambda a, b: float((a.float() - b.float()).norm() / b.float().norm())  # noqa: E731
    assert rel(vis, gold["vis_features"]) < EMB_REL_L2 and rel(txt, gold["text_features"]) < EMB_REL_L2
    assert torch.nn.functional.cosine_similarity(vis, gold["vis_features"]).min() > ROW_COSINE
    assert torch.nn.functional.cosine_similarity(txt, gold["text_features"]).min() > ROW_COSINE
    assert abs(float(loss) - float(gold["loss"])) < LOSS_REL * abs(float(gold["loss"]))
    loss.backward()
    torch.cuda.synchronize()
    named = dict(model.clipmodel.named_parameters())
    for k, gn in gold["grad_norms"].items():
        assert named[k].grad is not None, k
        if gn >= 1e-4:
            assert 0.85 < float(named[k].grad.norm()) / gn < 1.15, k
    for k, sample in gold["grad_samples"].items():
        if sample.norm() < 1e-6:
            continue
        got = named[k].grad.detach().flatten()[:256].cpu()
        assert float(torch.nn.functional.cosine_similarity(got, sample, dim=0)) > GRAD_COSINE, k


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
    model = _model(dev, 12, 12)
    B, T, Lt = 4, 12, 32
    video, ids, mask = _inputs(dev, B, T, Lt)
    model.clipmodel.gradient_checkpointing_enable()
    _step(model, video, ids, mask)                      # weight copies and streams exist before the measurement
    kept = _kept_by_forward(model, video, ids, mask)
    want = _predicted_kept_bytes(model.clipmodel.config, B, T, Lt)
    print(f"  checkpointed forward keeps {kept / 2**20:.1f} MiB, predicted {want / 2**20:.1f} MiB")
    assert abs(kept - want) <= 0.05 * want, (kept, want)


def _step_peak(model, video, ids, mask):
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    _step(model, video, ids, mask)
    return torch.cuda.max_memory_allocated() - base


def test_checkpointing_halves_peak_memory(dev):
    model = _model(dev, 12, 12)
    video, ids, mask = _inputs(dev, 4, 12, 32)
    _step(model, video, ids, mask)
    peak_off = _step_peak(model, video, ids, mask)
    model.clipmodel.gradient_checkpointing_enable()
    peak_on = _step_peak(model, video, ids, mask)
    print(f"  peak over forward + backward: {peak_off / 2**20:.0f} MiB off, {peak_on / 2**20:.0f} MiB on "
          f"({peak_on / peak_off:.2f})")
    assert peak_on <= 0.5 * peak_off, (peak_on, peak_off)


def test_checkpointing_is_ignored_in_eval_mode(dev):
    model = _model(dev, 2, 2)
    video, ids, mask = _inputs(dev, 4, 12, 24)
    model.eval()
    _step(model, video, ids, mask)
    kept_off = _kept_by_forward(model, video, ids, mask)
    off = _step(model, video, ids, mask)
    model.clipmodel.gradient_checkpointing_enable()
    kept_on = _kept_by_forward(model, video, ids, mask)
    out = model(video=video, text_input_ids=ids, text_input_mask=mask)
    ctx = out["vis_features"].grad_fn                  # the autograd node holds both towers' saved state
    for sv in (ctx.vis, ctx.txt):
        assert sv.recompute is None and all(isinstance(s, tuple) for s in sv.layers)
    del out, ctx, sv
    on = _step(model, video, ids, mask)
    # the same tensors are saved (checked above); two readings of the same code path are not exact to the byte (they have
    # differed by 0.2 MiB), which is far below one block's saved state (about 260 MiB here)
    assert abs(kept_on - kept_off) <= 2**20, (kept_on, kept_off)
    _assert_same(off, on)
    model.train()
    assert _kept_by_forward(model, video, ids, mask) < kept_off - 2**28      # the same flag takes effect in training mode


def test_checkpointing_hands_over_the_same_gradient_buffers(dev):
    model = _model(dev, 2, 2)
    video, ids, mask = _inputs(dev, 4, 12, 24)
    cm = model.clipmodel
    seen = {}
    for mode in ("off", "on"):
        (cm.gradient_checkpointing_enable if mode == "on" else cm.gradient_checkpointing_disable)()
        rec = seen[mode] = []
        cm.grad_ready_hook = lambda flat: rec.append(flat.detach().clone())
        _step(model, video, ids, mask)
    cm.grad_ready_hook = None
    assert [t.numel() for t in seen["on"]] == [t.numel() for t in seen["off"]]
    assert len(seen["off"]) == 2 * 2 + 2                  # one per layer, then the rest of each tower
    for a, b in zip(seen["off"], seen["on"]):      # flat buffers: the q/k/v bias gradient is one fused vector in them
        assert float((a - b).abs().max()) <= GRAD_REL * float(a.abs().max())
