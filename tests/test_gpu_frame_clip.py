"""H100: the per-frame CLIP video model (vision_additional_config.type != "ViP") end to end.  The reference goldens of
tests/golden/make_golden_frame_clip.py under the calibrated rule; the frame-mean head kernel against fp64 torch; the
proxy-token attention at M = 1, T = 1 as dense attention; uint8 frames; the reference's two failure modes; the frozen text
tower, the losses, the fused AdamW and the retrieval metrics.  Gradient checkpointing on each residual stream is in
test_gpu_checkpointing.py."""
from types import SimpleNamespace

import pytest
import torch

from clipvip_cases import (EMB_REL_L2, b16, golden_rule, low_rank_rows, ragged_batch, reference_golden_case, rel,
                           train_step, vidclip)
from contract_harness import FACTOR, reordering_violations

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


def _model(dev, v_layers, t_layers, sd=None):
    return vidclip(b16(v_layers, t_layers), sd=sd, per_frame=True, seed=0, dev=dev)


# ------------------------------------------------------------------------------------------ reference goldens
def _pooled_row_sums(meta):
    """Gradient vectors that are plain sums over the text tower's B pooled (EOS) rows: final_layer_norm.bias and the last
    layer's fc2.bias (only the EOS rows receive gradient from the head).  With B = 2 videos whose random-init features are
    nearly equal, InfoNCE makes those two rows' gradients nearly opposite (in the B/16 golden: norms 0.52 each, sum 0.011),
    so the sums measure the features' error over a 46-fold cancellation, not the kernels: they are left out, like the
    analytically zero k_proj.bias."""
    if meta["B"] != 2:
        return set()
    last = meta["text_layers"] - 1
    return {"text_model.final_layer_norm.bias", f"text_model.encoder.layers.{last}.mlp.fc2.bias"}


@pytest.mark.parametrize("name", ["frame_clip_b16_b2_t3_ragged", "frame_clip_b32_b8_t1", "frame_clip_l14_b8_t2"])
def test_frame_clip_golden_calibrated_against_reference_bf16(dev, golden_dir, name):
    """Features, logits and every sampled gradient within 1.5 x the deviation of the reference algorithm's own bf16-autocast
    run on the same inputs on this GPU.  B/16 and B/32 run the staged attention kernel (197 and 50 rows per frame), L/14 the
    streamed one (257 rows)."""
    ours, ref, meta = reference_golden_case(dev, golden_dir, name, skip=_pooled_row_sums)
    golden_rule(ours, ref, low_rank=low_rank_rows(meta))


# ------------------------------------------------------------------------------------------ frame-mean head kernel
def _pool(dev, proj, T, dfeat=None, scale=1.0):
    from xpretrain_b200 import ops
    rows, P = proj.shape
    B = rows // T
    feat = torch.full((B, P), float("nan"), dtype=f32, device=dev)
    inv_f = torch.full((rows,), float("nan"), dtype=f32, device=dev)
    inv_v = torch.full((B,), float("nan"), dtype=f32, device=dev)
    ops.frame_pool_fwd(proj, feat, inv_f, inv_v, T)
    if dfeat is None:
        return feat, inv_f, inv_v, None
    dproj = torch.full((rows, P), float("nan"), dtype=bf16, device=dev)
    ops.frame_pool_bwd(dfeat, feat, proj, inv_f, inv_v, dproj, T, scale)
    return feat, inv_f, inv_v, dproj


@pytest.mark.parametrize("P", [512, 768])
@pytest.mark.parametrize("T,B", [(1, 128), (2, 97), (12, 128), (32, 64)])
def test_frame_pool_kernel_against_fp64(dev, T, B, P):
    from oracle import frame_clip_oracle as F
    g = torch.Generator().manual_seed(T * 1000 + P + B)
    # rows of very different norms, and a shared direction so that the frame mean is not tiny
    proj = (torch.randn(B * T, P, generator=g, dtype=torch.float64) + 0.5 * torch.randn(1, P, generator=g, dtype=torch.float64)) \
        * torch.exp(2 * torch.randn(B * T, 1, generator=g, dtype=torch.float64))
    proj = proj.float()
    dfeat = torch.randn(B, P, generator=g)
    feat, inv_f, inv_v, dproj = _pool(dev, proj.to(dev), T, dfeat.to(dev))
    p64 = proj.double().requires_grad_(True)
    want = F.frame_mean_head(p64, B, T)
    (dwant,) = torch.autograd.grad(want, p64, dfeat.double())
    assert float((feat.cpu().double() - want.detach()).abs().max()) < 2e-6
    assert float((inv_f.cpu().double() * proj.double().norm(dim=1) - 1).abs().max()) < 2e-6
    m = torch.nn.functional.normalize(proj.double(), dim=1).reshape(B, T, P).mean(1)
    assert float((inv_v.cpu().double() * m.norm(dim=1) - 1).abs().max()) < 2e-6
    # bf16 output: within one bf16 rounding of the fp64 gradient, plus fp32 cancellation relative to each row's size
    row = dwant.abs().amax(dim=1, keepdim=True)
    err = (dproj.cpu().double() - dwant).abs()
    assert bool((err <= 2.0 ** -8 * dwant.abs() + 2e-5 * row).all()), float((err / row).max())
    # no atomics: a second call into fresh buffers gives the same bits; `scale` is a plain factor
    feat2, inv_f2, inv_v2, dproj2 = _pool(dev, proj.to(dev), T, dfeat.to(dev))
    assert torch.equal(feat, feat2) and torch.equal(inv_f, inv_f2) and torch.equal(inv_v, inv_v2) and torch.equal(dproj, dproj2)
    *_, half = _pool(dev, proj.to(dev), T, dfeat.to(dev), scale=0.5)
    assert torch.equal(half.float() * 2, dproj.float())


def test_frame_pool_zero_norm_frame_gives_nan_like_the_reference(dev):
    proj = torch.randn(3 * 4, 512, device=dev)
    proj[5] = 0.0                                 # video 1, frame 1
    feat, *_ = _pool(dev, proj, 4)
    assert bool(torch.isnan(feat[1]).all()) and bool(torch.isfinite(feat[0]).all()) and bool(torch.isfinite(feat[2]).all())


def test_frame_pool_bad_arguments_raise(dev):
    from xpretrain_b200 import _lib
    x = torch.zeros(4, 512, device=dev)
    f = torch.zeros(2, 512, device=dev)
    a, b = torch.zeros(4, device=dev), torch.zeros(2, device=dev)
    rc = _lib.lib().xp_frame_pool_fwd(x.data_ptr(), f.data_ptr(), a.data_ptr(), b.data_ptr(), 2, 0, 512,
                                      torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b"T >= 1" in _lib.lib().xp_last_error()
    rc = _lib.lib().xp_frame_pool_fwd(x.data_ptr(), f.data_ptr(), a.data_ptr(), b.data_ptr(), 2, 2, 20000,
                                      torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b"12288" in _lib.lib().xp_last_error()


# ------------------------------------------------------------------------------------------ attention at M = 1, T = 1
@pytest.mark.parametrize("L,H", [(49, 12), (196, 12), (256, 16)])
def test_vip_attention_single_frame_is_dense_attention(dev, L, H):
    """One frame and one global row per sequence: the ViP kernels (staged at 50 and 197 rows, streamed at 257) compute
    dense attention over the 1 + L rows, within 1.5 x the bf16 arm of oracle/attention_ref.vip_ref; and perturbing one
    image's qkv leaves every other image's out, lse and dqkv bit-identical."""
    from oracle import attention_ref as R
    from xpretrain_b200 import ops
    B, C, S = 5, 64 * H, 1 + L
    q_scale = 64 ** -0.5
    g = torch.Generator().manual_seed(L)
    qkv = torch.randn(B * S, 3 * C, generator=g)
    qkv[:, :C] *= q_scale * 4                                     # q as the QKV GEMM leaves it, scaled
    qkv = qkv.to(bf16)
    dout = torch.randn(B * S, C, generator=g).to(bf16)

    def run(qkv_h):
        out = torch.full((B * S, C), float("nan"), dtype=bf16, device=dev)
        lse = torch.full((B, H, S), float("nan"), dtype=f32, device=dev)
        dqkv = torch.full((B * S, 3 * C), float("nan"), dtype=bf16, device=dev)
        ws = ops.vip_attention_workspace(B, H, 1, 1, dev)
        q = qkv_h.to(dev)
        ops.vip_attention_fwd(q, out, lse, ws, B, H, 1, L, 1, C)
        ops.vip_attention_bwd(q, out, dout.to(dev), lse, dqkv, ws, B, H, 1, L, 1, C, q_scale)
        torch.cuda.synchronize()
        return out.cpu(), lse.cpu(), dqkv.cpu()

    out, lse, dqkv = run(qkv)
    exact = R.vip_ref(qkv.float(), dout.float(), B, H, 1, L, 1, q_scale)
    arm = R.vip_ref(qkv.float(), dout.float(), B, H, 1, L, 1, q_scale, arm="vip")
    # M = 1, T = 1 is dense attention over all S rows of a sequence
    x = qkv.double().reshape(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    dense = torch.softmax(x[0] @ x[1].transpose(-1, -2), dim=-1) @ x[2]
    assert float((exact["out"] - dense.permute(0, 2, 1, 3).reshape(B * S, C)).abs().max()) < 1e-12
    for b in range(B):
        rows = slice(b * S, (b + 1) * S)
        for key, got in (("out", out), ("dqkv", dqkv)):
            e_k = rel(got[rows], exact[key][rows])
            e_a = rel(arm[key][rows].float(), exact[key][rows])
            assert e_k <= FACTOR * e_a + 1e-6, (b, key, e_k, e_a)
        assert float(((lse[b] - exact["lse"][b]).abs() / exact["lse"][b].abs().clamp_min(1)).max()) < 1e-4
    assert torch.isfinite(out.float()).all() and torch.isfinite(dqkv.float()).all()
    # locality: image 2's rows perturbed by large finite values
    qkv2 = qkv.clone()
    qkv2[2 * S:3 * S] = (qkv2[2 * S:3 * S].float() * 7 + 3).to(bf16)
    out2, lse2, dqkv2 = run(qkv2)
    for b in range(B):
        rows = slice(b * S, (b + 1) * S)
        same = torch.equal(out[rows], out2[rows]) and torch.equal(lse[b], lse2[b]) and torch.equal(dqkv[rows], dqkv2[rows])
        assert same == (b != 2), b
    again = run(qkv)
    assert torch.equal(again[0], out) and torch.equal(again[1], lse) and torch.equal(again[2], dqkv)


# ------------------------------------------------------------------------------------------ model-level behaviour
def test_uint8_frames_match_float_path(dev):
    """Raw decoder frames [B, T, H, W, 3] give the same features, bit for bit, as the reference-transformed float video."""
    from xpretrain_b200 import ops
    model = _model(dev, 1, 1)
    model.eval()
    frames, ids, mask = ragged_batch(2, 3, 16, u8=True, dev=dev)
    mean = torch.tensor(ops.CLIP_MEAN, dtype=f32, device=dev)
    std = torch.tensor(ops.CLIP_STD, dtype=f32, device=dev)
    img = frames.reshape(6, 224, 224, 3).permute(0, 3, 1, 2).float() / 255.
    img = img.clone().sub_(mean[:, None, None]).div_(std[:, None, None]).reshape(2, 3, 3, 224, 224)
    with torch.no_grad():
        a = model(video=frames, text_input_ids=ids, text_input_mask=mask)
        b = model(video=img.contiguous(), text_input_ids=ids, text_input_mask=mask)
    assert torch.equal(a["vis_features"], b["vis_features"]) and torch.equal(a["text_features"], b["text_features"])


def test_image_branch_and_forward_video_fail_like_the_reference(dev):
    from xpretrain_b200 import ops
    model = _model(dev, 1, 1)
    video, ids, mask = ragged_batch(2, 2, 16, dev=dev)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(ValueError):
        model(video=video, text_input_ids=ids, text_input_mask=mask, image=video[:, :1], caption_ids=ids[:, None],
              caption_masks=mask[:, None])
    with pytest.raises(TypeError):
        model.forward_video(video)
    with pytest.raises(TypeError):
        model.forward_text(ids, mask)
    assert ops.launch_count() == n0                  # nothing was launched


def test_images_and_get_image_features_against_oracle(dev):
    """CLIP.py semantics on images [N, 3, H, W]: get_image_features returns each image's unnormalised projection, the
    forward returns it normalised."""
    from oracle import clipvip_oracle as O
    from oracle import frame_clip_oracle as F
    cfg = b16(2, 1)
    sd = F.init_state_dict(cfg, seed=4)
    model = _model(dev, 2, 1, sd=sd)
    images = torch.randn(5, 3, 224, 224, generator=torch.Generator().manual_seed(5))
    ids = torch.full((5, 8), 49407)
    ids[:, :4] = 320
    with torch.no_grad():
        proj = model.clipmodel.get_image_features(pixel_values=images.to(dev))
        out = model.clipmodel(pixel_values=images.to(dev), input_ids=ids.to(dev), attention_mask=torch.ones_like(ids).to(dev))
    want = F.frame_vision_tower(sd, images, cfg) @ sd["visual_projection.weight"].t()
    assert proj.shape == (5, 512) and rel(proj.cpu(), want) < EMB_REL_L2
    assert rel(out["image_embeds"].cpu(), O.l2_normalize(want)) < EMB_REL_L2
    assert rel(out["image_embeds"], torch.nn.functional.normalize(proj, dim=-1)) < 1e-6


def test_frozen_text_encoder(dev):
    """VidCLIP.freeze_text_encoder: no text gradient and no text backward; the loss and the vision-side gradients are those
    of the unfrozen model."""
    model = _model(dev, 1, 1)
    model.train()
    video, ids, mask = ragged_batch(4, 3, 16, dev=dev)
    full = train_step(model, video, ids, mask)
    model.freeze_text_encoder(freeze_text_proj=True)
    frozen = train_step(model, video, ids, mask)
    assert all(g is None for n, g in frozen[3].items() if n.startswith(("clipmodel.text_model.", "clipmodel.text_projection.")))
    trained = {n: g for n, g in frozen[3].items() if g is not None}
    bad, worst = reordering_violations({"loss": full[0], "vis": full[1]}, {"loss": frozen[0], "vis": frozen[1]},
                                       {n: full[3][n] for n in trained}, trained)
    print(f"  worst gradient difference {worst[0]:.2e} (relative to max |g|) at {worst[1]}")
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("name", ["gather_nce_loss", "NCEContrastiveLoss", "NCELearnableTempDSLLoss",
                                  "VidImgDivideNCELearnableTempLoss", "NCELearnableTempLoss_vsc_fc"])
def test_losses_on_per_frame_features(dev, name):
    """The contrastive losses on the per-frame model's features: video / subtitle from the video forward, image / caption
    features from a forward over single images (the model has no image/caption branch), against loss_family_oracle."""
    from oracle import loss_family_oracle as LF
    from xpretrain_b200.optimization.loss import build_loss_func, gather_nce_loss
    model = _model(dev, 1, 1)
    model.train()
    video, ids, mask = ragged_batch(6, 2, 16, dev=dev)
    out = model(video=video, text_input_ids=ids, text_input_mask=mask)
    feats = [out["vis_features"], out["text_features"]]
    temp = model.clipmodel.logit_scale
    if name in ("VidImgDivideNCELearnableTempLoss", "NCELearnableTempLoss_vsc_fc"):
        images, cap, cmask = ragged_batch(6, 1, 12, seed=2, dev=dev)
        o2 = model.clipmodel(pixel_values=images[:, 0], input_ids=cap, attention_mask=cmask)
        feats += [o2["image_embeds"], o2["text_embeds"]]
    if name == "gather_nce_loss":
        loss = gather_nce_loss(*feats, temp)
        want = LF.nce_family_loss("NCELearnableTempLoss", [f.detach().cpu() for f in feats], temp.detach().cpu())
    elif name == "NCEContrastiveLoss":
        loss = build_loss_func({"loss_name": name, "temp": 0.05})(*feats)
        want = LF.nce_family_loss(name, [f.detach().cpu() for f in feats], 0.05)
    else:
        loss = build_loss_func({"loss_name": name})(*feats, temp)
        want = LF.nce_family_loss(name, [f.detach().cpu() for f in feats], temp.detach().cpu())
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss) - float(want)) < 2e-3 * abs(float(want)) + 1e-4, (float(loss), float(want))
    named = dict(model.clipmodel.named_parameters())
    for k in ("vision_model.embeddings.patch_embedding.weight", "vision_model.embeddings.class_embedding",
              "vision_model.encoder.layers.0.self_attn.q_proj.weight", "visual_projection.weight"):
        assert named[k].grad is not None and bool(torch.isfinite(named[k].grad).all()) and float(named[k].grad.norm()) > 0, k


def test_full_depth_b16_t12_trains_with_adamw_and_feeds_metrics(dev):
    """The full 12 + 12-layer ViT-B/16 per-frame model built by name: a checkpointed training step at T = 12 through the
    driver's `model(**batch)` with gather_nce_loss and the fused AdamW, then the retrieval metrics on eval-mode features."""
    from xpretrain_b200.modeling import VidCLIP
    from xpretrain_b200.optimization.adamw import AdamW
    from xpretrain_b200.optimization.loss import gather_nce_loss
    from xpretrain_b200.utils import metrics
    torch.manual_seed(0)
    add = SimpleNamespace(type="meanP", temporal_size=12, if_use_temporal_embed=1, logit_scale_init_value=4.6, add_cls_num=3)
    model = VidCLIP(SimpleNamespace(clip_config="openai/clip-vit-base-patch16", clip_weights="",
                                    clip_vision_additional_config=add)).to(dev)
    cm = model.clipmodel
    assert cm.config.per_frame and cm.config.vision.num_hidden_layers == 12
    cm.gradient_checkpointing_enable()
    model.train()
    opt = AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-5, betas=(0.9, 0.98), weight_decay=0.2)
    video, ids, mask = ragged_batch(8, 12, 32, dev=dev)
    batch = {"video": video, "text_input_ids": ids, "text_input_mask": mask}
    before = cm.vision_model.embeddings.patch_embedding.weight.detach().clone()
    out = model(**batch)
    assert out["vis_features"].shape == (8, 512) and out["text_features"].shape == (8, 512)
    loss = gather_nce_loss(out["vis_features"], out["text_features"], cm.logit_scale)
    loss.backward()
    for n, p in model.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), n
    opt.step()
    torch.cuda.synchronize()
    assert torch.isfinite(loss) and not torch.equal(before, cm.vision_model.embeddings.patch_embedding.weight)
    model.eval()
    with torch.no_grad():
        ev = model(**batch)
    sim = metrics.cal_cossim(ev["text_features"].float().contiguous(), ev["vis_features"].float().contiguous())
    assert sim.shape == (8, 8) and bool(torch.isfinite(sim).all())
    assert len(metrics.compute_metrics(sim)) > 0
