"""H100: CLIP-ViP with ViT-L/14 towers (1024-wide vision tower with 16 heads and 14-pixel patches, 768-wide text tower and
projection) end to end: the reference goldens of tests/golden/make_golden_vit_l14.py under the calibrated rule, the
image/caption branch, the losses at d = 768, the fused AdamW and the retrieval metrics.  Gradient checkpointing on each
residual stream and on uint8 frames is in test_gpu_checkpointing.py."""
from types import SimpleNamespace

import pytest
import torch

from clipvip_cases import (EMB_REL_L2, GRAD_COSINE, golden_rule, l14, low_rank_rows, ragged_batch, reference_golden_case,
                           rel, vidclip)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


# ------------------------------------------------------------------------------------------ reference goldens
@pytest.mark.parametrize("name", ["l14_224_b2_t3_ragged", "l14_336_b2_t2"])
def test_vit_l14_golden_calibrated_against_reference_bf16(dev, golden_dir, name):
    """Features, logits and every sampled gradient within 1.5 x the deviation of the reference algorithm's own bf16-autocast
    run on the same inputs on this GPU (DESIGN.md §2).  The last layer's out_proj and fc2 weight gradients are rank-B outer
    products over the B = 2 CLS rows (low_rank_rows)."""
    ours, ref, meta = reference_golden_case(dev, golden_dir, name)
    golden_rule(ours, ref, low_rank=low_rank_rows(meta))


# ------------------------------------------------------------------------------------------ image/caption, losses
def test_vit_l14_image_caption_branch_against_oracle(dev):
    """Video pass plus a T = 1 image/caption pass (the streamed attention's single-frame case) at 336 px, six-term loss
    at d = 768, backward through both passes."""
    from oracle import clipvip_oracle as O
    from xpretrain_b200.optimization.loss import build_loss_func
    cfg = l14(336, 1, 1)
    sd = O.init_state_dict(cfg, seed=5)
    B, T, Lt = 3, 2, 16
    video, ids, mask = O.synthetic_batch(B, T, Lt, cfg, seed=21)
    image, cap_ids, cap_mask = O.synthetic_batch(B, 1, Lt, cfg, seed=22, ragged_text=True)
    model = vidclip(cfg, sd=sd, seed=0, dev=dev)
    out = model(video=video.to(dev), text_input_ids=ids.to(dev), text_input_mask=mask.to(dev), image=image.to(dev),
                caption_ids=cap_ids.to(dev), caption_masks=cap_mask.to(dev))
    loss = build_loss_func({"loss_name": "NCELearnableTempLoss_vsc_fc"})(
        out["vis_features"], out["text_features"], out["img_features"], out["cap_features"], model.clipmodel.logit_scale)
    loss.backward()
    sdo = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    o1 = O.clip_vip_forward(sdo, video, ids, mask, cfg)
    o2 = O.clip_vip_forward(sdo, image.reshape(-1, 1, *image.shape[2:]), cap_ids, cap_mask, cfg)
    want = O.nce_vsc_fc_loss(o1["vis_features"], o1["text_features"], o2["vis_features"], o2["text_features"],
                             sdo["logit_scale"])
    want.backward()
    for k, ref in (("vis_features", o1["vis_features"]), ("text_features", o1["text_features"]),
                   ("img_features", o2["vis_features"]), ("cap_features", o2["text_features"])):
        assert rel(out[k].detach().cpu(), ref.detach()) < EMB_REL_L2, k
    assert abs(float(loss) - float(want)) < 1e-2 * abs(float(want))
    named = dict(model.clipmodel.named_parameters())
    for k in ("vision_model.embeddings.temporal_embedding", "vision_model.embeddings.patch_embedding.weight",
              "vision_model.embeddings.position_embedding.weight", "vision_model.encoder.layers.0.self_attn.q_proj.weight",
              "text_model.encoder.layers.0.self_attn.q_proj.weight", "visual_projection.weight", "text_projection.weight"):
        cos = float(torch.nn.functional.cosine_similarity(named[k].grad.detach().flatten().cpu(), sdo[k].grad.flatten(), dim=0))
        assert cos > GRAD_COSINE, (k, cos)


@pytest.mark.parametrize("N", [16, 96])
def test_gather_nce_loss_d768_against_oracle(dev, N):
    from oracle import clipvip_oracle as O
    from xpretrain_b200.optimization.loss import gather_nce_loss
    g = torch.Generator().manual_seed(N)
    v = torch.nn.functional.normalize(torch.randn(N, 768, generator=g), dim=-1)
    t = torch.nn.functional.normalize(torch.randn(N, 768, generator=g), dim=-1)
    temp = torch.tensor(4.6)
    vd, td = v.to(dev).requires_grad_(True), t.to(dev).requires_grad_(True)
    pd = temp.to(dev).requires_grad_(True)
    loss = gather_nce_loss(vd, td, pd)
    loss.backward()
    want = O.nce_learnable_temp_loss(v, t, temp)
    dv, dt, dl = O.nce_closed_form_grads(v, t, temp)
    assert abs(float(loss) - float(want)) < 2e-3 * abs(float(want))
    assert rel(vd.grad.cpu(), dv) < 6e-3 and rel(td.grad.cpu(), dt) < 6e-3
    assert abs(float(pd.grad) - float(dl)) < 6e-3 * abs(float(dl)) + 1e-4


# ------------------------------------------------------------------------------------------ full model by name
def test_vit_l14_336_by_name_trains_and_evaluates(dev):
    """The full 24 + 12-layer ViT-L/14-336 model built from its name: a checkpointed training step (gather_nce_loss, fused
    AdamW), then the retrieval metrics on eval-mode features."""
    from xpretrain_b200.modeling import VidCLIP
    from xpretrain_b200.optimization.adamw import AdamW
    from xpretrain_b200.optimization.loss import gather_nce_loss
    from xpretrain_b200.utils import metrics
    add = SimpleNamespace(type="ViP", temporal_size=12, if_use_temporal_embed=1, logit_scale_init_value=4.6, add_cls_num=3)
    torch.manual_seed(0)
    model = VidCLIP(SimpleNamespace(clip_config="openai/clip-vit-large-patch14-336", clip_weights="",
                                    clip_vision_additional_config=add)).to(dev)
    cm = model.clipmodel
    assert cm.config.num_patches == 576 and cm.config.vision.num_hidden_layers == 24
    cm.gradient_checkpointing_enable()
    model.train()
    opt = AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-5, betas=(0.9, 0.98), weight_decay=0.2)
    video, ids, mask = ragged_batch(4, 3, 24, size=336, dev=dev)
    before = cm.vision_model.embeddings.patch_embedding.weight.detach().clone()
    out = model(video=video, text_input_ids=ids, text_input_mask=mask)
    assert out["vis_features"].shape == (4, 768) and out["text_features"].shape == (4, 768)
    loss = gather_nce_loss(out["vis_features"], out["text_features"], cm.logit_scale)
    loss.backward()
    for n, p in model.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), n
    opt.step()
    torch.cuda.synchronize()
    assert torch.isfinite(loss) and not torch.equal(before, cm.vision_model.embeddings.patch_embedding.weight)
    model.eval()
    with torch.no_grad():
        vf = model.forward_video(video)
        tf = model.forward_text(ids, mask)
    sim = metrics.cal_cossim(tf.float().contiguous(), vf.float().contiguous())
    assert sim.shape == (4, 4) and bool(torch.isfinite(sim).all())
    r = metrics.compute_metrics(sim)
    assert len(r) > 0
