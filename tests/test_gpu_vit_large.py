"""H100: CLIP-ViP with ViT-L/14 towers (1024-wide vision tower with 16 heads and 14-pixel patches, 768-wide text tower and
projection) end to end: the reference goldens of tests/golden/make_golden_vit_l14.py under the calibrated rule, gradient
checkpointing, the residual-stream and uint8 variants, the image/caption branch, the losses at d = 768, the fused AdamW
and the retrieval metrics."""
import os
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu

CALIBRATION = 1.5        # ours may deviate from the fp32 reference by at most 1.5 x what the reference's own bf16 run deviates
# The loss and the logit_scale gradient (sum G Z) are each ONE sample of the logits error: the reference's own two bf16
# runs differ on them by up to 15 x.  They are bounded by the larger of the two reference deviations, with a floor of 2e-3.
SCALAR_SAMPLES = ("loss", "d vec logit_scale")
EMB_REL_L2 = 1.2e-2
GRAD_COSINE = 0.97


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


def _ocfg(image_size, v_layers, t_layers):
    from oracle import clipvip_oracle as O
    return O.ClipVipCfg(vision=O.TowerCfg(1024, 16, v_layers, 4096), text=O.TowerCfg(768, 12, t_layers, 3072),
                        image_size=image_size, patch=14, proj_dim=768)


def _model(dev, image_size, v_layers, t_layers, sd=None, stream="fp32", seed=0):
    from xpretrain_b200.modeling import VidCLIP
    from xpretrain_b200.modeling.clip_vip import ClipVipConfig, TowerConfig
    add = SimpleNamespace(type="ViP", temporal_size=12, if_use_temporal_embed=1, logit_scale_init_value=4.6, add_cls_num=3)
    mc = ClipVipConfig(vision=TowerConfig(1024, 16, v_layers, 4096), text=TowerConfig(768, 12, t_layers, 3072),
                       image_size=image_size, patch_size=14, projection_dim=768, residual_fp32=(stream != "bf16"),
                       residual_dtype=("fp16" if stream == "fp16" else "fp32"))
    torch.manual_seed(seed)
    model = VidCLIP(SimpleNamespace(clip_config=mc, clip_weights="", clip_vision_additional_config=add))
    if sd is not None:
        missing, unexpected = model.clipmodel.load_state_dict(sd, strict=False)
        assert not missing and not unexpected, (missing, unexpected)
    return model.to(dev)


# ------------------------------------------------------------------------------------------ reference goldens
def _unpack(e):
    return e["data"].float() * e["scale"]


def _errors(gold, vis, txt, loss, grads):
    e = {"vis": _rel(vis, gold["vis_features"]), "txt": _rel(txt, gold["text_features"]),
         "logits": _rel(vis @ txt.t(), gold["vis_features"] @ gold["text_features"].t()),
         "loss": abs(loss - float(gold["loss"])) / abs(float(gold["loss"]))}
    for k, ent in gold["grad_full"].items():
        e["d " + k] = _rel(grads[k[:-len("[rows]")]][ent["rows"]], _unpack(ent))
    vec = [(k, _unpack(v)) for k, v in gold["grad_vectors"].items()]
    vec = [(k, g) for k, g in vec if float(g.norm()) > 1e-3 * gold["grad_norms"]["logit_scale"] and "k_proj.bias" not in k]
    for k, g in vec:            # each vector against its own bar (the same vector's error in the reference's bf16 runs)
        e["d vec " + k] = _rel(grads[k], g)
    return e


@pytest.mark.parametrize("name", ["l14_224_b2_t3_ragged", "l14_336_b2_t2"])
def test_vit_l14_golden_calibrated_against_reference_bf16(dev, golden_dir, name):
    """Features, logits and every sampled gradient within 1.5 x the deviation of the reference algorithm's own bf16-autocast
    run on the same inputs on this GPU (DESIGN.md §2)."""
    from oracle import clipvip_oracle as O
    from xpretrain_b200.optimization.loss import build_loss_func
    gold = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    meta = gold["meta"]
    cfg = _ocfg(meta["image_size"], meta["vision_layers"], meta["text_layers"])
    sd = O.init_state_dict(cfg, seed=meta["weight_seed"])
    video, ids, mask = O.synthetic_batch(meta["B"], meta["T"], meta["Lt"], cfg, seed=meta["data_seed"], ragged_text=meta["ragged"])
    assert torch.equal(ids, gold["input_ids"]) and abs(float(video.double().sum()) - gold["video_checksum"]) < 1e-6
    model = _model(dev, meta["image_size"], meta["vision_layers"], meta["text_layers"], sd)
    out = model(video=video.to(dev), text_input_ids=ids.to(dev), text_input_mask=mask.to(dev))
    loss = build_loss_func({"loss_name": "NCELearnableTempLoss"})(out["vis_features"], out["text_features"],
                                                                  model.clipmodel.logit_scale)
    loss.backward()
    torch.cuda.synchronize()
    grads = {n: p.grad.detach().float().cpu() for n, p in model.clipmodel.named_parameters()}
    ours = _errors(gold, out["vis_features"].detach().float().cpu(), out["text_features"].detach().float().cpu(),
                   float(loss), grads)
    del model, out, loss
    torch.cuda.empty_cache()
    ref = {}
    for mode in ("autocast", "pure"):
        rv, rt, rl, rg = O.run_reduced_precision(sd, video, ids, mask, cfg, dev, mode)
        ref[mode] = _errors(gold, rv, rt, rl, rg)
    print(f"\n[{name}] relative L2 vs the fp32 reference golden      ours   | reference bf16-autocast | reference all-bf16")
    for k in ours:
        print(f"  {k:72s} {ours[k]:.2e} | {ref['autocast'][k]:.2e} | {ref['pure'][k]:.2e}")
    # Only the CLS rows receive gradient from the head, so the weight gradients of the LAST layer's out_proj and fc2 are
    # rank-B outer products over the B = 2 CLS rows: like the loss, two samples of the CLS-row error, on which the
    # reference's own two bf16 runs differ up to 3x.  They are bounded by the larger of the two reference deviations.
    last = meta["vision_layers"] - 1
    rank_b = {f"d vision_model.encoder.layers.{last}.{m}.weight[rows]" for m in ("self_attn.out_proj", "mlp.fc2")}
    for k in ours:
        if k in SCALAR_SAMPLES:
            continue
        bar = max(ref["autocast"][k], ref["pure"][k]) if k in rank_b else ref["autocast"][k]
        assert ours[k] <= CALIBRATION * bar + 1e-6, (k, ours[k], ref["autocast"][k], ref["pure"][k])
    for k in (k for k in SCALAR_SAMPLES if k in ours):
        assert ours[k] <= max(CALIBRATION * max(ref["pure"][k], ref["autocast"][k]), 2e-3), (k, ours[k], ref)


# ------------------------------------------------------------------------------------------ checkpointing, streams
def _inputs(dev, B, T, Lt, size, u8=False, seed=1):
    g = torch.Generator().manual_seed(seed)
    if u8:
        video = torch.randint(0, 256, (B, T, size, size, 3), generator=g, dtype=torch.uint8)
    else:
        video = torch.randn(B, T, 3, size, size, generator=g)
    ids = torch.randint(1, 49406, (B, Lt), generator=g)
    mask = torch.ones(B, Lt, dtype=torch.long)
    eos = torch.randint(2, Lt, (B,), generator=g)
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
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    return loss.detach(), out["vis_features"].detach(), out["text_features"].detach(), grads


@pytest.mark.parametrize("stream,u8", [("fp32", False), ("fp16", False), ("bf16", False), ("fp32", True)])
def test_vit_l14_checkpointing_bit_identical(dev, stream, u8):
    """Gradient checkpointing reruns the forward kernels, the streamed attention included: loss and features are
    bit-identical with it on and off; gradients differ by atomic ordering only."""
    model = _model(dev, 224, 2, 2, stream=stream)
    model.train()
    video, ids, mask = _inputs(dev, 3, 3, 24, 224, u8=u8)
    cm = model.clipmodel
    cm.gradient_checkpointing_disable()
    off = _step(model, video, ids, mask)
    cm.gradient_checkpointing_enable()
    on = _step(model, video, ids, mask)
    assert torch.isfinite(off[0]) and torch.isfinite(off[1]).all()
    assert torch.equal(off[0], on[0]) and torch.equal(off[1], on[1]) and torch.equal(off[2], on[2])
    assert off[3].keys() == on[3].keys()
    for n, g in off[3].items():
        scale = float(g.abs().max())
        if n.endswith("k_proj.bias"):
            scale = max(scale, float(off[3][n.replace("k_proj", "q_proj")].abs().max()))
        assert float((on[3][n] - g).abs().max()) <= 1e-3 * scale + 1e-12, n


# ------------------------------------------------------------------------------------------ image/caption, losses
def test_vit_l14_image_caption_branch_against_oracle(dev):
    """Video pass plus a T = 1 image/caption pass (the streamed attention's single-frame case) at 336 px, six-term loss
    at d = 768, backward through both passes."""
    from oracle import clipvip_oracle as O
    from xpretrain_b200.optimization.loss import build_loss_func
    cfg = _ocfg(336, 1, 1)
    sd = O.init_state_dict(cfg, seed=5)
    B, T, Lt = 3, 2, 16
    video, ids, mask = O.synthetic_batch(B, T, Lt, cfg, seed=21)
    image, cap_ids, cap_mask = O.synthetic_batch(B, 1, Lt, cfg, seed=22, ragged_text=True)
    model = _model(dev, 336, 1, 1, sd)
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
        assert _rel(out[k].detach().cpu(), ref.detach()) < EMB_REL_L2, k
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
    assert _rel(vd.grad.cpu(), dv) < 6e-3 and _rel(td.grad.cpu(), dt) < 6e-3
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
    video, ids, mask = _inputs(dev, 4, 3, 24, 336)
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
