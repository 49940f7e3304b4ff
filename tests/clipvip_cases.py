"""The CLIP-ViP and per-frame CLIP model cases the model tests share, and the reference goldens with the rule they are held to.

  b16, l14              oracle configs (ViT-B and ViT-L/14 towers); golden_config maps a golden's meta to one, and
                        module_config maps an oracle config to the module's ClipVipConfig
  vidclip               the module built through the reference's VidCLIP(args) boundary
  ragged_batch          seeded video (float or uint8 frames) and ragged text
  train_step            one NCELearnableTempLoss step: (loss, vis, txt, {name: grad or None})
  load_golden           a golden made from the reference (tests/golden/make_golden*.py), with the seeded weights and batch
                        it was made from, checked against the ids, mask and video checksum it stores
  golden_errors         relative L2 against a golden: features, logits, loss, the grad_full rows and the kept grad_vectors
  golden_rule           the calibrated rule of DESIGN.md §2 against the reference's own bf16 runs on those errors
  reference_golden_case ours and the reference's own bf16 runs against one golden, printed as one table
  small_golden_case     the cfg1 / depth2 goldens (grad_norms / grad_samples) at the small-golden bars

The goldens come in two formats.  cfg1_b2_t4 and depth2_b3_t12_ragged hold grad_norms / grad_samples, which
small_golden_case reads; the frame-clip and ViT-L goldens hold grad_full / grad_vectors, which golden_errors reads;
full12_b4_t12_ragged holds both.
"""
import os
from types import SimpleNamespace

import torch

from contract_harness import FACTOR
from oracle import clipvip_oracle as O
from oracle import frame_clip_oracle as FC

# Small-golden bars, set from the deviation of the reference's own bf16-autocast run from its fp32 output at full depth
# (the reference-golden cases measure that deviation on the GPU they run on and calibrate against it).
EMB_REL_L2 = 1.2e-2      # about 1.5 x the reference's bf16 deviation of the text tower (the larger one)
ROW_COSINE = 1.0 - 1e-3
LOSS_REL = 1e-2          # a 2..4-pair loss at logit scale ~100 is one sample of the logits error (see golden_rule)
GRAD_COSINE = 0.97

# The loss and the logit_scale gradient (sum G Z) are each ONE sample of the logits error: the reference's own two bf16
# runs differ on them by up to 15 x.  They are bounded by the larger of the two reference deviations, with a floor.
SCALAR_SAMPLES = ("loss", "d vec logit_scale")
SCALAR_FLOOR = 2e-3


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


# ============================================================================================================ configs
def b16(v_layers, t_layers, **kw):
    return O.ClipVipCfg(vision=O.TowerCfg(768, 12, v_layers, 3072), text=O.TowerCfg(512, 8, t_layers, 2048), **kw)


def l14(image_size, v_layers, t_layers):
    return O.ClipVipCfg(vision=O.TowerCfg(1024, 16, v_layers, 4096), text=O.TowerCfg(768, 12, t_layers, 3072),
                        image_size=image_size, patch=14, proj_dim=768)


def golden_config(meta):
    """The oracle config of a CLIP-ViP or per-frame golden: ViT-L/14 towers where the patch is 14, ViT-B otherwise."""
    if meta.get("patch") == 14:
        return l14(meta["image_size"], meta["vision_layers"], meta["text_layers"])
    return b16(meta["vision_layers"], meta["text_layers"], image_size=meta.get("image_size", 224),
               patch=meta.get("patch", 16))


def module_config(cfg, stream="fp32", per_frame=False, temporal=True):
    """The module's ClipVipConfig of an oracle config, on the residual stream `stream` ("fp32", "fp16" or "bf16")."""
    from xpretrain_b200.modeling.clip_vip import ClipVipConfig, TowerConfig
    return ClipVipConfig(vision=TowerConfig(cfg.vision.width, cfg.vision.heads, cfg.vision.layers, cfg.vision.mlp),
                         text=TowerConfig(cfg.text.width, cfg.text.heads, cfg.text.layers, cfg.text.mlp),
                         image_size=cfg.image_size, patch_size=cfg.patch, projection_dim=cfg.proj_dim,
                         vocab_size=cfg.vocab, max_position_embeddings=cfg.max_text_pos, layer_norm_eps=cfg.ln_eps,
                         residual_fp32=stream != "bf16", residual_dtype="fp16" if stream == "fp16" else "fp32",
                         temporal_size=cfg.temporal_size, if_use_temporal_embed=int(temporal), add_cls_num=cfg.add_cls_num,
                         logit_scale_init_value=cfg.logit_scale_init, vision_type="meanP" if per_frame else "ViP")


# ====================================================================================================== model, batch
def vidclip(cfg, *, sd=None, stream="fp32", per_frame=False, seed=None, temporal_init=False, dev=None):
    """VidCLIP(args) for an oracle config, its vision_additional_config taken from that config.  seed: torch.manual_seed
    before construction.  temporal_init: temporal_embedding redrawn from N(0, 0.02) after construction (its init is 0,
    which would leave the temporal table's gradient path untested).  sd: loaded, every key of the module and of sd matched."""
    from xpretrain_b200.modeling import VidCLIP
    mc = module_config(cfg, stream, per_frame)
    add = SimpleNamespace(type=mc.vision_type, temporal_size=mc.temporal_size, if_use_temporal_embed=mc.if_use_temporal_embed,
                          logit_scale_init_value=mc.logit_scale_init_value, add_cls_num=mc.add_cls_num)
    if seed is not None:
        torch.manual_seed(seed)
    model = VidCLIP(SimpleNamespace(clip_config=mc, clip_weights="", clip_vision_additional_config=add))
    assert model.clipmodel.config.per_frame == per_frame
    if temporal_init:
        with torch.no_grad():
            model.clipmodel.vision_model.embeddings.temporal_embedding.normal_(0, 0.02)
    if sd is not None:
        missing, unexpected = model.clipmodel.load_state_dict(sd, strict=False)
        assert not missing and not unexpected, (missing, unexpected)        # state_dict names == the reference's
    return model if dev is None else model.to(dev)


def ragged_batch(B, T, Lt, *, size=224, u8=False, seed=1, dev=None):
    """Video [B, T, 3, size, size] from N(0, 1), or with u8 uint8 frames [B, T, size, size, 3]; text ids in [1, 49406) with
    EOS (49407) at a random position >= 2, then padding with mask 0."""
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
    if dev is not None:
        video, ids, mask = video.to(dev), ids.to(dev), mask.to(dev)
    return video, ids, mask


def train_step(model, video, ids, mask):
    """Gradients zeroed, forward, NCELearnableTempLoss, backward, synchronize.  -> (loss, vis, txt, {name: .grad clone or
    None}), named as model.named_parameters() names them."""
    from xpretrain_b200.optimization.loss import NCELearnableTempLoss
    model.zero_grad(set_to_none=True)
    out = model(video=video, text_input_ids=ids, text_input_mask=mask)
    loss = NCELearnableTempLoss()(out["vis_features"], out["text_features"], model.clipmodel.logit_scale)
    loss.backward()
    torch.cuda.synchronize()
    grads = {n: (p.grad.detach().clone() if p.grad is not None else None) for n, p in model.named_parameters()}
    return loss.detach(), out["vis_features"].detach(), out["text_features"].detach(), grads


# ============================================================================================================ goldens
def _per_frame(name):
    return name.startswith("frame_clip_")


def load_golden(golden_dir, name):
    """-> (gold, oracle config, state dict, video, ids, mask): the golden and the seeded weights and batch it was made from.
    Every golden stores its ids, mask and video checksum; they are checked here."""
    gold = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    meta = gold["meta"]
    cfg = golden_config(meta)
    sd = (FC if _per_frame(name) else O).init_state_dict(cfg, seed=meta["weight_seed"])
    video, ids, mask = O.synthetic_batch(meta["B"], meta["T"], meta["Lt"], cfg, seed=meta["data_seed"],
                                         ragged_text=meta["ragged"])
    assert torch.equal(ids, gold["input_ids"]) and torch.equal(mask, gold["attention_mask"])
    assert abs(float(video.double().sum()) - gold["video_checksum"]) < 1e-6
    return gold, cfg, sd, video, ids, mask


def _unpack(e):
    return e["data"].float() * e["scale"]


def golden_errors(gold, vis, txt, loss, grads, skip=()):
    """Relative L2 against the fp32 reference golden: features, the logits matrix, the loss (a float), every grad_full
    entry (rows of a gradient, keyed name[rows], the one form the generators write) and every gradient vector but
    k_proj.bias (analytically zero), those below 1e-3 x the logit_scale gradient's norm (round-off-sized) and `skip`.
    grads: {parameter name: gradient}."""
    e = {"vis": rel(vis, gold["vis_features"]), "txt": rel(txt, gold["text_features"]),
         "logits": rel(vis @ txt.t(), gold["vis_features"] @ gold["text_features"].t()),
         "loss": abs(loss - float(gold["loss"])) / abs(float(gold["loss"]))}
    for k, ent in gold["grad_full"].items():
        if not k.endswith("[rows]"):
            raise ValueError(f"grad_full key {k!r}: the goldens store rows of a gradient as name[rows]")
        e["d " + k] = rel(grads[k[:-len("[rows]")]][ent["rows"]], _unpack(ent))
    floor = 1e-3 * gold["grad_norms"]["logit_scale"]
    for k, ent in gold["grad_vectors"].items():
        g = _unpack(ent)
        if float(g.norm()) > floor and "k_proj.bias" not in k and k not in skip:
            e["d vec " + k] = rel(grads[k], g)          # each vector against its own bar
    return e


def low_rank_rows(meta):
    """Only the CLS rows receive gradient from the head, so the weight gradients of the last vision layer's out_proj and
    fc2 are low-rank outer products over those rows: like the loss, few samples of the CLS-row error, on which the
    reference's own two bf16 runs differ up to 3 x.  golden_rule bounds them by the larger of the two."""
    last = meta["vision_layers"] - 1
    return {f"d vision_model.encoder.layers.{last}.{m}.weight[rows]" for m in ("self_attn.out_proj", "mlp.fc2")}


def golden_rule(ours, ref, *, low_rank=(), against="autocast"):
    """ours, ref[mode]: golden_errors of the module and of the reference's own bf16 runs ("autocast": fp32 residual
    stream, bf16 matmul inputs; "pure": every tensor in bf16).  Each error is at most FACTOR x the reference's `against`
    error (+ 1e-6); the keys in low_rank against the larger of both modes; SCALAR_SAMPLES against
    max(FACTOR x the larger of both modes, SCALAR_FLOOR)."""
    bad = []
    for k, e in ours.items():
        both = max(ref["autocast"][k], ref["pure"][k])
        if k in SCALAR_SAMPLES:
            bar = max(FACTOR * both, SCALAR_FLOOR)
        else:
            bar = FACTOR * (both if k in low_rank else ref[against][k]) + 1e-6
        if not e <= bar:
            bad.append(f"{k}: {e:.3e} > {bar:.3e} (reference bf16-autocast {ref['autocast'][k]:.3e}, all-bf16 "
                       f"{ref['pure'][k]:.3e})")
    assert not bad, "\n".join(bad)


def reference_golden_case(dev, golden_dir, name, pad_to=None, skip=lambda meta: ()):
    """The module on a grad_full golden, then the reference's own bf16 runs on the same inputs on this GPU (both modes of
    run_reduced_precision); prints the three golden_errors (skip(the golden's meta) left out) as one table.  With pad_to
    the golden pairs are rows 0..B-1 of a pad_to-pair batch and the loss is taken on those rows only, so every gradient
    must still equal the reference's.  -> (ours, {"autocast": ..., "pure": ...}, the golden's meta)"""
    from xpretrain_b200.optimization.loss import build_loss_func
    gold, cfg, sd, video, ids, mask = load_golden(golden_dir, name)
    skip = skip(gold["meta"])
    B = ids.shape[0]
    model = vidclip(cfg, sd=sd, per_frame=_per_frame(name), dev=dev)
    v_in, i_in, m_in = video, ids, mask
    if pad_to is not None:
        pad = O.synthetic_batch(pad_to - B, video.shape[1], ids.shape[1], cfg, seed=777, ragged_text=True)
        v_in, i_in, m_in = (torch.cat([a, b]) for a, b in zip((video, ids, mask), pad))
    out = model(video=v_in.to(dev), text_input_ids=i_in.to(dev), text_input_mask=m_in.to(dev))
    vis, txt = out["vis_features"][:B], out["text_features"][:B]
    loss = build_loss_func({"loss_name": "NCELearnableTempLoss"})(vis, txt, model.clipmodel.logit_scale)
    loss.backward()
    torch.cuda.synchronize()
    grads = {n: p.grad.detach().float().cpu() for n, p in model.clipmodel.named_parameters()}
    ours = golden_errors(gold, vis.detach().float().cpu(), txt.detach().float().cpu(), float(loss), grads, skip)
    del model, out, vis, txt, loss
    torch.cuda.empty_cache()
    run = (FC if _per_frame(name) else O).run_reduced_precision
    ref = {mode: golden_errors(gold, *run(sd, video, ids, mask, cfg, dev, mode), skip) for mode in ("autocast", "pure")}
    tag = name if pad_to is None else f"{name}, batch {pad_to}"
    print(f"\n[{tag}] relative L2 vs the fp32 reference golden      ours   | reference bf16-autocast | reference all-bf16")
    for k in ours:
        print(f"  {k:72s} {ours[k]:.2e} | {ref['autocast'][k]:.2e} | {ref['pure'][k]:.2e}")
    return ours, ref, gold["meta"]


def small_golden_case(dev, golden_dir, name, checkpointing=False):
    """A grad_norms / grad_samples golden: features, their rows and the loss at the small-golden bars; every gradient
    present, its norm within 15 % where the golden's is at least 1e-4, and its first 256 elements at cosine > GRAD_COSINE
    with the golden's sample."""
    from xpretrain_b200.optimization.loss import build_loss_func
    gold, cfg, sd, video, ids, mask = load_golden(golden_dir, name)
    model = vidclip(cfg, sd=sd, dev=dev)
    if checkpointing:
        model.clipmodel.gradient_checkpointing_enable()
    out = model(video=video.to(dev), text_input_ids=ids.to(dev), text_input_mask=mask.to(dev))
    loss = build_loss_func({"loss_name": "NCELearnableTempLoss"})(out["vis_features"], out["text_features"],
                                                                  model.clipmodel.logit_scale)
    vis, txt = out["vis_features"].detach().cpu(), out["text_features"].detach().cpu()
    e_v, e_t = rel(vis, gold["vis_features"]), rel(txt, gold["text_features"])
    cos_v = torch.nn.functional.cosine_similarity(vis, gold["vis_features"]).min()
    cos_t = torch.nn.functional.cosine_similarity(txt, gold["text_features"]).min()
    e_l = abs(float(loss) - float(gold["loss"])) / abs(float(gold["loss"]))
    print(f"[{name}{', checkpointed' if checkpointing else ''}] vs reference golden: vis rel-L2 {e_v:.2e} (min cos "
          f"{cos_v:.6f})  txt rel-L2 {e_t:.2e} (min cos {cos_t:.6f})  loss {float(loss):.5f} vs {float(gold['loss']):.5f} "
          f"(rel {e_l:.2e})")
    assert e_v < EMB_REL_L2 and e_t < EMB_REL_L2
    assert cos_v > ROW_COSINE and cos_t > ROW_COSINE
    assert e_l < LOSS_REL
    loss.backward()
    torch.cuda.synchronize()
    named = dict(model.clipmodel.named_parameters())
    worst = (1.0, None)
    for k, gn in gold["grad_norms"].items():
        g = named[k].grad
        assert g is not None, k
        if gn < 1e-4:
            continue
        ratio = float(g.norm()) / gn
        assert 0.85 < ratio < 1.15, (k, ratio)
    for k, sample in gold["grad_samples"].items():
        got = named[k].grad.detach().flatten()[:256].cpu()
        if sample.norm() < 1e-6:
            continue
        cos = float(torch.nn.functional.cosine_similarity(got, sample, dim=0))
        if cos < worst[0]:
            worst = (cos, k)
        assert cos > GRAD_COSINE, (k, cos)
    print(f"  gradients: worst sampled cosine {worst[0]:.5f} at {worst[1]}")
