"""CPU: the per-frame CLIP video model (vision_additional_config.type != "ViP", CLIP.py under VidCLIP.py:54-65).  The oracle
replays the goldens made from the reference (tests/golden/make_golden_frame_clip.py); the config records the type; the
model has the reference's state_dict names, shapes and init statistics; a plain CLIP checkpoint loads whole; and there is
still no CPU forward path."""
import os
from types import SimpleNamespace

import pytest
import torch

from clipvip_cases import b16, golden_errors, load_golden, vidclip
from oracle import clipvip_oracle as O
from oracle import frame_clip_oracle as F

CASES = {"frame_clip_b16_b2_t3_ragged": "openai/clip-vit-base-patch16", "frame_clip_b32_b8_t1": "openai/clip-vit-base-patch32",
         "frame_clip_l14_b8_t2": "openai/clip-vit-large-patch14"}


def _add(kind="meanP"):
    return SimpleNamespace(type=kind, temporal_size=12, if_use_temporal_embed=1, logit_scale_init_value=4.6, add_cls_num=3)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_replays_frame_clip_golden(golden_dir, name):
    gold, cfg, sd, video, ids, mask = load_golden(golden_dir, name)
    sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    o = F.frame_clip_forward(sdg, video, ids, mask, cfg)
    loss = O.nce_learnable_temp_loss(o["vis_features"], o["text_features"], sdg["logit_scale"])
    loss.backward()
    assert set(gold["grad_norms"]) == {k for k, v in sd.items() if v.is_floating_point()}
    e = golden_errors(gold, o["vis_features"].detach(), o["text_features"].detach(), float(loss),
                      {k: v.grad for k, v in sdg.items() if v.is_floating_point()})
    assert e["vis"] < 2e-5 and e["txt"] < 2e-5 and e["loss"] < 1e-5, e
    bad = {k: v for k, v in e.items() if k.startswith("d ") and not v < 2e-3}             # fp16 storage of the golden
    assert not bad, bad


def test_frame_mean_head_matches_single_normalisation_at_one_frame():
    g = torch.Generator().manual_seed(0)
    p = torch.randn(5, 512, generator=g, dtype=torch.float64)
    assert torch.allclose(F.frame_mean_head(p, 5, 1), O.l2_normalize(p), rtol=0, atol=1e-15)


def test_config_from_args_records_the_vision_type():
    from xpretrain_b200.modeling.vidclip import config_from_args
    cfg = config_from_args(SimpleNamespace(clip_config="openai/clip-vit-base-patch16", clip_vision_additional_config=_add()))
    assert cfg.vision_type == "meanP" and cfg.per_frame and cfg.num_global_tokens == 1
    vip = config_from_args(SimpleNamespace(clip_config="openai/clip-vit-base-patch16", clip_vision_additional_config=_add("ViP")))
    assert vip.vision_type == "ViP" and not vip.per_frame and vip.num_global_tokens == 4
    assert config_from_args(SimpleNamespace(clip_config="openai/clip-vit-base-patch16")).vision_type == "ViP"
    l14 = config_from_args(SimpleNamespace(clip_config="openai/clip-vit-large-patch14", clip_vision_additional_config=_add("seqTransf")))
    assert l14.per_frame and (l14.patch_size, l14.vision.hidden_size, l14.projection_dim) == (14, 1024, 768)


@pytest.mark.parametrize("name", sorted(CASES))
def test_vidclip_per_frame_has_reference_state_dict(golden_dir, name):
    from xpretrain_b200.modeling import VidCLIP
    args = SimpleNamespace(clip_config=CASES[name], clip_weights="", clip_vision_additional_config=_add())
    with torch.device("meta"):
        model = VidCLIP(args)
    want = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)["reference_state_shapes"]
    got = {k: tuple(v.shape) for k, v in model.clipmodel.state_dict().items()}
    assert got == want
    assert "vision_model.embeddings.added_cls" not in got and "vision_model.embeddings.temporal_embedding" not in got
    assert got["vision_model.embeddings.position_ids"] == (1, model.clipmodel.config.num_patches + 1)


def test_per_frame_init_statistics_follow_clip_py():
    """CLIPPreTrainedModel._init_weights (CLIP.py:391-434) at the ViT-B/16 widths: the measured std of each initialised tensor
    within 3 % of its formula; LayerNorms at (1, 0), Linear biases at 0, position_ids = arange(L + 1)."""
    from xpretrain_b200.modeling import VidCLIP
    torch.manual_seed(0)
    model = VidCLIP(SimpleNamespace(clip_config="openai/clip-vit-base-patch16", clip_weights="", clip_vision_additional_config=_add()))
    cm = model.clipmodel
    sd = dict(cm.named_parameters())
    ve = "vision_model.embeddings."
    want = {ve + "class_embedding": 768 ** -0.5, ve + "patch_embedding.weight": 0.02, ve + "position_embedding.weight": 0.02,
            "text_model.embeddings.token_embedding.weight": 0.02, "text_model.embeddings.position_embedding.weight": 0.02,
            "visual_projection.weight": 768 ** -0.5, "text_projection.weight": 512 ** -0.5}
    for tower, C, n in (("vision_model", 768, 12), ("text_model", 512, 12)):
        for i in (0, n - 1):
            p = f"{tower}.encoder.layers.{i}."
            for q in ("q_proj", "k_proj", "v_proj"):
                want[p + f"self_attn.{q}.weight"] = C ** -0.5 * (2 * n) ** -0.5
            want[p + "self_attn.out_proj.weight"] = C ** -0.5
            want[p + "mlp.fc1.weight"] = (2 * C) ** -0.5
            want[p + "mlp.fc2.weight"] = C ** -0.5 * (2 * n) ** -0.5
    for k, std in want.items():
        got = float(sd[k].detach().double().std())
        assert abs(got - std) < 0.03 * std, (k, got, std)
        assert abs(float(sd[k].detach().double().mean())) < 0.05 * std, k
    for n, p in cm.named_parameters():
        if "layer_norm" in n or "layrnorm" in n:
            assert torch.all(p == (1.0 if n.endswith(".weight") else 0.0)), n
        elif n.endswith(".bias"):
            assert torch.all(p == 0.0), n
    assert torch.equal(cm.vision_model.embeddings.position_ids, torch.arange(197).unsqueeze(0))
    assert float(cm.logit_scale) == pytest.approx(4.6)


def test_plain_clip_checkpoint_loads_every_key(golden_dir, tmp_path):
    """A checkpoint with exactly the reference CLIPModel's keys (an OpenAI CLIP checkpoint converted to Hugging Face names)
    loads with no missing and no unexpected key, directly and through VidCLIP's `clip_weights`."""
    from xpretrain_b200.modeling import VidCLIP
    shapes = torch.load(os.path.join(golden_dir, "frame_clip_b32_b8_t1.pt"), weights_only=False)["reference_state_shapes"]
    g = torch.Generator().manual_seed(3)
    sd = {k: (torch.arange(s[1]).unsqueeze(0) if k.endswith("position_ids") else torch.randn(s, generator=g))
          for k, s in shapes.items()}
    args = SimpleNamespace(clip_config="openai/clip-vit-base-patch32", clip_weights="", clip_vision_additional_config=_add())
    model = VidCLIP(args)
    missing, unexpected = model.clipmodel.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    path = tmp_path / "pytorch_model.bin"
    torch.save(sd, path)
    loaded = VidCLIP(SimpleNamespace(clip_config="openai/clip-vit-base-patch32", clip_weights=str(path),
                                     clip_vision_additional_config=_add()))
    for k, v in loaded.clipmodel.state_dict().items():
        if k == "logit_scale":
            assert float(v) == pytest.approx(4.6)          # VidCLIP.py:25-27 refills it from the config
        else:
            assert torch.equal(v, sd[k]), k


def test_per_frame_model_has_no_cpu_path():
    from xpretrain_b200 import _lib
    model = vidclip(b16(1, 1), per_frame=True)
    assert model.clipmodel.config.per_frame
    video = torch.randn(1, 2, 3, 224, 224)
    ids = torch.full((1, 8), 49407)
    with pytest.raises(_lib.XpError):
        model(video, ids, torch.ones(1, 8, dtype=torch.long))
    with pytest.raises(ValueError):
        model(video, ids, torch.ones(1, 8, dtype=torch.long), image=video[:, :1], caption_ids=ids[:, None],
              caption_masks=torch.ones(1, 1, 8, dtype=torch.long))
    with pytest.raises(TypeError):
        model.forward_video(video)


def test_frame_clip_flops_per_pair_close_to_vip():
    """197 tokens per frame against ViP's 196 + 4/12: the per-pair training FLOPs agree within 2 %."""
    cfg = O.ClipVipCfg()
    frame, vip = F.flops_per_pair(cfg, 12, 32), O.flops_per_pair(cfg, 12, 32)
    assert abs(frame["train"] / vip["train"] - 1.0) < 0.02
    assert frame["frame_block_fwd"] > 0 and frame["train"] > 2.9 * frame["fwd"]
