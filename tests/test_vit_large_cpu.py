"""CPU: the ViT-L/14 configurations (openai/clip-vit-large-patch14 and -patch14-336).  The oracle replays the goldens made
from the reference (tests/golden/make_golden_vit_l14.py), a model built from each name has the reference's state_dict, and
the patch-matrix pitch rule keeps the existing patch sizes unchanged."""
import os
from types import SimpleNamespace

import pytest
import torch

from clipvip_cases import golden_errors, load_golden
from oracle import clipvip_oracle as O

CASES = ("l14_224_b2_t3_ragged", "l14_336_b2_t2")


@pytest.mark.parametrize("name", CASES)
def test_oracle_replays_vit_l14_golden(golden_dir, name):
    gold, cfg, sd, video, ids, mask = load_golden(golden_dir, name)
    sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    o = O.clip_vip_forward(sdg, video, ids, mask, cfg)
    loss = O.nce_learnable_temp_loss(o["vis_features"], o["text_features"], sdg["logit_scale"])
    loss.backward()
    e = golden_errors(gold, o["vis_features"].detach(), o["text_features"].detach(), float(loss),
                      {k: v.grad for k, v in sdg.items() if v.is_floating_point()})
    assert e["vis"] < 2e-5 and e["txt"] < 2e-5 and e["loss"] < 1e-5, e
    bad = {k: v for k, v in e.items() if k.startswith("d ") and not v < 2e-3}             # fp16 storage of the golden
    assert not bad, bad


@pytest.mark.parametrize("name,image_size,golden", [("openai/clip-vit-large-patch14", 224, CASES[0]),
                                                    ("openai/clip-vit-large-patch14-336", 336, CASES[1])])
def test_vidclip_from_l14_name_has_reference_state_dict(golden_dir, name, image_size, golden):
    from xpretrain_b200.modeling import VidCLIP
    from xpretrain_b200.modeling.vidclip import config_from_args
    add = SimpleNamespace(type="ViP", temporal_size=12, if_use_temporal_embed=1, logit_scale_init_value=4.6, add_cls_num=3)
    args = SimpleNamespace(clip_config=name, clip_weights="", clip_vision_additional_config=add)
    cfg = config_from_args(args)
    assert (cfg.vision.hidden_size, cfg.vision.num_attention_heads, cfg.vision.num_hidden_layers,
            cfg.vision.intermediate_size) == (1024, 16, 24, 4096)
    assert (cfg.text.hidden_size, cfg.text.num_attention_heads, cfg.text.num_hidden_layers,
            cfg.text.intermediate_size) == (768, 12, 12, 3072)
    assert (cfg.patch_size, cfg.image_size, cfg.projection_dim, cfg.num_patches) == (14, image_size, 768, (image_size // 14) ** 2)
    with torch.device("meta"):
        model = VidCLIP(args)
    want = torch.load(os.path.join(golden_dir, golden + ".pt"), weights_only=False)["reference_state_shapes"]
    got = {k: tuple(v.shape) for k, v in model.clipmodel.state_dict().items()}
    assert got == want


def test_base_names_unchanged():
    from xpretrain_b200.modeling.vidclip import config_from_args
    for name, patch in (("openai/clip-vit-base-patch16", 16), ("openai/clip-vit-base-patch32", 32)):
        cfg = config_from_args(SimpleNamespace(clip_config=name))
        assert (cfg.patch_size, cfg.image_size, cfg.projection_dim, cfg.vision.hidden_size, cfg.text.hidden_size) == \
            (patch, 224, 512, 768, 512)


def test_local_config_json_wins_over_l14_name(tmp_path):
    import json
    from xpretrain_b200.modeling.vidclip import config_from_args
    d = tmp_path / "clip-vit-large-patch14"
    d.mkdir()
    (d / "config.json").write_text(json.dumps({"vision_config": {"hidden_size": 512, "patch_size": 16}, "projection_dim": 256}))
    cfg = config_from_args(SimpleNamespace(clip_config=str(d)))
    assert (cfg.vision.hidden_size, cfg.patch_size, cfg.projection_dim) == (512, 16, 256)


def test_patch_pitch_rule():
    from xpretrain_b200 import ops
    assert ops.patch_pitch(16) == 3 * 16 * 16 and ops.patch_pitch(32) == 3 * 32 * 32
    assert ops.patch_pitch(14) == 592 and ops.patch_pitch(7) == 152
    assert all(ops.patch_pitch(p) % 8 == 0 and 0 <= ops.patch_pitch(p) - 3 * p * p < 8 for p in range(1, 40))
