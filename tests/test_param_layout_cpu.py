"""CPU: the parameter layout each model declares (modeling/_weights.py), built on the host for small configs of all four
models.  Every parameter the Function differentiates lies in exactly one row range of one operand, padding rows come after
all parameter rows, every gradient view is 16-byte aligned, and the parameter list keeps its name order and exclusions."""
import json
from types import SimpleNamespace

import pytest
import torch

LINEAR = lambda p: [p + ".weight", p + ".bias"]  # noqa: E731


def _clip(vision_type):
    from xpretrain_b200.modeling.clip_vip import CLIPModel, ClipVipConfig, TowerConfig
    cfg = ClipVipConfig(vision=TowerConfig(64, 2, 2, 256), text=TowerConfig(32, 2, 1, 128), projection_dim=16, vocab_size=100,
                        vision_type=vision_type)
    return CLIPModel(cfg)


def _clip_names(vision_type):
    def layers(tower, n):
        out = []
        for i in range(n):
            p = f"{tower}.encoder.layers.{i}."
            out += sum((LINEAR(p + "self_attn." + x) for x in ("k_proj", "v_proj", "q_proj", "out_proj")), [])
            out += LINEAR(p + "layer_norm1") + LINEAR(p + "mlp.fc1") + LINEAR(p + "mlp.fc2") + LINEAR(p + "layer_norm2")
        return out
    e = "vision_model.embeddings."
    emb = [e + "added_cls", e + "class_embedding", e + "temporal_embedding"] if vision_type == "ViP" else [e + "class_embedding"]
    emb += [e + "patch_embedding.weight", e + "position_embedding.weight"]
    return (emb + LINEAR("vision_model.pre_layrnorm") + layers("vision_model", 2) + LINEAR("vision_model.post_layernorm")
            + ["text_model.embeddings.token_embedding.weight", "text_model.embeddings.position_embedding.weight"]
            + layers("text_model", 1) + LINEAR("text_model.final_layer_norm")
            + ["visual_projection.weight", "text_projection.weight"])                        # logit_scale left out


def _tsf(attention_type):
    from xpretrain_b200.modeling.timesformer import TimeSformer
    return TimeSformer(depth=2, num_frames=2, H=2, W=2, embed_dim=128, num_heads=2, attention_type=attention_type)


def _tsf_names(attention_type):
    names = ["pos_embed"] + ([] if attention_type == "space_only" else ["time_embed"])
    for i in range(2):
        p = f"blocks.{i}."
        names += LINEAR(p + "norm1") + LINEAR(p + "attn.qkv") + LINEAR(p + "attn.proj")
        if attention_type == "divided_space_time":
            names += (LINEAR(p + "temporal_norm1") + LINEAR(p + "temporal_attn.qkv") + LINEAR(p + "temporal_attn.proj")
                      + LINEAR(p + "temporal_fc"))
        names += LINEAR(p + "norm2") + LINEAR(p + "mlp.fc1") + LINEAR(p + "mlp.fc2")
    return names                                                                             # norm.* left out


SWIN = dict(embed_dim=64, depths=[2, 1], num_heads=[2, 4], stages=[0, 1], downsample_stages=[0],
            window_size=[[2, 3, 5], [4, 3, 5]], patch_norm=True, local_window=4)


def _swin():
    from xpretrain_b200.modeling.swin3d import SwinTransformer3D
    return SwinTransformer3D(**SWIN)


def _swin_names(prefix=""):
    names = LINEAR("patch_embed.proj") + LINEAR("patch_embed.norm")
    for i, depth in enumerate(SWIN["depths"]):
        for j in range(depth):
            p = f"layers.{i}.blocks.{j}."
            names += (LINEAR(p + "norm1") + [p + "attn.relative_position_bias_table"] + LINEAR(p + "attn.qkv")
                      + LINEAR(p + "attn.proj") + LINEAR(p + "norm2") + LINEAR(p + "mlp.fc1") + LINEAR(p + "mlp.fc2"))
        if i in SWIN["downsample_stages"]:
            names += [f"layers.{i}.downsample.reduction.weight"] + LINEAR(f"layers.{i}.downsample.norm")
    return [prefix + n for n in names + LINEAR("norm")]                                      # norm_local / local_feat_proj left out


def _lfvila(tmp_path):
    from xpretrain_b200.modeling import LFVILA_Video_Classification
    path = tmp_path / "bert_config.json"
    path.write_text(json.dumps({"hidden_size": 128}))
    return LFVILA_Video_Classification(None, SimpleNamespace(VideoEncoder=SWIN, bert_config=str(path),
                                                             DATA=SimpleNamespace(classification_labels=5)))


CASES = {
    "clip_vip": (lambda tmp: _clip("ViP"), _clip_names("ViP")),
    "clip_per_frame": (lambda tmp: _clip("CLIP"), _clip_names("CLIP")),
    "tsf_divided": (lambda tmp: _tsf("divided_space_time"), _tsf_names("divided_space_time")),
    "tsf_joint": (lambda tmp: _tsf("joint_space_time"), _tsf_names("joint_space_time")),
    "tsf_space_only": (lambda tmp: _tsf("space_only"), _tsf_names("space_only")),
    "swin3d": (lambda tmp: _swin(), _swin_names()),
    "lfvila_head": (_lfvila, LINEAR("video_global_proj") + LINEAR("video_frame_proj") + LINEAR("classifier")),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_layout_covers_every_parameter_once(case, tmp_path):
    from xpretrain_b200.modeling._weights import param_layout
    build, names = CASES[case]
    model = build(tmp_path)
    lay = param_layout(model)
    assert param_layout(model) is lay                                    # built once per device
    assert lay.names == names
    named = dict(model.named_parameters())
    assert all(p is named[n] for n, p in zip(lay.names, lay.params))
    assert set(lay.rows) == set(names)
    ranges = {}
    for n in names:
        op, r0, r1 = lay.rows[n]
        assert (r1 - r0,) + tuple(lay.shapes[op][1:]) == tuple(named[n].shape), n
        ranges.setdefault(op, []).append((r0, r1))
    assert set(ranges) == set(lay.shapes)
    for op, rs in ranges.items():
        rs.sort()
        assert rs[0][0] == 0 and all(a[1] == b[0] for a, b in zip(rs, rs[1:])), (op, rs)     # no overlap, no gap
        pad = lay.shapes[op][0] - rs[-1][1]                                                   # padding rows come last
        assert 0 <= pad < 8 and (pad == 0 or lay.shapes[op][0] % 8 == 0), (op, pad)
    grads, flats = {}, {}
    for key in lay.groups:
        flats[key] = lay.alloc_grads(key, grads)
    assert set(grads) <= set(lay.shapes)
    for op, g in grads.items():
        assert g.data_ptr() % 16 == 0 and tuple(g.shape) == lay.shapes[op] and g.dtype == torch.float32, op
    spans = sorted((g.data_ptr(), g.data_ptr() + 4 * g.numel()) for g in grads.values())
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))                               # views do not overlap
    need = [True] * len(names)
    for n, g in zip(names, lay.grads_out(grads, need)):
        op = lay.rows[n][0]
        if op in grads:
            assert tuple(g.shape) == tuple(named[n].shape)
            assert g.data_ptr() == grads[op].data_ptr() + 4 * lay.rows[n][1] * grads[op][0].numel(), n


def test_clip_vip_fuses_qkv_and_keeps_its_gradient_groups(tmp_path):
    from xpretrain_b200.modeling._weights import param_layout
    model = _clip("ViP")
    lay = param_layout(model)
    p = "vision_model.encoder.layers.1.self_attn."
    assert lay.shapes[p + "qkv.weight"] == (192, 64) and lay.shapes[p + "qkv.bias"] == (192,)
    assert [lay.rows[p + x + "_proj.weight"] for x in "qkv"] == [(p + "qkv.weight", 64 * j, 64 * (j + 1)) for j in range(3)]
    assert lay[p + "qkv.weight"].dtype == torch.bfloat16 and lay[p + "qkv.bias"].dtype == torch.float32
    # one group per encoder layer and one per tower, each with the same members and size as the q/k/v-split parameters
    keys = sorted(lay.groups)
    assert keys == sorted(["vision_model", "text_model"] + [f"vision_model.encoder.layers.{i}." for i in range(2)]
                          + ["text_model.encoder.layers.0."])
    for key in keys:
        members = [n for n in lay.names if (n.startswith(key) if key.endswith(".") else
                   (n.startswith(key + ".") and ".encoder.layers." not in n) or
                   n == ("visual_projection.weight" if key == "vision_model" else "text_projection.weight"))]
        ops_ = {lay.rows[n][0] for n in members}
        assert ops_ == {op for op, _, _ in lay.groups[key][1]}, key
        assert lay.groups[key][0] == sum((int(torch.Size(lay.shapes[op]).numel()) + 3) // 4 * 4 for op in ops_)


def test_lfvila_classifier_is_padded_to_eight_labels(tmp_path):
    from xpretrain_b200.modeling._weights import param_layout
    lay = param_layout(_lfvila(tmp_path))
    assert lay.shapes["classifier.weight"] == (8, 128) and lay.shapes["classifier.bias"] == (8,)
    assert lay["classifier.weight"].dtype == torch.bfloat16 and lay["classifier.bias"].dtype == torch.float32
    assert not lay["classifier.weight"][5:].any() and not lay["classifier.bias"][5:].any()
    grads = {}
    lay.alloc_grads("", grads)
    out = dict(zip(lay.names, lay.grads_out(grads, [True] * len(lay.names))))
    assert out["classifier.weight"].shape == (5, 128) and out["classifier.bias"].shape == (5,)
    assert out["classifier.weight"].data_ptr() == grads["classifier.weight"].data_ptr()
