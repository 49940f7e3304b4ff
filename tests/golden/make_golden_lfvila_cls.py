"""Golden vectors for LF-VILA's video classification model (coin_cls.yaml, lvu_*_cls.yaml) from the REAL reference.

Needs a checkout of the reference, named by XP_REFERENCE_ROOT:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_lfvila_cls.py

Imports LF-VILA/src/models/lfvila_video_classification.py unmodified.  Its encoder is video_encoder.py behind the stub `timm`
/ `mmcv` modules of make_golden_swin3d.py; its other imports (the BERT tower, the text encoder, the logger, timm's ViT
Block) are stubs the model never calls, except `BertConfig`, which is transformers' own.  Loads the oracle's deterministic
weights into the reference model, runs forward + backward in fp32 on CPU (eval mode, and one training-mode case with the
reference's DropPath draws), asserts oracle/lfvila_cls_oracle.py agrees to fp32 round-off, and stores small numeric
fixtures plus the reference's state_dict names and shapes.
"""
import importlib.machinery
import importlib.util
import json
import os
import sys
import tempfile
import types
from types import SimpleNamespace

import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
REF = os.environ["XP_REFERENCE_ROOT"]     # a checkout of microsoft/XPretrain
sys.dont_write_bytecode = True

import make_golden_swin3d  # noqa: E402
from oracle import lfvila_cls_oracle as L  # noqa: E402
from oracle import swin3d_oracle as SO  # noqa: E402


def load_reference():
    ve = make_golden_swin3d.load_reference()            # stubs timm.models.layers, mmcv.runner, src, src.utils.dist
    from transformers import BertConfig

    def stub(name, **attrs):
        m = types.ModuleType(name)
        m.__spec__ = importlib.machinery.ModuleSpec(name, None)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    unused = type("Unused", (nn.Module,), {})
    stub("src.models", video_encoder=ve)
    sys.modules["src.models.video_encoder"] = ve
    stub("src.models.bert", BertConfig=BertConfig, BertModel=unused, BertOnlyMLMHead=unused, BertOnlyNSPHead=unused,
         BertForMaskedLM=unused)
    stub("src.models.text_encoder", TextEncoderForPretraining=unused)
    stub("src.utils.logger", LOGGER=SimpleNamespace(info=print, warning=print))
    stub("timm.models.vision_transformer", Block=unused)
    path = os.path.join(REF, "LF-VILA/src/models/lfvila_video_classification.py")
    spec = importlib.util.spec_from_file_location("ref_lfvila_video_classification", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def ref_config(cfg: SO.Swin3DCfg, n_labels: int, bert_json: str):
    enc = dict(patch_size=list(cfg.patch_size), embed_dim=cfg.embed_dim, depths=list(cfg.depths),
               downsample_stages=list(cfg.downsample_stages), stages=list(cfg.stages), num_heads=list(cfg.num_heads),
               window_size=[list(w) for w in cfg.window_size], patch_norm=cfg.patch_norm, local_window=cfg.local_window)
    return SimpleNamespace(VideoEncoder=enc, bert_config=bert_json, DATA=SimpleNamespace(classification_labels=n_labels))


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def head_weights(shape_out, seed):
    """Cotangents of the three feature outputs, so that every head branch (video_frame_feat included) has a gradient."""
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(s, generator=g) for k, s in shape_out.items()}


def objective(out, w):
    return out["loss"] + sum((out[k] * w[k]).sum() for k in w)


def run_case(mod, name, cfg, n_labels, B, D, H, W, weight_seed, data_seed, train=False, torch_seed=0):
    hidden = cfg.dim(len(cfg.depths) - 1)
    with tempfile.TemporaryDirectory() as tmp:
        bert_json = os.path.join(tmp, "bert_config.json")
        with open(bert_json, "w") as f:
            json.dump({"hidden_size": hidden, "model_type": "bert"}, f)
        model = mod.LFVILA_Video_Classification(None, ref_config(cfg, n_labels, bert_json))
    sd = L.init_state_dict(cfg, n_labels, seed=weight_seed)
    own = model.state_dict()
    shapes = {k: tuple(v.shape) for k, v in own.items()}
    assert shapes == L.param_shapes(cfg, n_labels), set(shapes) ^ set(L.param_shapes(cfg, n_labels))
    model.load_state_dict(sd, strict=True)
    if train:
        model.train()
    else:
        model.eval()
    video = SO.synthetic_video(B, D, H, W, cfg, seed=data_seed)
    labels = L.synthetic_labels(B, n_labels, seed=data_seed + 2)
    if train:
        torch.manual_seed(torch_seed)
    out = model(video, labels)
    w = head_weights({"video_global_feat": out["video_global_feat"].shape, "video_frame_feat": out["video_frame_feat"].shape,
                      "prediction": out["prediction"].shape}, data_seed + 1)
    objective(out, w).backward()
    ref_grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}

    masks = None
    if train:
        torch.manual_seed(torch_seed)
        masks = SO.draw_drop_masks(cfg, B, 0.2)          # SwinTransformer3D's default drop_path_rate
        assert sum(int((m == 0).sum()) for blk in masks if blk is not None for m in blk) > 0
    sdo = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    got = L.lfvila_cls_forward(sdo, video, labels, cfg, drop_masks=masks)
    objective(got, w).backward()
    for k in ("video_global_feat", "video_frame_feat", "prediction"):
        assert rel(got[k].detach(), out[k].detach()) < 2e-6, k
    assert abs(float(got["loss"].detach()) - float(out["loss"].detach())) < 2e-6 * abs(float(out["loss"].detach()))
    assert torch.equal(got["acc"], out["acc"]) and out["acc"].shape == (1,)
    worst, scale0 = 0.0, float(ref_grads["video_global_proj.weight"].norm())
    for n, gr in ref_grads.items():
        worst = max(worst, float((sdo[n].grad - gr).norm()) / max(float(gr.norm()), 1e-3 * scale0))
    assert set(ref_grads) == {n for n in sd if sd[n].is_floating_point() and sdo[n].grad is not None}
    print(f"{name}: logits {tuple(out['prediction'].shape)} loss {float(out['loss']):.5f} acc {float(out['acc']):.3f} "
          f"worst param grad {worst:.2e}")
    assert worst < 5e-5
    keep = [n for n in ref_grads if not n.startswith("video_encoder.")] + [
        "video_encoder.patch_embed.proj.weight", "video_encoder.layers.0.blocks.0.mlp.fc1.weight",
        "video_encoder.layers.2.blocks.1.attn.qkv.weight", "video_encoder.layers.5.blocks.0.attn.proj.weight",
        "video_encoder.layers.0.blocks.0.attn.relative_position_bias_table", "video_encoder.norm.weight"]
    torch.save({"cfg": vars(cfg), "n_labels": n_labels, "B": B, "D": D, "H": H, "W": W, "weight_seed": weight_seed,
                "data_seed": data_seed, "train": train, "torch_seed": torch_seed, "masks": masks, "labels": labels,
                "state_dict_shapes": shapes,
                "out": {k: out[k].detach().clone() for k in ("video_global_feat", "video_frame_feat", "prediction", "loss",
                                                               "acc")},
                # first 8 rows of the matrices, vectors and bias tables whole
                "grads": {n: (ref_grads[n][:8].clone() if ref_grads[n].dim() >= 2 and "bias_table" not in n
                              else ref_grads[n].clone()) for n in keep},
                "grad_norms": {n: float(g.norm()) for n, g in ref_grads.items()}},
               os.path.join(HERE, f"{name}.pt"))


def main():
    # the released encoder structure (embed 128, heads, windows, downsampling) at reduced depth; 4 frames of 128 x 192 px
    # end on a 2 x 3 grid, the smallest the (2, 3) pool takes
    cfg = SO.Swin3DCfg(depths=(1, 1, 2, 1, 1, 1))
    mod = load_reference()
    run_case(mod, "lfvila_cls_eval_b6", cfg, 6, B=6, D=4, H=128, W=192, weight_seed=11, data_seed=41)
    # training mode: the encoder's DropPath (drop_path_rate 0.2, the default the released configs keep) drawn in the
    # reference's torch.rand order; a 4-label head
    run_case(mod, "lfvila_cls_train_droppath", cfg, 4, B=4, D=4, H=128, W=192, weight_seed=12, data_seed=42, train=True,
             torch_seed=93)


if __name__ == "__main__":
    main()
