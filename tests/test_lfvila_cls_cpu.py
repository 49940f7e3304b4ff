"""CPU: LF-VILA's video classification model (lfvila_video_classification.py).  The oracle replays the goldens made from
the reference (tests/golden/make_golden_lfvila_cls.py); the module has the reference's state_dict; a stage-1-shaped
checkpoint lands in the encoder; the reference's failure modes stay errors; and there is no CPU forward path."""
import json
import os
from types import SimpleNamespace

import pytest
import torch

from oracle import lfvila_cls_oracle as L
from oracle import swin3d_oracle as SO

CASES = ("lfvila_cls_eval_b6", "lfvila_cls_train_droppath")


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


def make_config(tmp_path, cfg: SO.Swin3DCfg, n_labels: int, hidden=None):
    path = tmp_path / "bert_large_config.json"
    path.write_text(json.dumps({"hidden_size": hidden or cfg.dim(len(cfg.depths) - 1), "num_hidden_layers": 24}))
    enc = dict(patch_size=list(cfg.patch_size), embed_dim=cfg.embed_dim, depths=list(cfg.depths),
               downsample_stages=list(cfg.downsample_stages), stages=list(cfg.stages), num_heads=list(cfg.num_heads),
               window_size=[list(w) for w in cfg.window_size], patch_norm=cfg.patch_norm, local_window=cfg.local_window)
    return SimpleNamespace(VideoEncoder=enc, bert_config=str(path), DATA=SimpleNamespace(classification_labels=n_labels))


@pytest.mark.parametrize("name", CASES)
def test_oracle_replays_golden(golden_dir, name):
    gold = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    cfg = SO.Swin3DCfg(**gold["cfg"])
    sd = L.init_state_dict(cfg, gold["n_labels"], seed=gold["weight_seed"])
    video = SO.synthetic_video(gold["B"], gold["D"], gold["H"], gold["W"], cfg, seed=gold["data_seed"])
    labels = L.synthetic_labels(gold["B"], gold["n_labels"], seed=gold["data_seed"] + 2)
    assert torch.equal(labels, gold["labels"])
    if name == "lfvila_cls_eval_b6":
        assert sorted(labels.tolist()) == list(range(6))                # every class of the 6-label head
    sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    out = L.lfvila_cls_forward(sdg, video, labels, cfg, drop_masks=gold["masks"])
    g = torch.Generator().manual_seed(gold["data_seed"] + 1)
    w = {k: torch.randn(out[k].shape, generator=g) for k in ("video_global_feat", "video_frame_feat", "prediction")}
    (out["loss"] + sum((out[k] * w[k]).sum() for k in w)).backward()
    for k in ("video_global_feat", "video_frame_feat", "prediction"):
        assert _rel(out[k].detach(), gold["out"][k]) < 2e-6, k
    assert abs(float(out["loss"].detach()) - float(gold["out"]["loss"])) < 2e-6 * float(gold["out"]["loss"])
    assert torch.equal(out["acc"], gold["out"]["acc"])
    assert set(gold["grad_norms"]) == {k for k, v in sdg.items() if v.is_floating_point() and v.grad is not None}
    for n, ref in gold["grads"].items():
        got = sdg[n].grad
        got = got if got.shape == ref.shape else got[:ref.shape[0]]
        assert _rel(got, ref) < 5e-5, n


def test_module_has_the_reference_state_dict(tmp_path, golden_dir):
    from xpretrain_b200.modeling import LFVILA_Video_Classification
    gold = torch.load(os.path.join(golden_dir, "lfvila_cls_eval_b6.pt"), weights_only=False)
    cfg = SO.Swin3DCfg(**gold["cfg"])
    m = LFVILA_Video_Classification(None, make_config(tmp_path, cfg, gold["n_labels"]))
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == gold["state_dict_shapes"]
    m.load_state_dict(L.init_state_dict(cfg, gold["n_labels"], seed=0), strict=True)
    # the released config: 1024-wide features (bert_large_config.json), 180 COIN labels
    big = LFVILA_Video_Classification(None, make_config(tmp_path, SO.Swin3DCfg(), 180, hidden=1024))
    assert {k: tuple(v.shape) for k, v in big.state_dict().items()} == L.param_shapes(SO.Swin3DCfg(), 180)
    with pytest.raises(ValueError):                 # hidden_size must equal the encoder's num_features
        LFVILA_Video_Classification(None, make_config(tmp_path, cfg, 6, hidden=768))


def test_stage1_checkpoint_lands_in_the_encoder(tmp_path):
    """load_model_weights_with_mismatch (LF-VILA/src/utils/load.py:6-90 without window changes): the keys the model has,
    with the same shapes, are loaded; a stage-1 checkpoint's text tower and its heads are skipped, the classifier keeps its
    initialisation."""
    from xpretrain_b200.modeling import LFVILA_Video_Classification
    cfg = SO.Swin3DCfg(embed_dim=32, depths=(1, 1, 1), num_heads=(1, 2, 4), stages=(0, 1, 2), downsample_stages=(0, 1),
                       window_size=((2, 3, 5), (4, 3, 5), (8, 3, 5)))
    torch.manual_seed(0)
    model = LFVILA_Video_Classification(None, make_config(tmp_path, cfg, 5))
    head_before = {k: v.clone() for k, v in model.state_dict().items() if not k.startswith("video_encoder.")}
    stage1 = {"video_encoder." + k: v for k, v in SO.init_state_dict(cfg, seed=3).items()}
    g = torch.Generator().manual_seed(1)
    stage1.update({"text_encoder.bert.embeddings.word_embeddings.weight": torch.randn(30522, 128, generator=g),
                   "text_encoder.bert.encoder.layer.0.attention.self.query.weight": torch.randn(128, 128, generator=g),
                   "video_global_proj.weight": torch.randn(256, 256, generator=g),      # another width: skipped
                   "mlm_head.predictions.bias": torch.randn(30522, generator=g)})
    path = tmp_path / "lfvila_stage1.bin"
    torch.save(stage1, path)
    loaded = torch.load(path, map_location="cpu")
    own = model.state_dict()
    take = {k: v for k, v in loaded.items() if k in own and own[k].shape == v.shape}
    missing, unexpected = model.load_state_dict(take, strict=False)
    assert unexpected == [] and sorted(missing) == sorted(head_before)
    for k, v in model.state_dict().items():
        want = stage1[k] if k.startswith("video_encoder.") else head_before[k]
        assert torch.equal(v, want), k


def test_reference_failure_modes(tmp_path):
    from xpretrain_b200 import _lib
    from xpretrain_b200.modeling import LFVILA_Video_Classification
    cfg = SO.Swin3DCfg(embed_dim=32, depths=(1, 1, 1), num_heads=(1, 2, 4), stages=(0, 1, 2), downsample_stages=(0, 1),
                       window_size=((2, 3, 5), (4, 3, 5), (8, 3, 5)))
    model = LFVILA_Video_Classification(None, make_config(tmp_path, cfg, 4))
    video = torch.zeros(2, 3, 2, 64, 96)
    with pytest.raises(TypeError, match="target"):                 # CrossEntropyLoss(logits, None)
        model(video)
    with pytest.raises(TypeError, match="is_train"):               # the trainer's evaluate() call (trainer :115)
        model(video, labels=torch.zeros(2, dtype=torch.long), is_train=False)
    with pytest.raises(_lib.XpError):                              # no CPU path
        model(video, torch.zeros(2, dtype=torch.long))
