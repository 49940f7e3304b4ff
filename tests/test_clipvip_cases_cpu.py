"""The reference-golden reader and rule of clipvip_cases.py at their boundaries, on the CPU: golden_rule at exactly FACTOR x
the bar, the low-rank keys, the scalar samples' floor and the all-bf16 bar; golden_errors on a fabricated golden; and
load_golden on every CLIP-ViP and per-frame golden."""
import math

import pytest
import torch

from clipvip_cases import SCALAR_FLOOR, golden_errors, golden_rule, load_golden
from contract_harness import FACTOR

GOLDENS = ["cfg1_b2_t4", "depth2_b3_t12_ragged", "full12_b4_t12_ragged", "l14_224_b2_t3_ragged", "l14_336_b2_t2",
           "frame_clip_b16_b2_t3_ragged", "frame_clip_b32_b8_t1", "frame_clip_l14_b8_t2"]
ROWS = "d vision_model.encoder.layers.1.mlp.fc2.weight[rows]"


def _passes(ours, ref, **kw):
    try:
        golden_rule(ours, ref, **kw)
        return True
    except AssertionError:
        return False


def _ref(autocast, pure):
    return {"autocast": autocast, "pure": pure}


def test_rule_at_exactly_factor_times_the_bar_passes_and_just_above_fails():
    ref = _ref({"vis": 1e-3}, {"vis": 4e-3})
    at = FACTOR * 1e-3 + 1e-6
    assert _passes({"vis": at}, ref)
    assert not _passes({"vis": math.nextafter(at, 1.0)}, ref)
    assert not _passes({"vis": float("nan")}, ref)


def test_only_low_rank_keys_use_the_larger_mode():
    ref = _ref({"vis": 1e-3, ROWS: 1e-3}, {"vis": 4e-3, ROWS: 4e-3})
    at = FACTOR * 4e-3 + 1e-6
    assert _passes({ROWS: at}, ref, low_rank={ROWS})
    assert not _passes({ROWS: math.nextafter(at, 1.0)}, ref, low_rank={ROWS})
    assert not _passes({ROWS: at}, ref)
    assert not _passes({"vis": at}, ref, low_rank={ROWS})


@pytest.mark.parametrize("key", ["loss", "d vec logit_scale"])
def test_scalar_samples_use_the_larger_mode_with_a_floor(key):
    big = _ref({key: 1e-3}, {key: 4e-3})
    assert _passes({key: FACTOR * 4e-3}, big)
    assert not _passes({key: math.nextafter(FACTOR * 4e-3, 1.0)}, big)
    small = _ref({key: 1e-4}, {key: 2e-4})
    assert _passes({key: SCALAR_FLOOR}, small)
    assert not _passes({key: math.nextafter(SCALAR_FLOOR, 1.0)}, small)


def test_against_pure_switches_the_bar():
    ref = _ref({"vis": 1e-3}, {"vis": 4e-3})
    at = FACTOR * 4e-3 + 1e-6
    assert _passes({"vis": at}, ref, against="pure")
    assert not _passes({"vis": math.nextafter(at, 1.0)}, ref, against="pure")
    assert not _passes({"vis": at}, ref)


def _entry(t, rows=None):
    scale = float(t.abs().max())
    e = {"data": (t / scale).to(torch.float16), "scale": scale}
    if rows is not None:
        e["rows"] = rows
    return e


def _fabricated():
    """A two-pair golden: one weight gradient stored as rows 1 and 3, and four gradient vectors (a large one, k_proj.bias,
    one below 1e-3 x the logit_scale gradient's norm, one the caller skips) plus logit_scale's."""
    g = torch.Generator().manual_seed(0)
    vis, txt = torch.randn(2, 8, generator=g), torch.randn(2, 8, generator=g)
    w = torch.randn(4, 6, generator=g)
    vecs = {"logit_scale": torch.tensor([2.0]), "a.bias": torch.randn(6, generator=g),
            "layers.0.self_attn.k_proj.bias": torch.randn(6, generator=g), "tiny.bias": torch.full((6,), 1e-4),
            "skipped.bias": torch.randn(6, generator=g)}
    gold = {"vis_features": vis, "text_features": txt, "loss": torch.tensor(0.5),
            "grad_full": {"w[rows]": _entry(w[[1, 3]], torch.tensor([1, 3]))},
            "grad_vectors": {k: _entry(v) for k, v in vecs.items()},
            "grad_norms": {k: float(v.norm()) for k, v in vecs.items()}}
    grads = {"w": w.clone(), **{k: v.clone() for k, v in vecs.items()}}
    return gold, grads


def test_golden_errors_reads_the_rows_and_keeps_the_large_vectors():
    gold, grads = _fabricated()
    grads["w"][[0, 2]] = 7.0                                # rows the golden does not hold are not read
    grads["w"][3] *= 1.01
    grads["a.bias"] *= 0.98
    e = golden_errors(gold, gold["vis_features"] * 1.1, gold["text_features"], 0.55, grads, skip={"skipped.bias"})
    assert list(e) == ["vis", "txt", "logits", "loss", "d w[rows]", "d vec logit_scale", "d vec a.bias"]
    want_w = gold["grad_full"]["w[rows]"]
    stored = want_w["data"].float() * want_w["scale"]
    got_w = grads["w"][[1, 3]]
    assert e["d w[rows]"] == pytest.approx(float((got_w - stored).norm() / stored.norm()), rel=1e-6)
    assert e["vis"] == pytest.approx(0.1, rel=1e-5) and e["txt"] == 0.0 and e["loss"] == pytest.approx(0.1)
    assert 0.015 < e["d vec a.bias"] < 0.025
    assert "d vec skipped.bias" in golden_errors(gold, gold["vis_features"], gold["text_features"], 0.5, grads)


@pytest.mark.parametrize("key", ["w[:2]", "w", "w[rows][0]"])
def test_golden_errors_refuses_any_other_grad_full_key(key):
    gold, grads = _fabricated()
    gold["grad_full"] = {key: gold["grad_full"]["w[rows]"]}
    with pytest.raises(ValueError, match="name\\[rows\\]"):
        golden_errors(gold, gold["vis_features"], gold["text_features"], 0.5, grads)


@pytest.mark.parametrize("name", GOLDENS)
def test_load_golden_reads_every_clipvip_golden(golden_dir, name):
    """The ids, mask and video checksum are checked inside; the config and the state dict follow the meta."""
    gold, cfg, sd, video, ids, mask = load_golden(golden_dir, name)
    meta = gold["meta"]
    assert video.shape == (meta["B"], meta["T"], 3, cfg.image_size, cfg.image_size) and ids.shape == mask.shape
    assert (cfg.vision.layers, cfg.text.layers, cfg.patch) == (meta["vision_layers"], meta["text_layers"],
                                                                meta.get("patch", 16))
    assert sd["vision_model.embeddings.patch_embedding.weight"].shape == (cfg.vision.width, 3, cfg.patch, cfg.patch)
    assert ("vision_model.embeddings.temporal_embedding" in sd) == (not name.startswith("frame_clip_"))
