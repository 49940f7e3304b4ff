"""CPU: the bicubic frame-resize oracle (oracle/frame_resize_ref.py) against the reference transform, and the host-side
choice of patch extraction for decoded frames.

  golden       tests/golden/frame_resize_u8.pt (torchvision's Resize + CenterCrop + Normalize, composed as
               init_transform_dict_simple does) is replayed by the oracle within the derived bound of torch's fp32
               pipeline, sample by sample and as a whole-tensor sum; its bf16 roundings pass the midpoint rule
  interpolate  the oracle's resize agrees with F.interpolate(mode="bicubic") in fp32 at every golden shape
  routing      which (dtype, H, W, image_size) goes to the resize kernel, the unchanged kernel or ValueError
"""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import frame_resize_ref as E

GOLDEN = "frame_resize_u8.pt"
SHAPES = [(240, 320), (360, 640), (100, 150), (239, 317), (1, 1)]


def _golden(golden_dir):
    return torch.load(os.path.join(golden_dir, GOLDEN), weights_only=False)


def _frames(n, H, W, seed):
    return torch.randint(0, 256, (n, H, W, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def test_golden_covers_every_source_shape_and_size(golden_dir):
    gold = _golden(golden_dir)
    assert sorted((c["H"], c["W"], c["S"]) for c in gold["cases"]) == sorted((H, W, S) for H, W in SHAPES for S in (224, 336))


@pytest.mark.parametrize("k", range(10))
def test_oracle_replays_the_torchvision_golden(golden_dir, k):
    gold = _golden(golden_dir)
    c = gold["cases"][k]
    mean, std = gold["meta"]["mean"], gold["meta"]["std"]
    frames = _frames(gold["meta"]["frames"], c["H"], c["W"], c["seed"])
    assert int(frames.long().sum()) == c["frames_sum"], "the seeded frames changed"
    exact, bound = E.resize_frames_ref(frames, c["S"], mean, std, arithmetic="torch")
    idx = c["index"].long()
    ex, bd, got = exact.reshape(-1)[idx], bound.reshape(-1)[idx], c["values"]
    err = (got.double() - ex).abs()
    assert bool((err <= bd).all()), f"worst |err| / bound {float((err / bd).max()):.3g}"
    assert abs(c["sum"] - float(exact.sum())) <= float(bound.sum())
    ok, _ = E.bf16_allowed(got.to(torch.bfloat16), ex, bd)
    assert bool(ok.all()), f"{int((~ok).sum())} bf16 values break the midpoint rule"


@pytest.mark.parametrize("S", [224, 336])
@pytest.mark.parametrize("H,W", SHAPES)
def test_oracle_agrees_with_interpolate(H, W, S):
    frames = _frames(3, H, W, seed=H * 7 + W + S)
    r, r_abs, r_w = E.resize_ref(frames, S)
    x = frames.permute(0, 3, 1, 2).float() / 255.
    got = F.interpolate(x, size=(S, S), mode="bicubic", align_corners=False).double()
    bound = (E.TORCH_GAMMA * r_abs + E.E_W * r_w) * E.SLACK
    err = (got - r).abs()
    assert bool((err <= bound).all()), f"worst |err| / bound {float((err / bound).max()):.3g}"


def test_identity_size_is_exact():
    frames = _frames(2, 32, 32, seed=5)
    r, _, _ = E.resize_ref(frames, 32)
    assert torch.equal(r, frames.permute(0, 3, 1, 2).double() / 255.0)


def test_rne_bf16_rounds_once():
    x = torch.randn(10000, dtype=torch.float32) * 10
    assert torch.equal(E.rne_bf16(x.double()), x.to(torch.bfloat16).double())
    above_midpoint = torch.tensor([1 + 2.0 ** -8 + 2.0 ** -30], dtype=torch.float64)   # fp32 rounds it onto the midpoint
    assert float(E.rne_bf16(above_midpoint)) == 1 + 2.0 ** -7
    assert float(above_midpoint.to(torch.bfloat16)) == 1.0


def test_midpoint_rule_allows_either_neighbour_only_within_the_bound():
    mid = torch.tensor([1 + 2.0 ** -8], dtype=torch.float64)
    lo, hi = torch.tensor([1.0]), torch.tensor([1 + 2.0 ** -7])
    for b, want in ((1e-6, (True, True)), (0.0, (True, False))):      # RNE of the exact midpoint is the even 1.0
        ok = [bool(E.bf16_allowed(v.to(torch.bfloat16), mid, torch.tensor([b]))[0]) for v in (lo, hi)]
        assert tuple(ok) == want
    ok, multi = E.bf16_allowed(torch.tensor([1.0], dtype=torch.bfloat16), mid + 1e-3, torch.tensor([1e-6]))
    assert not bool(ok) and not bool(multi)


@pytest.mark.parametrize("dtype,H,W,size,want", [
    (torch.uint8, 224, 224, 224, "patchify_u8"),
    (torch.uint8, 336, 336, 336, "patchify_u8"),
    (torch.uint8, 240, 320, 224, "resize_u8"),
    (torch.uint8, 224, 224, 336, "resize_u8"),
    (torch.uint8, 224, 320, 224, "resize_u8"),
    (torch.uint8, 1, 1, 224, "resize_u8"),
    (torch.float32, 224, 224, 224, "patchify"),
    (torch.bfloat16, 336, 336, 336, "patchify"),
    (torch.float16, 224, 224, 224, "patchify"),
    (torch.float32, 240, 320, 224, ValueError),
    (torch.bfloat16, 224, 224, 336, ValueError),
    (torch.float16, 224, 225, 224, ValueError),
])
def test_frame_input_path(dtype, H, W, size, want):
    from xpretrain_b200.modeling.clip_vip import frame_input_path
    if want is ValueError:
        with pytest.raises(ValueError):
            frame_input_path(dtype, H, W, size)
    else:
        assert frame_input_path(dtype, H, W, size) == want
