"""CPU: LF-VILA's uint8 frame transform — the float64 oracle (oracle/lfvila_frames_ref.py) against the reference's own
init_transform_dict, and the crop draws of xpretrain_b200/modeling/lfvila_frames.py.

  golden       tests/golden/lfvila_frames_u8.pt (the reference's val and seeded train Compose on stored uint8 clips) is
               replayed by the oracle within the derived bound of torch's fp32 pipeline, sample by sample and as a
               whole-tensor sum; its bf16 roundings pass the midpoint rule
  draws        train_crops under the golden's seed gives the reference's boxes and flips, the central fallback included
  coordinate   torch's bilinear CPU loop rounds scale * (d + 0.5) - 0.5 once (a fused multiply-add), as the oracle and the
               kernel do; rounding the product first misses it
  taps         the kernel's 4 taps per output scatter to the oracle's composite matrix; rows sum to 1; at most 4 source
               indices per row; stage A at the frame's own size is the identity
"""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import lfvila_frames_ref as R
from xpretrain_b200.modeling import lfvila_frames as LF

GOLDEN = "lfvila_frames_u8.pt"
F32, F64 = torch.float32, torch.float64


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, GOLDEN), weights_only=False)


def _crops(gold, case, split):
    B, H, W = case["clips"].shape[0], case["H"], case["W"]
    if split == "val":
        return LF.eval_crops(B)
    return LF.train_crops(B, H, W, generator=torch.Generator().manual_seed(gold["meta"]["seed"]))


def test_golden_covers_upscales_downscales_and_the_fallback(gold):
    shapes = [(c["H"], c["W"]) for c in gold["cases"]]
    assert any(H < 240 and W < 428 for H, W in shapes) and any(H > 240 for H, W in shapes) and \
        any(W > 428 for H, W in shapes)
    assert (8, 200) in shapes and (200, 8) in shapes            # every RandomResizedCrop try fails: the central fallback
    assert gold["meta"]["input_res"] == list(LF.INPUT_RES)


@pytest.mark.parametrize("split", ["val", "train"])
@pytest.mark.parametrize("k", range(6))
def test_oracle_replays_the_reference_golden(gold, k, split):
    case = gold["cases"][k]
    crops = _crops(gold, case, split)
    exact, bound = R.transform_ref(case["clips"], crops.params, crops.stage_a, LF.INPUT_RES, gold["meta"]["mean"],
                                   gold["meta"]["std"], arithmetic="torch")
    g = case[split]
    idx = g["index"].long()
    ex, bd, got = exact.reshape(-1)[idx], bound.reshape(-1)[idx], g["values"]
    err = (got.double() - ex).abs()
    assert bool((err <= bd).all()), f"worst |err| / bound {float((err / bd).max()):.3g}"
    assert abs(g["sum"] - float(exact.sum())) <= float(bound.sum())
    ok, _ = R.bf16_allowed(got.to(torch.bfloat16), ex, bd)
    assert bool(ok.all()), f"{int((~ok).sum())} bf16 values break the midpoint rule"


@pytest.mark.parametrize("k", range(6))
def test_train_crops_reproduce_the_reference_draws(gold, k):
    case = gold["cases"][k]
    crops = _crops(gold, case, "train")
    assert crops.stage_a == (case["H"], case["W"])
    assert torch.equal(crops.params, case["train"]["draws"])


def test_fallback_boxes_are_central():
    for H, W, want in ((8, 200, [0, 94, 8, 11, 0]), (200, 8, [94, 0, 11, 8, 0])):
        got = LF.train_crops(3, H, W, generator=torch.Generator().manual_seed(7)).params
        assert torch.equal(got[:, :4], torch.tensor([want[:4]] * 3, dtype=torch.int32))


def test_train_crops_draw_from_the_default_generator_like_the_reference():
    torch.manual_seed(11)
    a = LF.train_crops(4, 360, 640).params
    b = LF.train_crops(4, 360, 640, generator=torch.Generator().manual_seed(11)).params
    assert torch.equal(a, b)


def test_eval_crops_are_the_center_crop():
    c = LF.eval_crops(3)
    assert c.stage_a == (240, 428) and c.params.dtype == torch.int32
    assert torch.equal(c.params, torch.tensor([[12, 22, 216, 385, 0]] * 3, dtype=torch.int32))


SIZES = [(1080, 240), (1920, 428), (720, 240), (1280, 428), (360, 240), (640, 428), (239, 240), (317, 428), (100, 240),
         (150, 428), (216, 192), (385, 320), (4096, 240), (3, 428), (1, 8)]


@pytest.mark.parametrize("n_in,n_out", SIZES)
def test_torch_bilinear_rounds_the_coordinate_once(n_in, n_out):
    """Impulse columns through F.interpolate give torch's weights: bit-equal to the single-rounding rule, on both axes."""
    eye = torch.eye(n_in, dtype=F32)
    got_h = F.interpolate(eye[None, None], size=(n_out, n_in), mode="bilinear", align_corners=False)[0, 0]
    got_w = F.interpolate(eye[None, None], size=(n_in, n_out), mode="bilinear", align_corners=False)[0, 0].t()
    want = R.linear_matrix(n_in, n_out).float()
    assert torch.equal(got_h, want) and torch.equal(got_w, want)


@pytest.mark.parametrize("n_in,n_out", [(1280, 428), (640, 428), (239, 240), (100, 240), (150, 428), (3, 428)])
def test_rounding_the_product_first_would_miss_torch(n_in, n_out):
    scale = torch.tensor(n_in, dtype=F32) / torch.tensor(n_out, dtype=F32)
    d = torch.arange(n_out, dtype=F32) + 0.5
    fused = (scale.to(F64) * d.to(F64) - 0.5).to(F32)
    assert not torch.equal(fused, scale * d - 0.5)          # so the bit-equality above tells the two rules apart


AXES = [  # (n_src, n_a, box0, length, n_out)
    (1080, 240, 12, 216, 192), (1920, 428, 22, 385, 320), (100, 240, 12, 216, 192), (317, 428, 22, 385, 320),
    (4096, 240, 0, 240, 8), (1, 240, 12, 216, 192), (640, 640, 0, 1, 320), (640, 640, 639, 1, 320), (640, 640, 0, 640, 320),
    (360, 360, 37, 300, 192), (4096, 4096, 0, 4096, 8), (3, 3, 1, 2, 4096)]


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("n_src,n_a,box0,length,n_out", AXES)
def test_taps_scatter_to_the_composite_matrix(n_src, n_a, box0, length, n_out, flip):
    idx, w = R.composite_taps(n_src, n_a, box0, length, n_out, flip)
    m = R.axis_matrix(n_src, n_a, box0, length, n_out, flip)
    assert idx.shape == (n_out, 4) and bool((idx >= 0).all()) and bool((idx < n_src).all())
    scattered = torch.zeros(n_out, n_src, dtype=F64).scatter_add_(1, idx, w)
    assert torch.allclose(scattered, m, rtol=0, atol=1e-15)
    assert torch.allclose(m.sum(1), torch.ones(n_out, dtype=F64), rtol=0, atol=1e-14)
    assert bool(((m != 0).sum(1) <= 4).all()) and bool((w >= 0).all())


def test_identity_stage_a_has_unit_weights():
    idx, w = R.composite_taps(360, 360, 30, 300, 192)
    assert bool((w[:, 1] == 0).all()) and bool((w[:, 3] == 0).all())
    assert torch.equal(w[:, 0] + w[:, 2], torch.ones(192, dtype=F64))
    assert torch.equal(R.linear_matrix(77, 77), torch.eye(77, dtype=F64))


def test_kernel_bound_is_below_torch_bound_and_positive():
    clips = torch.randint(0, 256, (2, 2, 30, 50, 3), generator=torch.Generator().manual_seed(3), dtype=torch.uint8)
    crops = LF.eval_crops(2)
    args = (clips, crops.params, crops.stage_a, (16, 24), (0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
    ek, bk = R.transform_ref(*args)
    et, bt = R.transform_ref(*args, arithmetic="torch")
    assert torch.equal(ek, et) and bool((bk <= bt).all()) and bool((bk > 0).all())
    p_exact, p_bound = R.patchify_ref(*args)
    assert p_exact.shape == (2 * 2 * 2 * 3, 192) and torch.equal(p_exact[0, :8], ek[0, 0, 0, 0, :8])
    assert torch.equal(p_exact[1, 64:72], ek[0, 0, 1, 0, 8:16]) and torch.equal(p_bound[0, :8], bk[0, 0, 0, 0, :8])
