"""H100: LF-VILA's uint8 frame transform (xp_lfvila_frames_patchify_u8) against oracle/lfvila_frames_ref.py's float64
composite, pinned on the CPU by test_lfvila_frames_cpu.py, and through LFVILA_Video_Classification.

  midpoint     every output bf16 is RNE of the float64 oracle, except where that value lies within the derived bound
               KERNEL_GAMMA (r + |mean|) / std of a bf16 midpoint, where either neighbour passes
  shapes       val and train (boxes touching each border, flip on and off, a 1 x 1 box), downscales from 1080 x 1920,
               upscales from sources smaller than 240 x 428, odd, tall, wide and 1 x 1 frames, the 4096 limits
  coverage     every element written, guards intact, bitwise repeatable; more than 65535 work items; an input past
               2^31 bytes (16 x 32 x 1080 x 1920)
  alignment    a misaligned input is copied and gives the same bits; bad arguments are refused before any launch
  model        uint8 frames in eval and with train_crops: the patch matrix equals the float path's fed the oracle-transformed
               frames except at midpoint-allowed elements; features, loss and every gradient hold the calibrated rule of
               DESIGN.md §2 against the fp32 oracle on those frames; torch.no_grad() evaluation keeps no activations
"""
import json
import os
from types import SimpleNamespace

import pytest
import torch

from contract_harness import Guarded, Report, calibrated_model_rows, no_tf32, same_bits
from encoder_cases import _arm_core, frame_slices, param_slices
from oracle import lfvila_cls_oracle as L
from oracle import lfvila_frames_ref as R
from oracle import swin3d_oracle as SO

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
REPORT = Report("LF-VILA frames: midpoint-allowed elements (either neighbour passes) per case", width=50,
                fmt=lambda v: f"{v}")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "these tests need the H100"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    REPORT.print()


def _ops():
    from xpretrain_b200 import ops
    return ops


def _LF():
    from xpretrain_b200.modeling import lfvila_frames
    return lfvila_frames


def _clips(dev, B, N, H, W, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(0, 256, (B, N, H, W, 3), generator=g, device=dev, dtype=torch.uint8)


def _check(key, got, clips, params, stage_a, out_size):
    ops = _ops()
    exact, bound = R.patchify_ref(clips, params, stage_a, out_size, ops.IMAGENET_MEAN, ops.IMAGENET_STD)
    ok, multi = R.bf16_allowed(got, exact, bound)
    REPORT.record(key, int(multi.sum()))
    if not bool(ok.all()):
        w = int((~ok).reshape(-1).nonzero()[0])
        raise AssertionError(f"{key}: {int((~ok).sum())} of {ok.numel()} elements break the midpoint rule; the first at "
                             f"flat index {w}: got {float(got.reshape(-1)[w]):.7e}, exact {float(exact.reshape(-1)[w]):.7e},"
                             f" bound {float(bound.reshape(-1)[w]):.3e}")


def _run(dev, clips, crops, out_size, key):
    """The kernel into a guarded patch matrix: every element written, guards intact, a second run bit-identical."""
    ops = _ops()
    B, N = clips.shape[:2]
    rows = B * N * (out_size[0] // 8) * (out_size[1] // 8)
    out = Guarded(dev, (rows, 192), bf16)
    ops.lfvila_frames_patchify_u8(clips, crops.params, crops.stage_a, out_size, out.t)
    got = out.written(key)
    again = torch.empty_like(got)
    ops.lfvila_frames_patchify_u8(clips, crops.params, crops.stage_a, out_size, again)
    assert same_bits(got, again), f"{key}: not bitwise repeatable"
    return got


def _border_boxes(H, W):
    """Train boxes on an H x W frame: each corner (so each border) with flip off and on, the whole frame, a 1 x 1 box."""
    h, w = max(1, (H * 3) // 4), max(1, (W * 2) // 3)
    return [[0, 0, h, w, 0], [0, W - w, h, w, 1], [H - h, 0, h, w, 1], [H - h, W - w, h, w, 0], [0, 0, H, W, 1],
            [H // 2, W // 2, 1, 1, 0]]


# ======================================================================================================== kernel
VAL = [  # (B, N, H, W, Ho, Wo)
    (1, 2, 1080, 1920, 192, 320),
    (2, 2, 720, 1280, 192, 320),
    (2, 3, 360, 640, 192, 320),
    (2, 2, 100, 150, 192, 320),      # upscale in both stages' first step
    (2, 2, 239, 317, 192, 320),      # odd
    (3, 1, 1, 1, 192, 320),
    (1, 2, 1000, 90, 192, 320),      # tall
    (1, 2, 90, 1000, 192, 320),      # wide
    (1, 1, 4096, 2, 192, 320),
    (1, 1, 2, 4096, 192, 320),
    (1, 1, 60, 80, 4096, 8),
    (1, 1, 60, 80, 8, 4096),
    (2, 2, 240, 428, 224, 400),      # stage A the identity on the val path
]


@pytest.mark.parametrize("B,N,H,W,Ho,Wo", VAL, ids=[f"{b}x{n}x{h}x{w}-{ho}x{wo}" for b, n, h, w, ho, wo in VAL])
def test_val_follows_the_midpoint_rule(dev, B, N, H, W, Ho, Wo):
    clips = _clips(dev, B, N, H, W, seed=B + N + H + W + Ho)
    crops = _LF().eval_crops(B)
    key = f"val {B}x{N}x{H}x{W} -> {Ho}x{Wo}"
    _check(key, _run(dev, clips, crops, (Ho, Wo), key), clips, crops.params, crops.stage_a, (Ho, Wo))


TRAIN = [(1080, 1920), (360, 640), (100, 150), (239, 317), (1, 1), (1000, 90), (90, 1000), (4096, 3), (3, 4096)]


@pytest.mark.parametrize("H,W", TRAIN, ids=[f"{h}x{w}" for h, w in TRAIN])
def test_train_boxes_follow_the_midpoint_rule(dev, H, W):
    LF = _LF()
    boxes = _border_boxes(H, W)
    crops = LF.Crops(torch.tensor(boxes, dtype=torch.int32), (H, W))
    clips = _clips(dev, len(boxes), 2, H, W, seed=H * 3 + W)
    key = f"train {H}x{W} border boxes"
    _check(key, _run(dev, clips, crops, LF.INPUT_RES, key), clips, crops.params, crops.stage_a, LF.INPUT_RES)
    drawn = LF.train_crops(4, H, W, generator=torch.Generator().manual_seed(H + W))
    clips = clips[:4]
    key = f"train {H}x{W} drawn"
    _check(key, _run(dev, clips, drawn, LF.INPUT_RES, key), clips, drawn.params, drawn.stage_a, LF.INPUT_RES)


def test_more_than_65535_work_items(dev):
    B, N, H, W = 200, 8, 24, 40                          # 1600 frames x 24 bands x 2 column tiles = 76800 items
    clips = _clips(dev, B, N, H, W, seed=5)
    crops = _LF().train_crops(B, H, W, generator=torch.Generator().manual_seed(5))
    got = _run(dev, clips, crops, (192, 320), "76800 items")
    _check("76800 work items", got, clips, crops.params, crops.stage_a, (192, 320))


@pytest.mark.parametrize("mode", ["val", "train"])
def test_input_past_2_31_bytes(dev, mode):
    """The COIN batch at 1080p: 16 clips x 32 frames x 1080 x 1920 x 3 = 3.2e9 bytes.  Every clip is held to the oracle,
    the last ones lie wholly past 2^31 bytes."""
    LF, ops = _LF(), _ops()
    B, N, H, W = 16, 32, 1080, 1920
    clips = _clips(dev, B, N, H, W, seed=11)
    assert clips.numel() > 2 ** 31
    crops = LF.eval_crops(B) if mode == "val" else LF.train_crops(B, H, W, generator=torch.Generator().manual_seed(12))
    per_clip = N * 24 * 40
    out = Guarded(dev, (B * per_clip, 192), bf16)
    ops.lfvila_frames_patchify_u8(clips, crops.params, crops.stage_a, LF.INPUT_RES, out.t)
    got = out.written(f"{mode} 16x32x1080x1920")
    for b in range(B):
        _check(f"{mode} 16x32x1080x1920", got[b * per_clip:(b + 1) * per_clip], clips[b:b + 1], crops.params[b:b + 1],
               crops.stage_a, LF.INPUT_RES)


def test_misaligned_input_is_copied_and_gives_the_same_bits(dev, monkeypatch):
    from xpretrain_b200 import _lib
    LF, ops = _LF(), _ops()
    clips = _clips(dev, 2, 2, 60, 90, seed=4)
    crops = LF.train_crops(2, 60, 90, generator=torch.Generator().manual_seed(4))
    want = torch.empty(2 * 2 * 24 * 40, 192, dtype=bf16, device=dev)
    ops.lfvila_frames_patchify_u8(clips, crops.params, crops.stage_a, LF.INPUT_RES, want)
    h = _lib.lib()
    orig, calls = h.xp_lfvila_frames_patchify_u8, []

    def wrapper(*args):
        assert args[0] % 16 == 0, "the frames reach the kernel misaligned"
        calls.append(args)
        return orig(*args)
    monkeypatch.setattr(h, "xp_lfvila_frames_patchify_u8", wrapper)
    buf = torch.empty(clips.numel() + 3, dtype=torch.uint8, device=dev)
    mis = buf[3:].view(clips.shape)
    mis.copy_(clips)
    assert mis.is_contiguous() and mis.data_ptr() % 16 != 0
    got = torch.empty_like(want)
    ops.lfvila_frames_patchify_u8(mis, crops.params, crops.stage_a, LF.INPUT_RES, got)
    assert len(calls) == 1 and same_bits(got, want)


REFUSALS = ["misaligned_output", "H0", "H4097", "Wa4097", "Ho4097", "Ho_not_multiple_of_8", "patch16", "box_past_bottom",
            "box_past_right", "negative_top", "empty_box", "params_int64", "params_on_the_gpu", "params_wrong_rows"]


@pytest.mark.parametrize("case", REFUSALS)
def test_bad_arguments_are_refused_before_any_launch(dev, case):
    from xpretrain_b200 import _lib
    ops = _ops()
    H, W, stage_a, out_size, patch = 24, 40, (24, 40), (16, 32), 8
    params = torch.tensor([[0, 0, 24, 40, 0], [2, 3, 10, 20, 1]], dtype=torch.int32)
    H = {"H0": 0, "H4097": 4097}.get(case, H)
    stage_a = (24, 4097) if case == "Wa4097" else stage_a
    out_size = {"Ho4097": (4097, 32), "Ho_not_multiple_of_8": (20, 32)}.get(case, out_size)
    patch = 16 if case == "patch16" else patch
    box = {"box_past_bottom": [15, 0, 10, 5, 0], "box_past_right": [0, 31, 5, 10, 0], "negative_top": [-1, 0, 5, 5, 0],
           "empty_box": [0, 0, 0, 5, 0]}.get(case)
    if box is not None:
        params[1] = torch.tensor(box, dtype=torch.int32)
    if case == "params_int64":
        params = params.long()
    elif case == "params_on_the_gpu":
        params = params.to(dev)
    elif case == "params_wrong_rows":
        params = params[:1]
    clips = torch.zeros(2, 1, H, W, 3, dtype=torch.uint8, device=dev)
    out = torch.zeros(2 * 2 * 4 * 192 + 8, dtype=bf16, device=dev)
    out = out[4:] if case == "misaligned_output" else out
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(_lib.XpError):
        ops.lfvila_frames_patchify_u8(clips, params, stage_a, out_size, out, patch)
    assert ops.launch_count() == n0


# ========================================================================================================= model
FEATS = ("video_global_feat", "video_frame_feat", "prediction")


def _config(tmp, cfg, n_labels):
    path = os.path.join(tmp, "bert_config.json")
    with open(path, "w") as f:
        json.dump({"hidden_size": cfg.dim(len(cfg.depths) - 1)}, f)
    enc = dict(patch_size=list(cfg.patch_size), embed_dim=cfg.embed_dim, depths=list(cfg.depths),
               downsample_stages=list(cfg.downsample_stages), stages=list(cfg.stages), num_heads=list(cfg.num_heads),
               window_size=[list(w) for w in cfg.window_size], patch_norm=cfg.patch_norm, local_window=cfg.local_window)
    return SimpleNamespace(VideoEncoder=enc, bert_config=path,
                           DATA=SimpleNamespace(classification_labels=n_labels, input_res=[192, 320]))


def _oracle(sd, video, labels, w, cfg, masks, mode):
    """The classification oracle on float video: 'fp32' (the truth) or 'bf16' (the arm) -> ({output}, {name: grad})."""
    dt = bf16 if mode == "bf16" else f32
    sdo = {k: (v.detach().to(dt).requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    if masks is not None and mode == "bf16":
        masks = [None if m is None else tuple(t.to(dt) for t in m) for m in masks]
    with _arm_core(SO, mode), no_tf32():
        out = L.lfvila_cls_forward(sdo, video.to(dt), labels, cfg, drop_masks=masks)
        out = {k: v.float() for k, v in out.items()}
        (out["loss"] + sum((out[k] * w[k]).sum() for k in FEATS)).backward()
    return ({k: v.detach() for k, v in out.items()},
            {n: p.grad for n, p in sdo.items() if p.is_floating_point() and p.grad is not None})


class _Captured:
    """The patch matrices Swin-3D's patch extraction writes, in call order."""

    def __init__(self, monkeypatch):
        ops = _ops()
        self.patches = []
        for fn in ("vip_patchify", "lfvila_frames_patchify_u8"):
            orig = getattr(ops, fn)

            def wrapper(*a, _orig=orig, _fn=fn, **k):
                _orig(*a, **k)
                self.patches.append((a[1] if _fn == "vip_patchify" else a[4]).clone())
            monkeypatch.setattr(ops, fn, wrapper)


MODEL_CASES = {  # name: (B, D, H, W, train)
    "eval_360x640": (2, 4, 360, 640, False),
    "train_crops_300x500": (2, 4, 300, 500, True),
}


def _model_case(dev, tmp, name, n_labels=4):
    from xpretrain_b200.modeling import LFVILA_Video_Classification
    LF = _LF()
    B, D, H, W, train = MODEL_CASES[name]
    cfg = SO.Swin3DCfg()
    sd = L.init_state_dict(cfg, n_labels, seed=31)
    model = LFVILA_Video_Classification(None, _config(tmp, cfg, n_labels))
    model.load_state_dict(sd, strict=True)
    model = model.to(dev)
    clips = _clips(dev, B, D, H, W, seed=32)
    labels = L.synthetic_labels(B, n_labels, seed=33).to(dev)
    masks, crops = None, None
    if train:
        model.train()
        crops = LF.train_crops(B, H, W, generator=torch.Generator().manual_seed(34))
        masks = model.video_encoder.draw_drop_masks(B, dev, f32)
        model.video_encoder.forced_drop_masks = masks
    else:
        model.eval()
    used = crops if crops is not None else LF.eval_crops(B)
    ops = _ops()
    exact, bound = R.transform_ref(clips, used.params, used.stage_a, LF.INPUT_RES, ops.IMAGENET_MEAN, ops.IMAGENET_STD)
    video = exact.float().permute(0, 2, 1, 3, 4).contiguous()            # the transformed float video [B, 3, D, Ho, Wo]
    return cfg, sd, model, clips, labels, crops, masks, video, (exact, bound)


@pytest.mark.parametrize("name", list(MODEL_CASES))
def test_model_patch_matrix_matches_the_float_path(dev, tmp_path, monkeypatch, name):
    _, _, model, clips, labels, crops, _, video, (exact, bound) = _model_case(dev, str(tmp_path), name)
    cap = _Captured(monkeypatch)
    with torch.no_grad():
        model(clips, labels, crops=crops)
        model(video, labels)
    assert len(cap.patches) == 2
    u8, fl = cap.patches
    e, b = (R._im2col(t.reshape(-1, 3, 192, 320), 8) for t in (exact, bound))
    ok, multi = R.bf16_allowed(u8, e, b)
    assert bool(ok.all()), f"{name}: {int((~ok).sum())} elements break the midpoint rule"
    differ = u8.view(torch.int16) != fl.view(torch.int16)
    assert not bool((differ & ~multi).any()), f"{name}: {int((differ & ~multi).sum())} elements differ off the midpoints"
    REPORT.record(f"model {name}", int(multi.sum()))


@pytest.mark.parametrize("name", list(MODEL_CASES))
def test_model_calibrated_against_the_oracle_on_transformed_frames(dev, tmp_path, name):
    cfg, sd, model, clips, labels, crops, masks, video, _ = _model_case(dev, str(tmp_path), name)
    B = clips.shape[0]
    out = model(clips, labels, crops=crops)
    g = torch.Generator().manual_seed(35)
    w = {k: torch.randn(out[k].shape, generator=g).to(dev) for k in FEATS}
    (out["loss"] + sum((out[k] * w[k]).sum() for k in FEATS)).backward()
    assert out["prediction"].shape == (B, 4) and out["video_frame_feat"].dtype == f32
    ours = ({k: out[k].detach() for k in FEATS + ("loss",)},
            {n: p.grad for n, p in model.named_parameters() if p.grad is not None})
    sd = {k: v.to(dev) for k, v in sd.items()}
    want, arm = (_oracle(sd, video, labels, w, cfg, masks, mode) for mode in ("fp32", "bf16"))
    assert set(ours[1]) == set(want[1]), set(ours[1]) ^ set(want[1])
    rows = [(k, ours[0][k], want[0][k], arm[0][k], None) for k in FEATS]
    rows += [(n, ours[1][n], want[1][n], arm[1][n], None) for n in sorted(want[1])]
    slices = {"video_frame_feat": frame_slices(want[0]["video_frame_feat"]), **param_slices(want[1])}
    bad, _, _ = calibrated_model_rows(f"uint8 {name}", rows, slices)
    e = abs(float(ours[0]["loss"]) - float(want[0]["loss"])) / abs(float(want[0]["loss"]))
    ea = abs(float(arm[0]["loss"]) - float(want[0]["loss"])) / abs(float(want[0]["loss"]))
    if e > max(1.5 * ea, 2e-3):
        bad.append(f"{name}: loss: error {e:.3e} vs the bf16 oracle's {ea:.3e}")
    assert not bad, "\n".join(bad)


def test_float_frames_with_crops_and_other_uint8_layouts_raise_before_any_launch(dev, tmp_path):
    _, _, model, clips, labels, _, _, video, _ = _model_case(dev, str(tmp_path), "eval_360x640")
    ops, LF = _ops(), _LF()
    crops = LF.eval_crops(clips.shape[0])
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    for x, c in ((video, crops), (clips.permute(0, 4, 1, 2, 3).contiguous(), None), (clips[:, 0], None),
                 (clips[..., :2].contiguous(), None)):
        with pytest.raises(ValueError):
            model(x, labels, crops=c)
        with pytest.raises(ValueError):
            model.video_encoder(x, crops=c)
    assert ops.launch_count() == n0


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def test_no_grad_evaluation_of_uint8_frames_keeps_no_activations(dev, tmp_path):
    """Under torch.no_grad() the peak above the resident memory stays below the patch matrix + 6 x the largest activation
    (the first stage's MLP hidden layer), far under the training forward's; the outputs are those of a forward with grad."""
    from xpretrain_b200.modeling import LFVILA_Video_Classification
    cfg = SO.Swin3DCfg()
    B, D, H, W = 2, 32, 360, 640
    model = LFVILA_Video_Classification(None, _config(str(tmp_path), cfg, 180)).to(dev).eval()
    clips = _clips(dev, B, D, H, W, seed=3)
    labels = L.synthetic_labels(B, 180).to(dev)
    rows0 = B * D * 24 * 40
    bound = rows0 * 192 * 2 + 6 * rows0 * 4 * cfg.embed_dim * 2
    fn = lambda: model(clips, labels)                                      # noqa: E731
    with torch.no_grad():
        fn()                                                                # index tables and weight copies
    with torch.no_grad():
        ev, peak_eval = _peak(fn)
    tr, peak_train = _peak(fn)
    print(f"uint8 360x640: peak above resident, no_grad {peak_eval / 2**20:.0f} MiB (bound {bound / 2**20:.0f}), "
          f"training forward {peak_train / 2**20:.0f} MiB")
    assert peak_eval < bound and peak_eval < 0.35 * peak_train, (peak_eval, bound, peak_train)
    assert all(same_bits(ev[k], tr[k].detach()) for k in FEATS + ("loss", "acc"))
