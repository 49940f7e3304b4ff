"""H100: decoded uint8 frames of any size (xp_vip_resize_patchify_u8) against oracle/frame_resize_ref.py's float64 bicubic
resize, pinned on the CPU by test_frame_resize_cpu.py, and through every model entry that takes uint8 frames.

  midpoint     every output bf16 is RNE of the float64 oracle, except where that value lies within the derived bound
               KERNEL_GAMMA (r_abs + |mean|) / std of a bf16 midpoint, where either neighbour passes
  shapes       p = 14 / 16 / 32, S = 224 / 336, down- and upscaling, odd, tall, wide and 1 x 1 sources, 1 to 1536 frames,
               and a frame count whose band count exceeds 65535
  coverage     every element written, guards intact, pad columns +0; bitwise repeatable; at H = W = S the bits of
               xp_vip_patchify_u8
  alignment    misaligned frames are copied (checked on the host) and give the same bits; a misaligned output and
               out-of-range sizes are refused before any launch
  model        ViP B/16 at T = 12, the per-frame model (4-D and 5-D), L/14-336 and the uint8 image= branch: with uint8
               240 x 320 frames the patch matrix equals the float path's, fed the oracle-transformed frames, except at
               midpoint-allowed elements; features and every gradient hold the calibrated rule of DESIGN.md §2 against the
               fp32 oracle on those frames; gradient checkpointing leaves loss and features bit-identical; float frames of
               another size raise ValueError before any launch
"""
import pytest
import torch

from clipvip_arm import features_objective, oracle_run, rule_violations
from clipvip_cases import b16, l14, module_config, vidclip
from contract_harness import Guarded, Report, same_bits
from oracle import clipvip_oracle as O
from oracle import embed_ref as EMB
from oracle import frame_resize_ref as E
from oracle import frame_clip_oracle as FC

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
REPORT = Report("frame resize: midpoint-allowed elements (either neighbour passes) per case", width=40,
                fmt=lambda v: f"{v}")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    REPORT.print()


def _ops():
    from xpretrain_b200 import ops
    return ops


def _frames(dev, n, H, W, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(0, 256, (n, H, W, 3), generator=g, device=dev, dtype=torch.uint8)


def _check(key, got, frames, S, p):
    """got: the kernel's patch matrix; the midpoint rule against the oracle, pad columns +0."""
    ops = _ops()
    exact, bound = E.resize_patchify_u8_ref(frames, S, p, ops.CLIP_MEAN, ops.CLIP_STD)
    ok, multi = E.bf16_allowed(got, exact, bound)
    REPORT.record(key, int(multi.sum()))
    if not bool(ok.all()):
        w = int((~ok).reshape(-1).nonzero()[0])
        raise AssertionError(f"{key}: {int((~ok).sum())} of {ok.numel()} elements break the midpoint rule; the first at "
                             f"flat index {w}: got {float(got.reshape(-1)[w]):.7e}, exact {float(exact.reshape(-1)[w]):.7e},"
                             f" bound {float(bound.reshape(-1)[w]):.3e}")
    assert torch.all(got[:, 3 * p * p:].view(torch.int16) == 0), f"{key}: pad columns must be +0"


# ======================================================================================================== kernel
CASES = [  # (frames, H, W, S, p)
    (3, 240, 320, 224, 16),      # the retrieval configs' video_res
    (2, 240, 320, 336, 14),
    (2, 360, 640, 224, 32),
    (2, 100, 150, 336, 16),      # upscaling
    (2, 239, 317, 224, 14),      # odd
    (5, 1, 1, 224, 16),
    (1, 720, 1280, 224, 16),     # a band needs more source rows than one pass stages
    (1, 4096, 3, 224, 32),
    (1, 2, 4096, 336, 14),
    (1536, 24, 40, 32, 16),
]


@pytest.mark.parametrize("frames,H,W,S,p", CASES, ids=[f"{f}x{h}x{w}-S{s}-p{p}" for f, h, w, s, p in CASES])
def test_resize_follows_the_midpoint_rule_and_writes_exactly_the_patch_matrix(dev, frames, H, W, S, p):
    ops = _ops()
    video = _frames(dev, frames, H, W, seed=frames + H + W + S + p)
    rows, ld = frames * (S // p) ** 2, EMB.patch_pitch(p)
    out = Guarded(dev, (rows, ld), bf16)
    ops.vip_resize_patchify_u8(video, out.t, S, p)
    got = out.written(f"resize {H}x{W}->{S} p={p}")
    _check(f"{frames}x{H}x{W} -> {S} p{p}", got, video, S, p)
    again = torch.empty_like(got)
    ops.vip_resize_patchify_u8(video, again, S, p)
    assert same_bits(got, again), "not bitwise repeatable"


def test_more_than_65535_bands(dev):
    ops = _ops()
    frames, S, p = 33000, 32, 16                          # 2 bands per frame: 66000 bands
    video = _frames(dev, frames, 2, 3, seed=3)
    out = Guarded(dev, (frames * 4, EMB.patch_pitch(p)), bf16)
    ops.vip_resize_patchify_u8(video, out.t, S, p)
    _check("33000 frames (66000 bands)", out.written("66000 bands"), video, S, p)


@pytest.mark.parametrize("S,p", [(224, 14), (224, 16), (224, 32), (336, 14), (336, 16)])
def test_identity_size_has_the_bits_of_patchify_u8(dev, S, p):
    ops = _ops()
    video = _frames(dev, 3, S, S, seed=S + p)
    want = torch.empty(3 * (S // p) ** 2, EMB.patch_pitch(p), dtype=bf16, device=dev)
    ops.vip_patchify_u8(video, want, p)
    got = torch.empty_like(want)
    ops.vip_resize_patchify_u8(video, got, S, p)
    assert same_bits(got, want)


def _misaligned(t, offset_elems):
    buf = torch.empty(t.numel() + offset_elems, dtype=t.dtype, device=t.device)
    view = buf[offset_elems:].view(t.shape)
    view.copy_(t)
    return view


def _checked(monkeypatch, arg_align):
    from xpretrain_b200 import _lib
    h = _lib.lib()
    orig = h.xp_vip_resize_patchify_u8
    calls = []

    def wrapper(*args):
        for i, a in arg_align:
            assert args[i] % a == 0, f"argument {i} is misaligned ({args[i] % a} mod {a})"
        calls.append(args)
        return orig(*args)
    monkeypatch.setattr(h, "xp_vip_resize_patchify_u8", wrapper)
    return calls


def test_misaligned_frames_are_copied(dev, monkeypatch):
    ops = _ops()
    video = _frames(dev, 2, 60, 90, seed=4)
    want = torch.empty(2 * 4, 768, dtype=bf16, device=dev)
    ops.vip_resize_patchify_u8(video, want, 32, 16)
    calls = _checked(monkeypatch, [(0, 16), (1, 16)])
    got = torch.empty_like(want)
    mis = _misaligned(video, 3)
    assert mis.is_contiguous() and mis.data_ptr() % 16 != 0
    ops.vip_resize_patchify_u8(mis, got, 32, 16)
    assert len(calls) == 1 and same_bits(got, want)


@pytest.mark.parametrize("case", ["misaligned_output", "H0", "H4097", "W4097", "S4097", "S_not_multiple_of_p"])
def test_refusals_launch_nothing(dev, case):
    from xpretrain_b200 import _lib
    ops = _ops()
    H, W, S, p = 24, 40, 32, 16
    if case == "H0":
        H = 0
    elif case == "H4097":
        H = 4097
    elif case == "W4097":
        W = 4097
    elif case == "S4097":
        S, p = 4097, 17
    elif case == "S_not_multiple_of_p":
        S = 40
    video = torch.zeros(2, H, W, 3, dtype=torch.uint8, device=dev)
    out = torch.zeros(2 * 4 * 768 + 8, dtype=bf16, device=dev)      # the sizes are refused before it is written
    out = out[4:] if case == "misaligned_output" else out
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    with pytest.raises(_lib.XpError):
        ops.vip_resize_patchify_u8(video, out, S, p)
    assert ops.launch_count() == n0


# ========================================================================================================= model
MODELS = {  # name: (oracle config, per frame, B, T)
    "vip_b16_t12": (b16(2, 1), False, 2, 12),
    "frame_b16": (b16(2, 1), True, 2, 3),
    "vip_l14_336": (l14(336, 1, 1), False, 2, 2),
}


def _setup(dev, name, seed=0):
    from xpretrain_b200.modeling.clip_vip import CLIPModel
    cfg, per_frame, B, T = MODELS[name]
    sd = (FC if per_frame else O).init_state_dict(cfg, seed=seed)
    model = CLIPModel(module_config(cfg, per_frame=per_frame))
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    _, ids, mask = O.synthetic_batch(B, T, 16, cfg, seed=seed + 1, ragged_text=True)
    frames = _frames(dev, B * T, 240, 320, seed=seed + 2).reshape(B, T, 240, 320, 3)
    ops = _ops()
    exact, bound = E.resize_frames_ref(frames, cfg.image_size, ops.CLIP_MEAN, ops.CLIP_STD)
    S = cfg.image_size
    transformed = exact.float().reshape(B, T, 3, S, S)
    return cfg, sd, model.to(dev), frames, transformed, (exact, bound), ids.to(dev), mask.to(dev)


class _Captured:
    """The patch matrices the model's patch extraction writes, in call order."""

    def __init__(self, monkeypatch):
        ops = _ops()
        self.patches = []
        for fn in ("vip_patchify", "vip_patchify_u8", "vip_resize_patchify_u8"):
            orig = getattr(ops, fn)

            def wrapper(video, patches, *a, _orig=orig, **k):
                _orig(video, patches, *a, **k)
                self.patches.append(patches.clone())
            monkeypatch.setattr(ops, fn, wrapper)


def _patch_matrices_agree(key, u8_patches, float_patches, ref, p):
    """The uint8 path's patch matrix equals the float path's except where the midpoint rule allows either neighbour."""
    exact, bound = EMB._im2col(ref[0], p), EMB._im2col(ref[1], p)
    ok, multi = E.bf16_allowed(u8_patches, exact, bound)
    assert bool(ok.all()), f"{key}: {int((~ok).sum())} elements break the midpoint rule"
    differ = u8_patches.view(torch.int16) != float_patches.view(torch.int16)
    assert not bool((differ & ~multi).any()), f"{key}: {int((differ & ~multi).sum())} elements differ off the midpoints"
    REPORT.record(f"model {key}", int(multi.sum()))


@pytest.mark.parametrize("name", list(MODELS))
def test_model_patch_matrix_matches_the_float_path(dev, monkeypatch, name):
    cfg, _, model, frames, transformed, ref, ids, mask = _setup(dev, name)
    cap = _Captured(monkeypatch)
    with torch.no_grad():
        model(input_ids=ids, pixel_values=frames, attention_mask=mask)
        model(input_ids=ids, pixel_values=transformed, attention_mask=mask)
    assert len(cap.patches) == 2
    _patch_matrices_agree(name, *cap.patches, ref, cfg.patch)


def test_per_frame_model_takes_4d_uint8_images(dev, monkeypatch):
    cfg, _, model, frames, transformed, ref, _, _ = _setup(dev, "frame_b16")
    S = cfg.image_size
    cap = _Captured(monkeypatch)
    with torch.no_grad():
        model.get_image_features(pixel_values=frames.reshape(-1, 240, 320, 3))
        model.get_image_features(pixel_values=transformed.reshape(-1, 3, S, S))
        model.get_image_features(pixel_values=frames)
    assert len(cap.patches) == 3 and same_bits(cap.patches[0], cap.patches[2])
    _patch_matrices_agree("frame_b16 4-D", cap.patches[0], cap.patches[1], ref, cfg.patch)


def test_image_branch_takes_uint8_frames(dev, monkeypatch):
    cfg, sd, _, frames, transformed, ref, ids, mask = _setup(dev, "vip_b16_t12")
    vid = vidclip(cfg, sd=sd, dev=dev)
    image, image_f = frames[:, :1].contiguous(), transformed[:, :1].contiguous()    # [B, 1, H, W, 3] / [B, 1, 3, S, S]
    cap = _Captured(monkeypatch)
    with torch.no_grad():
        vid(video=frames, text_input_ids=ids, text_input_mask=mask, image=image, caption_ids=ids[:, None],
            caption_masks=mask[:, None])
        vid.forward_video(image.reshape(-1, 1, 240, 320, 3))
        vid(video=transformed, text_input_ids=ids, text_input_mask=mask, image=image_f, caption_ids=ids[:, None],
            caption_masks=mask[:, None])
    assert len(cap.patches) == 5
    assert same_bits(cap.patches[1], cap.patches[2])
    ref_img = tuple(t.reshape(2, 12, 3, 224, 224)[:, :1].reshape(-1, 3, 224, 224) for t in ref)
    _patch_matrices_agree("image= branch", cap.patches[1], cap.patches[4], ref_img, cfg.patch)


@pytest.mark.parametrize("name", list(MODELS))
def test_model_calibrated_against_the_oracle_on_transformed_frames(dev, name):
    cfg, sd, model, frames, transformed, _, ids, mask = _setup(dev, name)
    per_frame = MODELS[name][1]
    B = ids.shape[0]
    obj = features_objective(B, cfg.proj_dim, seed=3)
    want = oracle_run(sd, transformed, ids, mask, cfg, obj, "fp32", per_frame=per_frame)
    model.train()
    out = model(input_ids=ids, pixel_values=frames, attention_mask=mask)
    obj(out["image_embeds"], out["text_embeds"], None).backward()
    ours = (out["image_embeds"].detach().float(), out["text_embeds"].detach().float(),
            {n: p.grad.detach().float() for n, p in model.named_parameters() if p.grad is not None})
    del model, out
    arm = oracle_run(sd, transformed, ids, mask, cfg, obj, "bf16", per_frame=per_frame)
    bad, _, _ = rule_violations(f"{name} uint8 240x320", ours, want, arm, None, ids)
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("name", list(MODELS))
def test_gradient_checkpointing_is_bit_identical(dev, name):
    cfg, _, model, frames, _, _, ids, mask = _setup(dev, name)
    obj = features_objective(ids.shape[0], cfg.proj_dim, seed=4)
    model.train()
    runs = []
    for ckpt in (False, True):
        (model.gradient_checkpointing_enable if ckpt else model.gradient_checkpointing_disable)()
        out = model(input_ids=ids, pixel_values=frames, attention_mask=mask)
        loss = obj(out["image_embeds"], out["text_embeds"], None)
        loss.backward()
        runs.append((loss.detach(), out["image_embeds"].detach(), out["text_embeds"].detach()))
        model.zero_grad(set_to_none=True)
    for a, b in zip(*runs):
        assert same_bits(a, b)


@pytest.mark.parametrize("name", list(MODELS))
def test_float_frames_of_another_size_raise_before_any_launch(dev, name):
    cfg, _, model, frames, _, _, ids, mask = _setup(dev, name)
    ops = _ops()
    B, T = frames.shape[:2]
    wrong = torch.zeros(B, T, 3, 240, 320, dtype=f32, device=dev)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    for video in (wrong, wrong.to(bf16), wrong.to(torch.float16)):
        with pytest.raises(ValueError):
            model(input_ids=ids, pixel_values=video, attention_mask=mask)
        with pytest.raises(ValueError):
            model.get_image_features(pixel_values=video)
    assert ops.launch_count() == n0
