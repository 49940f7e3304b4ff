"""H100: CLIP-ViP (BASELINE.json configs[0] / [1]) and the per-frame CLIP video model under the calibrated rule of DESIGN.md
§2, every gradient whole and per slice, on each residual stream.

Each case compares three runs with the fp32 oracle (oracle/clipvip_oracle.py, frame_clip_oracle.py) on this GPU, TF32 off:
  ours      the module (modeling/clip_vip.py)
  arm       the same oracle with Bf16Arm swapped into its arithmetic points: it rounds exactly where the module does, on the
            module's residual stream (fp32, fp16 or bf16), with the float64 attention arms of oracle/attention_ref.py
  autocast  the oracle under bf16 autocast: printed, never asserted
The objective is a seeded cotangent on both normalised feature matrices, sum(vis * w_v) + sum(txt * w_t), so that every row
gets a gradient of its own and nothing cancels (NCELearnableTempLoss at B <= 4 makes every gradient a projection of 16
logits' error scaled by ~100; its logit_scale gradient is held by the reference-golden tests).  Asserted:
  params    the parameters that receive a gradient are exactly the oracle's
  whole     both feature matrices and every parameter gradient: err(ours) <= 1.5 x err(arm), nothing left out
  slices    contract_harness.calibrated, with its floors: features per sample; q / k / v weight and bias per head;
            out_proj.weight per input-head column block; the vision position table per row (row 0 carries the CLS row
            and every proxy); temporal_embedding per table row; added_cls per row; patch_embedding.weight per
            (64 output channels, colour); the projections per 64 output rows; the text position table per position;
            token_embedding per id present in the batch
  zeros     token-embedding rows of ids absent from the batch, text position rows >= Lt, and text position rows past the
            longest EOS (causality: no pooled row sees them) are exactly 0
  k bias    the k third of every qkv bias gradient is zero exactly; it is held whole and per head to 1.5 x the arm plus
            a bound on the two roundings it is made of (k_bias_violations)
`pytest -s` prints each case's worst whole-tensor and slice ratio and, at the end of the module, the worst of every case.
These cases are separate tests from the reference-golden comparisons of test_gpu_parity.py, test_gpu_vit_large.py and
test_gpu_frame_clip.py: those compare with the real reference's numbers and its own bf16 runs, these with the fp32 oracle
and the module's rounding; one failing does not hide the other.  The arm and the rule live in clipvip_arm.py.
"""
import pytest
import torch

from clipvip_arm import features_objective, oracle_run, rule_violations
from clipvip_cases import b16, load_golden, module_config
from contract_harness import Report
from oracle import clipvip_oracle as O

pytestmark = pytest.mark.gpu

f32 = torch.float32
REPORT = Report("CLIP-ViP calibration: worst err / bf16-arm err per case (whole tensor, slice)", width=30,
                fmt=lambda v: f"whole {v[0][0]:.3f} ({v[0][1]})  slice {v[1][0]:.3f} ({v[1][1]})")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    REPORT.print()


def normalised_frames(u8):
    """uint8 [B, T, H, W, 3] -> the fp32 frames [B, T, 3, H, W] the module's patchify_u8 computes before rounding."""
    from xpretrain_b200 import ops
    m = torch.tensor(ops.CLIP_MEAN, dtype=f32, device=u8.device)
    s = torch.tensor(ops.CLIP_STD, dtype=f32, device=u8.device)
    return ((u8.to(f32) / 255.0 - m) / s).permute(0, 1, 4, 2, 3).contiguous()


def check_case(tag, ours, want, arm, ac, ids):
    bad, worst, worst_sl = rule_violations(tag, ours, want, arm, ac, ids)
    REPORT.record(tag, (worst, worst_sl))
    assert not bad, "\n".join(bad)


def clipvip_case(dev, tag, cfg, sd, video, ids, mask, streams=("fp32",), per_frame=False, temporal=True, pad=None, seed=0):
    """One model under the rule on each residual stream in `streams`.  video: fp32 [B, T, 3, H, W] or uint8 [B, T, H, W, 3]
    (the module takes it as is, the oracles the module's normalised frames).  pad = (video, ids, mask) of extra pairs that
    follow the case's in the module's batch only (the objective reads rows 0..B-1).  -> {stream: (ours, fp32 oracle)},
    each (vis, txt, {name: grad}) on the device."""
    from xpretrain_b200.modeling.clip_vip import CLIPModel
    B = ids.shape[0]
    if not temporal:
        sd = {k: v for k, v in sd.items() if not k.endswith("temporal_embedding")}
    video_o = normalised_frames(video.to(dev)) if video.dtype == torch.uint8 else video.to(dev)
    obj = features_objective(B, cfg.proj_dim, seed)
    want = oracle_run(sd, video_o, ids, mask, cfg, obj, "fp32", per_frame=per_frame)
    ac = oracle_run(sd, video_o, ids, mask, cfg, obj, "autocast", per_frame=per_frame)
    result = {}
    for stream in streams:
        model = CLIPModel(module_config(cfg, stream, per_frame, temporal))
        missing, unexpected = model.load_state_dict(sd, strict=False)
        assert not missing and not unexpected, (missing, unexpected)
        model = model.to(dev).train()
        v_in, i_in, m_in = video, ids, mask
        if pad is not None:
            v_in, i_in, m_in = (torch.cat([a, b]) for a, b in zip((video, ids, mask), pad))
        out = model(input_ids=i_in.to(dev), pixel_values=v_in.to(dev), attention_mask=m_in.to(dev))
        vis, txt = out["image_embeds"][:B], out["text_embeds"][:B]
        loss = obj(vis, txt, None)
        loss.backward()
        ours = (vis.detach().float(), txt.detach().float(),
                {n: p.grad.detach().float() for n, p in model.named_parameters() if p.grad is not None})
        del model, out, loss
        arm = oracle_run(sd, video_o, ids, mask, cfg, obj, "bf16", stream=stream, per_frame=per_frame)
        check_case(f"{tag} {stream}", ours, want, arm, ac, ids.to(dev))
        result[stream] = (ours, want)
    torch.cuda.empty_cache()
    return result


# ========================================================================================================== cases
GOLDEN_CASES = {  # name: (golden, streams, per frame)
    "b16_depth2_ragged": ("depth2_b3_t12_ragged", ("fp32", "fp16", "bf16"), False),
    "b16_cfg1_t4": ("cfg1_b2_t4", ("fp32",), False),
    "b16_full12": ("full12_b4_t12_ragged", ("fp32",), False),
    "l14_224": ("l14_224_b2_t3_ragged", ("fp32", "fp16"), False),
    "l14_336": ("l14_336_b2_t2", ("fp32",), False),
    "frame_b16": ("frame_clip_b16_b2_t3_ragged", ("fp32", "fp16", "bf16"), True),
    "frame_b32": ("frame_clip_b32_b8_t1", ("fp32",), True),
    "frame_l14": ("frame_clip_l14_b8_t2", ("fp32",), True),
}


def golden_case(dev, golden_dir, name, pad_to=None):
    golden, streams, per_frame = GOLDEN_CASES[name]
    _, cfg, sd, video, ids, mask = load_golden(golden_dir, golden)
    pad = None
    if pad_to is not None:
        pad = O.synthetic_batch(pad_to - ids.shape[0], video.shape[1], ids.shape[1], cfg, seed=777, ragged_text=True)
        name = name.replace("full12", f"bench{pad_to}")
    return clipvip_case(dev, name, cfg, sd, video, ids, mask, streams, per_frame, pad=pad)


@pytest.mark.parametrize("name", [n for n in GOLDEN_CASES if n not in ("b16_full12",)])
def test_golden_inputs_calibrated(dev, golden_dir, name):
    golden_case(dev, golden_dir, name)


@pytest.mark.parametrize("pad_to", [None, 64], ids=["b16_full12", "b16_bench64"])
def test_full_depth_calibrated(dev, golden_dir, pad_to):
    """The bench model, 12 + 12 layers at T = 12; with pad_to = 64 the four pairs are rows 0..3 of a 64-pair batch."""
    golden_case(dev, golden_dir, "b16_full12", pad_to)


SEEDED_CASES = {  # name: (cfg, B, T, Lt, video as uint8, temporal table, weight seed)
    "b16_t1": (b16(2, 2), 4, 1, 20, False, True, 51),
    "b16_m1": (b16(2, 2, add_cls_num=0), 3, 4, 20, False, True, 52),      # M = 1: no added_cls rows
    "b16_m8": (b16(2, 2, add_cls_num=7), 3, 4, 20, False, True, 53),
    "b16_no_temporal": (b16(2, 2), 3, 4, 20, False, False, 54),
    "b16_u8": (b16(2, 2), 3, 4, 20, True, True, 55),
    "b32": (b16(2, 2, patch=32), 4, 6, 20, False, True, 56),              # L = 49
}


@pytest.mark.parametrize("name", list(SEEDED_CASES))
def test_seeded_configs_calibrated(dev, name):
    cfg, B, T, Lt, u8, temporal, seed = SEEDED_CASES[name]
    sd = O.init_state_dict(cfg, seed=seed)
    video, ids, mask = O.synthetic_batch(B, T, Lt, cfg, seed=41, ragged_text=True)
    if u8:
        video = torch.randint(0, 256, (B, T, cfg.image_size, cfg.image_size, 3), dtype=torch.uint8,
                              generator=torch.Generator().manual_seed(42))
    clipvip_case(dev, name, cfg, sd, video, ids, mask, temporal=temporal)
