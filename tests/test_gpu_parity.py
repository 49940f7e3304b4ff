"""H100: the CUDA path (VidCLIP module -> C ABI kernels) against the CPU oracle and the golden vectors that were
generated from the real reference (tests/golden/make_golden.py).

Tolerances (bf16 compute, fp32 oracle).  BASELINE.md §3 calibrates what bf16 costs the REFERENCE ITSELF
(autocast vs its own fp32, 12 layers): embeddings rel-L2 4.4e-3 (video) / 7.9e-3 (text), loss rel-err 9.4e-4.
SURVEY.md §8c sets the bar at 2x that for tensors and cosine >= 1 - 1e-3 per row.  Integer paths (patch /
sequence order, EOS argmax, token gather) are bit-exact and covered in test_gpu_kernels.py.
"""
import os

import pytest
import torch

from clipvip_cases import (EMB_REL_L2, GRAD_COSINE, LOSS_REL, b16, golden_rule, reference_golden_case, rel,
                           small_golden_case, vidclip)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda", 0)


def test_depth2_ragged_against_reference_golden(dev, golden_dir):
    small_golden_case(dev, golden_dir, "depth2_b3_t12_ragged")


def test_cfg1_full_depth_against_reference_golden(dev, golden_dir):
    """BASELINE.json configs[0]: ViT-B/16, batch 2, 4 frames (temporal interpolation 12 -> 4), 32 tokens."""
    small_golden_case(dev, golden_dir, "cfg1_b2_t4")


def _assert_calibrated(ours, ref):
    """Full tensors (features, logits matrix, whole gradient tensors): our deviation from the fp32 reference golden may be at
    most FACTOR = 1.5 x the deviation of the REFERENCE's own bf16 path (autocast: fp32 residual stream, bf16 matmul inputs)
    on the same inputs on this GPU — tighter than SURVEY.md §8c's 2x.  With `residual_fp32=False` (bf16 residual stream) only
    the all-bf16 bar holds, which is why the fp32 stream is the default."""
    golden_rule(ours, ref, against="pure" if os.environ.get("XP_RESIDUAL_BF16") == "1" else "autocast")


def test_full_depth_t12_full_gradients_calibrated_against_reference_bf16(dev, golden_dir):
    """T = 12, 12 + 12 layers, ragged text — the BENCH model — against the golden made from the real reference
    (tests/golden/make_golden.py full12): relative L2 of the features, the logits matrix, a fixed seeded sample of whole rows
    (~12 k elements each) of fifteen weight-gradient tensors and all bias / LayerNorm gradient vectors, each CALIBRATED
    against the deviation the reference algorithm itself shows in bf16 on the same inputs on this GPU (autocast and
    all-bf16), not against a hand-set number."""
    ours, ref, _ = reference_golden_case(dev, golden_dir, "full12_b4_t12_ragged")
    _assert_calibrated(ours, ref)


def test_bench_batch64_rows_against_reference_golden(dev, golden_dir):
    """BASELINE.json configs[1] (batch 64 x 12 frames, 12 layers): the golden pairs ride in rows 0..3 of the 64-pair batch."""
    ours, ref, _ = reference_golden_case(dev, golden_dir, "full12_b4_t12_ragged", pad_to=64)
    _assert_calibrated(ours, ref)


def test_hidden_states_against_oracle(dev):
    """Layer-by-layer hidden states of a 2-layer model vs the oracle run on the host (seeded, not from goldens)."""
    from oracle import clipvip_oracle as O
    from xpretrain_b200.modeling import clip_vip as M
    from xpretrain_b200.modeling._weights import param_layout
    cfg = b16(2, 2)
    sd = O.init_state_dict(cfg, seed=11)
    video, ids, mask = O.synthetic_batch(2, 3, 16, cfg, seed=5, ragged_text=True)
    _, vh = O.vision_tower(sd, video, cfg, return_hidden=True)
    model = vidclip(cfg, sd=sd, dev=dev)
    param_layout(model.clipmodel).refresh()
    proj, sv = M._vision_fwd(model.clipmodel, video.to(dev), save=True)
    S = sv.S
    for i, want in enumerate(vh[:-1]):
        got = sv.layers[i][0].view(2, S, 768).cpu()          # saved input of layer i == hidden state i
        assert rel(got, want) < 8e-3, i
    xl, pend = sv.x_last                                          # fp32 residual stream + the last block's bf16 branch output
    last = xl.float() + (pend.float() if pend is not None else 0)
    assert rel(last.view(2, S, 768).cpu(), vh[-1]) < 1e-2


def test_full_size_properties(dev):
    """BASELINE.json configs[1] shapes (12 frames, 12 layers) at a batch the test can afford: size-independent
    properties — unit-norm rows, row i of text pairs with row i of video (permutation equivariance), determinism,
    and the loss of identical towers' outputs under a row permutation."""
    from oracle import clipvip_oracle as O
    from xpretrain_b200.optimization.loss import NCELearnableTempLoss
    cfg = O.ClipVipCfg()
    sd = O.init_state_dict(cfg, seed=0)
    model = vidclip(cfg, sd=sd, dev=dev)
    B = 8
    video, ids, mask = O.synthetic_batch(B, 12, 32, cfg, seed=77)
    video, ids, mask = video.to(dev), ids.to(dev), mask.to(dev)
    with torch.no_grad():
        o1 = model(video=video, text_input_ids=ids, text_input_mask=mask)
        o2 = model(video=video, text_input_ids=ids, text_input_mask=mask)
        perm = torch.randperm(B, device=dev)
        o3 = model(video=video[perm], text_input_ids=ids[perm], text_input_mask=mask[perm])
    for k in ("vis_features", "text_features"):
        assert torch.equal(o1[k], o2[k])                                           # deterministic
        assert float((o1[k].norm(dim=-1) - 1).abs().max()) < 1e-5                 # L2-normalised rows
        assert float((o1[k][perm] - o3[k]).abs().max()) < 1e-6                    # samples are independent
    temp = model.clipmodel.logit_scale.detach()
    l1 = NCELearnableTempLoss()(o1["vis_features"], o1["text_features"], temp)
    l3 = NCELearnableTempLoss()(o3["vis_features"], o3["text_features"], temp)
    assert abs(float(l1) - float(l3)) < 1e-4 * abs(float(l1))


def test_state_dict_round_trip(dev):
    """Checkpoint compatibility (SURVEY.md §8b): keys / shapes / dtypes equal the reference CLIPModel's."""
    from oracle import clipvip_oracle as O
    cfg = O.ClipVipCfg()
    sd = O.init_state_dict(cfg, seed=0)
    model = vidclip(cfg, sd=sd, dev=dev)
    own = model.state_dict()
    assert set(own) == {"clipmodel." + k for k in sd}
    for k, v in sd.items():
        assert own["clipmodel." + k].shape == v.shape and own["clipmodel." + k].dtype == v.dtype, k


def test_image_caption_branch_and_vsc_fc_loss_against_oracle(dev):
    """The released pre-training path (VidCLIP.py:70-79 + loss.py:288-324): video/subtitle pass plus a T = 1 frame/caption
    pass through the same towers (temporal table interpolated 12 -> 1), six-term loss, backward through both passes."""
    from oracle import clipvip_oracle as O
    from xpretrain_b200.optimization.loss import build_loss_func
    cfg = b16(1, 1)
    sd = O.init_state_dict(cfg, seed=5)
    B, T, Lt = 4, 2, 16
    video, ids, mask = O.synthetic_batch(B, T, Lt, cfg, seed=21)
    image, cap_ids, cap_mask = O.synthetic_batch(B, 1, Lt, cfg, seed=22, ragged_text=True)
    model = vidclip(cfg, sd=sd, dev=dev)
    out = model(video=video.to(dev), text_input_ids=ids.to(dev), text_input_mask=mask.to(dev), image=image.to(dev),
                caption_ids=cap_ids.to(dev), caption_masks=cap_mask.to(dev))
    assert set(out) == {"text_features", "vis_features", "img_features", "cap_features"}
    loss_fn = build_loss_func({"loss_name": "NCELearnableTempLoss_vsc_fc"})
    loss = loss_fn(out["vis_features"], out["text_features"], out["img_features"], out["cap_features"],
                   model.clipmodel.logit_scale)
    loss.backward()
    # oracle (fp32, host): the same two passes share the weights, gradients accumulate over both
    sdo = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    o1 = O.clip_vip_forward(sdo, video, ids, mask, cfg)
    o2 = O.clip_vip_forward(sdo, image.reshape(-1, 1, *image.shape[2:]), cap_ids, cap_mask, cfg)
    want = O.nce_vsc_fc_loss(o1["vis_features"], o1["text_features"], o2["vis_features"], o2["text_features"],
                             sdo["logit_scale"])
    want.backward()
    for k, ref in (("vis_features", o1["vis_features"]), ("text_features", o1["text_features"]),
                   ("img_features", o2["vis_features"]), ("cap_features", o2["text_features"])):
        assert rel(out[k].detach().cpu(), ref.detach()) < EMB_REL_L2, k
    assert abs(float(loss) - float(want)) < LOSS_REL * abs(float(want))
    named = dict(model.clipmodel.named_parameters())
    for k in ("vision_model.embeddings.temporal_embedding", "vision_model.encoder.layers.0.mlp.fc1.weight",
              "text_model.encoder.layers.0.self_attn.q_proj.weight", "visual_projection.weight", "text_projection.weight",
              "vision_model.embeddings.patch_embedding.weight"):
        got, ref = named[k].grad.detach().flatten().cpu(), sdo[k].grad.flatten()
        cos = float(torch.nn.functional.cosine_similarity(got, ref, dim=0))
        assert cos > GRAD_COSINE, (k, cos)
    assert abs(float(model.clipmodel.logit_scale.grad) - float(sdo["logit_scale"].grad)) < 0.05 * abs(float(sdo["logit_scale"].grad)) + 1e-3
