"""Generate the per-frame CLIP golden vectors under tests/golden/ from the REAL reference.

Needs a checkout of the reference (microsoft/XPretrain), named by XP_REFERENCE_ROOT:

    XP_REFERENCE_ROOT=<path to XPretrain> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_frame_clip.py

The model VidCLIP builds when `vision_additional_config.type` is not "ViP": the reference's own CLIP.CLIPModel, imported
unmodified (its unused `easydict` import is satisfied by a stub module), with VidCLIP.py:54-65 reproduced around it: the
frames folded into the batch, each frame's pooled output projected and normalised, the mean over the frames normalised
again.  It loads the oracle's deterministic synthetic weights, runs forward / NCELearnableTempLoss / backward in fp32 on
CPU, asserts that oracle/frame_clip_oracle.py reproduces it to fp32 round-off, and stores numbers only:
    frame_clip_b16_b2_t3_ragged.pt   ViT-B/16, 2 + 2 layers, batch 2, 3 frames, ragged text
    frame_clip_b32_b8_t1.pt          ViT-B/32, 1 + 1 layers, batch 8, 1 frame
    frame_clip_l14_b8_t2.pt          ViT-L/14 at 224 px (1 + 256 rows per frame), 1 + 1 layers, batch 8, 2 frames
(batch 8 gives the loss and the logits 64 entries, so their calibrated bars are not single-sample noise)
Features, loss, gradient norms and fp16 gradients after a per-tensor max-normalisation (a seeded sample of whole rows of
the large tensors, every small tensor whole), so each file stays under 1 MB.  Each file also keeps the names and shapes
of the reference CLIPModel's state_dict at the full depth of its checkpoint.
"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as G  # noqa: E402  (puts the repository and the reference on sys.path)
from oracle import clipvip_oracle as O  # noqa: E402
from oracle import frame_clip_oracle as F  # noqa: E402


def build_reference(cfg: O.ClipVipCfg):
    if "easydict" not in sys.modules:          # imported by CLIP.py, not used by the model
        stub = types.ModuleType("easydict")
        stub.EasyDict = dict
        sys.modules["easydict"] = stub
    from transformers.models.clip.configuration_clip import CLIPConfig
    import src.modeling.CLIP as ref

    tc = dict(vocab_size=cfg.vocab, hidden_size=cfg.text.width, intermediate_size=cfg.text.mlp,
              num_hidden_layers=cfg.text.layers, num_attention_heads=cfg.text.heads,
              max_position_embeddings=cfg.max_text_pos, hidden_act="quick_gelu")
    vc = dict(hidden_size=cfg.vision.width, intermediate_size=cfg.vision.mlp, num_hidden_layers=cfg.vision.layers,
              num_attention_heads=cfg.vision.heads, image_size=cfg.image_size, patch_size=cfg.patch,
              hidden_act="quick_gelu")
    hf = CLIPConfig(text_config=tc, vision_config=vc, projection_dim=cfg.proj_dim)
    hf.vision_additional_config = types.SimpleNamespace(type="meanP", temporal_size=cfg.temporal_size,
                                                        if_use_temporal_embed=1,
                                                        logit_scale_init_value=cfg.logit_scale_init,
                                                        add_cls_num=cfg.add_cls_num)
    return ref.CLIPModel(hf)


def reference_forward(model, video, ids, mask):
    """VidCLIP.forward's non-ViP branch, VidCLIP.py:54-68."""
    B, N, C, H, W = video.shape
    outputs = model(input_ids=ids, attention_mask=mask, pixel_values=video.reshape(-1, C, H, W))
    vis = model.visual_projection(outputs["vision_model_output"][1])
    vis = vis / vis.norm(dim=-1, keepdim=True)
    vis = vis.reshape(B, N, -1).mean(1)
    vis = vis / vis.norm(dim=-1, keepdim=True)
    return vis, outputs["text_embeds"]


def cfg_b(patch, vision_layers, text_layers):
    return O.ClipVipCfg(vision=O.TowerCfg(768, 12, vision_layers, 3072), text=O.TowerCfg(512, 8, text_layers, 2048),
                        patch=patch)


def cfg_l14(vision_layers, text_layers):
    return O.ClipVipCfg(vision=O.TowerCfg(1024, 16, vision_layers, 4096), text=O.TowerCfg(768, 12, text_layers, 3072),
                        patch=14, proj_dim=768)


def row_keys(cfg):
    v, t = cfg.vision.layers - 1, cfg.text.layers - 1
    return (
        "vision_model.embeddings.patch_embedding.weight", "vision_model.embeddings.position_embedding.weight",
        "vision_model.encoder.layers.0.self_attn.q_proj.weight", "vision_model.encoder.layers.0.self_attn.k_proj.weight",
        "vision_model.encoder.layers.0.self_attn.v_proj.weight", "vision_model.encoder.layers.0.mlp.fc1.weight",
        f"vision_model.encoder.layers.{v}.self_attn.out_proj.weight", f"vision_model.encoder.layers.{v}.mlp.fc2.weight",
        "text_model.encoder.layers.0.mlp.fc1.weight", f"text_model.encoder.layers.{t}.self_attn.q_proj.weight",
        "visual_projection.weight", "text_projection.weight",
    )


def run_case(name, cfg, full_cfg, B, T, Lt, ragged, weight_seed, data_seed):
    from src.optimization.loss import NCELearnableTempLoss

    sd = F.init_state_dict(cfg, seed=weight_seed)
    model = build_reference(cfg)
    missing, unexpected = model.load_state_dict(sd, strict=True)
    assert not missing and not unexpected, (missing, unexpected)
    video, ids, mask = O.synthetic_batch(B, T, Lt, cfg, seed=data_seed, ragged_text=ragged)
    vis, txt = reference_forward(model, video, ids, mask)
    loss = NCELearnableTempLoss(None)(vis, txt, model.logit_scale)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}

    # --- pin the oracle against the reference (fp32 round-off only) ---
    sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    o = F.frame_clip_forward(sdg, video, ids, mask, cfg)
    oloss = O.nce_learnable_temp_loss(o["vis_features"], o["text_features"], sdg["logit_scale"])
    oloss.backward()
    e_vis, e_txt = G.rel(o["vis_features"].detach(), vis.detach()), G.rel(o["text_features"].detach(), txt.detach())
    e_loss = abs(float(oloss) - float(loss)) / abs(float(loss))
    scale = {k: max(float(g.norm()), 1e-4 * float(sd[k].numel()) ** 0.5 * float(loss)) for k, g in grads.items()}
    errs = {k: float((sdg[k].grad - g).norm()) / scale[k] for k, g in grads.items()}
    worst_key = max(errs, key=errs.get)
    print(f"[{name}] oracle vs reference: vis {e_vis:.2e} txt {e_txt:.2e} loss {e_loss:.2e} "
          f"worst-grad {errs[worst_key]:.2e} ({worst_key})")
    assert e_vis < 2e-5 and e_txt < 2e-5 and e_loss < 1e-5 and errs[worst_key] < 5e-4, "oracle does not match the reference"

    full = {k + "[rows]": G.pack_rows(grads[k], torch.arange(grads[k].shape[0])) for k in row_keys(cfg)}
    tk = "text_model.embeddings.token_embedding.weight"
    full[tk + "[rows]"] = G.pack_rows(grads[tk], torch.unique(ids))
    gold = {
        "meta": dict(name=name, B=B, T=T, Lt=Lt, ragged=ragged, weight_seed=weight_seed, data_seed=data_seed,
                     image_size=cfg.image_size, patch=cfg.patch, vision_width=cfg.vision.width,
                     vision_layers=cfg.vision.layers, text_layers=cfg.text.layers, torch=torch.__version__),
        "input_ids": ids, "attention_mask": mask, "video_checksum": float(video.double().sum()),
        "vis_features": vis.detach(), "text_features": txt.detach(), "loss": loss.detach(),
        "grad_norms": {k: float(g.norm()) for k, g in grads.items()},
        "grad_full": full,
        "grad_vectors": {k: G._pack_f16(g) for k, g in grads.items() if g.dim() <= 1 or g.numel() <= 4096},
    }
    with torch.device("meta"):
        full_model = build_reference(full_cfg)
    gold["reference_state_shapes"] = {k: tuple(v.shape) for k, v in full_model.state_dict().items()}
    path = os.path.join(HERE, f"{name}.pt")
    torch.save(gold, path)
    print(f"  wrote {path} ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    run_case("frame_clip_b16_b2_t3_ragged", cfg_b(16, 2, 2), cfg_b(16, 12, 12), B=2, T=3, Lt=32, ragged=True,
             weight_seed=7, data_seed=1616)
    run_case("frame_clip_b32_b8_t1", cfg_b(32, 1, 1), cfg_b(32, 12, 12), B=8, T=1, Lt=24, ragged=False,
             weight_seed=8, data_seed=3232)
    run_case("frame_clip_l14_b8_t2", cfg_l14(1, 1), cfg_l14(24, 12), B=8, T=2, Lt=24, ragged=True,
             weight_seed=9, data_seed=1402)
