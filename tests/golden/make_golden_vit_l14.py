"""Generate the ViT-L/14 golden vectors under tests/golden/ from the REAL reference.

Needs a checkout of the reference (microsoft/XPretrain), named by XP_REFERENCE_ROOT:

    XP_REFERENCE_ROOT=<path to XPretrain> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_vit_l14.py

The pattern of make_golden.py at the openai/clip-vit-large-patch14(-336) shapes: 1024-wide vision tower with 16 heads and
14-pixel patches, 768-wide text tower, 768-wide projection.  It imports the reference's own CLIP_ViP.CLIPModel unmodified,
loads the oracle's deterministic synthetic weights, runs forward / NCELearnableTempLoss / backward in fp32 on CPU, asserts
that oracle/clipvip_oracle.py reproduces it to fp32 round-off, and stores numbers only:
    l14_224_b2_t3_ragged.pt   224 px (L = 256 patches per frame), 2 + 2 layers, batch 2, 3 frames, ragged text
    l14_336_b2_t2.pt          336 px (L = 576), 1 + 1 layers, batch 2, 2 frames
Features, loss, gradient norms, and fp16 gradients after a per-tensor max-normalisation: a seeded sample of whole rows of
the large tensors and every small (bias / LayerNorm / embedding-vector) tensor whole, so each file stays under 1 MB.  Each
file also keeps the names and shapes of the reference's state_dict at the full 24 + 12-layer depth of its checkpoint.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as G  # noqa: E402  (puts the repository and the reference on sys.path)
from oracle import clipvip_oracle as O  # noqa: E402


def l14_cfg(image_size, vision_layers, text_layers):
    return O.ClipVipCfg(vision=O.TowerCfg(1024, 16, vision_layers, 4096), text=O.TowerCfg(768, 12, text_layers, 3072),
                        image_size=image_size, patch=14, proj_dim=768)


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


def run_case(name, cfg, B, T, Lt, ragged, weight_seed, data_seed):
    from src.optimization.loss import NCELearnableTempLoss

    sd = O.init_state_dict(cfg, seed=weight_seed)
    model = G.build_reference(cfg)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all("position_ids" in m for m in missing), missing
    video, ids, mask = O.synthetic_batch(B, T, Lt, cfg, seed=data_seed, ragged_text=ragged)
    out = model(input_ids=ids, attention_mask=mask, pixel_values=video, return_loss=False, return_dict=True)
    vis, txt = out["image_embeds"], out["text_embeds"]
    loss = NCELearnableTempLoss(None)(vis, txt, model.logit_scale)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}

    # --- pin the oracle against the reference (fp32 round-off only) ---
    sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    o = O.clip_vip_forward(sdg, video, ids, mask, cfg)
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
                     image_size=cfg.image_size, patch=cfg.patch, vision_layers=cfg.vision.layers,
                     text_layers=cfg.text.layers, torch=torch.__version__),
        "input_ids": ids, "attention_mask": mask, "video_checksum": float(video.double().sum()),
        "vis_features": vis.detach(), "text_features": txt.detach(), "loss": loss.detach(),
        "grad_norms": {k: float(g.norm()) for k, g in grads.items()},
        "grad_full": full,
        "grad_vectors": {k: G._pack_f16(g) for k, g in grads.items() if g.dim() <= 1 or g.numel() <= 4096},
    }
    # the reference CLIPModel's state_dict (names and shapes) at the full depth of the checkpoint this case stands for
    with torch.device("meta"):
        full_model = G.build_reference(l14_cfg(cfg.image_size, 24, 12))
    gold["reference_state_shapes"] = {k: tuple(v.shape) for k, v in full_model.state_dict().items()}
    path = os.path.join(HERE, f"{name}.pt")
    torch.save(gold, path)
    print(f"  wrote {path} ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    run_case("l14_224_b2_t3_ragged", l14_cfg(224, 2, 2), B=2, T=3, Lt=32, ragged=True, weight_seed=5, data_seed=1414)
    run_case("l14_336_b2_t2", l14_cfg(336, 1, 1), B=2, T=2, Lt=24, ragged=False, weight_seed=6, data_seed=3336)
