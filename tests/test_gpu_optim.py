"""H100: the fused optimizer step (SURVEY.md §8(f).1) against the reference trajectory golden and the oracle."""
import os

import pytest
import torch

from oracle import adamw_oracle as AO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "these tests need the H100"
    return torch.device("cuda", 0)


def _grads(shapes, step):
    scale = 0.01 if step % 3 == 0 else 1.0
    return {n: torch.randn(s, generator=torch.Generator().manual_seed(1000 * step + i)) * scale
            for i, (n, s) in enumerate(shapes.items())}


@pytest.mark.parametrize("fused_clip", [True, False])
def test_adamw_replays_the_reference_trajectory(dev, golden_dir, fused_clip):
    from xpretrain_b200.optimization.adamw import AdamW, build_e2e_optimizer_w_lr_mul, clip_grad_norm_, get_lr_sched

    gold = torch.load(os.path.join(golden_dir, "adamw_8steps.pt"), weights_only=False)
    cfg, shapes = gold["cfg"], gold["shapes"]
    g0 = torch.Generator().manual_seed(0)
    params = {n: torch.nn.Parameter(torch.randn(s, generator=g0).to(dev)) for n, s in shapes.items()}
    groups = build_e2e_optimizer_w_lr_mul(list(params.items()), cfg["learning_rate"], cfg["weight_decay"],
                                          lr_mul=cfg["lr_mul"], lr_mul_prefix=cfg["lr_mul_prefix"])
    name_of = {id(p): n for n, p in params.items()}
    assert [[name_of[id(p)] for p in g["params"]] for g in groups] == gold["group_names"]
    opt = AdamW(groups, lr=cfg["learning_rate"], betas=tuple(cfg["betas"]))
    versions = {n: p._version for n, p in params.items()}
    for step in range(1, cfg["steps"] + 1):
        lr = get_lr_sched(step, cfg["decay"], cfg["learning_rate"], cfg["num_train_steps"], warmup_ratio=cfg["warmup_ratio"])
        assert lr == gold["lrs"][step - 1]
        for i, pg in enumerate(opt.param_groups):          # run_pretrain.py:395-401
            pg["lr"] = cfg["lr_mul"] * lr if i in (0, 1) else lr
        for n, g in _grads(shapes, step).items():
            params[n].grad = g.to(dev)
        if fused_clip:
            opt.step(max_grad_norm=cfg["grad_norm"])
            norm = float(opt.last_grad_norm)
        else:
            norm = float(clip_grad_norm_(params.values(), cfg["grad_norm"]))
            opt.step()
        assert abs(norm - gold["norms"][step - 1]) < 1e-5 * gold["norms"][step - 1]
    for n in shapes:
        p, m, v = params[n].data.cpu(), opt.state[params[n]]["exp_avg"].cpu(), opt.state[params[n]]["exp_avg_sq"].cpu()
        assert torch.allclose(p, gold["final_p"][n], rtol=2e-5, atol=2e-6), n
        assert torch.allclose(m, gold["final_m"][n], rtol=2e-5, atol=1e-7), n
        assert torch.allclose(v, gold["final_v"][n], rtol=2e-5, atol=1e-9), n
        assert params[n]._version > versions[n]            # raw-pointer update is visible to version-keyed caches
        assert opt.state[params[n]]["step"] == cfg["steps"]


def test_large_multi_chunk_tensors_bf16_targets_and_unaligned_views(dev):
    from xpretrain_b200.optimization.adamw import AdamW

    torch.manual_seed(0)
    flat = torch.randn(3_000_001 + 7, device=dev)
    big = torch.nn.Parameter(torch.randn(3_000_001, device=dev))         # 367 chunks, ragged tail
    odd = torch.nn.Parameter(torch.randn(1001, device=dev))
    big.grad = flat[:3_000_001]
    odd.grad = torch.randn(1001 + 1, device=dev)[1:]                      # 4-byte aligned only: scalar path
    opt = AdamW([{"params": [big], "weight_decay": 0.1}, {"params": [odd], "weight_decay": 0.0}], lr=3e-4, betas=(0.9, 0.98))
    tgt = torch.zeros(3_000_001, dtype=torch.bfloat16, device=dev)
    opt.bf16_targets[id(big)] = tgt
    ref = {}
    for name, p, wd in (("big", big, 0.1), ("odd", odd, 0.0)):
        rp, rm, rv = p.data.clone(), torch.zeros_like(p.data), torch.zeros_like(p.data)
        ref[name] = (rp, rm, rv, p.grad.clone(), wd)
    total, coef = AO.clip_coef([big.grad, odd.grad], 1.0)
    for t in (1, 2):
        opt.step(max_grad_norm=1.0)
        for name in ref:
            rp, rm, rv, g, wd = ref[name]
            AO.adamw_step(rp, g * coef, rm, rv, t, 3e-4, (0.9, 0.98), 1e-6, wd, True)
    assert abs(float(opt.last_grad_norm) - float(total)) < 1e-4 * float(total)
    assert torch.allclose(big.data, ref["big"][0], rtol=1e-5, atol=1e-6)
    assert torch.allclose(odd.data, ref["odd"][0], rtol=1e-5, atol=1e-6)
    assert torch.equal(tgt, big.data.to(torch.bfloat16))


def test_no_cpu_path():
    from xpretrain_b200 import _lib
    from xpretrain_b200.optimization.adamw import AdamW

    p = torch.nn.Parameter(torch.zeros(4))
    p.grad = torch.ones(4)
    with pytest.raises(_lib.XpError):
        AdamW([p]).step()


def test_training_step_on_the_dual_encoder_matches_the_oracle_update(dev):
    """fwd + InfoNCE + bwd + fused clip + AdamW on VidCLIP (depth 1): every parameter moves exactly as adamw.py says for
    the gradients the backward produced, and the next forward really uses the updated weights (bf16 copies refreshed)."""
    from clipvip_cases import b16, vidclip
    from oracle import clipvip_oracle as O
    from xpretrain_b200.optimization import build_loss_func
    from xpretrain_b200.optimization.adamw import AdamW, build_e2e_optimizer_w_lr_mul

    ocfg = b16(1, 1)
    model = vidclip(ocfg, dev=dev)
    video, ids, mask = O.synthetic_batch(8, 2, 16, ocfg, seed=3)
    video, ids, mask = video.to(dev), ids.to(dev), mask.to(dev)
    loss_fn = build_loss_func({"loss_name": "NCELearnableTempLoss"})
    lr, wd, betas = 1e-4, 0.2, (0.9, 0.98)
    named = list(model.named_parameters())
    opt = AdamW(build_e2e_optimizer_w_lr_mul(named, lr, wd), lr=lr, betas=betas)

    def loss_of():
        out = model(video=video, text_input_ids=ids, text_input_mask=mask)
        return loss_fn(out["vis_features"], out["text_features"], model.clipmodel.logit_scale)

    loss0 = loss_of()
    loss0.backward()
    before = {n: (p.detach().cpu().clone(), p.grad.detach().cpu().clone()) for n, p in named}
    total, coef = AO.clip_coef([g for _, g in before.values()], 5.0)
    opt.step(max_grad_norm=5.0)
    assert abs(float(opt.last_grad_norm) - float(total)) < 1e-4 * float(total)
    for n, p in named:
        rp, g = before[n]
        m, v = torch.zeros_like(rp), torch.zeros_like(rp)
        decayed = not any(k in n for k in AO.NO_DECAY)
        AO.adamw_step(rp, g * coef, m, v, 1, lr, betas, 1e-6, wd if decayed else 0.0, True)
        assert torch.allclose(p.detach().cpu(), rp, rtol=1e-5, atol=1e-7), n
    with torch.no_grad():
        loss1 = loss_of()
    assert float(loss1) != float(loss0)        # the bf16 compute copies were refreshed from the updated masters
