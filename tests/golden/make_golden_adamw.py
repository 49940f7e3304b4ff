"""Golden vectors for the optimizer step (SURVEY.md §8(f).1) from the REAL reference.

Needs a checkout of the reference, named by XP_REFERENCE_ROOT:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_adamw.py

Drives the reference's own `AdamW` (optimization/adamw.py), `build_e2e_optimizer_w_lr_mul` (optimization/utils.py),
`get_lr_sched` (optimization/sched.py) and torch's `clip_grad_norm_` exactly as run_pretrain.py:388-423 does, for a few
steps on a small named parameter set, asserts oracle/adamw_oracle.py reproduces every tensor bit-for-bit, and stores the
trajectory (no reference source) for tests/test_oracle_golden.py (CPU) and tests/test_gpu_optim.py (GPU).
"""
import os
import sys
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ["XP_REFERENCE_ROOT"]     # a checkout of microsoft/XPretrain
sys.path.insert(0, os.path.join(REF, "CLIP-ViP"))
sys.dont_write_bytecode = True

from oracle import adamw_oracle as O  # noqa: E402

SHAPES = {
    "clipmodel.vision_model.encoder.layers.0.mlp.fc1.weight": (96, 40),
    "clipmodel.vision_model.encoder.layers.0.mlp.fc1.bias": (96,),
    "clipmodel.vision_model.encoder.layers.0.layer_norm1.weight": (40,),    # decayed: 'LayerNorm' is not in the name
    "clipmodel.vision_model.embeddings.added_cls": (3, 40),
    "clipmodel.text_projection.weight": (24, 40),
    "clipmodel.logit_scale": (),
    "odd.sized.weight": (7, 13),                                            # 91 elements: not a multiple of 4
}
CFG = dict(learning_rate=1e-3, weight_decay=0.2, betas=(0.9, 0.98), decay="cosine", num_train_steps=20, warmup_ratio=0.2,
           grad_norm=2.0, lr_mul=10.0, lr_mul_prefix="text_projection", steps=8)


def make_params(seed):
    g = torch.Generator().manual_seed(seed)
    return {n: torch.randn(s, generator=g) for n, s in SHAPES.items()}


def make_grad(step, name_index, shape, scale):
    g = torch.Generator().manual_seed(1000 * step + name_index)
    return torch.randn(shape, generator=g) * scale


def grad_scale(step):
    return 0.01 if step % 3 == 0 else 1.0        # some steps below the clipping threshold, most above


def main():
    warnings.simplefilter("ignore")
    from torch.nn.utils import clip_grad_norm_
    from src.optimization.adamw import AdamW
    from src.optimization.sched import get_lr_sched
    from src.optimization.utils import build_e2e_optimizer_w_lr_mul

    init = make_params(0)
    params = {n: torch.nn.Parameter(v.clone()) for n, v in init.items()}
    groups = build_e2e_optimizer_w_lr_mul(list(params.items()), CFG["learning_rate"], CFG["weight_decay"],
                                          lr_mul=CFG["lr_mul"], lr_mul_prefix=CFG["lr_mul_prefix"])
    opt = AdamW(groups, lr=CFG["learning_rate"], betas=CFG["betas"])

    # oracle state
    o_p = {n: v.clone() for n, v in init.items()}
    o_m = {n: torch.zeros_like(v) for n, v in init.items()}
    o_v = {n: torch.zeros_like(v) for n, v in init.items()}
    o_groups = O.param_groups([(n, params[n]) for n in SHAPES], CFG["learning_rate"], CFG["weight_decay"],
                              CFG["lr_mul"], CFG["lr_mul_prefix"])
    name_of = {id(p): n for n, p in params.items()}
    assert [[name_of[id(p)] for p in g["params"]] for g in o_groups] == [[name_of[id(p)] for p in g["params"]] for g in groups]

    lrs, norms = [], []
    for step in range(1, CFG["steps"] + 1):
        lr = get_lr_sched(step, CFG["decay"], CFG["learning_rate"], CFG["num_train_steps"], warmup_ratio=CFG["warmup_ratio"])
        assert lr == O.lr_schedule(step, CFG["decay"], CFG["learning_rate"], CFG["num_train_steps"], CFG["warmup_ratio"])
        for i, pg in enumerate(opt.param_groups):      # run_pretrain.py:395-401
            pg["lr"] = CFG["lr_mul"] * lr if i in (0, 1) else lr
        grads = {n: make_grad(step, i, s, grad_scale(step)) for i, (n, s) in enumerate(SHAPES.items())}
        for n, p in params.items():
            p.grad = grads[n].clone()
        total = clip_grad_norm_(list(params.values()), CFG["grad_norm"])
        opt.step()
        # ---- oracle
        o_total, coef = O.clip_coef([grads[n] for n in SHAPES], CFG["grad_norm"])
        assert float(o_total) == float(total)
        for gi, pg in enumerate(opt.param_groups):
            for p in pg["params"]:
                n = name_of[id(p)]
                O.adamw_step(o_p[n], grads[n] * coef, o_m[n], o_v[n], step, pg["lr"], CFG["betas"], 1e-6,
                             pg["weight_decay"], True)
        for n in SHAPES:
            assert torch.equal(o_p[n], params[n].data), (step, n)
            assert torch.equal(o_m[n], opt.state[params[n]]["exp_avg"]) and torch.equal(o_v[n], opt.state[params[n]]["exp_avg_sq"])
        lrs.append(lr)
        norms.append(float(total))
    print("oracle == reference AdamW/clip/sched for", CFG["steps"], "steps; norms", [round(x, 3) for x in norms])
    torch.save({"cfg": CFG, "shapes": SHAPES, "lrs": lrs, "norms": norms,
                "group_names": [[name_of[id(p)] for p in g["params"]] for g in groups],
                "final_p": {n: params[n].data.clone() for n in SHAPES},
                "final_m": {n: opt.state[params[n]]["exp_avg"].clone() for n in SHAPES},
                "final_v": {n: opt.state[params[n]]["exp_avg_sq"].clone() for n in SHAPES}},
               os.path.join(HERE, "adamw_8steps.pt"))


if __name__ == "__main__":
    main()
