"""CPU: pin oracle/embed_ref.py and oracle/optim_ref.py, which the GPU contract suites (test_gpu_embed_contract.py,
test_gpu_optim_contract.py) hold the kernels to, against independent statements of the same operations: F.conv2d / unfold
for the im2col, F.interpolate and float64 autograd for the ViP tables, nn.Embedding autograd for the text embeddings,
the TimeSformer reference's rearranges for the tokens, and oracle/adamw_oracle.py plus the adamw_8steps golden for AdamW."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import adamw_oracle as AO
from oracle import clipvip_oracle as CO
from oracle import embed_ref as E
from oracle import optim_ref as O

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16


# ------------------------------------------------------------------------------------------- im2col
@pytest.mark.parametrize("p", [4, 14, 16, 32])
def test_im2col_is_the_stride_p_convolution(p):
    g = torch.Generator().manual_seed(p)
    H, W = 2 * p, 3 * p
    video = torch.randn(3, 3, H, W, generator=g, dtype=F64)
    cols = E._im2col(video, p)
    Kp = 3 * p * p
    assert cols.shape == (3 * 2 * 3, E.patch_pitch(p)) and E.patch_pitch(p) % 8 == 0
    assert torch.all(cols[:, Kp:] == 0)
    unf = F.unfold(video, kernel_size=p, stride=p).transpose(1, 2).reshape(-1, Kp)     # [F*L, 3*p*p], same column order
    assert torch.equal(cols[:, :Kp], unf)
    w = torch.randn(5, 3, p, p, generator=g, dtype=F64)
    conv = F.conv2d(video, w, stride=p).flatten(2).transpose(1, 2).reshape(-1, 5)       # patch order row-major (flatten(2))
    torch.testing.assert_close(cols[:, :Kp] @ w.reshape(5, -1).t(), conv, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("dtype", [F32, BF16, torch.float16])
def test_patchify_ref_rounds_once(dtype):
    g = torch.Generator().manual_seed(1)
    video = (torch.randn(2, 3, 28, 42, generator=g) * 3).to(dtype)
    got = E.patchify_ref(video, 14)
    want = E._im2col(video.to(F64), 14).to(F32).to(BF16)                                  # f16 / bf16 -> f32 are exact
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_u8_transform_is_the_reference_fp32_chain():
    g = torch.Generator().manual_seed(2)
    frames = torch.randint(0, 256, (2, 32, 48, 3), generator=g, dtype=torch.uint8)
    mean, std = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)
    # dataset_pretrain_stage1_all_source.py:182 then torchvision Normalize, all fp32
    x = frames.permute(0, 3, 1, 2).float() / 255.
    x = (x - torch.tensor(mean).view(1, 3, 1, 1)) / torch.tensor(std).view(1, 3, 1, 1)
    want = E._im2col(x, 16).to(BF16)
    assert torch.equal(E.patchify_u8_ref(frames, 16, mean, std).view(torch.int16), want.view(torch.int16))


# ------------------------------------------------------------------------------------------- ViP tables
@pytest.mark.parametrize("Tsz,T", [(12, 12), (12, 1), (12, 5), (12, 7), (12, 13), (12, 32), (1, 1), (1, 4), (3, 12)])
def test_taps_are_f_interpolate(Tsz, T):
    x = torch.randn(1, 6, Tsz, dtype=F64)
    want = x if T == Tsz else F.interpolate(x, size=T, mode="linear", align_corners=False)
    torch.testing.assert_close(E.tap_matrix(Tsz, T) @ x[0].t(), want[0].t(), rtol=1e-14, atol=1e-14)
    i0, i1, lam = E.linear_taps(Tsz, T)
    assert all(0 <= a <= b < Tsz and 0.0 <= w < 1.0 for a, b, w in zip(i0, i1, lam))
    assert E.weight_error(Tsz, T) < 2e-5


def _vip_params(C, M, Tsz, seed, temporal=True):
    g = torch.Generator().manual_seed(seed)
    L = 4
    pos = torch.randn(L + 1, C, generator=g)
    tmp = torch.randn(Tsz, C, generator=g) if temporal else None
    cls = torch.randn(C, generator=g)
    added = torch.randn(max(M - 1, 0), C, generator=g)
    return L, pos, tmp, cls, added


@pytest.mark.parametrize("M", [1, 4])
@pytest.mark.parametrize("Tsz,T", [(12, 12), (12, 5), (12, 16), (1, 3)])
@pytest.mark.parametrize("temporal", [True, False])
def test_vip_tables_against_the_clipvip_oracle(M, Tsz, T, temporal):
    C, B = 24, 2
    L, pos, tmp, cls, added = _vip_params(C, M, Tsz, seed=T * 7 + M, temporal=temporal)
    exact, bound, t32, glob = E.vip_tables_ref(pos, tmp, cls, added, B, T, L, M, Tsz)
    # oracle: the whole embedding with a zero patch conv is exactly the tables
    sd = {"vision_model.embeddings.patch_embedding.weight": torch.zeros(C, 3, 2, 2, dtype=F64),
          "vision_model.embeddings.position_embedding.weight": pos.to(F64),
          "vision_model.embeddings.temporal_embedding": (tmp if temporal else torch.zeros(Tsz, C)).to(F64)[None],
          "vision_model.embeddings.class_embedding": cls.to(F64),
          "vision_model.embeddings.added_cls": added.to(F64)}
    cfg = type("Cfg", (), {"patch": 2})()
    x, (Mo, To, Lo) = CO.vip_embeddings(sd, torch.zeros(B, T, 3, 4, 4, dtype=F64), cfg)
    assert (Mo, To, Lo) == (M, T, L)
    torch.testing.assert_close(exact, x[0, M:], rtol=1e-13, atol=1e-13)
    assert torch.all((glob.to(F64) - x[:, :M]).abs() <= 0.5 * E.ulp_bf16(x[:, :M]))
    if t32 is not None:
        assert torch.all(bound == 0) and torch.all((t32.to(F64) - exact).abs() <= 0.5 * E.ulp_bf16(exact) + 1e-6 * exact.abs())
    else:
        assert torch.all(bound > 0)
        assert torch.all(bound <= 0.5 * E.ulp_bf16(exact.abs() + 1e-3) + 1e-4 * (1 + exact.abs()))   # far below one bf16 step + noise


@pytest.mark.parametrize("M", [1, 4])
@pytest.mark.parametrize("Tsz,T", [(12, 12), (12, 5), (12, 16)])
def test_vip_bwd_is_float64_autograd(M, Tsz, T):
    C, B = 16, 3
    L, pos, tmp, cls, added = _vip_params(C, M, Tsz, seed=11 + T)
    g = torch.Generator().manual_seed(5)
    d_patch = torch.randn(B, T * L, C, generator=g).to(BF16)
    d_glob = torch.randn(B, M, C, generator=g).to(BF16)
    init = {"pos": torch.randn(L + 1, C, generator=g), "temporal": torch.randn(Tsz, C, generator=g),
            "cls": torch.randn(C, generator=g), "added": torch.randn(max(M - 1, 0), C, generator=g)}
    ref = E.vip_bwd_ref(d_patch, d_glob, init, B, T, L, M, Tsz)
    leaves = {k: v.to(F64).requires_grad_() for k, v in
              (("pos", pos), ("temporal", tmp), ("cls", cls), ("added", added))}
    tv = F.interpolate(leaves["temporal"].t()[None], size=T, mode="linear", align_corners=False)[0].t() \
        if T != Tsz else leaves["temporal"]
    patch = (tv[:, None] + leaves["pos"][1:1 + L][None]).reshape(T * L, C)
    glob = torch.cat([leaves["cls"][None], leaves["added"]], 0) + leaves["pos"][0]
    out = torch.cat([glob[None].expand(B, M, C), patch[None].expand(B, T * L, C)], 1)
    out.backward(torch.cat([d_glob, d_patch], 1).to(F64))
    for k in ("pos", "temporal", "cls") + (("added",) if M > 1 else ()):
        exact, bound = ref[k]
        torch.testing.assert_close(exact, init[k].to(F64) + leaves[k].grad, rtol=1e-12, atol=1e-12)
        assert torch.all(bound > 0)
    assert "added" not in ref or M > 1
    # the derived atomic bound: n - 1 roundings of the running sum of the addends' magnitudes
    n = 1 + B * T
    assert torch.allclose(ref["pos"][1][1], (n - 1) * E.U * (init["pos"][1].abs().to(F64) + d_patch.to(F64).abs()[:, 0::L].sum((0, 1)))
                          * E.SLACK)


# ------------------------------------------------------------------------------------------- text
def test_text_embeddings_against_nn_embedding():
    vocab, C, Lt, B = 50, 20, 7, 6
    g = torch.Generator().manual_seed(3)
    tok = torch.randn(vocab, C, generator=g)
    pos = torch.randn(Lt, C, generator=g)
    ids = torch.randint(0, vocab, (B, Lt), generator=g)
    ids[0, 0], ids[1, 3] = 0, vocab - 1
    x, err = E.text_fwd_ref(ids, tok, pos, Lt)
    want = (tok[ids] + pos[None]).reshape(-1, C).to(BF16)        # CLIP_ViP.py:222-225 in fp32, one rounding
    assert err == 0 and torch.equal(x.view(torch.int16), want.view(torch.int16))
    emb_t = torch.nn.Embedding(vocab, C).double()
    emb_p = torch.nn.Embedding(Lt, C).double()
    dx = torch.randn(B * Lt, C, generator=g).to(BF16)
    (emb_t(ids) + emb_p(torch.arange(Lt))[None]).reshape(-1, C).backward(dx.to(F64))
    t0, p0 = torch.randn(vocab, C, generator=g), torch.randn(Lt, C, generator=g)
    ref = E.text_bwd_ref(ids, dx, t0, p0, Lt)
    torch.testing.assert_close(ref["tok"][0], t0.to(F64) + emb_t.weight.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["pos"][0], p0.to(F64) + emb_p.weight.grad, rtol=1e-12, atol=1e-12)
    bad = ids.clone()
    bad[2, 2] = vocab
    bad[3, 0] = -1
    x2, err2 = E.text_fwd_ref(bad, tok, pos, Lt)
    assert err2 == 1 and torch.equal(x2[2 * Lt + 2].float(), (tok[0] + pos[2]).to(BF16).float())
    ref2 = E.text_bwd_ref(bad, dx, t0, p0, Lt)
    keep = torch.ones(B * Lt, dtype=torch.bool)
    keep[2 * Lt + 2] = keep[3 * Lt] = False
    torch.testing.assert_close(ref2["pos"][0][2], p0[2].to(F64) + dx.to(F64)[keep.view(B, Lt)[:, 2].nonzero()[:, 0] * Lt + 2].sum(0))


def test_eos_first_maximum():
    ids = torch.tensor([[1, 9, 9, 3], [7, 7, 7, 7], [-5, -3, -3, -9], [0, 0, 0, 2]])
    off, idx = E.eos_ref(ids, 10)
    assert idx.tolist() == [1, 0, 1, 3] == ids.argmax(dim=-1).tolist()       # torch.argmax: first maximal index
    assert off.tolist() == [(b * 4 + i) * 10 for b, i in enumerate([1, 0, 1, 3])]


# ------------------------------------------------------------------------------------------- TimeSformer
@pytest.mark.parametrize("use_pos,use_time", [(True, True), (False, False), (True, False)])
def test_tokens_are_the_timesformer_rearranges(use_pos, use_time):
    B, T, C, Hh, Ww = 2, 3, 5, 2, 3
    g = torch.Generator().manual_seed(4)
    x = torch.randn(B, T, C, Hh, Ww, generator=g)
    pos = torch.randn(Hh * Ww, C, generator=g) if use_pos else None
    time = torch.randn(T, C, generator=g) if use_time else None
    tok = E.tsf_tokens_ref(x.reshape(B, T, C, -1), pos, time)
    # timesformer.py:481-509: '(b t) (h w) c' + pos, '(b n) t m' + time, 'b (n t) m'
    y = x.permute(0, 1, 3, 4, 2).reshape(B * T, Hh * Ww, C)
    if pos is not None:
        y = y + pos[None]
    y = y.reshape(B, T, Hh * Ww, C).permute(0, 2, 1, 3).reshape(B * Hh * Ww, T, C)
    if time is not None:
        y = y + time[None]
    want = y.reshape(B, Hh * Ww * T, C).reshape(-1, C).to(BF16)
    assert torch.equal(tok.view(torch.int16), want.view(torch.int16))
    back = E.tsf_untokenize_ref(tok, B, T, C, Hh * Ww, F32)
    # timesformer.py:523: x.reshape(B, H, W, T, C).permute(0, 3, 4, 1, 2)
    assert torch.equal(back, tok.float().reshape(B, Hh, Ww, T, C).permute(0, 3, 4, 1, 2).reshape(B, T, C, -1))


# ------------------------------------------------------------------------------------------- optimizer
def test_clip_coef_matches_clip_grad_norm():
    g = torch.Generator().manual_seed(6)
    grads = [torch.randn(n, generator=g) for n in (3, 100, 7)]
    norm, rel = O.grad_norm_ref(grads)
    total, coef = AO.clip_coef(grads, 1.0)
    assert abs(norm - float(total)) <= rel * norm and rel < 3e-6
    assert O.clip_coef_f32(1.0, float(total)) == pytest.approx(float(coef), rel=1e-6)
    assert O.clip_coef_f32(1e9, 1.0) == 1.0 and O.clip_coef_f32(0.0, 5.0) == 1.0 and O.clip_coef_f32(-1.0, 5.0) == 1.0
    assert math.isnan(O.clip_coef_f32(1.0, float("nan"))) and O.clip_coef_f32(1.0, float("inf")) == 0.0
    p = torch.nn.Parameter(torch.ones(3))
    p.grad = torch.tensor([1.0, float("nan"), 2.0])
    torch.nn.utils.clip_grad_norm_([p], 1.0)
    assert torch.isnan(p.grad).all()          # the NaN coefficient reaches every gradient


@pytest.mark.parametrize("wd", [0.0, 0.2])
def test_adamw_ref_bounds_the_oracle(wd):
    g = torch.Generator().manual_seed(7)
    n, lr, betas, eps = 4096, 3e-4, (0.9, 0.98), 1e-6
    p = torch.randn(n, generator=g)
    m, v = torch.zeros(n), torch.zeros(n)
    for step in range(1, 4):
        grad = torch.randn(n, generator=g) * (0.01 if step == 2 else 1.0)
        grad[:4] = 0.0
        ss = O.step_size_of(lr, betas, step)
        # adamw.py's constants: 1 - beta in double, step_size and lr * wd in double, each rounded to fp32 by the tensor op
        ref = O.adamw_ref(p, grad, m, v, 1.0, betas[0], betas[1], eps, O.f32(ss), O.f32(lr * wd),
                          one_minus=(1.0 - betas[0], 1.0 - betas[1]))
        AO.adamw_step(p, grad, m, v, step, lr, betas, eps, wd, True)
        for name, t in (("p", p), ("m", m), ("v", v)):
            exact, bound = ref[name]
            err = (t.to(F64) - exact).abs()
            assert torch.all(err <= bound), (name, step, float((err - bound).max()))
        assert float(ref["p"][1].max()) < 1e-2 * ss          # far below one step of lr


def test_adamw_ref_replays_the_golden_trajectory(golden_dir):
    gold = torch.load(os.path.join(golden_dir, "adamw_8steps.pt"), weights_only=False)
    cfg, shapes = gold["cfg"], gold["shapes"]
    g0 = torch.Generator().manual_seed(0)
    params = {n: torch.randn(s, generator=g0) for n, s in shapes.items()}
    names = [n for grp in gold["group_names"] for n in grp]
    lr_of, wd_of = {}, {}
    for i, grp in enumerate(gold["group_names"]):
        for n in grp:
            lr_of[n] = (cfg["lr_mul"] if i in (0, 1) else 1.0)
            wd_of[n] = cfg["weight_decay"] if i in (0, 2) else 0.0
    state = {n: (params[n].clone(), torch.zeros(shapes[n]), torch.zeros(shapes[n])) for n in names}
    betas = tuple(cfg["betas"])
    for step in range(1, cfg["steps"] + 1):
        lr = gold["lrs"][step - 1]
        gs = {n: torch.randn(s, generator=torch.Generator().manual_seed(1000 * step + i)) * (0.01 if step % 3 == 0 else 1.0)
              for i, (n, s) in enumerate(shapes.items())}
        norm, rel = O.grad_norm_ref([gs[n] for n in names])
        assert abs(norm - gold["norms"][step - 1]) <= 2 * rel * norm + 1e-6 * norm
        coef = O.clip_coef_f32(cfg["grad_norm"], float(np.float32(norm)))
        for n in names:
            p, m, v = state[n]
            glr = lr_of[n] * lr
            ref = O.adamw_ref(p, gs[n], m, v, coef, betas[0], betas[1], 1e-6, O.f32(O.step_size_of(glr, betas, step)),
                              O.f32(glr * wd_of[n]))
            state[n] = tuple(ref[k][0].to(F32) for k in ("p", "m", "v"))
    for n in names:
        torch.testing.assert_close(state[n][0], gold["final_p"][n], rtol=2e-5, atol=2e-6)
        torch.testing.assert_close(state[n][1], gold["final_m"][n], rtol=2e-5, atol=1e-7)
        torch.testing.assert_close(state[n][2], gold["final_v"][n], rtol=2e-5, atol=1e-9)
