"""H100: LF-VILA's video classification model (lfvila_video_classification.py) — the head kernels element by element against
float64, the module against the fp32 oracle under the calibrated bf16 rule (DESIGN.md §2) on the reference goldens' cases and
at the released geometry, and the peak memory of evaluation under torch.no_grad()."""
import json
import os
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from contract_harness import Guarded, Report, calibrated_model_rows, no_tf32, same_bits, within
from encoder_cases import _arm_core, frame_slices, param_slices
from oracle import lfvila_cls_oracle as L
from oracle import swin3d_oracle as SO

pytestmark = pytest.mark.gpu

bf16, f16, f32, f64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
U32 = 2.0 ** -24
UNIT = {f32: 2.0 ** -24, f16: 2.0 ** -11, bf16: 2.0 ** -8}
REPORT = Report("LF-VILA head kernels: worst |err| / bound")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "these tests need the H100"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    REPORT.print()


# ------------------------------------------------------------------------------------------------ pool kernel
def _plant(x, gen):
    """Ties and NaN / +-inf where two windows overlap: per frame a random kind, placed at an interior column (w = 1, which
    every column window of a 3-wide grid covers) of row 0 or of an interior row (h = 1 is covered by two row windows)."""
    B, N, Hp, Wp, C = x.shape
    kind = torch.randint(0, 10, (B, N, C), generator=gen)          # 5..9: untouched
    h = torch.randint(0, min(Hp, 2), (B, N, C), generator=gen)
    w = torch.randint(1, Wp - 1, (B, N, C), generator=gen)
    b, n, c = torch.meshgrid(torch.arange(B), torch.arange(N), torch.arange(C), indexing="ij")
    top = x.abs().amax(dim=(2, 3)) + 1.0                              # above every value of the frame
    v = x[b, n, h, w, c]
    v = torch.where(kind == 0, top, v)                                 # tie: the same maximum twice, in two windows
    v = torch.where(kind == 1, torch.tensor(float("nan")), v)
    v = torch.where(kind == 2, torch.tensor(float("inf")), v)
    v = torch.where(kind == 3, torch.tensor(float("-inf")), v)
    x[b, n, h, w, c] = v
    tie_w = torch.where(w + 1 < Wp, w + 1, w - 1)
    x[b, n, h, tie_w, c] = torch.where(kind == 0, top, x[b, n, h, tie_w, c])
    # kind 4: a second NaN in the same frame (the later one of a window must win)
    x[b, n, torch.minimum(h + 1, torch.tensor(Hp - 1)), w, c] = torch.where(
        kind == 4, torch.tensor(float("nan")), x[b, n, torch.minimum(h + 1, torch.tensor(Hp - 1)), w, c])
    x[b, n, h, w, c] = torch.where(kind == 4, torch.tensor(float("nan")), x[b, n, h, w, c])
    return x


def _torch_pool(x64):
    """torch's own max_pool2d (float64, NCHW) and its indices converted to window positions kh * 3 + kw."""
    B, N, Hp, Wp, C = x64.shape
    y, idx = F.max_pool2d(x64.permute(0, 1, 4, 2, 3).reshape(B * N, C, Hp, Wp).contiguous(), (2, 3), stride=1,
                          return_indices=True)
    Ho, Wo = Hp - 1, Wp - 2
    i = torch.arange(Ho, device=x64.device).view(1, 1, Ho, 1)
    j = torch.arange(Wo, device=x64.device).view(1, 1, 1, Wo)
    k = (idx // Wp - i) * 3 + (idx % Wp - j)
    to_last = lambda t: t.reshape(B, N, C, Ho * Wo).permute(0, 1, 3, 2)     # noqa: E731  [B, N, X, C]
    return to_last(y), to_last(k)


@pytest.mark.parametrize("B,N,Hp,Wp,C,dt", [
    (2, 1, 2, 3, 128, f32),          # the smallest grid the pool takes: one window
    (3, 4, 2, 3, 1000, f16),
    (32, 4, 3, 5, 128, f32),         # the released grid, B = 32
    (2, 32, 3, 5, 1024, f16),        # released: 32 frames, 1024 channels, the trainer's fp16
    (2, 32, 3, 5, 1024, f32),
    (1, 4, 7, 7, 1000, f32),
    (4, 1, 7, 7, 1024, f16),
])
def test_pool_against_float64(dev, B, N, Hp, Wp, C, dt):
    from xpretrain_b200 import ops
    tag = f"pool B{B} N{N} {Hp}x{Wp} C{C} {str(dt)[6:]}"
    gen = torch.Generator().manual_seed(B * 1000 + N * 10 + C)
    x = _plant(torch.randn(B, N, Hp, Wp, C, generator=gen).to(dt).float(), gen).to(dt).to(dev)
    X = (Hp - 1) * (Wp - 2)
    outs = dict(frame=Guarded(dev, (B * N, C), f32), frame_bf=Guarded(dev, (B * N, C), bf16),
                glob=Guarded(dev, (B, C), f32), glob_bf=Guarded(dev, (B, C), bf16),
                argmax=Guarded(dev, (B, N, X, C), torch.uint8))
    run = lambda: ops.lfvila_pool_fwd(x, *(outs[k].t for k in ("frame", "frame_bf", "glob", "glob_bf", "argmax")))  # noqa
    run()
    torch.cuda.synchronize()
    for k, o in outs.items():      # coverage: NaN only where the exact mean is NaN, every arg-max equal to torch's (below)
        o.guards(f"{tag}: {k}")
    first = {k: o.t.clone() for k, o in outs.items()}
    run()
    assert all(same_bits(first[k], outs[k].t) for k in outs if k != "argmax") and torch.equal(first["argmax"], outs["argmax"].t)

    x64 = x.double()
    m, k_ref = _torch_pool(x64)
    assert torch.equal(outs["argmax"].t.long(), k_ref), f"{tag}: arg-max positions differ from max_pool2d's indices"
    # the maximum is a copy: the float64 means of the exact maxima, within the fp32 summation bound
    for name, got, exact, absum, terms in (
            ("frame", outs["frame"].t.view(B, N, C), m.mean(2), m.abs().mean(2), X),
            ("global", outs["glob"].t, m.mean(dim=(1, 2)), m.abs().mean(dim=(1, 2)), N * X + 8)):
        fin = torch.isfinite(exact)
        assert torch.equal(torch.isnan(got), torch.isnan(exact)), f"{tag}: {name}: NaN placement"
        assert torch.equal(got[~fin & ~torch.isnan(exact)], exact[~fin & ~torch.isnan(exact)].float()), f"{tag}: {name}: inf"
        within(REPORT, f"{tag}: {name}", got[fin], exact[fin], (terms * U32 * absum + U32 * exact.abs())[fin] + 1e-30)
        bf = (outs["frame_bf"].t.view(B, N, C) if name == "frame" else outs["glob_bf"].t)
        assert same_bits(bf[fin], got[fin].to(bf16)), f"{tag}: {name}: the bf16 copy is not the rounded fp32 value"

    # backward: the gradient routing of torch's max_pool2d autograd, values within the rounding of g to x's dtype
    d_frame = torch.randn(B * N, C, generator=gen).to(dev)
    d_global = torch.randn(B, C, generator=gen).to(dev)
    for df, dg in ((d_frame, d_global), (d_frame, None), (None, d_global)):
        xr = x64.clone().requires_grad_(True)
        mm, _ = _torch_pool(xr)
        obj = 0
        if df is not None:
            obj = obj + (mm.mean(2) * df.double().view(B, N, C)).sum()
        if dg is not None:
            obj = obj + (mm.mean(dim=(1, 2)) * dg.double()).sum()
        obj.backward()
        dx = Guarded(dev, (B, N, Hp, Wp, C), dt)
        ops.lfvila_pool_bwd(df, dg, outs["argmax"].t, dx.t)
        torch.cuda.synchronize()
        got = dx.written(f"{tag}: dx").clone()
        assert torch.equal(got != 0, xr.grad != 0), f"{tag}: dx routing differs from max_pool2d's autograd"
        g_abs = torch.zeros(B, N, C, dtype=f64, device=dev)
        if df is not None:
            g_abs += df.double().abs().view(B, N, C) / X
        if dg is not None:
            g_abs += dg.double().abs().view(B, 1, C) / (N * X)
        bound = UNIT[dt] * xr.grad.abs() + 8 * U32 * 6 * g_abs.view(B, N, 1, 1, C) + (2.0 ** -25 if dt == f16 else 0.0)
        within(REPORT, f"{tag}: dx", got, xr.grad, bound)
        ops.lfvila_pool_bwd(df, dg, outs["argmax"].t, dx.t)
        assert same_bits(got, dx.t), f"{tag}: dx is not bitwise repeatable"


def test_pool_refusals(dev):
    from xpretrain_b200 import _lib, ops
    for Hp, Wp in ((1, 5), (3, 2)):              # the reference's MaxPool2d((2, 3)) raises on these grids
        x = torch.zeros(1, 2, Hp, Wp, 64, device=dev)
        X = max(Hp - 1, 0) * max(Wp - 2, 0)
        with pytest.raises(_lib.XpError, match="Hp >= 2 and Wp >= 3"):
            ops.lfvila_pool_fwd(x, torch.empty(2, 64, device=dev), torch.empty(2, 64, dtype=bf16, device=dev),
                                torch.empty(1, 64, device=dev), torch.empty(1, 64, dtype=bf16, device=dev),
                                torch.empty(1, 2, X, 64, dtype=torch.uint8, device=dev))
    x = torch.zeros(1, 2, 3, 5, 64, device=dev)
    buf = torch.empty(2 * 64 + 1, device=dev)
    with pytest.raises(_lib.XpError, match="16-byte aligned"):
        ops.lfvila_pool_fwd(x, buf[1:].view(2, 64), torch.empty(2, 64, dtype=bf16, device=dev), torch.empty(1, 64, device=dev),
                            torch.empty(1, 64, dtype=bf16, device=dev), torch.empty(1, 2, 6, 64, dtype=torch.uint8, device=dev))
    dx = torch.empty(2 * 3 * 5 * 64 + 1, device=dev)[1:].view(1, 2, 3, 5, 64)
    with pytest.raises(_lib.XpError, match="16-byte aligned"):
        ops.lfvila_pool_bwd(None, torch.zeros(1, 64, device=dev), torch.zeros(1, 2, 6, 64, dtype=torch.uint8, device=dev), dx)


# ------------------------------------------------------------------------------------------- head row kernels
def test_normalize_against_float64(dev):
    from xpretrain_b200 import ops
    gen = torch.Generator().manual_seed(5)
    rows, C = 37, 1024
    x = torch.randn(rows, C, generator=gen) * 3
    x[0] = 0.0                                   # the 1e-12 clamp: y = 0, dx = g / 1e-12
    x[1] = 1e-16                                 # ||x|| = 3.2e-15 < 1e-12: clamped too
    x[2, :5] = 1e-3
    x[2, 5:] = 0.0
    x = x.to(dev)
    y, ybf, nrm = Guarded(dev, (rows, C), f32), Guarded(dev, (rows, C), bf16), Guarded(dev, (rows,), f32)
    ops.lfvila_normalize_fwd(x, y.t, ybf.t, nrm.t)
    torch.cuda.synchronize()
    xr = x.double().requires_grad_(True)
    ref = F.normalize(xr, dim=-1)
    got = y.written("normalize y").clone()
    within(REPORT, "normalize y", got, ref.detach(), 4 * U32 * ref.detach().abs() + 1e-45)
    assert same_bits(ybf.written("normalize y bf16"), got.to(bf16))
    within(REPORT, "normalize norm", nrm.written("norm"), xr.detach().norm(dim=-1), 4 * U32 * xr.detach().norm(dim=-1))
    dy, dy2 = torch.randn(rows, C, generator=gen).to(dev), torch.randn(rows, C, generator=gen).to(dev)
    ref.backward((dy + dy2).double())
    for a, b in ((dy, dy2), ((dy + dy2), None), (None, dy + dy2)):
        dx = Guarded(dev, (rows, C), bf16)
        ops.lfvila_normalize_bwd(a, b, y.t, nrm.t, dx.t)
        torch.cuda.synchronize()
        g = dx.written("normalize dx").clone()
        scale = ((dy + dy2).double().abs().sum(-1, keepdim=True) / xr.detach().norm(dim=-1, keepdim=True).clamp_min(1e-12))
        within(REPORT, "normalize dx", g, xr.grad, 2.0 ** -8 * xr.grad.abs() + 16 * U32 * scale)
    assert float(g[0].float().abs().max()) > 1e11                        # below the clamp: g / 1e-12


@pytest.mark.parametrize("n,B", [(4, 2), (5, 16), (6, 33), (180, 16)])
def test_cross_entropy_against_float64(dev, n, B):
    from xpretrain_b200 import ops
    tag = f"ce n{n} B{B}"
    gen = torch.Generator().manual_seed(n * 100 + B)
    n_pad = (n + 7) // 8 * 8
    z = torch.randn(B, n, generator=gen) * 4
    labels = torch.randint(0, n, (B,), generator=gen)
    # argmax ties: rows with the maximum twice; the label is the first index on even rows, the second on odd rows
    for r in range(0, B, 3):
        a, b = sorted(torch.randperm(n, generator=gen)[:2].tolist())
        z[r, a] = z[r, b] = float(z[r].max()) + 1.0
        labels[r] = a if r % 2 == 0 else b
    logits = torch.full((B, n_pad), 1e30)
    logits[:, :n] = z                                  # the pad columns are never read
    logits, labels = logits.to(dev), labels.to(dev)
    pred, lse = Guarded(dev, (B, n), f32), Guarded(dev, (B,), f32)
    loss, acc = Guarded(dev, (), f32), Guarded(dev, (1,), f32)
    ops.lfvila_ce_fwd(logits, n, labels, pred.t, lse.t, loss.t, acc.t)
    torch.cuda.synchronize()
    assert same_bits(pred.written(f"{tag}: pred"), logits[:, :n])
    zr = logits[:, :n].double().requires_grad_(True)
    ref = F.cross_entropy(zr, labels)
    want_acc = (zr.max(dim=-1)[1] == labels).float().mean(dim=0, keepdim=True)
    assert torch.equal(acc.written(f"{tag}: acc"), want_acc), (acc.t, want_acc)
    within(REPORT, f"{tag}: loss", loss.written(f"{tag}: loss").view(1), ref.detach().view(1),
           torch.tensor([16 * U32 * (1 + float(ref.detach()))], dtype=f64, device=dev))
    within(REPORT, f"{tag}: lse", lse.written(f"{tag}: lse"), torch.logsumexp(zr.detach(), -1),
           16 * U32 * torch.logsumexp(zr.detach(), -1).abs().clamp_min(1.0))
    d_loss = torch.tensor(0.75, device=dev)
    d_pred = torch.randn(B, n, generator=gen).to(dev) * 0.1
    (ref * 0.75 + (zr * d_pred.double()).sum()).backward()
    for dl_, dp_, want in ((d_loss, d_pred, zr.grad), (d_loss, None, None), (None, d_pred, d_pred.double())):
        if want is None:
            zz = zr.detach().clone().requires_grad_(True)
            (F.cross_entropy(zz, labels) * 0.75).backward()
            want = zz.grad
        out = Guarded(dev, (B, n_pad), bf16)
        ops.lfvila_ce_bwd(logits, n, lse.t, labels, dl_, dp_, out.t)
        torch.cuda.synchronize()
        got = out.written(f"{tag}: dlogits").clone()
        assert float(got[:, n:].float().abs().max()) == 0.0 if n_pad > n else True
        within(REPORT, f"{tag}: dlogits", got[:, :n], want, 2.0 ** -8 * want.abs() + 1e-6)
    # ignore_index -100: the row leaves the loss mean and gets no loss gradient
    lab2 = labels.clone()
    lab2[0] = -100
    ops.lfvila_ce_fwd(logits, n, lab2, None, lse.t, loss.t, acc.t)
    ref2 = F.cross_entropy(logits[:, :n].double(), lab2)
    assert abs(float(loss.t) - float(ref2)) <= 16 * U32 * (1 + float(ref2))


# ------------------------------------------------------------------------------------------------- module
def _config(tmp, cfg, n_labels):
    path = os.path.join(tmp, "bert_config.json")
    with open(path, "w") as f:
        json.dump({"hidden_size": cfg.dim(len(cfg.depths) - 1)}, f)
    enc = dict(patch_size=list(cfg.patch_size), embed_dim=cfg.embed_dim, depths=list(cfg.depths),
               downsample_stages=list(cfg.downsample_stages), stages=list(cfg.stages), num_heads=list(cfg.num_heads),
               window_size=[list(w) for w in cfg.window_size], patch_norm=cfg.patch_norm, local_window=cfg.local_window)
    return SimpleNamespace(VideoEncoder=enc, bert_config=path, DATA=SimpleNamespace(classification_labels=n_labels))


FEATS = ("video_global_feat", "video_frame_feat", "prediction")


def _oracle(sd, video, labels, w, cfg, masks, mode):
    """mode 'fp32' (the truth), 'bf16' (bf16 weights, input and activations; the kernels' attention backward) or
    'autocast' -> ({output: tensor}, {name: grad})."""
    dt = bf16 if mode == "bf16" else f32
    sdo = {k: (v.detach().to(dt).requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    if masks is not None and mode == "bf16":
        masks = [None if m is None else tuple(t.to(dt) for t in m) for m in masks]
    with torch.autocast(device_type="cuda", dtype=bf16, enabled=mode == "autocast"), _arm_core(SO, mode), no_tf32():
        out = L.lfvila_cls_forward(sdo, video.to(dt), labels, cfg, drop_masks=masks)
        out = {k: v.float() for k, v in out.items()}
        (out["loss"] + sum((out[k] * w[k]).sum() for k in FEATS)).backward()
    return ({k: v.detach() for k, v in out.items()},
            {n: p.grad for n, p in sdo.items() if p.is_floating_point() and p.grad is not None})


def cls_case(dev, tmp, tag, cfg, n_labels, B, D, H, W, weight_seed, data_seed, masks=None, video_dtype=f32, autocast=True):
    """Our model and the oracle runs on one case; the calibrated rule asserted on every output and parameter gradient,
    whole and per slice.  Returns (ours, fp32 oracle), each ({output: tensor}, {name: grad})."""
    from xpretrain_b200.modeling import LFVILA_Video_Classification
    sd = L.init_state_dict(cfg, n_labels, seed=weight_seed)
    model = LFVILA_Video_Classification(None, _config(tmp, cfg, n_labels))
    model.load_state_dict(sd, strict=True)
    model = model.to(dev)
    if masks is not None:
        masks = [None if m is None else tuple(t.to(dev) for t in m) for m in masks]
        model.train()
        model.video_encoder.forced_drop_masks = masks
    else:
        model.eval()
    video = SO.synthetic_video(B, D, H, W, cfg, seed=data_seed).to(video_dtype).to(dev)
    labels = L.synthetic_labels(B, n_labels, seed=data_seed + 2).to(dev)
    out = model(video, labels)
    g = torch.Generator().manual_seed(data_seed + 1)
    w = {k: torch.randn(out[k].shape, generator=g).to(dev) for k in FEATS}
    (out["loss"] + sum((out[k] * w[k]).sum() for k in FEATS)).backward()
    assert out["acc"].shape == (1,) and out["loss"].shape == () and out["prediction"].shape == (B, n_labels)
    assert float(out["acc"]) == float((out["prediction"].argmax(-1) == labels).float().mean())
    ours = ({k: out[k].detach() for k in FEATS + ("loss",)},
            {n: p.grad for n, p in model.named_parameters() if p.grad is not None})
    sd = {k: v.to(dev) for k, v in sd.items()}
    modes = ("fp32", "bf16", "autocast") if autocast else ("fp32", "bf16")
    runs = [_oracle(sd, video.float(), labels, w, cfg, masks, mode) for mode in modes]
    want, arm, ac = runs[0], runs[1], (runs[2] if autocast else None)
    assert set(ours[1]) == set(want[1]), set(ours[1]) ^ set(want[1])
    rows = [(k, ours[0][k], want[0][k], arm[0][k], ac and ac[0][k]) for k in FEATS]
    rows += [(n, ours[1][n], want[1][n], arm[1][n], ac and ac[1][n]) for n in sorted(want[1])]
    slices = {"video_frame_feat": frame_slices(want[0]["video_frame_feat"]), **param_slices(want[1])}
    bad, _, _ = calibrated_model_rows(tag, rows, slices)
    # the loss is one scalar: one sample of the logits' error, which a lucky bf16 rounding of the arm can make arbitrarily
    # small, so it is held to 1.5 x the arm's error or 2e-3 relative, whichever is larger
    e = abs(float(ours[0]["loss"]) - float(want[0]["loss"])) / abs(float(want[0]["loss"]))
    ea = abs(float(arm[0]["loss"]) - float(want[0]["loss"])) / abs(float(want[0]["loss"]))
    print(f"{tag}: loss rel err {e:.2e} (bf16 oracle {ea:.2e})")
    if e > max(1.5 * ea, 2e-3):
        bad.append(f"{tag}: loss: error {e:.3e} vs the bf16 oracle's {ea:.3e}")
    assert not bad, "\n".join(bad)
    return ours, want


@pytest.mark.parametrize("name", ["lfvila_cls_eval_b6", "lfvila_cls_train_droppath"])
def test_module_against_golden_under_the_calibrated_rule(dev, tmp_path, golden_dir, name):
    gold = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    cfg = SO.Swin3DCfg(**gold["cfg"])
    ours, want = cls_case(dev, str(tmp_path), name, cfg, gold["n_labels"], gold["B"], gold["D"], gold["H"], gold["W"],
                          gold["weight_seed"], gold["data_seed"], masks=gold["masks"])
    # the fp32 oracle on the GPU is the reference's own result (the golden, made on the CPU)
    for k in FEATS:
        assert float((want[0][k].cpu() - gold["out"][k]).norm() / gold["out"][k].norm()) < 1e-4, k
    for n, ref in gold["grads"].items():
        got = want[1][n].cpu()
        got = got if got.shape == ref.shape else got[:ref.shape[0]]
        assert float((got - ref).norm() / ref.norm().clamp_min(1e-30)) < 1e-3, n


@pytest.mark.parametrize("n_labels,video_dtype", [(180, f32), (4, f16)])
def test_released_geometry_against_fp32_oracle(dev, tmp_path, n_labels, video_dtype):
    """coin_cls.yaml / lvu_*_cls.yaml: the released encoder at full depth, 2 clips x 32 frames x 192 x 320 (a 3 x 5 final
    grid), a 180-label and a 4-label head; fp16 video as the trainer's --fp16 casts it (the oracle takes the same fp16
    values)."""
    cls_case(dev, str(tmp_path), f"released {n_labels} labels {str(video_dtype)[6:]}", SO.Swin3DCfg(), n_labels, 2, 32,
             192, 320, weight_seed=21, data_seed=22, video_dtype=video_dtype, autocast=False)


# ------------------------------------------------------------------------------------------ evaluation memory
def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def test_no_grad_evaluation_keeps_no_activations(dev, tmp_path):
    """Under torch.no_grad() (the trainer's @torch.no_grad() evaluate) the encoder keeps nothing for a backward: the peak
    above the resident memory stays below the video's frame copy + the patch matrix + 6 x the largest activation (the
    first stage's MLP hidden layer), far under the training forward's; the outputs are bitwise those of a forward with grad."""
    from xpretrain_b200.modeling import LFVILA_Video_Classification
    cfg = SO.Swin3DCfg()
    B, D, H, W = 2, 32, 192, 320
    model = LFVILA_Video_Classification(None, _config(str(tmp_path), cfg, 180)).to(dev).eval()
    video = SO.synthetic_video(B, D, H, W, cfg, seed=3).to(dev)
    labels = L.synthetic_labels(B, 180).to(dev)
    rows0 = B * D * (H // 8) * (W // 8)
    bound = video.numel() * 4 + rows0 * 192 * 2 + 6 * rows0 * 4 * cfg.embed_dim * 2
    for name, fn in (("classifier", lambda: model(video, labels)), ("encoder", lambda: model.video_encoder(video)[0])):
        with torch.no_grad():
            fn()                                                         # index tables and weight copies
        with torch.no_grad():
            ev, peak_eval = _peak(fn)
        tr, peak_train = _peak(fn)
        print(f"{name}: peak above resident, no_grad {peak_eval / 2**20:.0f} MiB (bound {bound / 2**20:.0f}), "
              f"training forward {peak_train / 2**20:.0f} MiB")
        assert peak_eval < bound, (name, peak_eval, bound)
        assert peak_eval < 0.35 * peak_train, (name, peak_eval, peak_train)
        pairs = [(ev[k], tr[k]) for k in FEATS + ("loss", "acc")] if isinstance(ev, dict) else [(ev, tr)]
        assert all(same_bits(a, b.detach()) for a, b in pairs)
        del tr
