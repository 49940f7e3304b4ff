"""The bf16 arm of CLIP-ViP and the per-frame CLIP model, and the calibrated rule they are held to: shared by
test_gpu_clipvip_calibration.py and the CPU negative controls of test_clipvip_calibration_cpu.py.

  Bf16Arm            the oracle (oracle/clipvip_oracle.py, frame_clip_oracle.py) rounded exactly where
                     modeling/clip_vip.py rounds, on the module's residual stream
  oracle_run         one run of the oracle: fp32 (the truth), the arm, or bf16 autocast
  rule_violations    the rule on both feature matrices and every parameter gradient, whole and per slice, the k third of
                     every qkv bias against its rounding bound, and the exact zeros of the text embeddings
"""
import contextlib

import torch
import torch.nn.functional as F

from contract_harness import ABS_FLOOR, FACTOR, FLOOR, calibrated_model_rows, no_tf32
from oracle import attention_ref as R
from oracle import clipvip_oracle as O
from oracle import frame_clip_oracle as FC

bf16, f16, f32 = torch.bfloat16, torch.float16, torch.float32
KB_U = 2.0 ** -8           # bf16's largest relative rounding error


# ============================================================================================================ the arm
class _Round(torch.autograd.Function):
    """Forward: the value rounded to `fwd` (None: unchanged).  Backward: the gradient rounded to bf16 when `bwd`."""

    @staticmethod
    def forward(ctx, x, fwd, bwd):
        ctx.bwd = bwd
        return x.clone() if fwd is None else x.to(fwd).to(x.dtype)

    @staticmethod
    def backward(ctx, g):
        return (R.bf(g) if ctx.bwd else g), None, None


def rnd(x, fwd=bf16, bwd=False):
    return _Round.apply(x, fwd, bwd)


class _QuickGelu(torch.autograd.Function):
    """fc1's epilogue: the activation of the fp32 accumulator rounded once; the pre-activation stored in bf16, and the
    backward (the dgrad epilogue) takes dQuickGELU at that stored value and rounds dpre."""

    @staticmethod
    def forward(ctx, acc):
        pre = R.bf(acc)
        ctx.save_for_backward(pre)
        return R.bf(acc * torch.sigmoid(1.702 * acc))

    @staticmethod
    def backward(ctx, g):
        (pre,) = ctx.saved_tensors
        s = torch.sigmoid(1.702 * pre)
        return R.bf(g * (s + 1.702 * pre * s * (1 - s)))


def _rows(t):
    B, H, S, d = t.shape
    return t.transpose(1, 2).reshape(B * S, H * d)


def _heads(t, B, H):
    return t.reshape(B, -1, H, t.shape[1] // H).transpose(1, 2)


class _Attention(torch.autograd.Function):
    """The attention kernels' arithmetic: oracle/attention_ref's float64 vip_ref / text_ref with arm "vip" / "text" (the
    rounding test_gpu_attention_contract pins), on the bf16 q (scaled), k, v.  The backward rounds the incoming gradient
    (da, the out_proj dgrad) and returns the rounded dq / dk / dv of the kernels, dq with respect to the scaled q."""

    @staticmethod
    def forward(ctx, q, k, v, kind, geo, mask, sink=None):
        B, H = q.shape[:2]
        qkv = torch.cat([_rows(q), _rows(k), _rows(v)], dim=1)
        ctx.save_for_backward(qkv)
        ctx.meta = kind, geo, mask, B, H, q.dtype
        ctx.sink = sink
        return _heads(_Attention._ref(qkv, None, *ctx.meta[:5])["out"], B, H).to(q.dtype)

    @staticmethod
    def _ref(qkv, dout, kind, geo, mask, B, H):
        if kind == "vip":
            M, T, L = geo
            return R.vip_ref(qkv, dout, B, H, T, L, M, arm="vip")
        return R.text_ref(qkv, mask, dout, B, H, geo, arm="text")

    @staticmethod
    def backward(ctx, g):
        (qkv,) = ctx.saved_tensors
        kind, geo, mask, B, H, dt = ctx.meta
        dout = R.bf(_rows(g))
        res = _Attention._ref(qkv, dout, kind, geo, mask, B, H)
        d = res["dqkv"]
        C = qkv.shape[1] // 3
        if ctx.sink is not None:
            floors, name = ctx.sink
            floors[name] = k_bias_bound(qkv, dout, res["out"], d[:, C:2 * C], H, kind == "vip")
        return tuple(_heads(d[:, i * C:(i + 1) * C], B, H).to(dt) for i in range(3)) + (None, None, None, None)


def k_bias_bound(qkv, dout, out, dk, H, delta_from_o):
    """A bound on what rounding alone puts into the k third of the qkv bias gradient, sum_j dk_j, whose exact value is 0:
    the bf16 store of every dk row (KB_U sum_j |dk_j|) and, where the kernel takes delta = rowsum(dO * O) from the stored
    bf16 O (the proxy-token kernels), that O's rounding: sum_j dk_j = sum_i q_i (delta_exact_i - delta_used_i), and
    |delta_exact_i - delta_used_i| <= KB_U sum_d |dO_id O_id|.  The text kernel forms delta in fp32 from P and dP."""
    C = dk.shape[1]
    bound = KB_U * dk.double().abs().sum(0)
    if delta_from_o:
        rows = dout.shape[0]
        dd = (dout.double() * out.double()).abs().view(rows, H, -1).sum(-1, keepdim=True)        # [rows, H, 1]
        bound = bound + KB_U * (qkv[:, :C].double().abs().view(rows, H, -1) * dd).sum(0).reshape(C)
    return bound


_ORACLE_VIP_CORE, _ORACLE_TEXT_EMBEDDINGS = O.vip_core, O.text_embeddings


class Bf16Arm:
    """The oracle rounded where modeling/clip_vip.py rounds (_layer_fwd, _layer_bwd, _vision_fwd, _text_fwd, the heads and
    the embedding kernels of embed.cu), on the residual stream `stream`:

    forward
      - GEMMs: bf16 weight mirrors and bf16 inputs, fp32 accumulation, fp32 bias.  Rounded to bf16: qkv, the attention
        output, the out_proj and fc2 branches (fp32 / fp16 streams) and f1 = QuickGELU(fc1) taken from the fp32 accumulator;
        the pre-activation is stored in bf16.  q's scale 0.125 is a power of two: rounding before or after it is the same.
        The projections write fp32.
      - LayerNorm: fp32 statistics of the stream, output in bf16; pre_layrnorm writes the stream itself.
      - residual stream: "fp32" the add happens in fp32 inside the next LayerNorm and stays fp32; "fp16" the same sum stored
        as fp16; "bf16" the add happens in the out_proj / fc2 epilogue (accumulator + bias + stream) and is rounded to bf16.
      - attention: _Attention (vip_ref / text_ref with their kernel arms); the per-frame vision tower runs the proxy-token
        kernel at M = 1, T = 1.
      - embeddings: frames rounded to bf16 (the patchify kernels); the patch GEMM's epilogue adds the bf16 table
        bf16(temporal + position) and rounds; the CLS / proxy rows are bf16(embedding + position row 0); the text rows
        bf16(token + position).
    backward
      - bf16 gradient at every block boundary and at every residual sum (dx1, dxin: the LayerNorm backward adds the
        residual gradient in fp32 and rounds once).
      - dpre: dQuickGELU at the stored bf16 pre-activation, rounded; dh2, da, dh (one fused q / k / v dgrad) rounded at the
        LayerNorm / attention outputs; dqkv rounded by the attention arm.
      - weight and bias gradients: fp32 sums of bf16 operands (autograd over the rounded values).
      - the l2-norm and frame-pool backwards write dproj in bf16; dpooled and the embedding-sum gradients are bf16.

    `mistake` plants one deliberate error (the negative controls of test_clipvip_calibration_cpu.py)."""

    MISTAKES = ("proxy_no_pos0", "align_corners", "global_sees_frame0", "patch_grid_transposed", "q_bias_unscaled",
                "temporal_reversed")

    def __init__(self, stream="fp32", mistake=None):
        assert stream in ("fp32", "fp16", "bf16") and (mistake is None or mistake in self.MISTAKES)
        self.stream, self.mistake = stream, mistake
        self.stream_dt = {"fp32": None, "fp16": f16, "bf16": bf16}[stream]
        self.k_floors = {}                  # k_proj.bias name -> k_bias_bound of its layer, filled by the backward
        self._layers = {}

    def _sink(self, tower):
        i = self._layers[tower] = self._layers.get(tower, -1) + 1
        return self.k_floors, f"{tower}_model.encoder.layers.{i}.self_attn.k_proj.bias"

    # ---------------------------------------------------------------------------------------------- arithmetic points
    def linear(self, x, sd, prefix):
        w, b = rnd(sd[prefix + ".weight"]), sd.get(prefix + ".bias")
        if self.mistake == "q_bias_unscaled" and prefix.endswith("q_proj"):
            b = b / 0.125                               # after the caller's * 0.125 the bias is left unscaled
        acc = F.linear(rnd(x), w, b)
        if prefix.endswith("projection"):
            return rnd(acc, None, True)                 # fp32 out; dproj from the l2-norm / frame-pool backward in bf16
        if prefix.endswith("fc1"):
            return acc                                  # rounded by quick_gelu
        if prefix.endswith(("out_proj", "fc2")) and self.stream == "bf16":
            return acc                                  # the epilogue adds the stream before rounding: residual_add
        return rnd(acc)

    def quick_gelu(self, acc):
        return _QuickGelu.apply(acc)

    def layer_norm(self, x, sd, prefix, eps):
        y = F.layer_norm(x, (x.shape[-1],), sd[prefix + ".weight"], sd[prefix + ".bias"], eps)
        if prefix.endswith("pre_layrnorm"):
            return rnd(y, self.stream_dt, True)
        return rnd(y, bf16, True)

    def residual_add(self, x, h):
        return rnd(x + h, self.stream_dt, True)

    def vip_core(self, q, k, v, size):
        if self.mistake == "global_sees_frame0":
            M, T, L = size
            o = _ORACLE_VIP_CORE(q, k, v, size)
            og = torch.softmax(q[:, :, :M] @ k[:, :, :M + L].transpose(-1, -2), dim=-1) @ v[:, :, :M + L]
            return rnd(torch.cat([og, o[:, :, M:]], dim=2), bf16, True)
        return _Attention.apply(rnd(q), rnd(k), rnd(v), "vip", size, None, self._sink("vision"))

    def dense_core(self, q, k, v, add_mask):
        if add_mask is None:                            # the per-frame vision tower: M = 1, T = 1
            return _Attention.apply(q, k, v, "vip", (1, 1, q.shape[2] - 1), None, self._sink("vision"))
        mask = (add_mask[:, 0, -1, :] == 0).long()      # the last row of the causal mask keeps every unpadded key
        return _Attention.apply(q, k, v, "text", q.shape[2], mask, self._sink("text"))

    def text_embeddings(self, sd, ids):
        x = rnd(_ORACLE_TEXT_EMBEDDINGS(sd, ids), bf16, True)
        return rnd(x, f16) if self.stream == "fp16" else x     # the bf16 rows enter an fp16 stream converted

    def _patch_rows(self, frames, sd, cfg, pre):
        """frames [N, 3, H, W] -> the patch GEMM's fp32 accumulator [N, L, C] over bf16 frames and weights."""
        N, C, H, W = frames.shape
        p = cfg.patch
        x = R.bf(frames).reshape(N, C, H // p, p, W // p, p)
        x = x.permute(0, 4, 2, 1, 3, 5) if self.mistake == "patch_grid_transposed" else x.permute(0, 2, 4, 1, 3, 5)
        w = rnd(sd[pre + "patch_embedding.weight"])
        return x.reshape(N, -1, C * p * p) @ w.reshape(w.shape[0], -1).t()

    def temporal_table(self, sd, T, pre):
        table = sd[pre + "temporal_embedding"]
        if T != table.shape[1]:
            table = F.interpolate(table.transpose(1, 2), size=T, mode="linear",
                                  align_corners=self.mistake == "align_corners").transpose(1, 2)
        return table.flip(1) if self.mistake == "temporal_reversed" else table

    def vip_embeddings(self, sd, video, cfg, pre="vision_model.embeddings."):
        B, T = video.shape[:2]
        patches = self._patch_rows(video.reshape(B * T, *video.shape[2:]), sd, cfg, pre)
        L, C = patches.shape[1], patches.shape[2]
        pos = sd[pre + "position_embedding.weight"]
        table = pos[1:].reshape(1, 1, L, C)
        if pre + "temporal_embedding" in sd:
            table = self.temporal_table(sd, T, pre).unsqueeze(2) + table              # [1, T, L, C]
        rows = patches.reshape(B, T, L, C) + rnd(table)
        cls = (sd[pre + "class_embedding"] + pos[0]).expand(B, 1, -1)
        added = sd[pre + "added_cls"]
        proxies = (added if self.mistake == "proxy_no_pos0" else added + pos[0]).unsqueeze(0).expand(B, -1, -1)
        x = torch.cat([cls, proxies, rows.reshape(B, T * L, C)], dim=1)
        return rnd(x, bf16, True), (1 + added.shape[0], T, L)

    def frame_embeddings(self, sd, images, cfg, pre="vision_model.embeddings."):
        patches = self._patch_rows(images, sd, cfg, pre)
        pos = sd[pre + "position_embedding.weight"]
        rows = patches + rnd(pos[1:], bf16)
        cls = (sd[pre + "class_embedding"] + pos[0]).expand(images.shape[0], 1, -1)
        return rnd(torch.cat([cls, rows], dim=1), bf16, True)

    # -------------------------------------------------------------------------------------------------- swapping in
    @contextlib.contextmanager
    def installed(self):
        swaps = [(O, n) for n in ("linear", "quick_gelu", "layer_norm", "residual_add", "vip_core", "dense_core",
                                  "text_embeddings", "vip_embeddings")] + [(FC, "frame_embeddings")]
        saved = [(mod, n, getattr(mod, n)) for mod, n in swaps]
        for mod, n, _ in saved:
            setattr(mod, n, getattr(self, n))
        try:
            yield
        finally:
            for mod, n, f in saved:
                setattr(mod, n, f)


# ======================================================================================================= the runs
def features_objective(B, P, seed):
    """(vis, txt, logit_scale) -> sum(vis * w_v) + sum(txt * w_t), seeded cotangents of unit scale per row."""
    g = torch.Generator().manual_seed(seed)
    w_v, w_t = torch.randn(B, P, generator=g), torch.randn(B, P, generator=g)

    def obj(vis, txt, scale):
        return (vis * w_v.to(vis.device)).sum() + (txt * w_t.to(txt.device)).sum()
    return obj


def oracle_run(sd, video, ids, mask, cfg, objective, mode, stream="fp32", per_frame=False, arm=None):
    """mode: 'fp32' (the truth), 'bf16' (the arm of `stream`, or `arm`) or 'autocast'.  Every tensor lives on the device of
    `video`.  -> (vis, txt, {name: grad}, {k_proj.bias name: k_bias_bound}) in fp32; the bounds come from the arm only."""
    dv = video.device
    sdo = {k: (v.detach().to(dv, f32, copy=True).requires_grad_(True) if v.is_floating_point() else v.to(dv))
           for k, v in sd.items()}
    if mode == "bf16":
        arm = arm or Bf16Arm(stream)
        ctx = arm.installed()
    else:
        ctx = contextlib.nullcontext()
    with ctx, torch.autocast(dv.type, dtype=bf16, enabled=mode == "autocast"), no_tf32():
        fwd = FC.frame_clip_forward if per_frame else O.clip_vip_forward
        o = fwd(sdo, video.to(dv, f32), ids.to(dv), mask.to(dv), cfg)
        vis, txt = o["vis_features"].float(), o["text_features"].float()
        objective(vis, txt, sdo["logit_scale"]).backward()
    grads = {k: t.grad for k, t in sdo.items() if t.is_floating_point() and t.grad is not None}
    return vis.detach(), txt.detach(), grads, (arm.k_floors if mode == "bf16" else {})


# ======================================================================================================= the rule
def _head_ids(g, width, dim):
    """Slice ids per 64-wide block of dimension `dim` of g."""
    n = g.shape[dim]
    ids = torch.arange(n, device=g.device) // width
    return ids.view(*[n if i == dim else 1 for i in range(g.dim())]).expand(g.shape)


def param_slices(grads):
    out = {}
    for n, g in grads.items():
        if g.numel() == 0:
            continue
        if n.endswith(("q_proj.weight", "k_proj.weight", "v_proj.weight", "q_proj.bias", "k_proj.bias", "v_proj.bias")):
            out[n] = (_head_ids(g, 64, 0), lambda i: f"head {i}")
        elif n.endswith("out_proj.weight"):
            out[n] = (_head_ids(g, 64, 1), lambda i: f"input head {i}")
        elif n.endswith(("position_embedding.weight", "added_cls")):
            out[n] = (_head_ids(g, 1, 0), lambda i: f"row {i}")
        elif n.endswith("temporal_embedding"):
            out[n] = (_head_ids(g, 1, 1), lambda i: f"table row {i}")
        elif n.endswith("patch_embedding.weight"):
            ids = (_head_ids(g, 64, 0) * 3 + _head_ids(g, 1, 1))
            out[n] = (ids, lambda i: f"(channels {64 * (i // 3)}.., colour {i % 3})")
        elif n.endswith("projection.weight"):
            out[n] = (_head_ids(g, 64, 0), lambda i: f"output rows {64 * i}..")
    return out


def k_bias_violations(tag, name, got, ref, arm, bound):
    """The k third of every qkv bias gradient is zero exactly (a shift of every key leaves each softmax row unchanged), so
    ours and the arm's are rounding alone, mostly that of the O each side's delta reads, carried by the few global rows
    with the largest dO.  Fed the module's own qkv, O and da, the proxy-token backward matches vip_ref's arm per head to
    1.03 x (H100, full-depth inputs), but at model level each side rounds its own O, and per head the two draws differed
    up to 17 x while the whole tensors agreed to 1.6 x.  So each head and the whole tensor are held to 1.5 x the arm plus
    k_bias_bound, whose O term allows each delta_i only KB_U of sum_d |dO_id O_id|: a stale or wrong O, or a dropped
    delta term, moves delta_i by the order of that sum itself."""
    bad = []
    b = bound if bound is not None else torch.zeros_like(ref, dtype=torch.float64)
    d = lambda x: x.double().reshape(-1, 64)                  # noqa: E731   per head
    e_k, e_a, fl = (d(got) - d(ref)).norm(dim=1), (d(arm) - d(ref)).norm(dim=1), d(b).norm(dim=1)
    fl = fl + FLOOR * d(ref).norm(dim=1) + ABS_FLOOR * 8
    ratio = e_k / (FACTOR * e_a + fl)
    w = int(ratio.argmax())
    if float(ratio[w]) > 1:
        bad.append(f"{tag}: {name}: head {w}: error {float(e_k[w]):.3e} against the arm's {float(e_a[w]):.3e} and the "
                   f"rounding bound {float(fl[w]):.3e}")
    ew, ea, bw = (float((x.double() - ref.double()).norm()) for x in (got, arm, ref + b))
    if ew > FACTOR * ea + bw:
        bad.append(f"{tag}: {name}: error {ew:.3e} against the arm's {ea:.3e} and the rounding bound {bw:.3e}")
    print(f"{tag}: {name}: err / (1.5 x arm err + bound) {ew / (FACTOR * ea + bw):.3f} whole, {float(ratio[w]):.3f} worst head")
    return bad


def rule_violations(tag, ours, want, arm, ac, ids):
    """ours / want / arm / ac (ac may be None): oracle_run's (vis, txt, {name: grad}, ...).  The rule on every tensor, whole
    and per slice; the k bias against its bound; the exact zeros of the text embeddings.  -> (violations, worst
    whole-tensor ratio, worst slice ratio)."""
    assert set(ours[2]) == set(want[2]), f"{tag}: gradients received differ from the oracle's: {set(ours[2]) ^ set(want[2])}"
    dv = want[0].device
    if ac is None:
        ac = (None, None, {n: None for n in want[2]})
    ours = (ours[0].to(dv), ours[1].to(dv), {n: g.to(dv) for n, g in ours[2].items()})
    rows = [("vis", ours[0], want[0], arm[0], ac[0]), ("txt", ours[1], want[1], arm[1], ac[1])]
    assert "logit_scale" not in want[2] and "logit_scale" not in ours[2]
    names = sorted(want[2])
    rows += [(n, ours[2][n], want[2][n], arm[2][n], ac[2][n]) for n in names]
    per_sample = lambda x: (_head_ids(x, 1, 0), lambda i: f"sample {i}")        # noqa: E731
    slices = {"vis": per_sample(want[0]), "txt": per_sample(want[1]), **param_slices(want[2])}
    tok, tpos = "text_model.embeddings.token_embedding.weight", "text_model.embeddings.position_embedding.weight"
    present = torch.unique(ids.to(dv))
    slices.pop(tok, None)
    rows.append((tok + "[ids]",) + tuple(r[2][tok][present] for r in (ours, want, arm))
                + (ac[2][tok] if ac[2][tok] is None else ac[2][tok][present],))
    slices[tok + "[ids]"] = (_head_ids(want[2][tok][present], 1, 0), lambda i: f"id {int(present[i])}")
    kb = [r for r in rows if r[0].endswith("k_proj.bias")]
    bad, worst, worst_sl = calibrated_model_rows(tag, [r for r in rows if r not in kb], slices)
    for name, got, ref, a, _ in kb:
        bad += k_bias_violations(tag, name, got, ref, a, arm[3].get(name))
    # exact zeros
    absent = torch.ones(want[2][tok].shape[0], dtype=torch.bool, device=dv)
    absent[present] = False
    Lt = ids.shape[1]
    eos = int(ids.argmax(dim=-1).max())
    for what, g in (("token rows of ids absent from the batch", ours[2][tok][absent]),
                    (f"text position rows >= Lt = {Lt}", ours[2][tpos][Lt:]),
                    (f"text position rows past the longest EOS ({eos})", ours[2][tpos][eos + 1:])):
        if int((g != 0).sum()):
            bad.append(f"{tag}: {what}: {int((g != 0).sum())} elements are not exactly 0")
    return bad, worst, worst_sl
