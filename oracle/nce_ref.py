"""High-precision references of the contrastive-loss kernels, their bf16 arms and a derived element-wise error bound.

Every function takes the kernels' own operands: the fp32 embeddings that the fused kernel (nce_fused.cu) and the hi/lo
split logits GEMM (nce.cu:20-34) read, or the fp32 unscaled logits z that xp_nce_terms / xp_nce_dsl receive.  It returns
float64 tensors.  `exact` is the float64 value of the operation on those inputs; the arm rounds only where the kernel
rounds (file:line next to each point), so that |arm - exact| is what the kernel's own rounding costs.  DESIGN.md §2 holds
a kernel to a small multiple of it slice by slice.

The element bound is derived, not tuned.  Every intermediate value is carried as an `Err`: its float64 value and a bound
on how far the kernel's fp32 value of it can lie from that value, propagated by the usual first-order running error
analysis with the kernels' own operations:
  - every fp32 operation rounds once, by at most 2^-24 of its result, and may flush a result below 2^-126 to zero
    (the library is built with --use_fast_math, Makefile NVFLAGS);
  - expf / __expf is ex2.approx.ftz(x log2 e): 2^-22 relative (PTX ISA) plus the rounding of its result, and the rounding
    of x log2 e, which costs 2^-23 |x| relative;
  - logf / __logf is lg2.approx x ln 2: 2^-21.4 absolute near 1, 3 ulp relative elsewhere;
  - a log-sum-exp over n entries kept as (max, sum-exp) partials merged tile by tile (nce_fused.cu:246-311,
    nce.cu:79-85, 122-187, 242-263): the largest input error, the sum's n + merges roundings, one exp error per entry
    and per merge, and the log;
  - a fixed-order sum whose longest chain of additions is `depth`: depth 2^-24 sum |x_j|.
An error in an exponent argument therefore reaches dL/dZ weighted by the probabilities (p_row + p_col) / n of the terms
it enters.  d logit_scale = sum G Z cancels, so its bound is carried by sum |G Z|.

  split_logits   V T^T, its split arm hi*hi + hi*lo + lo*hi (nce_fused.cu:186-187, 210; nce.cu:26-27), the logits error
  terms          any XpNceTerms table (two-term InfoNCE included): loss, s dL/dZ, d logit_scale
  dsl            NCELearnableTempDSLLoss (xp_nce_dsl)
  feature_grads  dX = (sG) Y, dY = (sG)^T X of the gradient GEMMs
Pure torch; runs on the CPU or on a GPU (where the tests compute it)."""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import torch

from oracle.embed_ref import ulp_bf16

F64 = torch.float64
U = 2.0 ** -24
EXP_ABS = 2.0 ** -21      # ex2.approx: 2^-22 relative, plus the rounding of its fp32 result
LOG_ABS = 2.0 ** -21      # lg2.approx x ln 2: 2^-21.41 absolute on [0.5, 2]
TINY = 2.0 ** -126        # fp32 results below the normal range may flush to zero
ROW, COL = 0, 1


def bf(x: torch.Tensor) -> torch.Tensor:
    """Round to bf16 (nearest even), keeping the tensor's dtype."""
    return x.to(torch.bfloat16).to(x.dtype)


def ftz(x: torch.Tensor) -> torch.Tensor:
    """Flush values below the fp32 normal range to zero, as the kernels' fast-math arithmetic does."""
    return torch.where(x.abs() < TINY, torch.zeros_like(x), x)


# ------------------------------------------------------------------------------------------ running error bound
class Err:
    """A float64 value `v` and a bound `e` on |kernel's fp32 value - v|."""

    def __init__(self, v: torch.Tensor, e: Optional[torch.Tensor] = None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e


def _rnd(v):
    return U * v.abs() + TINY


def const(x, like: torch.Tensor) -> Err:
    """A value the kernel holds exactly (an exact 0, 1 or 2)."""
    return Err(torch.as_tensor(x, dtype=F64, device=like.device).expand_as(like).clone())


def add(a: Err, b: Err, sign: float = 1.0) -> Err:
    v = a.v + sign * b.v
    return Err(v, a.e + b.e + _rnd(v))


def mul(a: Err, b: Err) -> Err:
    v = a.v * b.v
    return Err(v, a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e + _rnd(v))


def exp(a: Err) -> Err:
    """__expf of an argument known to within a.e."""
    v = torch.exp(a.v)
    eta = EXP_ABS + 2 * U * (a.v.abs() + a.e)
    return Err(v, v * (torch.expm1(a.e) + eta * torch.exp(a.e)) + TINY)


def lse(x: Err, keep: torch.Tensor) -> Err:
    """log sum exp along dim 1 over the entries `keep` marks, as (max, sum-exp) partials merged in tile order."""
    xm = x.v.masked_fill(~keep, -math.inf)
    m = xm.amax(1)
    L = torch.logsumexp(xm, 1)
    p = torch.exp(xm - L[:, None])
    cnt = keep.sum(1).to(F64)
    spread = torch.nan_to_num(p * (xm - m[:, None]).abs(), nan=0.0).sum(1)       # E_p |x - max|
    merges = 16 + cnt / 64                                                         # 8 warps + one merge per tile
    e_in = x.e.masked_fill(~keep, 0.0).amax(1)
    e = (e_in + (merges + 2) * EXP_ABS + 4 * U * spread + (3 * cnt + 8) * U + cnt * TINY
         + LOG_ABS + 4 * U * (L - m).abs() + U * L.abs())
    return Err(L, e)


def total(x: Err, depth: float) -> Err:
    """A fixed-order fp32 sum of every element whose longest addition chain is `depth` long."""
    v = x.v.sum()
    return Err(v, x.e.sum() + depth * U * x.v.abs().sum() + TINY * x.v.numel())


def _sel(x: Err, mask: torch.Tensor) -> Err:
    """x where mask, an exact 0 elsewhere."""
    return Err(x.v.masked_fill(~mask, 0.0), x.e.masked_fill(~mask, 0.0))


# ------------------------------------------------------------------------------------------------ logits
def split_logits(V: torch.Tensor, T: torch.Tensor) -> Dict[str, torch.Tensor]:
    """V [N, d], T [M, d] fp32.  exact = V T^T in float64; arm = hi*hi + hi*lo + lo*hi with hi = bf16(v),
    lo = bf16(v - hi) (nce_fused.cu:186-187 and the bf16 pack at :190; nce.cu:26-27), lo*lo dropped (nce_fused.cu:206-214;
    [hi|hi|lo] . [hi|lo|hi], nce.cu:29-31); err = |arm - exact| + the fp32 accumulation bound (3d + 1) 2^-24 sum |products|
    of the K = 3d products, each exact in fp32."""
    def parts(x):
        x = x.float()
        hi = x.to(torch.bfloat16).float()
        lo = (x - hi).to(torch.bfloat16).float()
        return hi.to(F64), lo.to(F64)
    vh, vl = parts(V)
    th, tl = parts(T)
    exact = V.to(F64) @ T.to(F64).T
    arm = vh @ th.T + (vh @ tl.T + vl @ th.T)
    absprod = vh.abs() @ th.abs().T + vh.abs() @ tl.abs().T + vl.abs() @ th.abs().T
    K = 3 * V.shape[1]
    return {"exact": exact, "arm": arm, "err": (arm - exact).abs() + (K + 1) * U * absprod,
            "vis_hi": vh, "txt_hi": th}


def scale_of(logit_scale: Optional[torch.Tensor] = None, scale: Optional[float] = None, device=None) -> Err:
    """s = expf(logit_scale) of the fp32 device log-scale (nce_fused.cu:230, nce.cu:75), or the host fp32 constant."""
    if logit_scale is not None:
        ls = logit_scale.reshape(()).to(F64).to(device)
        v = torch.exp(ls)
        return Err(v, v * (EXP_ABS + 2 * U * ls.abs()))
    return Err(torch.tensor(float(torch.tensor(scale, dtype=torch.float32)), dtype=F64, device=device))


# ------------------------------------------------------------------------------------------ term tables
def terms(z: Sequence[torch.Tensor], table, s: Err, z_err: Optional[Sequence[torch.Tensor]] = None,
          z_arm: Optional[Sequence[torch.Tensor]] = None, reduce_depth: Optional[float] = None) -> Dict[str, object]:
    """xp_nce_terms (nce.cu:192-361) and the fused kernel (nce_fused.cu:229-359, the table ((ROW, 1, 0, 0),
    (COL, 1, 0, 0))) on unscaled logits z[m] [n_m, n_m] (float64 values), each known to within z_err[m].
    table: (axis, members, excl_diag, target) with bit masks over the matrices, as XpNceTerms.

    Returns lists over the matrices of `exact` (s dL/dZ), `arm` (bf16 of s dL/dZ computed in float64 from z_arm, or from
    z; nce.cu:322, nce_fused.cu:327), `bound` (element bound of the kernel's bf16 s dL/dZ), `G` (dL/dZ), and the scalars
    `loss`, `loss_bound`, `dscale` (dL/d logit_scale = sum G Z), `dscale_bound`."""
    n_m = [x.shape[0] for x in z]
    dev = z[0].device
    z_err = z_err or [torch.zeros_like(x) for x in z]
    Z = [mul(Err(x.to(F64), e.to(F64)), Err(s.v.expand_as(x), s.e.expand_as(x))) for x, e in zip(z, z_err)]
    eye = [torch.eye(n, dtype=torch.bool, device=dev) for n in n_m]

    def lses(Zs):
        out = []
        for axis, members, excl, target in table:
            vs, es, ks = [], [], []
            for m, Zm in enumerate(Zs):
                if not (members >> m) & 1:
                    continue
                X = Zm if axis == ROW else Err(Zm.v.T, Zm.e.T)
                vs.append(X.v)
                es.append(X.e)
                ks.append(~eye[m] if (excl >> m) & 1 else torch.ones_like(eye[m]))
            out.append(lse(Err(torch.cat(vs, 1), torch.cat(es, 1)), torch.cat(ks, 1)))
        return out

    def grads(Zs, L):
        G = []
        for m, Zm in enumerate(Zs):
            gg = const(0.0, Zm.v)
            for t, (axis, members, excl, target) in enumerate(table):
                if not (members >> m) & 1:
                    continue
                Lt = L[t]
                Lb = Err(Lt.v[:, None].expand_as(Zm.v), Lt.e[:, None].expand_as(Zm.v)) if axis == ROW else \
                    Err(Lt.v[None, :].expand_as(Zm.v), Lt.e[None, :].expand_as(Zm.v))
                ex = exp(add(Zm, Lb, -1.0))
                gg = add(gg, _sel(ex, ~eye[m]) if (excl >> m) & 1 else ex)
                if target == m:
                    gg = add(gg, Err(eye[m].to(F64)), -1.0)
            G.append(mul(gg, Err(torch.full_like(Zm.v, 1.0 / n_m[m]), torch.full_like(Zm.v, U / n_m[m]))))
        return G

    L = lses(Z)
    G = grads(Z, L)
    sG = [mul(g, Err(s.v.expand_as(g.v), s.e.expand_as(g.v))) for g in G]
    n_tiles = sum(((n + 63) // 64) * ((n + 127) // 128) for n in n_m)
    depth = reduce_depth if reduce_depth is not None else 64 + n_tiles / 256 + max(n_m) / 256
    loss = None
    for t, (axis, members, excl, target) in enumerate(table):
        diag = Err(Z[target].v.diagonal(), Z[target].e.diagonal())
        lt = total(add(L[t], diag, -1.0), depth)
        lt = mul(lt, Err(torch.tensor(1.0 / n_m[target], dtype=F64, device=dev)))
        loss = lt if loss is None else add(loss, lt)
    ds = None
    for g, Zm in zip(G, Z):
        dm = total(mul(g, Zm), depth)
        ds = dm if ds is None else add(ds, dm)
    # the arm: the same float64 computation from the arm's logits, one bf16 rounding (flushed as the kernel's ftz)
    if z_arm is None:
        arm = [ftz(bf(x.v)) for x in sG]
    else:
        Za = [Err(x.to(F64) * s.v) for x in z_arm]
        arm = [ftz(bf(g.v * s.v)) for g in grads(Za, lses(Za))]
    bound = [x.e + ulp_bf16(x.v.abs() + x.e) + TINY for x in sG]
    return {"exact": [x.v for x in sG], "arm": arm, "bound": bound, "G": [g.v for g in G],
            "loss": loss.v, "loss_bound": loss.e, "dscale": ds.v, "dscale_bound": ds.e}


INFONCE = ((ROW, 1, 0, 0), (COL, 1, 0, 0))


def fused_depth(N: int) -> float:
    """Longest addition chain of the fused kernel's loss / d logit_scale: 128 rows per thread, the warp and warpgroup
    reductions, then the last CTA's sum over the (N/128)^2 tile shares (nce_fused.cu:319-352)."""
    nt = (N + 127) // 128
    return 136 + nt * nt


# ------------------------------------------------------------------------------------------------- DSL
def dsl(z: torch.Tensor, s: Err, z_err: Optional[torch.Tensor] = None, z_arm: Optional[torch.Tensor] = None
        ) -> Dict[str, object]:
    """xp_nce_dsl (nce.cu:192-361, 485-533) on the unscaled fp32 logits z [n, n], in the kernel's order:
    lse_r, lse_c of Z; la = row LSE of A' = Z Pc, lb = column LSE of B' = Z Pr; GA = (exp(A' - la) - I)/n,
    GB = (exp(B' - lb) - I)/n, u_j = sum_i GA Z Pc, w_i = sum_j GB Z Pr; G_Z = Pc (GA (1 + Z) - u_j) + Pr (GB (1 + Z) - w_i);
    loss = mean_i(la_i - Z_ii Pc_ii + lb_i - Z_ii Pr_ii); d logit_scale = sum G_Z Z.  z known to within z_err; the arm
    from z_arm, or from z.  Same keys as `terms` (one matrix)."""
    n = z.shape[0]
    dev = z.device
    keep = torch.ones(n, n, dtype=torch.bool, device=dev)
    eye = torch.eye(n, dtype=F64, device=dev)
    inv_n = Err(torch.full((n, n), 1.0 / n, dtype=F64, device=dev), torch.full((n, n), U / n, dtype=F64, device=dev))

    def row(x):
        return Err(x.v[:, None].expand(n, n), x.e[:, None].expand(n, n))

    def col(x):
        return Err(x.v[None, :].expand(n, n), x.e[None, :].expand(n, n))

    def T(x):
        return Err(x.v.T, x.e.T)

    def chain(Z):
        lr, lc = lse(Z, keep), lse(T(Z), keep)
        pc, pr = exp(add(Z, col(lc), -1.0)), exp(add(Z, row(lr), -1.0))
        a, b = mul(Z, pc), mul(Z, pr)
        la, lb = lse(a, keep), lse(T(b), keep)
        I = Err(eye)
        ga = mul(add(exp(add(a, row(la), -1.0)), I, -1.0), inv_n)
        gb = mul(add(exp(add(b, col(lb), -1.0)), I, -1.0), inv_n)
        cv, rv = mul(mul(ga, Z), pc), mul(mul(gb, Z), pr)
        depth = 64 + n / 64
        u = Err(cv.v.sum(0), cv.e.sum(0) + depth * U * cv.v.abs().sum(0) + n * TINY)
        w = Err(rv.v.sum(1), rv.e.sum(1) + depth * U * rv.v.abs().sum(1) + n * TINY)
        one_z = add(const(1.0, Z.v), Z)
        G = add(mul(pc, add(mul(ga, one_z), col(u), -1.0)), mul(pr, add(mul(gb, one_z), row(w), -1.0)))
        return G, (lr, lc, la, lb)

    Z = mul(Err(z.to(F64), None if z_err is None else z_err.to(F64)), Err(s.v.expand(n, n), s.e.expand(n, n)))
    G, (lr, lc, la, lb) = chain(Z)
    sG = mul(G, Err(s.v.expand(n, n), s.e.expand(n, n)))
    d = Err(Z.v.diagonal(), Z.e.diagonal())
    li = add(add(la, mul(d, exp(add(d, lc, -1.0))), -1.0), add(lb, mul(d, exp(add(d, lr, -1.0))), -1.0))
    li = mul(li, Err(torch.full((n,), 1.0 / n, dtype=F64, device=dev), torch.full((n,), U / n, dtype=F64, device=dev)))
    depth = 64 + n / 256
    loss = total(li, depth)
    n_tiles = ((n + 63) // 64) * ((n + 127) // 128)
    ds = total(mul(G, Z), 64 + n_tiles / 256)
    if z_arm is None:
        arm = ftz(bf(sG.v))
    else:
        Ga, _ = chain(Err(z_arm.to(F64) * s.v))
        arm = ftz(bf(Ga.v * s.v))
    return {"exact": [sG.v], "arm": [arm], "bound": [sG.e + ulp_bf16(sG.v.abs() + sG.e) + TINY], "G": [G.v],
            "loss": loss.v, "loss_bound": loss.e, "dscale": ds.v, "dscale_bound": ds.e}


# ------------------------------------------------------------------------------------------ gradient GEMMs
def feature_grads(pairs, sG: Sequence[torch.Tensor], feats: Sequence[Optional[torch.Tensor]]) -> Dict[int, torch.Tensor]:
    """dL/d feature of every feature a logits matrix reads: for matrix k = X_r X_c^T, d X_r += (sG_k) X_c and
    d X_c += (sG_k)^T X_r (optimization/loss.py, _nce_backward and _NceTermsFunction.backward), in float64.
    exact: sG the float64 s dL/dZ, feats the fp32 features.  GEMM arm: sG the bf16 arm and feats the bf16 hi copies the
    GEMMs take (nce_fused.cu:196, nce.cu:32); the GEMM's own fp32 accumulation is exact here."""
    out: Dict[int, torch.Tensor] = {}
    for g, (r, c) in zip(sG, pairs):
        g = g.to(F64)
        for i, add_ in ((r, g @ feats[c].to(F64)), (c, g.T @ feats[r].to(F64))):
            out[i] = add_ if i not in out else out[i] + add_
    return out
