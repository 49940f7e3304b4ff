"""The contrastive losses of CLIP-ViP/src/optimization/loss.py on the H100 kernels.

API mirrors CLIP-ViP/src/optimization/loss.py: `build_loss_func(cfg)` (:326-328) returns a module whose
`forward(vis_feat, text_feat, temp)` equals `NCELearnableTempLoss.forward` (:134-141):
    logits = vis @ text.T * exp(temp);  loss = CE(logits, arange) + CE(logits.T, arange)      (sum, no 1/2)
The logits GEMM and both gradient GEMMs run on the wgmma GEMM; softmax / loss / dL/dZ in nce.cu.
`gather_nce_loss` is the fused multi-GPU form (embedding all-gather + loss, backward without a collective).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from .. import _lib, ops

bf16, f32 = torch.bfloat16, torch.float32


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


FUSED_MAX_N = 1536      # (N / 128)^2 tiles of the fused kernel must be co-resident: up to two per SM on the 132 SMs of an H100


def _split_logits(vis: torch.Tensor, txt: torch.Tensor):
    """The unscaled logits V T^T of fp32 [N, d] rows as one hi/lo-split GEMM (fp32-grade on bf16 tensor cores).
    Returns (z fp32 [N, Np], vis_hi [N, d], txt_hi [N, d]); the pad columns N..Np of z are zero."""
    N, d = vis.shape
    Np = _pad8(N)
    v3, vh = _split_hi(vis, N, 0)
    t3, th = _split_hi(txt, Np, 1)
    z = torch.empty(N, Np, dtype=f32, device=vis.device)
    ops.gemm(v3, t3, z, M=N, N=Np, K=3 * d, lda=3 * d, ldb=3 * d, ldc=Np, out_mode=_lib.OUT_F32)
    return z, vh, th


def _nce_forward_unfused(vis: torch.Tensor, txt: torch.Tensor, temp: torch.Tensor):
    """Global batches above FUSED_MAX_N, and widths the fused kernel does not take: the split logits GEMM, then
    xp_nce_terms with the two-term table at the device logit_scale (fixed-order reductions, so loss and d logit_scale are
    bit-identical across calls and across ranks).  vis, txt: [N, d] fp32 (gathered).
    Returns (loss[1], g_scaled[N, Np] bf16, vis_hi, txt_hi, dscale[1])."""
    z, vh, th = _split_logits(vis, txt)
    g = torch.empty(z.shape, dtype=bf16, device=z.device)
    loss = torch.empty(1, dtype=f32, device=z.device)
    dscale = torch.empty(1, dtype=f32, device=z.device)
    ops.nce_terms([z], [g], TERM_TABLES["NCEContrastiveLoss"][1], loss, logit_scale=temp.detach().reshape(1).to(f32),
                  d_logit_scale=dscale)
    return loss, g, vh, th, dscale


class _Exchange:
    """Per (process group, b, d, device) state of the fused exchange: this rank's exchange buffer in SYMMETRIC MEMORY
    (torch.distributed._symmetric_memory: cuMem allocation mapped by every peer over NVLink), the device array of all
    ranks' base pointers, the kernel's zeroed workspace and the epoch counter.  world == 1 needs none of it."""

    _cache = {}

    def __init__(self, group, world: int, rank: int, b: int, d: int, dev: torch.device):
        import torch.distributed as dist
        self.world, self.rank, self.epoch = world, rank, 0
        nbytes = ops.nce_gather_exchange_bytes(b, d, world)
        self.mode = 0
        try:
            import torch.distributed._symmetric_memory as symm
            self.buf = symm.empty(nbytes, dtype=torch.uint8, device=dev)
            self.buf.zero_()
            self.handle = symm.rendezvous(self.buf, group if group is not None else dist.group.WORLD)
            ptrs = [int(x) for x in self.handle.buffer_ptrs]
            torch.cuda.synchronize(dev)
            self.handle.barrier()                     # every rank's flags are zero before anyone raises one
        except Exception as e:  # noqa: BLE001 — no P2P mapping on this machine: NCCL carries the rows, the kernel still fuses the rest
            import warnings
            warnings.warn(f"xpretrain_b200: symmetric-memory rendezvous failed ({type(e).__name__}: {e}); the embedding exchange "
                          f"falls back to ncclAllGather + the fused kernel in pre-gathered mode")
            self.mode = 1
            self.gathered = torch.empty(world, 2, b, d, dtype=f32, device=dev)
            ptrs = [self.gathered[r, 0].data_ptr() for r in range(world)] + [self.gathered[r, 1].data_ptr() for r in range(world)]
        self.ptrs = torch.tensor(ptrs, dtype=torch.int64, device=dev)
        self.ws = ops.nce_gather_workspace(world * b, dev)

    @classmethod
    def get(cls, group, world, rank, b, d, dev):
        key = (id(group) if group is not None else 0, world, rank, b, d, dev)
        ex = cls._cache.get(key)
        if ex is None:
            ex = cls._cache[key] = cls(group, world, rank, b, d, dev)
        return ex


_local_ws = {}


def _nce_forward_fused(vis: torch.Tensor, txt: torch.Tensor, temp: torch.Tensor, exchange: "_Exchange" = None, group=None):
    """One launch of csrc/nce_fused.cu.  vis, txt: this rank's [b, d] fp32 rows.  Returns (loss[1], g_scaled[N, Np] bf16,
    vis_hi[N, d], txt_hi[N, d], dscale[1]) for the global batch N = world * b."""
    b, d = vis.shape
    dev = vis.device
    world = exchange.world if exchange is not None else 1
    N = world * b
    Np = _pad8(N)
    vis, txt = ops.aligned_input(vis), ops.aligned_input(txt)      # the kernel reads rows with 16-byte vector loads
    g = (torch.zeros if Np != N else torch.empty)(N, Np, dtype=bf16, device=dev)
    vh = torch.empty(N, d, dtype=bf16, device=dev)
    th = torch.empty(N, d, dtype=bf16, device=dev)
    loss = torch.empty(1, dtype=f32, device=dev)
    dscale = torch.empty(1, dtype=f32, device=dev)
    scale = temp.detach().reshape(1).to(f32)
    if exchange is None:                                  # single process: rows are read in place
        key = (N, dev)
        ws = _local_ws.get(key)
        if ws is None:
            ws = _local_ws[key] = (ops.nce_gather_workspace(N, dev), torch.empty(2, dtype=torch.int64, device=dev))
        keep = torch.tensor([vis.data_ptr(), txt.data_ptr()], dtype=torch.int64).pin_memory()
        ws[1].copy_(keep, non_blocking=True)
        ops.nce_gather_fused(vis, txt, ws[1], scale, g, vh, th, loss, dscale, ws[0], rank=0, world=1, b=b, d=d, epoch=0,
                             mode=1)
    else:
        if exchange.mode == 1:
            import torch.distributed as dist
            dist.all_gather_into_tensor(exchange.gathered, torch.stack([vis, txt]), group=group)
        exchange.epoch += 1
        ops.nce_gather_fused(vis, txt, exchange.ptrs, scale, g, vh, th, loss, dscale, exchange.ws, rank=exchange.rank,
                             world=world, b=b, d=d, epoch=exchange.epoch, mode=exchange.mode)
    return loss, g, vh, th, dscale


def _nce_forward(vis: torch.Tensor, txt: torch.Tensor, temp: torch.Tensor):
    """vis, txt: [N, d] fp32 of ONE process (already gathered, or world == 1)."""
    if vis.shape[0] <= FUSED_MAX_N and vis.shape[1] % 64 == 0:
        return _nce_forward_fused(vis, txt, temp)
    return _nce_forward_unfused(vis, txt, temp)


def _nce_backward(g, vh, th, row0: int, nrows: int, scale: float):
    """d_vis[row0:row0+nrows] = scale * (sG) T ;  d_txt[row0:row0+nrows] = scale * (sG)^T V   (fp32 [nrows, d])."""
    N, d = vh.shape
    Np = g.shape[1]
    dev = g.device
    d_vis = torch.empty(nrows, d, dtype=f32, device=dev)
    # A = G rows (K-major), B = T stored [K=N, d] (MN-major)
    ops.gemm(g, th, d_vis, M=nrows, N=d, K=N, lda=Np, ldb=d, ldc=d, b_layout=1, out_mode=_lib.OUT_F32, alpha=scale,
             a_offset=row0 * Np)
    # A = G^T: stored [K=N(i), M=N(j)] -> MN-major A, columns row0.. ; B = V stored [K=N, d].  The TMA base must be
    # 16-byte aligned, so the column window starts at row0 rounded down to 8 and the slack rows are sliced off
    # (ADVICE r1: a per-rank batch that is not a multiple of 8 used to fail on ranks >= 1).
    r0 = row0 // 8 * 8
    ext = row0 - r0 + nrows
    d_txt = torch.empty(ext, d, dtype=f32, device=dev)
    ops.gemm(g, vh, d_txt, M=ext, N=d, K=N, lda=Np, ldb=d, ldc=d, a_layout=1, b_layout=1, out_mode=_lib.OUT_F32,
             alpha=scale, a_offset=r0)
    return d_vis, d_txt[row0 - r0:]


class _NceFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vis, txt, temp):
        loss, g, vh, th, dscale = _nce_forward(vis.to(f32), txt.to(f32), temp)
        ctx.saved = (g, vh, th, dscale)
        ctx.in_dtypes = (vis.dtype, txt.dtype, temp.dtype, temp.shape)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, dloss):
        g, vh, th, dscale = ctx.saved
        N = vh.shape[0]
        d_vis, d_txt = _nce_backward(g, vh, th, 0, N, 1.0)
        vd, td, pd, pshape = ctx.in_dtypes
        return (d_vis * dloss).to(vd), (d_txt * dloss).to(td), (dscale * dloss).reshape(pshape).to(pd)


class NCELearnableTempLoss(nn.Module):
    """Drop-in for loss.py:126-141 (the cfg argument is accepted and unused, as in the reference)."""

    def __init__(self, cfg=None):
        super().__init__()

    def forward(self, vis_feat, text_feat, temp):
        return _NceFunction.apply(vis_feat, text_feat, temp)


class _GatherNceFunction(torch.autograd.Function):
    """allgather(vis), allgather(txt) -> loss, as one autograd node (run_pretrain.py:344-356).

    Forward: ONE cooperative kernel (csrc/nce_fused.cu) — device-side flag barrier over symmetric memory, logits tiles
    whose operands are read straight from the peers' memory over NVLink, softmaxes, loss and dL/dZ.  No NCCL call.
    Backward: every rank already holds all embeddings and computes the same scalar loss, so the local rows of
    dV / dT are produced locally — no backward collective.  `grad_scale` = world size reproduces
    all_reduce(SUM)-then-slice (LF-VILA/src/utils/dist.py:35-41), which a gradient-AVERAGING data-parallel
    optimizer turns back into the true global-batch gradient (SURVEY.md §5)."""

    @staticmethod
    def forward(ctx, vis, txt, temp, group, grad_scale):
        import torch.distributed as dist

        b, d = vis.shape
        world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        rank = dist.get_rank(group) if world > 1 else 0
        if world > 1 and world * b <= FUSED_MAX_N and d % 64 == 0 and (b * d) % 4 == 0:
            ex = _Exchange.get(group, world, rank, b, d, vis.device)
            loss, g, vh, th, dscale = _nce_forward_fused(vis.to(f32), txt.to(f32), temp, ex, group)
        elif world > 1:                                  # global batch beyond one wave of tiles: NCCL gather + separate launches
            local = torch.stack([vis.to(f32), txt.to(f32)]).contiguous()          # [2, b, d]
            gathered = torch.empty(world, 2, b, d, dtype=f32, device=vis.device)
            dist.all_gather_into_tensor(gathered, local, group=group)
            loss, g, vh, th, dscale = _nce_forward(gathered[:, 0].reshape(world * b, d).contiguous(),
                                                   gathered[:, 1].reshape(world * b, d).contiguous(), temp)
        else:
            loss, g, vh, th, dscale = _nce_forward(vis.to(f32).contiguous(), txt.to(f32).contiguous(), temp)
        ctx.saved = (g, vh, th, dscale)
        ctx.meta = (rank * b, b, float(world if grad_scale is None else grad_scale), vis.dtype, txt.dtype, temp.dtype,
                    temp.shape)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, dloss):
        g, vh, th, dscale = ctx.saved
        row0, b, scale, vd, td, pd, pshape = ctx.meta
        d_vis, d_txt = _nce_backward(g, vh, th, row0, b, scale)
        return (d_vis * dloss).to(vd), (d_txt * dloss).to(td), (dscale * dloss).reshape(pshape).to(pd), None, None


def gather_nce_loss(vis_feat, text_feat, temp, group=None, grad_scale: Optional[float] = None):
    """Fused replacement for `hvd.allgather` x2 + `NCELearnableTempLoss` (run_pretrain.py:344-356)."""
    return _GatherNceFunction.apply(vis_feat, text_feat, temp, group, grad_scale)


def _split_hi(x: torch.Tensor, rows_pad: int, pattern: int):
    """bf16 hi/lo split of an fp32 [N, d] matrix: ([rows_pad, 3d] K-concatenated operand, [N, d] hi copy)."""
    N, d = x.shape
    x3 = (torch.zeros if rows_pad != N else torch.empty)(rows_pad, 3 * d, dtype=bf16, device=x.device)
    hi = torch.empty(N, d, dtype=bf16, device=x.device)
    ops.nce_split(x.contiguous(), x3, hi, pattern)
    return x3, hi


# ------------------------------------------------------------------------------------------------------------------------
# The other contrastive losses of loss.py.  Each one is a table: the logits matrices as (row features, column features)
# indices into the forward's arguments, and the cross-entropy terms as (axis, members, excl_diag, target) with members /
# excl_diag bit masks over the matrices (include/xpretrain_b200.h, XpNceTerms).  Forward: one hi/lo-split logits GEMM per
# matrix, then xp_nce_terms (loss, d logit_scale and s * dL/dZ per matrix); backward: two gradient GEMMs per matrix.
ROW, COL = 0, 1
_A, _B, _D = 1, 2, 4          # matrix bits: A = s V T^T, B = s V C^T, D = s I C^T (in this order in each table below)
_VTCI = ((0, 1), (0, 3), (2, 3))

TERM_TABLES = {
    # loss.py:76-83 (fixed temperature) and :162-183: rows and columns of V T^T (and of I C^T, whose n may differ)
    "NCEContrastiveLoss": (((0, 1),), ((ROW, _A, 0, 0), (COL, _A, 0, 0))),
    "VidImgDivideNCELearnableTempLoss": (((0, 1), (2, 3)), ((ROW, 1, 0, 0), (COL, 1, 0, 0), (ROW, 2, 0, 1), (COL, 2, 0, 1))),
    # loss.py:212-225, :235-254: rows and columns of each matrix
    "NCELearnableTempLoss_vs_vc": (_VTCI[:2], ((ROW, _A, 0, 0), (COL, _A, 0, 0), (ROW, _B, 0, 1), (COL, _B, 0, 1))),
    "NCELearnableTempLoss_vs_vc_fc": (_VTCI, ((ROW, _A, 0, 0), (COL, _A, 0, 0), (ROW, _B, 0, 1), (COL, _B, 0, 1),
                                              (ROW, _D, 0, 2), (COL, _D, 0, 2))),
    # loss.py:264-286: columns of A and B; per row i, [A_ii | A_i,j!=i | B_i,j!=i] and [B_ii | A_i,j!=i | B_i,j!=i]
    "NCELearnableTempLoss_vsc": (_VTCI[:2], ((COL, _A, 0, 0), (COL, _B, 0, 1), (ROW, _A | _B, _B, 0),
                                             (ROW, _A | _B, _A, 1))),
    # loss.py:296-324: the _vsc terms plus the columns and rows of D
    "NCELearnableTempLoss_vsc_fc": (_VTCI, ((COL, _A, 0, 0), (COL, _B, 0, 1), (ROW, _A | _B, _B, 0), (ROW, _A | _B, _A, 1),
                                            (COL, _D, 0, 2), (ROW, _D, 0, 2))),
}


def _check_square(name: str, feats, pairs) -> None:
    """ValueError (before any launch) unless every features matrix used is 2-D with one width and every logits matrix
    X Y^T is square, as the reference's arange labels require."""
    used = sorted({i for pr in pairs for i in pr})
    for i in used:
        if feats[i].dim() != 2:
            raise ValueError(f"{name}: argument {i} must be a 2-D [rows, dim] feature matrix, got shape {tuple(feats[i].shape)}")
    if len({feats[i].shape[1] for i in used}) != 1:
        raise ValueError(f"{name}: feature widths differ: {[tuple(feats[i].shape) for i in used]}")
    for r, c in pairs:
        if feats[r].shape[0] != feats[c].shape[0]:
            raise ValueError(f"{name}: argument {r} has {feats[r].shape[0]} rows but argument {c} has {feats[c].shape[0]}; "
                             f"their logits matrix must be square")


class _NceTermsFunction(torch.autograd.Function):
    """Any TERM_TABLES entry.  temp: the learnable log-scale tensor (s = exp(temp)), or None with s = `scale`."""

    @staticmethod
    def forward(ctx, table, scale, temp, *feats):
        pairs, terms = table
        d, dev = next(feats[i] for pr in pairs for i in pr).shape[1], feats[pairs[0][0]].device
        role = {}
        for r, c in pairs:
            role[r], role[c] = 0, 1
        assert len(role) == len({i for pr in pairs for i in pr})                # no feature is both a row and a column side
        split = {i: _split_hi(feats[i].to(f32), feats[i].shape[0] if pat == 0 else _pad8(feats[i].shape[0]), pat)
                 for i, pat in role.items()}
        z, g = [], []
        for r, c in pairs:
            n = feats[r].shape[0]
            Np = _pad8(n)
            zk = torch.empty(n, Np, dtype=f32, device=dev)
            ops.gemm(split[r][0], split[c][0], zk, M=n, N=Np, K=3 * d, lda=3 * d, ldb=3 * d, ldc=Np, out_mode=_lib.OUT_F32)
            z.append(zk)
            g.append(torch.empty(n, Np, dtype=bf16, device=dev))
        loss = torch.empty(1, dtype=f32, device=dev)
        dscale = torch.empty(1, dtype=f32, device=dev) if temp is not None else None
        ops.nce_terms(z, g, terms, loss, logit_scale=temp.detach().reshape(1).to(f32) if temp is not None else None,
                      scale=scale, d_logit_scale=dscale)
        ctx.saved = (g, {i: hi for i, (_, hi) in split.items()}, dscale)
        ctx.meta = (pairs, len(feats), [f.dtype for f in feats], None if temp is None else (temp.dtype, temp.shape))
        return loss.reshape(())

    @staticmethod
    def backward(ctx, dloss):
        g, hi, dscale = ctx.saved
        pairs, n_feats, dtypes, tmeta = ctx.meta
        out = {i: torch.zeros(h.shape[0], h.shape[1], dtype=f32, device=h.device) for i, h in hi.items()}
        for gk, (r, c) in zip(g, pairs):
            n, Np, d = gk.shape[0], gk.shape[1], hi[r].shape[1]
            # d_row += G_k @ col_feats (A = G_k rows, K-major);  d_col += G_k^T @ row_feats (A = G_k^T, MN-major)
            ops.gemm(gk, hi[c], out[r], M=n, N=d, K=n, lda=Np, ldb=d, ldc=d, b_layout=1, out_mode=_lib.OUT_F32_ATOMIC)
            ops.gemm(gk, hi[r], out[c], M=n, N=d, K=n, lda=Np, ldb=d, ldc=d, a_layout=1, b_layout=1,
                     out_mode=_lib.OUT_F32_ATOMIC)
        grads = [(out[i] * dloss).to(dtypes[i]) if i in out else None for i in range(n_feats)]
        dtemp = None if tmeta is None else (dscale * dloss).reshape(tmeta[1]).to(tmeta[0])
        return (None, None, dtemp, *grads)


def _table_loss(name: str, feats, temp=None, scale: float = 1.0):
    table = TERM_TABLES[name]
    _check_square(name, feats, table[0])
    return _NceTermsFunction.apply(table, scale, temp, *feats)


class _NceDslFunction(torch.autograd.Function):
    """NCELearnableTempDSLLoss (loss.py:185-202): hi/lo-split logits GEMM, the DSL chain of xp_nce_dsl, and the two
    gradient GEMMs of the plain InfoNCE in backward (the re-weighting's own gradient is inside G_Z)."""

    @staticmethod
    def forward(ctx, vis, txt, temp):
        z, vh, th = _split_logits(vis.to(f32), txt.to(f32))
        N, Np, dev = z.shape[0], z.shape[1], z.device
        g = torch.empty(N, Np, dtype=bf16, device=dev)
        loss = torch.empty(1, dtype=f32, device=dev)
        dscale = torch.empty(1, dtype=f32, device=dev)
        ops.nce_dsl(z, temp.detach().reshape(1).to(f32), g, loss, dscale)
        ctx.saved = (g, vh, th, dscale)
        ctx.in_dtypes = (vis.dtype, txt.dtype, temp.dtype, temp.shape)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, dloss):
        g, vh, th, dscale = ctx.saved
        d_vis, d_txt = _nce_backward(g, vh, th, 0, vh.shape[0], 1.0)
        vd, td, pd, pshape = ctx.in_dtypes
        return (d_vis * dloss).to(vd), (d_txt * dloss).to(td), (dscale * dloss).reshape(pshape).to(pd)


def _cfg_value(cfg, key):
    return cfg[key] if isinstance(cfg, dict) else getattr(cfg, key)


class NCEContrastiveLoss(nn.Module):
    """Drop-in for loss.py:67-83: InfoNCE at the fixed temperature cfg.temp (logits / temp), no temperature gradient."""

    def __init__(self, cfg):
        super().__init__()
        self.temp = _cfg_value(cfg, "temp")

    def forward(self, vis_feat, text_feat):
        return _table_loss("NCEContrastiveLoss", (vis_feat, text_feat), scale=1.0 / float(self.temp))


class NCELearnableTempDSLLoss(nn.Module):
    """Drop-in for loss.py:185-202: InfoNCE over the dual-softmax re-weighted logits Z * softmax(Z, 0) (rows) and
    Z^T * softmax(Z^T, 0) (columns); the retrieval fine-tuning loss (run_video_retrieval.py:333-338)."""

    def __init__(self, cfg=None):
        super().__init__()

    def forward(self, vis_feat, text_feat, temp):
        _check_square("NCELearnableTempDSLLoss", (vis_feat, text_feat), ((0, 1),))
        return _NceDslFunction.apply(vis_feat, text_feat, temp)


class VidImgNCELearnableTempLoss(nn.Module):
    """Drop-in for loss.py:143-160: NCELearnableTempLoss over [V; I] x [T; C]."""

    def __init__(self, cfg=None):
        super().__init__()

    def forward(self, vis_feat, text_feat, img_feat, cap_feat, temp):
        feats = (vis_feat, text_feat, img_feat, cap_feat)
        for f in feats:
            if f.dim() != 2 or f.shape[1] != vis_feat.shape[-1]:
                raise ValueError(f"VidImgNCELearnableTempLoss: every input must be [rows, {vis_feat.shape[-1]}], got "
                                 f"{[tuple(x.shape) for x in feats]}")
        if vis_feat.shape[0] + img_feat.shape[0] != text_feat.shape[0] + cap_feat.shape[0]:
            raise ValueError("VidImgNCELearnableTempLoss: len(vis) + len(img) must equal len(text) + len(cap)")
        if not all(f.is_cuda for f in feats):
            raise _lib.XpError("xpretrain_b200 kernels need CUDA tensors (there is no CPU path)")
        return _NceFunction.apply(torch.cat([vis_feat, img_feat], 0), torch.cat([text_feat, cap_feat], 0), temp)


def _table_module(name: str, doc: str):
    class _M(nn.Module):
        __doc__ = doc

        def __init__(self, cfg=None):
            super().__init__()

        def forward(self, vis_feat, text_feat, img_feat, cap_feat, temp):
            return _table_loss(name, (vis_feat, text_feat, img_feat, cap_feat), temp)

    _M.__name__ = _M.__qualname__ = name
    return _M


VidImgDivideNCELearnableTempLoss = _table_module(
    "VidImgDivideNCELearnableTempLoss", "Drop-in for loss.py:162-183: InfoNCE of V T^T plus InfoNCE of I C^T (I, C may have "
    "their own batch size).")
NCELearnableTempLoss_vs_vc = _table_module(
    "NCELearnableTempLoss_vs_vc", "Drop-in for loss.py:204-225: InfoNCE of video x subtitle plus video x caption.")
NCELearnableTempLoss_vs_vc_fc = _table_module(
    "NCELearnableTempLoss_vs_vc_fc", "Drop-in for loss.py:227-254: InfoNCE of video x subtitle, video x caption and frame x "
    "caption.")
NCELearnableTempLoss_vsc = _table_module(
    "NCELearnableTempLoss_vsc", "Drop-in for loss.py:256-286: column InfoNCE of V T^T and V C^T, and per video the joint "
    "softmax over its subtitle and caption negatives.")
NCELearnableTempLoss_vsc_fc = _table_module(
    "NCELearnableTempLoss_vsc_fc", "Drop-in for loss.py:288-324 — the released pre-training default "
    "(pretrain_vip_base_16.json:74-77): the _vsc terms plus InfoNCE of frame x caption.")

_LOSSES = {c.__name__: c for c in (
    NCELearnableTempLoss, NCEContrastiveLoss, NCELearnableTempDSLLoss, VidImgNCELearnableTempLoss,
    VidImgDivideNCELearnableTempLoss, NCELearnableTempLoss_vs_vc, NCELearnableTempLoss_vs_vc_fc, NCELearnableTempLoss_vsc,
    NCELearnableTempLoss_vsc_fc)}


def build_loss_func(cfg):
    """loss.py:326-328: `cfg.loss_name` selects the class.  TripletContrastiveLoss, HardNegLoss and MILNCEContrastiveLoss
    (legacy two-argument losses no released config selects) are not built."""
    name = cfg["loss_name"] if isinstance(cfg, dict) else cfg.loss_name
    if name not in _LOSSES:
        raise NotImplementedError(f"loss {name!r} is not built on the H100 path; available: {sorted(_LOSSES)}")
    return _LOSSES[name](cfg)
