"""In-batch video<->text InfoNCE with learnable temperature on the H100 kernels.

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


def _nce_forward_unfused(vis: torch.Tensor, txt: torch.Tensor, temp: torch.Tensor):
    """Global batches above FUSED_MAX_N: split / GEMM / softmax-grad as separate launches.
    vis, txt: [N, d] fp32 (gathered).  Returns (loss[1], g_scaled[N, Np] bf16, vis_hi, txt_hi, dscale[1])."""
    N, d = vis.shape
    Np = _pad8(N)
    dev = vis.device
    a3 = torch.empty(N, 3 * d, dtype=bf16, device=dev)
    b3 = torch.zeros(Np, 3 * d, dtype=bf16, device=dev) if Np != N else torch.empty(N, 3 * d, dtype=bf16, device=dev)
    vh = torch.empty(N, d, dtype=bf16, device=dev)
    th = torch.empty(N, d, dtype=bf16, device=dev)
    ops.nce_split(vis.contiguous(), a3, vh, 0)
    ops.nce_split(txt.contiguous(), b3, th, 1)
    z = torch.empty(N, Np, dtype=f32, device=dev)
    ops.gemm(a3, b3, z, M=N, N=Np, K=3 * d, lda=3 * d, ldb=3 * d, ldc=Np, out_mode=_lib.OUT_F32)
    lse_r = torch.empty(N, dtype=f32, device=dev)
    lse_c = torch.empty(N, dtype=f32, device=dev)
    g = torch.empty(N, Np, dtype=bf16, device=dev)
    loss = torch.empty(1, dtype=f32, device=dev)
    dscale = torch.zeros(1, dtype=f32, device=dev)
    ops.nce_softmax_grad(z, temp.detach().reshape(1).to(f32), lse_r, lse_c, g, loss, dscale)
    return loss, g, vh, th, dscale


class _Exchange:
    """Per (process group, b, d, device) state of the fused exchange: this rank's exchange buffer in SYMMETRIC MEMORY
    (torch.distributed._symmetric_memory: cuMem allocation mapped by every peer over NVLink), the device array of all
    ranks' base pointers, the kernel's zeroed workspace and the epoch counter.  world == 1 needs none of it."""

    _cache = {}

    def __init__(self, group, world: int, rank: int, b: int, d: int, dev: torch.device):
        import torch.distributed as dist
        self.world, self.rank, self.epoch = world, rank, 0
        nbytes = int(_lib.lib().xp_nce_gather_exchange_bytes(b, d, world))
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
        self.ws = torch.zeros(int(_lib.lib().xp_nce_gather_workspace_bytes(world * b)) // 4, dtype=f32, device=dev)

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
    vis, txt = vis.contiguous(), txt.contiguous()
    g = (torch.zeros if Np != N else torch.empty)(N, Np, dtype=bf16, device=dev)
    vh = torch.empty(N, d, dtype=bf16, device=dev)
    th = torch.empty(N, d, dtype=bf16, device=dev)
    loss = torch.empty(1, dtype=f32, device=dev)
    dscale = torch.empty(1, dtype=f32, device=dev)
    scale = temp.detach().reshape(1).to(f32)
    a = _lib.XpNceGather()
    a.vis_local, a.txt_local = vis.data_ptr(), txt.data_ptr()
    a.logit_scale, a.g_scaled, a.vis_hi, a.txt_hi = scale.data_ptr(), g.data_ptr(), vh.data_ptr(), th.data_ptr()
    a.loss, a.d_logit_scale = loss.data_ptr(), dscale.data_ptr()
    a.b, a.d, a.ld_g = b, d, Np
    keep = None
    if exchange is None:                                  # single process: rows are read in place
        key = (N, dev)
        ws = _local_ws.get(key)
        if ws is None:
            ws = _local_ws[key] = (torch.zeros(int(_lib.lib().xp_nce_gather_workspace_bytes(N)) // 4, dtype=f32, device=dev),
                                   torch.empty(2, dtype=torch.int64, device=dev))
        keep = torch.tensor([vis.data_ptr(), txt.data_ptr()], dtype=torch.int64).pin_memory()
        ws[1].copy_(keep, non_blocking=True)
        a.rank, a.world, a.mode, a.epoch = 0, 1, 1, 0
        a.peer_bufs, a.workspace = ws[1].data_ptr(), ws[0].data_ptr()
    else:
        if exchange.mode == 1:
            import torch.distributed as dist
            dist.all_gather_into_tensor(exchange.gathered, torch.stack([vis, txt]), group=group)
        exchange.epoch += 1
        a.rank, a.world, a.mode, a.epoch = exchange.rank, world, exchange.mode, exchange.epoch
        a.peer_bufs, a.workspace = exchange.ptrs.data_ptr(), exchange.ws.data_ptr()
    ops.check(_lib.lib().xp_nce_gather_fused(ops.C.byref(a), ops._stream()), "xp_nce_gather_fused")
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


class _NceVscFcFunction(torch.autograd.Function):
    """NCELearnableTempLoss_vsc_fc (loss.py:288-324): three hi/lo-split logits GEMMs (V T^T, V C^T, I C^T), the
    six-term softmax / loss / dL/dZ kernels of nce.cu, and six gradient GEMMs in backward."""

    @staticmethod
    def forward(ctx, vis, txt, img, cap, temp):
        assert txt.shape[0] == cap.shape[0]                                   # loss.py:290
        N, d = vis.shape
        Np, dev = _pad8(N), vis.device
        v3, vh = _split_hi(vis.to(f32), N, 0)
        i3, ih = _split_hi(img.to(f32), N, 0)
        t3, th = _split_hi(txt.to(f32), Np, 1)
        c3, ch = _split_hi(cap.to(f32), Np, 1)
        z = torch.empty(3, N, Np, dtype=f32, device=dev)
        for k, (a, b) in enumerate(((v3, t3), (v3, c3), (i3, c3))):
            ops.gemm(a, b, z[k], M=N, N=Np, K=3 * d, lda=3 * d, ldb=3 * d, ldc=Np, out_mode=_lib.OUT_F32)
        g = torch.empty(3, N, Np, dtype=bf16, device=dev)
        stats = torch.empty(6 * N, dtype=f32, device=dev)
        loss = torch.empty(1, dtype=f32, device=dev)
        dscale = torch.zeros(1, dtype=f32, device=dev)
        ops.nce_vsc_fc(z[0], z[1], z[2], temp.detach().reshape(1).to(f32), stats, g[0], g[1], g[2], loss, dscale)
        ctx.saved = (g, vh, th, ih, ch, dscale)
        ctx.in_meta = (vis.dtype, txt.dtype, img.dtype, cap.dtype, temp.dtype, temp.shape)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, dloss):
        g, vh, th, ih, ch, dscale = ctx.saved
        N, d = vh.shape
        Np, dev = g.shape[2], g.device
        out = torch.zeros(4, N, d, dtype=f32, device=dev)                     # d_vis, d_txt, d_img, d_cap (atomic accumulation)

        def rows_times(gk, feat, dst):       # dst += G_k  @ feat   (A = G_k rows, K-major; B = feat [K=N, d] MN-major)
            ops.gemm(gk, feat, dst, M=N, N=d, K=N, lda=Np, ldb=d, ldc=d, b_layout=1, out_mode=_lib.OUT_F32_ATOMIC)

        def cols_times(gk, feat, dst):       # dst += G_k^T @ feat  (A = G_k^T: MN-major)
            ops.gemm(gk, feat, dst, M=N, N=d, K=N, lda=Np, ldb=d, ldc=d, a_layout=1, b_layout=1,
                     out_mode=_lib.OUT_F32_ATOMIC)

        rows_times(g[0], th, out[0]); rows_times(g[1], ch, out[0])            # dV = s (G_a T + G_b C)
        cols_times(g[0], vh, out[1])                                          # dT = s G_a^T V
        rows_times(g[2], ch, out[2])                                          # dI = s G_d C
        cols_times(g[1], vh, out[3]); cols_times(g[2], ih, out[3])            # dC = s (G_b^T V + G_d^T I)
        vd, td, idt, cd, pd, pshape = ctx.in_meta
        return ((out[0] * dloss).to(vd), (out[1] * dloss).to(td), (out[2] * dloss).to(idt), (out[3] * dloss).to(cd),
                (dscale * dloss).reshape(pshape).to(pd))


class NCELearnableTempLoss_vsc_fc(nn.Module):
    """Drop-in for loss.py:280-324 — the released pre-training default (pretrain_vip_base_16.json:74-77):
    forward(vis_feat, text_feat, img_feat, cap_feat, temp) on the (gathered) feature matrices."""

    def __init__(self, cfg=None):
        super().__init__()

    def forward(self, vis_feat, text_feat, img_feat, cap_feat, temp):
        return _NceVscFcFunction.apply(vis_feat, text_feat, img_feat, cap_feat, temp)


_LOSSES = {"NCELearnableTempLoss": NCELearnableTempLoss, "NCELearnableTempLoss_vsc_fc": NCELearnableTempLoss_vsc_fc}


def build_loss_func(cfg):
    """loss.py:326-328: `cfg.loss_name` selects the class."""
    name = cfg["loss_name"] if isinstance(cfg, dict) else cfg.loss_name
    if name not in _LOSSES:
        raise NotImplementedError(f"loss {name!r} is outside the H100 hot path (SURVEY.md §8f lists it as 'next'); "
                                  f"available: {sorted(_LOSSES)}")
    return _LOSSES[name](cfg)
