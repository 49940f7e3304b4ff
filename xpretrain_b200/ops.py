"""Tensor-level wrappers over the C ABI.  PyTorch supplies device memory and the current stream only;
every computation below runs in the hand-written sm_90a kernels of libxpretrain_b200.so.
This is the only module that calls the library; `_lib.py` declares it."""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List, Optional

import torch

from . import _lib
from ._lib import XpDenseAttn, XpGemm, XpRowMap, XpSegAttn, check, lib

bf16, f32 = torch.bfloat16, torch.float32
_DT = {torch.float32: _lib.DTYPE_F32, torch.bfloat16: _lib.DTYPE_BF16, torch.float16: _lib.DTYPE_F16}


def _p(t: Optional[torch.Tensor]):
    if t is None:
        return None
    if not t.is_cuda:
        raise _lib.XpError("xpretrain_b200 kernels need CUDA tensors (there is no CPU path)")
    return t.data_ptr()


def _call(name: str, *args) -> None:
    """lib().<name>(*args, the current CUDA stream); XpError with the library's message on a nonzero return."""
    check(getattr(lib(), name)(*args, torch.cuda.current_stream().cuda_stream), name)


def _workspace(what: str, nbytes: int, device, workspace: Optional[torch.Tensor] = None, zero: bool = False):
    """fp32 scratch of the queried nbytes for `what`: the caller's buffer, checked, or a new (zeroed) one."""
    if nbytes < 0:
        raise _lib.XpError(f"{what}: invalid sizes (the workspace query returned {nbytes})")
    if workspace is None:
        return (torch.zeros if zero else torch.empty)((nbytes + 3) // 4, dtype=f32, device=device)
    if workspace.numel() * 4 < nbytes:
        raise _lib.XpError(f"{what}: the workspace needs {nbytes} bytes")
    return workspace


def ptrs(tensors: Iterable[Optional[torch.Tensor]]) -> List[int]:
    """Device pointers of CUDA tensors (0 for None), for the pointer columns of an OptTable."""
    return [0 if t is None else _p(t) for t in tensors]


def launch_count() -> int:
    return int(lib().xp_launch_count())


def reset_launch_count() -> None:
    lib().xp_launch_count_reset()


# ------------------------------------------------------------------------------------------ GEMM
def gemm(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, *, M: int, N: int, K: int, lda: int, ldb: int, ldc: int,
         a_layout: int = 0, b_layout: int = 0, bias: Optional[torch.Tensor] = None,
         residual: Optional[torch.Tensor] = None, ldr: int = 0, aux: Optional[torch.Tensor] = None, ld_aux: int = 0,
         act: int = _lib.ACT_NONE, out_mode: int = _lib.OUT_BF16, splits: int = 1, scale_cols: int = 0,
         col_scale: float = 1.0, alpha: float = 1.0, c_group: int = 0, c_group_stride: int = 0, r_group: int = 0,
         r_group_stride: int = 0, block_n: int = 0, a_offset: int = 0, b_offset: int = 0, c_offset: int = 0) -> None:
    """out = epilogue(alpha * A @ B^T); offsets are in elements from the tensors' data pointers."""
    assert a.dtype == bf16 and b.dtype == bf16
    if bias is not None:
        assert bias.dtype == f32 and bias.is_contiguous()
    g = XpGemm()
    g.a = _p(a) + a_offset * 2
    g.b = _p(b) + b_offset * 2
    g.c = _p(out) + c_offset * out.element_size()
    g.bias = _p(bias)
    g.residual = _p(residual)
    g.aux = _p(aux)
    g.M, g.N, g.K = M, N, K
    g.lda, g.ldb, g.ldc, g.ldr, g.ld_aux = lda, ldb, ldc, ldr, ld_aux
    g.a_layout, g.b_layout, g.act, g.out = a_layout, b_layout, act, out_mode
    g.splits, g.scale_cols, g.alpha, g.col_scale = splits, scale_cols, alpha, col_scale
    g.c_group, g.c_group_stride, g.r_group, g.r_group_stride = c_group, c_group_stride, r_group, r_group_stride
    g.block_n, g.max_ctas = block_n, _sm_limit
    if _gemm_timer is None:
        return _call("xp_gemm", C.byref(g))
    # bench.py's roofline leg: CUDA events on the launching stream around this launch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _call("xp_gemm", C.byref(g))
    e1.record()
    _gemm_timer.append((2.0 * M * N * K, e0, e1))


_gemm_timer = None
_sm_limit = 0


def set_sm_limit(n: int) -> None:
    """Cap the persistent GEMM grids at n CTAs (0 = all SMs).  A data-parallel job reserves a few SMs this way for the NCCL
    kernels of the overlapped gradient all-reduce (NCCL_MAX_CTAS), so that they never displace a persistent GEMM CTA — whose
    tiles would then run as a second, nearly empty wave (VERDICT r1: `gemm_ms_per_step` 71.3 -> 74.7 ms from 1 to 8 GPUs)."""
    global _sm_limit
    _sm_limit = max(0, int(n))


def set_gemm_timer(records) -> None:
    """records: a list receiving (flops, start_event, end_event) per GEMM launch, or None to switch timing off."""
    global _gemm_timer
    _gemm_timer = records


def linear_fwd(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor, **kw) -> None:
    """out[M,N] = x[M,K] @ w[N,K]^T (+bias, epilogue)."""
    M, K = x.shape
    N = w.shape[0]
    gemm(x, w, out, M=M, N=N, K=K, lda=x.stride(0), ldb=w.stride(0), ldc=out.stride(0), bias=bias, **kw)


def linear_dgrad(dy: torch.Tensor, w: torch.Tensor, dx: torch.Tensor, **kw) -> None:
    """dx[M,K] = dy[M,N] @ w[N,K]   (w in its nn.Linear layout: MN-major B operand)."""
    M, N = dy.shape
    K = w.shape[1]
    gemm(dy, w, dx, M=M, N=K, K=N, lda=dy.stride(0), ldb=w.stride(0), ldc=dx.stride(0), b_layout=1, **kw)


def wgrad_plan(n_out: int, n_in: int, rows: int, sms: int = 0):
    """(block_n, splits) for a weight-gradient GEMM: the split-K factor that fills whole waves of the persistent grid
    (one 128 x block_n tile per CTA, one CTA per SM; H100 SXM has 132 SMs)."""
    sms = sms or _sm_limit or 132
    bn = 256 if n_in >= 256 else 128
    tiles, slots = ((n_out + 127) // 128) * ((n_in + bn - 1) // bn), sms
    best, best_eff = 1, 0.0
    for s in range(1, 33):
        if s > 1 and rows // s < 1024:
            break
        total = tiles * s
        eff = total / (((total + slots - 1) // slots) * slots)
        if eff > best_eff + 0.02:
            best, best_eff = s, eff
    return bn, best


def linear_wgrad(dy: torch.Tensor, x: torch.Tensor, dw: torch.Tensor, alpha: float = 1.0) -> None:
    """dw[N,K] += dy[rows,N]^T @ x[rows,K]  (fp32 atomics; both operands MN-major, split-K over the rows)."""
    rows, N = dy.shape
    K = x.shape[1]
    assert dw.dtype == f32
    bn, splits = wgrad_plan(N, K, rows)
    gemm(dy, x, dw, M=N, N=K, K=rows, lda=dy.stride(0), ldb=x.stride(0), ldc=dw.stride(0), a_layout=1, b_layout=1,
         out_mode=_lib.OUT_F32_ATOMIC, splits=splits, block_n=bn, alpha=alpha)


# ------------------------------------------------------------------------------------ row kernels
def rowmap(ld: int, group: int = 0, group_stride: int = 0, offsets: Optional[torch.Tensor] = None) -> XpRowMap:
    return XpRowMap(group=group, group_stride=group_stride, ld=ld, offsets=_p(offsets))


def layernorm_fwd(x, xmap, y, ymap, gamma, beta, mean, rstd, rows: int, C_: int, eps: float, x_off=0, y_off=0,
                  add=None, addmap=None, add_off=0, sum_out=None, summap=None):
    """y = LayerNorm(x (+ add)); offsets in ELEMENTS of the respective tensor.  x / y may be bf16 or fp32 (the fp32 residual
    stream); `add` is the bf16 branch output folded in before the normalisation, `sum_out` (fp32) receives x + add."""
    assert add is None or add.dtype == bf16
    assert sum_out is None or sum_out.dtype == (torch.float16 if x.dtype == torch.float16 else f32)
    _call("xp_layernorm_add_fwd", _p(x) + x_off * x.element_size(), C.byref(xmap), _DT[x.dtype],
          (_p(add) + add_off * 2) if add is not None else None, C.byref(addmap) if addmap is not None else None,
          _p(sum_out), C.byref(summap) if summap is not None else None, _p(y) + y_off * y.element_size(), C.byref(ymap),
          _DT[y.dtype], _p(gamma), _p(beta), _p(mean), _p(rstd), rows, C_, eps)


def layernorm_bwd(dy, dymap, x, xmap, gamma, mean, rstd, dres, drmap, dx, dxmap, dgamma, dbeta, rows: int, C_: int,
                  dy_off=0, x_off=0, dres_off=0, dx_off=0, dres_colsum=None):
    """x: the saved LayerNorm input, bf16, fp32 or fp16; dy / dres / dx bf16.  Offsets in elements."""
    _call("xp_layernorm_bwd", _p(dy) + dy_off * 2, C.byref(dymap), _p(x) + x_off * x.element_size(), C.byref(xmap),
          _DT[x.dtype], _p(gamma), _p(mean), _p(rstd), (_p(dres) + dres_off * 2) if dres is not None else None,
          C.byref(drmap) if drmap is not None else None, _p(dx) + dx_off * 2, C.byref(dxmap), _p(dgamma), _p(dbeta),
          _p(dres_colsum), rows, C_)


def l2norm_fwd(x, y, inv_norm):
    rows, C_ = x.shape
    _call("xp_l2norm_fwd", _p(x), _p(y), _p(inv_norm), rows, C_)


def l2norm_bwd(dy, y, inv_norm, dx_bf16, scale: float = 1.0):
    rows, C_ = y.shape
    _call("xp_l2norm_bwd", _p(dy), _p(y), _p(inv_norm), _p(dx_bf16), rows, C_, scale)


def frame_pool_fwd(proj, feat, inv_frame, inv_video, T: int):
    """Frame-mean head (VidCLIP.py:62-65): proj fp32 [B*T, P] -> feat fp32 [B, P] = normalise(mean_t normalise(p_t)),
    with the inverse norms inv_frame [B*T] and inv_video [B] saved for the backward."""
    rows, P = proj.shape
    B = feat.shape[0]
    assert proj.dtype == f32 and feat.dtype == f32 and proj.is_contiguous() and feat.is_contiguous()
    assert rows == B * T and feat.shape[1] == P and inv_frame.numel() == rows and inv_video.numel() == B
    _call("xp_frame_pool_fwd", _p(proj), _p(feat), _p(inv_frame), _p(inv_video), B, T, P)


def frame_pool_bwd(dfeat, feat, proj, inv_frame, inv_video, dproj_bf16, T: int, scale: float = 1.0):
    """dproj bf16 [B*T, P] = scale * gradient of the frame-mean head w.r.t. proj, given dfeat fp32 [B, P]."""
    B, P = feat.shape
    assert dfeat.dtype == f32 and dfeat.is_contiguous() and dfeat.shape == feat.shape
    assert dproj_bf16.dtype == bf16 and dproj_bf16.is_contiguous() and dproj_bf16.shape == (B * T, P)
    _call("xp_frame_pool_bwd", _p(dfeat), _p(feat), _p(proj), _p(inv_frame), _p(inv_video), _p(dproj_bf16), B, T, P, scale)


def lfvila_pool_fwd(x, frame_raw, frame_bf16, global_raw, global_bf16, argmax):
    """LF-VILA's MaxPool2d((2, 3), stride 1) + frame / clip means (lfvila_video_classification.py:32-43) on the encoder
    output x [B, N, Hp, Wp, C] (fp32, fp16 or bf16): frame_raw fp32 [B*N, C], global_raw fp32 [B, C], their bf16 copies,
    and the winning window position of every (b, n, window, c) in argmax uint8 [B, N, X, C]."""
    B, N, Hp, Wp, C_ = x.shape
    X = max(Hp - 1, 0) * max(Wp - 2, 0)
    assert frame_raw.dtype == f32 and global_raw.dtype == f32 and frame_bf16.dtype == bf16 and global_bf16.dtype == bf16
    assert argmax.dtype == torch.uint8 and argmax.numel() == B * N * X * C_
    assert frame_raw.numel() == frame_bf16.numel() == B * N * C_ and global_raw.numel() == global_bf16.numel() == B * C_
    x = aligned_input(x)
    _call("xp_lfvila_pool_fwd", _p(x), _DT[x.dtype], _p(frame_raw), _p(frame_bf16), _p(global_raw), _p(global_bf16),
          _p(argmax), B, N, Hp, Wp, C_)


def lfvila_pool_bwd(d_frame, d_global, argmax, dx):
    """dx [B, N, Hp, Wp, C] (the dtype of x) from d_frame fp32 [B*N, C] and / or d_global fp32 [B, C] (None: no gradient)."""
    B, N, Hp, Wp, C_ = dx.shape
    for t, n in ((d_frame, B * N * C_), (d_global, B * C_)):
        assert t is None or (t.dtype == f32 and t.is_contiguous() and t.numel() == n)
    assert dx.is_contiguous()
    _call("xp_lfvila_pool_bwd", _p(d_frame), _p(d_global), _p(argmax), _p(dx), _DT[dx.dtype], B, N, Hp, Wp, C_)


def lfvila_normalize_fwd(x, y, y_bf16, norm):
    """y = F.normalize(x, dim=-1) (x / max(||x||, 1e-12)) on fp32 rows, with an optional bf16 copy; norm [rows] = ||x||."""
    rows, C_ = x.shape
    assert x.dtype == f32 and y.dtype == f32 and x.is_contiguous() and y.is_contiguous() and y.shape == x.shape
    assert y_bf16 is None or (y_bf16.dtype == bf16 and y_bf16.is_contiguous() and y_bf16.shape == x.shape)
    assert norm.dtype == f32 and norm.numel() == rows
    _call("xp_lfvila_normalize_fwd", _p(x), _p(y), _p(y_bf16), _p(norm), rows, C_)


def lfvila_normalize_bwd(dy, dy2, y, norm, dx_bf16):
    """dx bf16 = gradient of lfvila_normalize_fwd for the sum of dy and dy2 (fp32 [rows, C], either may be None)."""
    rows, C_ = y.shape
    for t in (dy, dy2):
        assert t is None or (t.dtype == f32 and t.is_contiguous() and t.shape == y.shape)
    assert dx_bf16.dtype == bf16 and dx_bf16.is_contiguous() and dx_bf16.shape == y.shape
    _call("xp_lfvila_normalize_bwd", _p(dy), _p(dy2), _p(y), _p(norm), _p(dx_bf16), rows, C_)


def lfvila_ce_fwd(logits, n_labels: int, labels, pred, lse, loss, acc):
    """nn.CrossEntropyLoss() and (argmax == label).float().mean(0, keepdim=True) of logits fp32 [B, >= n_labels] (row pitch
    logits.stride(0)); pred (or None) receives the logits as a contiguous [B, n_labels], lse fp32 [B] is kept for the
    backward, loss and acc are fp32 one-element tensors."""
    B = logits.shape[0]
    assert logits.dtype == f32 and logits.stride(1) == 1 and labels.dtype == torch.int64 and labels.numel() == B
    assert pred is None or (pred.dtype == f32 and pred.is_contiguous() and pred.shape == (B, n_labels))
    assert lse.dtype == f32 and lse.numel() == B and loss.dtype == f32 and acc.dtype == f32
    labels = aligned_input(labels)
    _call("xp_lfvila_ce_fwd", _p(logits), logits.stride(0), _p(labels), B, n_labels, _p(pred), _p(lse), _p(loss), _p(acc))


def lfvila_ce_bwd(logits, n_labels: int, lse, labels, d_loss, d_logits, dlogits_bf16):
    """dlogits bf16 [B, ld] = d_loss * d(loss)/d(logits) + d_logits (d_loss: fp32 scalar tensor or None; d_logits: fp32
    [B, n_labels] or None); the columns past n_labels are written as zeros."""
    B = logits.shape[0]
    assert dlogits_bf16.dtype == bf16 and dlogits_bf16.stride(1) == 1 and dlogits_bf16.shape[0] == B
    if d_loss is not None:
        d_loss = d_loss.reshape(1).to(f32).contiguous()
    if d_logits is not None:
        d_logits = aligned_input(d_logits.to(f32))
        assert d_logits.shape == (B, n_labels)
    labels = aligned_input(labels)
    _call("xp_lfvila_ce_bwd", _p(logits), logits.stride(0), _p(lse), _p(labels), _p(d_loss), _p(d_logits),
          d_logits.stride(0) if d_logits is not None else 0, _p(dlogits_bf16), dlogits_bf16.stride(0), B, n_labels)


def colsum(x: torch.Tensor, out: torch.Tensor, scale: float = 1.0):
    rows, C_ = x.shape
    _call("xp_colsum_bf16", _p(x), x.stride(0), _p(out), rows, C_, scale)


def cast_bf16(src: torch.Tensor, dst: torch.Tensor, dst_offset: int = 0):
    assert src.dtype == f32 and dst.dtype == bf16 and src.is_contiguous()
    _call("xp_cast_f32_bf16", _p(src), _p(dst) + dst_offset * 2, src.numel())


# ------------------------------------------------------------------------------------- embeddings
def patch_pitch(patch: int) -> int:
    """Row pitch (elements) of the bf16 patch matrix: 3*p*p rounded up to a multiple of 8, so that rows are 16-byte aligned
    for TMA; the pad columns are zero.  Equal to 3*p*p for p = 16 and 32; 592 for p = 14."""
    return (3 * patch * patch + 7) // 8 * 8


def aligned_input(x: torch.Tensor, nbytes: int = 16) -> torch.Tensor:
    """x contiguous with an nbytes-aligned data pointer: the embedding and fused-NCE kernels read their inputs in vectors,
    and a contiguous view (e.g. `video[:, 1:]` of a one-frame-longer buffer, or an offset slice of a flat buffer) need not
    start aligned.  A misaligned input is copied; the kernel computes the same bits from the copy."""
    x = x.contiguous()
    return x if x.data_ptr() % nbytes == 0 else x.clone()


def _aligned_output(x: torch.Tensor, nbytes: int, what: str) -> None:
    """Outputs are written in place, so a misaligned one cannot be copied: it is refused before any launch."""
    if x.data_ptr() % nbytes != 0:
        raise _lib.XpError(f"{what}: the output must be {nbytes}-byte aligned (got data_ptr % {nbytes} = "
                           f"{x.data_ptr() % nbytes})")


def vip_patchify(video: torch.Tensor, patches: torch.Tensor, patch: int):
    _aligned_output(patches, 16, "vip_patchify")
    video = aligned_input(video)
    frames = video.numel() // (3 * video.shape[-2] * video.shape[-1])
    _call("xp_vip_patchify", _p(video), _DT[video.dtype], _p(patches), frames, video.shape[-2], video.shape[-1], patch)


CLIP_MEAN, CLIP_STD = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)   # dataloader.py:213-214


def vip_patchify_u8(frames_hwc: torch.Tensor, patches: torch.Tensor, patch: int, mean=CLIP_MEAN, std=CLIP_STD):
    """frames_hwc uint8 [..., H, W, 3] -> normalised bf16 patch matrix (the reference's /255 + Normalize fused in)."""
    assert frames_hwc.dtype == torch.uint8 and frames_hwc.is_contiguous() and frames_hwc.shape[-1] == 3
    _aligned_output(patches, 16, "vip_patchify_u8")
    frames_hwc = aligned_input(frames_hwc, 8)
    H, W = frames_hwc.shape[-3], frames_hwc.shape[-2]
    n = frames_hwc.numel() // (3 * H * W)
    m3, s3 = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
    _call("xp_vip_patchify_u8", _p(frames_hwc), _p(patches), n, H, W, patch, m3, s3)


def vip_resize_patchify_u8(frames_hwc: torch.Tensor, patches: torch.Tensor, size: int, patch: int, mean=CLIP_MEAN,
                           std=CLIP_STD):
    """frames_hwc uint8 [..., H, W, 3] of any size -> the bf16 patch matrix of vip_patchify_u8 at size x size: the
    reference's bicubic Resize([size, size]) + CenterCrop + /255 + Normalize fused into the patch extraction."""
    assert frames_hwc.dtype == torch.uint8 and frames_hwc.dim() >= 3 and frames_hwc.shape[-1] == 3
    _aligned_output(patches, 16, "vip_resize_patchify_u8")
    frames_hwc = aligned_input(frames_hwc)
    H, W = frames_hwc.shape[-3], frames_hwc.shape[-2]
    n = frames_hwc.numel() // (3 * H * W) if H * W else 0
    m3, s3 = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
    _call("xp_vip_resize_patchify_u8", _p(frames_hwc), _p(patches), n, H, W, size, patch, m3, s3)


IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)   # LF-VILA dataloader.py:94-99


def lfvila_frames_patchify_u8(frames_hwc: torch.Tensor, params: torch.Tensor, stage_a, out_size, patches: torch.Tensor,
                              patch: int = 8, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """frames_hwc uint8 [B, N, H, W, 3] -> Swin-3D's bf16 patch matrix [B*N*(Ho/8)*(Wo/8), 192] of the transformed video:
    resize to stage_a = (Ha, Wa), crop the box params[b] = (top, left, h, w, flip) (a CPU int32 [B, 5] tensor), resize the
    box to out_size = (Ho, Wo), mirror if flip, /255 + Normalize.  The boxes are checked here and uploaded without a device
    synchronise."""
    if frames_hwc.dtype != torch.uint8 or frames_hwc.dim() != 5 or frames_hwc.shape[-1] != 3:
        raise ValueError(f"lfvila_frames_patchify_u8: frames must be uint8 [B, N, H, W, 3] (got {frames_hwc.dtype} "
                         f"{list(frames_hwc.shape)})")
    B, N, H, W, _ = frames_hwc.shape
    (Ha, Wa), (Ho, Wo) = (int(v) for v in stage_a), (int(v) for v in out_size)
    if params.device.type != "cpu" or params.dtype != torch.int32 or tuple(params.shape) != (B, 5):
        raise _lib.XpError(f"lfvila_frames_patchify_u8: params must be a CPU int32 [{B}, 5] tensor (got {params.device} "
                           f"{params.dtype} {list(params.shape)})")
    top, left, h, w = (params[:, k] for k in range(4))
    bad = (top < 0) | (left < 0) | (h < 1) | (w < 1) | (top + h > Ha) | (left + w > Wa)
    if bool(bad.any()):
        b = int(bad.nonzero()[0])
        raise _lib.XpError(f"lfvila_frames_patchify_u8: clip {b}'s box {params[b, :4].tolist()} is not inside the "
                           f"{Ha} x {Wa} stage-A image")
    _aligned_output(patches, 16, "lfvila_frames_patchify_u8")
    frames_hwc = aligned_input(frames_hwc)
    dev_params = params.pin_memory().to(frames_hwc.device, non_blocking=True) if B else params
    m3, s3 = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
    _call("xp_lfvila_frames_patchify_u8", _p(frames_hwc), dev_params.data_ptr(), _p(patches), B, N, H, W, Ha, Wa, Ho, Wo,
          patch, m3, s3)


def vip_embed_tables(pos, temporal, cls, added, table, x, B, T, L, M, C_, temporal_size):
    _call("xp_vip_embed_tables", _p(pos), _p(temporal), _p(cls), _p(added), _p(table), _p(x), B, T, L, M, C_, temporal_size)


def vip_embed_bwd(d_patch, d_global, d_pos, d_temporal, d_cls, d_added, B, T, L, M, C_, temporal_size):
    """Adds (fp32 atomics: not bitwise repeatable) the embedding gradients into d_pos and the optional d_temporal, d_cls,
    d_added (None = not wanted)."""
    d_patch, d_global = aligned_input(d_patch), aligned_input(d_global)
    _call("xp_vip_embed_bwd", _p(d_patch), _p(d_global), _p(d_pos), _p(d_temporal), _p(d_cls), _p(d_added), B, T, L, M, C_,
          temporal_size)


def text_embed_fwd(ids, tok, pos, x, Lt, err_flag):
    _aligned_output(x, 8, "text_embed_fwd")
    tok, pos = aligned_input(tok), aligned_input(pos)
    rows = ids.numel()
    _call("xp_text_embed_fwd", _p(ids), _p(tok), _p(pos), _p(x), rows, Lt, tok.shape[1], tok.shape[0], _p(err_flag))


def text_embed_bwd(ids, dx, d_tok, d_pos, Lt, C_, vocab):
    _call("xp_text_embed_bwd", _p(ids), _p(dx), _p(d_tok), _p(d_pos), ids.numel(), Lt, C_, vocab)


def eos_offsets(ids, offsets, index, C_):
    B, Lt = ids.shape
    _call("xp_eos_offsets", _p(ids), _p(offsets), _p(index), B, Lt, C_)


# -------------------------------------------------------------------------------------- attention
def vip_attention_workspace(B, H, T, M, device) -> torch.Tensor:
    return _workspace("xp_vip_attention", lib().xp_vip_attention_workspace_bytes(B, H, T, M), device)


def vip_attention_fwd(qkv, out, lse, ws, B, H, T, L, M, C_):
    _call("xp_vip_attention_fwd", _p(qkv), _p(out), _p(lse), _p(ws), B, H, T, L, M, C_)


def vip_attention_bwd(qkv, out, dout, lse, dqkv, ws, B, H, T, L, M, C_, q_scale):
    _call("xp_vip_attention_bwd", _p(qkv), _p(out), _p(dout), _p(lse), _p(dqkv), _p(ws), B, H, T, L, M, C_, q_scale)


def text_attention_fwd(qkv, mask, out, probs, B, H, Lt, C_):
    _call("xp_text_attention_fwd", _p(qkv), _p(mask), _p(out), _p(probs), B, H, Lt, C_)


def text_attention_bwd(qkv, dout, probs, dqkv, B, H, Lt, C_, q_scale):
    _call("xp_text_attention_bwd", _p(qkv), _p(dout), _p(probs), _p(dqkv), B, H, Lt, C_, q_scale)


# -------------------------------------------------------------------------------------------- NCE
def nce_split(x, x3, hi, pattern: int):
    rows, d = x.shape
    _call("xp_nce_split", _p(x), _p(x3), _p(hi), rows, d, pattern)


def nce_terms(z, g, terms, loss, *, logit_scale=None, scale: float = 1.0, d_logit_scale=None, workspace=None):
    """Loss, d logit_scale and s * dL/dZ of a table of cross-entropy terms over up to three logits matrices (xp_nce_terms).
    z: fp32 [n_m, ld_m] unscaled logits; g: matching bf16 outputs; terms: (axis, members, excl_diag, target) per term, with
    members / excl_diag as bit masks over the matrices.  The scale is exp(logit_scale[0]) or, without logit_scale, `scale`.
    workspace: fp32, at least xp_nce_terms_workspace_bytes; allocated here when None."""
    a = _lib.XpNceTerms()
    a.n_mats, a.n_terms = len(z), len(terms)
    for m, (zm, gm) in enumerate(zip(z, g)):
        assert zm.dtype == f32 and gm.dtype == bf16 and zm.stride(1) == 1 and gm.stride(0) == zm.stride(0)
        a.z[m], a.g[m], a.ld[m], a.n[m] = _p(zm), _p(gm), zm.stride(0), zm.shape[0]
    for t, (axis, members, excl, target) in enumerate(terms):
        a.term[t].axis, a.term[t].members, a.term[t].excl_diag, a.term[t].target = axis, members, excl, target
    a.logit_scale, a.scale, a.loss, a.d_logit_scale = _p(logit_scale), scale, _p(loss), _p(d_logit_scale)
    a.workspace = _p(_workspace("xp_nce_terms", lib().xp_nce_terms_workspace_bytes(C.byref(a)), z[0].device, workspace))
    _call("xp_nce_terms", C.byref(a))


def nce_dsl(z, logit_scale, g, loss, d_logit_scale, workspace=None):
    """NCELearnableTempDSLLoss on the unscaled logits z fp32 [n, ld]: loss, d logit_scale and s * dL/dZ (bf16, pitch ld).
    workspace: fp32, at least xp_nce_dsl_workspace_bytes(n); allocated here when None."""
    n, ld = z.shape[0], z.stride(0)
    assert z.dtype == f32 and g.dtype == bf16 and g.stride(0) == ld
    ws = _workspace("xp_nce_dsl", lib().xp_nce_dsl_workspace_bytes(n), z.device, workspace)
    _call("xp_nce_dsl", _p(z), ld, n, _p(logit_scale), _p(g), _p(loss), _p(d_logit_scale), _p(ws))


def nce_gather_exchange_bytes(b: int, d: int, world: int) -> int:
    """Size of one rank's exchange buffer of the fused gather + InfoNCE (mode 0)."""
    return int(lib().xp_nce_gather_exchange_bytes(b, d, world))


def nce_gather_workspace(N: int, device) -> torch.Tensor:
    """Zeroed workspace of the fused gather + InfoNCE for N global rows; every launch leaves its counters zero again."""
    return _workspace("xp_nce_gather_fused", lib().xp_nce_gather_workspace_bytes(N), device, zero=True)


def nce_gather_fused(vis_local, txt_local, peer_bufs, logit_scale, g, vis_hi, txt_hi, loss, d_logit_scale, workspace, *,
                     rank: int, world: int, b: int, d: int, epoch: int, mode: int):
    """The fused embedding exchange + InfoNCE over N = world * b rows (xp_nce_gather_fused; modes as in the header);
    g: bf16 [N, ld_g] receives exp(logit_scale) * dL/dZ.  Every row pointer must be 16-byte aligned."""
    a = _lib.XpNceGather(vis_local=_p(vis_local), txt_local=_p(txt_local), peer_bufs=_p(peer_bufs),
                         logit_scale=_p(logit_scale), g_scaled=_p(g), vis_hi=_p(vis_hi), txt_hi=_p(txt_hi), loss=_p(loss),
                         d_logit_scale=_p(d_logit_scale), workspace=_p(workspace), rank=rank, world=world, b=b, d=d,
                         epoch=epoch, mode=mode, ld_g=g.stride(0))
    _call("xp_nce_gather_fused", C.byref(a))


# ------------------------------------------------------------- config #4: TimeSformer (HD-VILA)
def seg_desc(n_rows: int, heads: int, ld_qkv: int, ld_out: int, *, n_seq: int, seq_len: int, seg_len: int, inner: int,
             outer_stride: int, inner_stride: int, tok_stride: int) -> XpSegAttn:
    return XpSegAttn(n_rows=n_rows, ld_qkv=ld_qkv, ld_out=ld_out, outer_stride=outer_stride, inner_stride=inner_stride,
                     tok_stride=tok_stride, heads=heads, n_seq=n_seq, seq_len=seq_len, seg_len=seg_len, inner=inner)


def window_desc(n_rows: int, heads: int, head_dim: int, ld_qkv: int, ld_out: int, row_index: torch.Tensor,
                bias: Optional[torch.Tensor], ds_out: Optional[torch.Tensor] = None) -> XpSegAttn:
    """Window attention of LF-VILA's Swin-3D (video_encoder.py:135-164,214-243): row_index int32 [n_windows, L] gives the token
    row of every window position; bias fp32 [nW, heads, L, L] is the relative-position bias (+ shift mask per window type).
    The descriptor keeps references to the tensors (their memory must outlive the launches)."""
    n_win, L = row_index.shape
    assert row_index.dtype == torch.int32 and row_index.is_contiguous()
    d = seg_desc(n_rows, heads, ld_qkv, ld_out, n_seq=n_win, seq_len=L, seg_len=L, inner=1, outer_stride=0, inner_stride=0,
                 tok_stride=1)
    d.row_index = _p(row_index)
    d.head_dim = head_dim
    if bias is not None:
        assert bias.dtype == f32 and bias.is_contiguous() and bias.shape[1:] == (heads, L, L)
        d.bias, d.bias_windows = _p(bias), bias.shape[0]
    if ds_out is not None:
        assert ds_out.dtype == bf16 and ds_out.is_contiguous() and ds_out.shape == (n_win, heads, L, L)
        d.ds_out = _p(ds_out)
    d._keep = (row_index, bias, ds_out)
    return d


def temporal_desc(n_rows: int, T: int, heads: int, ld_qkv: int, ld_out: int) -> XpSegAttn:
    """'(b h w) t m' groups of timesformer.py:210: T consecutive rows each; 64 // T groups share one CTA tile."""
    G = max(1, 64 // T)
    return seg_desc(n_rows, heads, ld_qkv, ld_out, n_seq=(n_rows + G * T - 1) // (G * T), seq_len=G * T, seg_len=T,
                    inner=1, outer_stride=G * T, inner_stride=0, tok_stride=1)


def spatial_desc(B: int, T: int, HW: int, heads: int, ld_qkv: int, ld_out: int) -> XpSegAttn:
    """'(b t) (h w) m' groups of timesformer.py:217: H*W tokens, T rows apart."""
    return seg_desc(B * HW * T, heads, ld_qkv, ld_out, n_seq=B * T, seq_len=HW, seg_len=HW, inner=T,
                    outer_stride=HW * T, inner_stride=1, tok_stride=T)


def seg_attention_fwd(qkv, out, lse, desc: XpSegAttn):
    _call("xp_seg_attention_fwd", _p(qkv), _p(out), _p(lse), C.byref(desc))


def seg_attention_bwd(qkv, out, dout, lse, delta, dqkv, desc: XpSegAttn, q_scale: float):
    _call("xp_seg_attention_bwd", _p(qkv), _p(out), _p(dout), _p(lse), _p(delta), _p(dqkv), C.byref(desc), q_scale)


def dense_desc(n_rows: int, heads: int, ld_qkv: int, ld_out: int, *, n_seq: int, seq_len: int) -> XpDenseAttn:
    """n_seq sequences of seq_len consecutive rows, every row attending to every row of its sequence: one clip of H*W*T
    tokens ('joint_space_time', timesformer.py:202-205) or one frame of H*W tokens ('space_only')."""
    return XpDenseAttn(n_rows=n_rows, ld_qkv=ld_qkv, ld_out=ld_out, heads=heads, n_seq=n_seq, seq_len=seq_len)


def dense_attention_fwd(qkv, out, lse, desc: XpDenseAttn):
    _call("xp_dense_attention_fwd", _p(qkv), _p(out), _p(lse), C.byref(desc))


def dense_attention_bwd(qkv, out, dout, lse, delta, dqkv, desc: XpDenseAttn, q_scale: float):
    _call("xp_dense_attention_bwd", _p(qkv), _p(out), _p(dout), _p(lse), _p(delta), _p(dqkv), C.byref(desc), q_scale)


def tsf_embed_fwd(x, pos, time, tokens, B, T, C_, HW):
    _call("xp_tsf_embed_fwd", _p(x), _DT[x.dtype], _p(pos), _p(time), _p(tokens), B, T, C_, HW)


def rowscale(x, scale, out, residual=None):
    """out = (residual or 0) + scale[:, None] * x  (DropPath on a residual branch); out may alias x."""
    rows, C_ = x.shape
    assert scale.dtype == f32 and scale.numel() == rows and x.is_contiguous() and out.is_contiguous()
    _call("xp_rowscale_bf16", _p(x), _p(scale), _p(residual), _p(out), rows, C_)


def layernorm_any_fwd(x, y, gamma, beta, mean, rstd, rows: int, C_: int, eps: float):
    """LayerNorm over contiguous [rows, C] (the wide kernel above 1024 columns)."""
    if C_ <= 1024:
        m = rowmap(C_)
        layernorm_fwd(x, m, y, m, gamma, beta, mean, rstd, rows, C_, eps)
    else:
        _call("xp_layernorm_wide_fwd", _p(x), _p(y), _p(gamma), _p(beta), _p(mean), _p(rstd), rows, C_, eps)


def layernorm_any_bwd(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, rows: int, C_: int):
    if C_ <= 1024:
        m = rowmap(C_)
        layernorm_bwd(dy, m, x, m, gamma, mean, rstd, dres, m if dres is not None else None, dx, m, dgamma, dbeta, rows, C_)
    else:
        assert dres is None
        _call("xp_layernorm_wide_bwd", _p(dy), _p(x), _p(gamma), _p(mean), _p(rstd), _p(dx), _p(dgamma), _p(dbeta), rows,
              C_)


def gather_rows(src, index, out, C_: int):
    """out.view(-1, C)[i] = src[index[i]] (zeros for index < 0); index int32."""
    assert index.dtype == torch.int32 and index.is_contiguous() and out.numel() == index.numel() * C_
    _call("xp_gather_rows_bf16", _p(src), _p(index), _p(out), index.numel(), C_)


def scatter_rows(inp, index, dst, C_: int):
    """dst[index[i]] = inp.view(-1, C)[i] for index >= 0."""
    assert index.dtype == torch.int32 and index.is_contiguous() and inp.numel() == index.numel() * C_
    _call("xp_scatter_rows_bf16", _p(inp), _p(index), _p(dst), index.numel(), C_)


def tsf_untokenize(tokens, x, B, T, C_, HW):
    _call("xp_tsf_untokenize", _p(tokens), _p(x), _DT[x.dtype], B, T, C_, HW)


# ------------------------------------------------------------------------------------- retrieval
def _require(ok: bool, what: str, msg: str) -> None:
    if not ok:
        raise _lib.XpError(f"{what}: {msg}")


def _rows_f32(t, what: str, name: str) -> None:
    """t: a 2-D fp32 matrix with unit column stride (its row pitch t.stride(0) goes to the kernel)."""
    _require(t.dtype == f32 and t.dim() == 2 and t.stride(1) == 1, what,
             f"{name} must be a 2-D fp32 matrix with unit column stride (got {t.dtype}, strides {tuple(t.stride())})")


def sim_f32(a, b, out):
    """out[Na, Nb] (row pitch out.stride(0)) = a[Na, d] @ b[Nb, d]^T, fp32 FFMA accumulation.  a and b are read with
    row pitch d, so they must be contiguous."""
    for name, t in (("a", a), ("b", b), ("out", out)):
        _rows_f32(t, "sim_f32", name)
    _require(a.is_contiguous() and b.is_contiguous(), "sim_f32", "a and b must be contiguous")
    _require(a.shape[1] == b.shape[1], "sim_f32", f"a and b widths differ ({a.shape[1]} vs {b.shape[1]})")
    _require(tuple(out.shape) == (a.shape[0], b.shape[0]), "sim_f32",
             f"out must be [{a.shape[0]}, {b.shape[0]}] (got {list(out.shape)})")
    _call("xp_sim_f32", _p(a), _p(b), _p(out), a.shape[0], b.shape[0], a.shape[1], out.stride(0))


def dsl_reweight(sim, theta: float, scratch):
    """sim *= softmax(theta * sim, axis=0) in place; scratch: at least 2 * cols fp32."""
    _rows_f32(sim, "dsl_reweight", "sim")
    _require(scratch.dtype == f32 and scratch.is_contiguous() and scratch.numel() >= 2 * sim.shape[1], "dsl_reweight",
             f"scratch must be contiguous fp32 of at least 2 * cols = {2 * sim.shape[1]} elements")
    _call("xp_dsl_reweight", _p(sim), sim.shape[0], sim.shape[1], sim.stride(0), float(theta), _p(scratch))


def rank_counts(sim, transpose: bool, greater, equal):
    """greater[i] / equal[i] = entries of row (column) i of the square sim larger than / equal to sim[i, i]."""
    _rows_f32(sim, "rank_counts", "sim")
    n = sim.shape[0]
    _require(sim.shape[1] == n, "rank_counts", f"sim must be square (got {list(sim.shape)})")
    for name, t in (("greater", greater), ("equal", equal)):
        _require(t.dtype == torch.int32 and t.is_contiguous() and t.numel() == n, "rank_counts",
                 f"{name} must be contiguous int32 of {n} elements")
    _call("xp_rank_counts", _p(sim), n, sim.stride(0), 1 if transpose else 0, _p(greater), _p(equal))


# ------------------------------------------------------------------------------------- optimizer
class OptTable:
    """Device-side XpOptTensor table + block map for a fixed list of tensors (sizes never change; pointers, step sizes
    and decays are rewritten every step through a pinned staging buffer)."""

    def __init__(self, numels: List[int], device: torch.device):
        chunk = int(lib().xp_opt_chunk_elems())
        blocks = [(i, c) for i, n in enumerate(numels) for c in range((n + chunk - 1) // chunk)]
        self.n_blocks = len(blocks)
        self.block_map = torch.tensor(blocks, dtype=torch.int32).reshape(-1, 2).to(device)
        self.host = torch.empty(len(numels) * _lib.XpOptTensor.itemsize, dtype=torch.uint8).pin_memory()
        self.rows = self.host.numpy().view(_lib.XpOptTensor)
        self.dev = torch.empty(self.host.shape, dtype=torch.uint8, device=device)
        self.partial = torch.empty(max(self.n_blocks, 1), dtype=torch.float32, device=device)
        self.norm = torch.zeros(2, dtype=torch.float32, device=device)
        self.rows["n"] = numels
        self.copied = torch.cuda.Event()
        self.copied.record()
        self.launch_args = (_p(self.dev), _p(self.block_map), self.n_blocks)     # leading arguments of every launch

    def begin(self):
        """Wait until the previous asynchronous upload has left the pinned staging buffer before rewriting it."""
        self.copied.synchronize()
        return self.rows

    def upload(self):
        self.dev.copy_(self.host, non_blocking=True)
        self.copied.record()


def opt_grad_norm(tab: OptTable, max_norm: float):
    """tab.norm = (2-norm over every g of the table, clip coefficient for max_norm)."""
    _call("xp_opt_grad_norm", *tab.launch_args, _p(tab.partial), float(max_norm), _p(tab.norm))


def opt_scale_grads(tab: OptTable):
    """g *= tab.norm[1] in place for every g of the table."""
    _call("xp_opt_scale_grads", *tab.launch_args, _p(tab.norm))


def opt_adamw_step(tab: OptTable, beta1: float, beta2: float, eps: float, clip: bool):
    """The fused AdamW update of every row; with clip, g is scaled by the coefficient opt_grad_norm left in tab.norm."""
    _call("xp_opt_adamw_step", *tab.launch_args, _p(tab.norm) if clip else None, beta1, beta2, eps)


def cast_table(tab: OptTable):
    """Per row: g (fp32 source) -> p_bf16 (bf16 destination) or, if that is null, p (fp32 copy)."""
    _call("xp_cast_table", *tab.launch_args)
