/*
 * xpretrain_b200 — C ABI of the H100-native CLIP-ViP / HD-VILA hot path.
 *
 * The reference (microsoft/XPretrain) is 100 % Python: it has no FFI or
 * plugin boundary for this path, so the seam a maintainer binds is the set of
 * torch ops its nn.Modules call.  Each entry point below names the reference
 * lines it replaces.  Conventions:
 *   - every pointer is a raw DEVICE pointer owned by the caller (PyTorch
 *     allocates; nothing here allocates or frees device memory);
 *   - `stream` is a cudaStream_t passed as void*;
 *   - bf16 = __nv_bfloat16 bits, f32 = IEEE float, i64 = int64_t;
 *   - return 0 on success, negative on error; xp_last_error() gives the text.
 *     There is no CPU fallback: without an H100 (sm_90a) every call fails loudly.
 */
#ifndef XPRETRAIN_B200_H
#define XPRETRAIN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XP_ABI_VERSION 1

int xp_version(void);
const char* xp_last_error(void);
/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
int64_t xp_launch_count(void);
void xp_launch_count_reset(void);

/* ------------------------------------------------------------------ GEMM --
 * C[M,N] = epilogue( alpha * sum_k A[m,k] * B[n,k] )      (wgmma / TMA)
 * Replaces every nn.Linear on the path and its autograd:
 *   forward  y = x W^T + b         CLIP_ViP.py:341-343,379 (q/k/v/out_proj), :393-395 (fc1/fc2),
 *                                   :1141-1145 (visual/text projection), :178 (patch conv as im2col GEMM)
 *   dgrad    dx = dy W             a_layout=0, b_layout=1
 *   wgrad    dW += dy^T x          a_layout=1, b_layout=1, out=XP_OUT_F32_ATOMIC
 * a_layout: 0 = A stored [M,K] (K contiguous), 1 = A stored [K,M] (M contiguous)
 * b_layout: 0 = B stored [N,K] (K contiguous, nn.Linear.weight), 1 = B stored [K,N]
 * Epilogue, in this order:  v = alpha*acc; v += bias[n]; if n < scale_cols: v *= col_scale
 *   (CLIP_ViP.py:341 scales q AFTER the bias); then EITHER act OR v += residual[m,n]; store.
 * Refused with an error: a residual together with any activation, aux together with c_group > 0, an odd or negative
 * scale_cols, split-K without XP_OUT_F32_ATOMIC, an activation with an fp32 output.  Any K >= 1 is computed exactly as
 * K rounded up to the 64-wide k-block with zeros (TMA fills the missing k-columns with 0), so K < 64 is supported.
 */
enum { XP_ACT_NONE = 0, XP_ACT_QUICK_GELU = 1, XP_ACT_DQUICK_GELU = 2, XP_ACT_GELU_ERF = 3, XP_ACT_DGELU_ERF = 4 };
enum { XP_OUT_BF16 = 0, XP_OUT_F32 = 1, XP_OUT_F32_ATOMIC = 2 };

typedef struct XpGemm {
  const void* a;        /* bf16 */
  const void* b;        /* bf16 */
  void* c;              /* bf16 or f32 per `out` */
  const float* bias;    /* f32 [N] or NULL */
  const void* residual; /* bf16 [M, ldr] or NULL */
  void* aux;            /* bf16 [M, ld_aux]: QUICK_GELU/GELU_ERF store the pre-activation here (may be NULL);
                           DQUICK_GELU/DGELU_ERF read the pre-activation from here */
  int64_t M, N, K;
  int64_t lda, ldb, ldc, ldr, ld_aux; /* leading dimensions in elements */
  int32_t a_layout, b_layout;
  int32_t act, out;
  int32_t splits;     /* split-K factor (>1 only with XP_OUT_F32_ATOMIC) */
  int32_t scale_cols; /* columns [0, scale_cols) are multiplied by col_scale */
  float alpha, col_scale;
  /* Optional grouped row addressing (0 = plain row*ld): element offset of row r is
   *   (r / group) * group_stride + (r % group) * ld.
   * C uses c_group (aux is always addressed row * ld_aux, so it is refused with c_group > 0); residual uses r_group
   * (r_group_stride = 0 makes the residual a
   * periodic [r_group, N] table, used for the patch-embedding position+temporal add). */
  int64_t c_group, c_group_stride, r_group, r_group_stride;
  int32_t block_n;    /* 0 = auto, 128 = ping-pong 128x128 tiles, 256 = cooperative 128x256 tiles */
  int32_t max_ctas;   /* 0 = one persistent CTA per SM */
  int32_t cta_pair;   /* 0 or 1: single-CTA tiles (sm_90 has no CTA pairs; other values are rejected) */
  int32_t reserved;
} XpGemm;

int xp_gemm(const XpGemm* g, void* stream);

/* ------------------------------------------------------------- row kernels --
 * Row addressing shared by the row-wise kernels: element offset of logical row r is
 *   offsets[r]                                            if offsets != NULL (device i64 array)
 *   (r / group) * group_stride + (r % group) * ld         if group > 0
 *   r * ld                                                otherwise.
 * This is how the kernels skip the M global tokens of each video, pick the CLS row
 * (CLIP_ViP.py:891) or the EOS row (CLIP_ViP.py:776) without a gather copy.
 * The row kernels move 16-byte vectors, so every row must start at a 16-byte-aligned address: the base pointer,
 * ld * elsize and (when group > 0) group_stride * elsize must be multiples of 16 bytes, or the call is refused before any
 * launch (a map whose operand is NULL is not read, and not checked).
 * offsets[] lives in device memory and is not read by the host: each entry times elsize must be a multiple of 16 bytes
 * as well (xp_eos_offsets emits multiples of C, and C % 8 == 0 is required). */
typedef struct XpRowMap {
  int64_t group, group_stride, ld;
  const int64_t* offsets;
} XpRowMap;

/* nn.LayerNorm forward (CLIP_ViP.py:447,458,881,892,771): bf16 in/out, fp32 gamma/beta/statistics. */
int xp_layernorm_fwd(const void* x, const XpRowMap* xmap, void* y, const XpRowMap* ymap, const float* gamma,
                     const float* beta, float* mean, float* rstd, int64_t rows, int32_t C, float eps, void* stream);
/* LayerNorm fused with the residual add of the block it opens (CLIPEncoderLayer, CLIP_ViP.py:445-460: `hidden = residual +
 * branch; hidden = layer_normN(hidden)`), with the residual stream kept in fp32 as under the reference's autocast:
 *   s = x (+ add_bf16);  sum_out = s (optional);  y = LayerNorm(s).
 * x is bf16, fp32 or fp16 (x_dtype) and so is y (y_dtype); sum_out is fp32, or fp16 when x is fp16 (saturating; the
 * reference's own training precision under apex O2, run_pretrain.py:234-236).  add / sum_out / their maps may be NULL. */
int xp_layernorm_add_fwd(const void* x, const XpRowMap* xmap, int32_t x_dtype, const void* add_bf16, const XpRowMap* addmap,
                         void* sum_out, const XpRowMap* summap, void* y, const XpRowMap* ymap, int32_t y_dtype,
                         const float* gamma, const float* beta, float* mean, float* rstd, int64_t rows, int32_t C, float eps,
                         void* stream);
/* LayerNorm backward; dx = LN'(dy) + dres (the residual-branch gradient, may be NULL);
 * dgamma/dbeta are ACCUMULATED (fp32 atomics) so they can point at .grad buffers.  dres_colsum (optional, needs dres):
 * ACCUMULATES sum_rows dres — the bias gradient of the Linear that closes the other branch of that residual add
 * (fc2.bias / out_proj.bias of CLIPEncoderLayer, CLIP_ViP.py:445-460), so no separate column-sum pass reads dres again.
 * x (the saved LayerNorm input) is bf16 or fp32 (x_dtype); dy, dres, dx are bf16. */
int xp_layernorm_bwd(const void* dy, const XpRowMap* dymap, const void* x, const XpRowMap* xmap, int32_t x_dtype,
                     const float* gamma, const float* mean, const float* rstd, const void* dres, const XpRowMap* drmap, void* dx,
                     const XpRowMap* dxmap, float* dgamma, float* dbeta, float* dres_colsum, int64_t rows, int32_t C,
                     void* stream);
/* x / x.norm(dim=-1, keepdim=True) (CLIP_ViP.py:1148-1149), fp32. */
int xp_l2norm_fwd(const float* x, float* y, float* inv_norm, int32_t rows, int32_t C, void* stream);
int xp_l2norm_bwd(const float* dy, const float* y, const float* inv_norm, void* dx_bf16, int32_t rows, int32_t C,
                  float scale, void* stream);
/* Frame-mean head of the per-frame CLIP model (VidCLIP.py:62-65), fp32: for each of B videos with T frame projections
 * proj [B*T, P], u_t = p_t/||p_t||, m = mean_t u_t, feat [B, P] = m/||m||; inv_frame [B*T] = 1/||p_t|| and
 * inv_video [B] = 1/||m|| are saved for the backward.  The backward writes dproj [B*T, P] bf16 = scale * d(feat)/d(proj)^T
 * dfeat, exact through both normalisations.  One CTA per video, no atomics: repeated calls are bitwise equal.
 * T + P <= 12288. */
int xp_frame_pool_fwd(const float* proj, float* feat, float* inv_frame, float* inv_video, int32_t B, int32_t T, int32_t P,
                      void* stream);
int xp_frame_pool_bwd(const float* dfeat, const float* feat, const float* proj, const float* inv_frame,
                      const float* inv_video, void* dproj_bf16, int32_t B, int32_t T, int32_t P, float scale, void* stream);
/* Head of LF-VILA's video classification model (lfvila_video_classification.py:32-62).  Every reduction runs in a fixed
 * order without atomics: repeated calls are bitwise equal.  Every pointer must be 16-byte aligned (optional ones may be
 * NULL); refused before any launch.
 * pool: x [B, N, Hp, Wp, C] of x_dtype (XP_DTYPE_F32 / _F16 / _BF16) -> MaxPool2d((2, 3), stride 1) per frame over the
 * X = (Hp-1)(Wp-2) windows, torch's arg-max rule (first maximum of a tie in window scan order; a NaN replaces the running
 * maximum); frame_raw [B*N, C] = mean over the X window maxima, global_raw [B, C] = mean over all N*X of them (one sum,
 * one division), fp32 plus bf16 copies; argmax [B, N, X, C] uint8 = the winning position kh*3+kw of every window.
 * Needs Hp >= 2, Wp >= 3, B*N < 2^31.  The backward writes every element of dx [B, N, Hp, Wp, C] (x_dtype) by gathering
 * over the windows that cover it; d_frame [B*N, C] and d_global [B, C] may each be NULL (no gradient). */
int xp_lfvila_pool_fwd(const void* x, int32_t x_dtype, float* frame_raw, void* frame_bf16, float* global_raw,
                       void* global_bf16, uint8_t* argmax, int32_t B, int32_t N, int32_t Hp, int32_t Wp, int32_t C,
                       void* stream);
int xp_lfvila_pool_bwd(const float* d_frame, const float* d_global, const uint8_t* argmax, void* dx, int32_t x_dtype,
                       int32_t B, int32_t N, int32_t Hp, int32_t Wp, int32_t C, void* stream);
/* F.normalize(x, dim=-1) on fp32 rows [rows, C]: y = x / max(||x||, 1e-12), optional bf16 copy, norm [rows] = ||x||.
 * Backward of dy (+ dy2, either may be NULL), written as bf16: (g - y (y . g)) / ||x||, or g / 1e-12 below the clamp. */
int xp_lfvila_normalize_fwd(const float* x, float* y, void* y_bf16, float* norm, int32_t rows, int32_t C, void* stream);
int xp_lfvila_normalize_bwd(const float* dy, const float* dy2, const float* y, const float* norm, void* dx_bf16,
                            int32_t rows, int32_t C, void* stream);
/* nn.CrossEntropyLoss (mean) and accuracy (argmax == label, first index of a tie, mean over B) of fp32 logits [B, n_labels]
 * with row pitch ld, int64 labels [B]; 1 <= B <= 4096.  pred (optional) receives the logits with row pitch n_labels;
 * lse [B] is kept for the backward.  Label -100 is ignored by the
 * loss (ignore_index); any other label outside [0, n_labels) gives a NaN loss.  The backward writes dlogits bf16 [B, ld_out]
 * = d_loss[0] / count * (softmax - onehot) (+ d_logits, pitch ld_d, if not NULL), the columns past n_labels zero; a NULL
 * d_loss means no loss gradient. */
int xp_lfvila_ce_fwd(const float* logits, int64_t ld, const int64_t* labels, int32_t B, int32_t n_labels, float* pred,
                     float* lse, float* loss, float* acc, void* stream);
int xp_lfvila_ce_bwd(const float* logits, int64_t ld, const float* lse, const int64_t* labels, const float* d_loss,
                     const float* d_logits, int64_t ld_d, void* dlogits_bf16, int64_t ld_out, int32_t B, int32_t n_labels,
                     void* stream);
/* out[c] += scale * sum_r x[r,c]: bias gradients of every nn.Linear.  x must be 16-byte aligned. */
int xp_colsum_bf16(const void* x, int64_t ld, float* out, int64_t rows, int32_t C, float scale, void* stream);
/* fp32 master parameter -> bf16 compute copy. */
int xp_cast_f32_bf16(const float* src, void* dst_bf16, int64_t n, void* stream);

/* ------------------------------------------------------------- embeddings --*/
enum { XP_DTYPE_F32 = 0, XP_DTYPE_BF16 = 1, XP_DTYPE_F16 = 2 };

/* im2col of nn.Conv2d(3, width, kernel=stride=patch, bias=False) (CLIP_ViP.py:157-159,178-179):
 * video [frames,3,H,W] -> patches bf16 [frames*(H/p)*(W/p), ld]; the conv itself then runs as xp_gemm with K = 3*p*p.
 * Row pitch ld = round_up(3*p*p, 8) elements (16-byte rows, as TMA and xp_gemm need); columns [3*p*p, ld) are written
 * as zero.  ld = 3*p*p for p = 16 and 32; p = 14 (ViT-L/14) gives 588 columns in a pitch of 592.  Any p dividing H and W.
 * Overwrites exactly the frames*(H/p)*(W/p) x ld patch matrix (pad columns included) and nothing else; every element is one
 * conversion of an input value to bf16 (round to nearest even), bit-exact.  Alignment: patches_bf16 16 bytes (16-byte
 * stores); for p % 8 == 0 also video 16 bytes (16-byte loads).  Misaligned pointers are refused before any launch. */
int xp_vip_patchify(const void* video, int32_t dtype, void* patches_bf16, int64_t frames, int32_t H, int32_t W,
                    int32_t patch, void* stream);
/* The reference's input transform fused into the patch extraction (SURVEY.md §8f.4): frames_hwc uint8 [frames, H, W, 3] as
 * the decoder delivers them -> `.permute(0,3,1,2).float() / 255.` (CLIP-ViP/src/datasets/dataset_pretrain_stage1_all_source.py:182)
 * -> Normalize(mean, std) (init_transform_dict_simple, CLIP-ViP/src/datasets/dataloader.py:209-233; Resize / CenterCrop are
 * the identity at the input resolution) -> the bf16 patch matrix of xp_vip_patchify (same pitch).  IEEE fp32 arithmetic, one rounding to
 * bf16: bit-identical to casting the reference's fp32 tensor.  mean3 / std3 are HOST arrays of 3 floats.  Overwrites the
 * patch matrix as xp_vip_patchify does.  Alignment: patches_bf16 16 bytes; for p % 8 == 0 also frames_hwc 8 bytes. */
int xp_vip_patchify_u8(const uint8_t* frames_hwc, void* patches_bf16, int64_t frames, int32_t H, int32_t W, int32_t patch,
                       const float* mean3, const float* std3, void* stream);
/* xp_vip_patchify_u8 for frames of any size 1 <= H, W <= 4096: the reference's Resize([S, S], BICUBIC) + CenterCrop(S)
 * (init_transform_dict_simple, CLIP-ViP/src/datasets/dataloader.py:209-233) fused in as well.  The pinned torchvision 0.9.0
 * runs it as F.interpolate(x / 255, size=(S, S), mode="bicubic", align_corners=False): A = -0.75, border-clamped taps, no
 * antialias, no clamp of the result.  The source coordinate scale * (d + 0.5) - 0.5, scale = in / out, is torch's fp32
 * value bit for bit (one rounding: a fused multiply-add); the cubic weights are float64 of its t rounded to fp32; taps are accumulated in fp32 in a fixed order
 * (bitwise repeatable), then Normalize, one rounding to bf16.  At H = W = S the bits equal xp_vip_patchify_u8's.  Writes
 * the frames*(S/p)^2 x round_up(3p^2, 8) patch matrix of xp_vip_patchify (pad columns zero) and nothing else.  mean3 /
 * std3 are HOST arrays of 3 floats.  Refused before any launch: H, W or S outside [1, 4096], S % patch != 0, a
 * patches_bf16 not 16-byte aligned.  frames_hwc may have any alignment. */
int xp_vip_resize_patchify_u8(const uint8_t* frames_hwc, void* patches_bf16, int64_t frames, int32_t H, int32_t W, int32_t S,
                              int32_t patch, const float* mean3, const float* std3, void* stream);
/* LF-VILA's input transform (init_transform_dict, LF-VILA/src/datasets/dataloader.py:94-121, as torchvision 0.11 runs it
 * on float tensors) fused into Swin-3D's patch extraction.  frames_hwc uint8 [clips, N, H, W, 3]; params int32 [clips, 5]
 * (device) = top, left, h, w, flip per clip.  Per frame: /255, resize to Ha x Wa (stage A), crop the box (top, left, h, w),
 * resize the box to Ho x Wo (stage B, taps clamped to the box), mirror the columns if flip != 0, Normalize, one rounding to
 * bf16.  Both resizes are F.interpolate(mode="bilinear", align_corners=False) without antialias, with torch's fp32 source
 * coordinate (one rounding: a fused multiply-add); the composite weights are float64 rounded to fp32, accumulated in fp32
 * in a fixed order (bitwise repeatable).  Writes exactly the clips*N*(Ho/8)*(Wo/8) x 192 patch matrix xp_vip_patchify
 * writes for the transformed video: rows (clip, frame, h, w), columns (c, kh, kw).  mean3 / std3 are HOST arrays of 3
 * floats.  Refused before any launch: H, W, Ha, Wa, Ho or Wo outside [1, 4096], patch != 8, Ho or Wo not a multiple of 8,
 * a patches_bf16 not 16-byte aligned.  Boxes are the caller's to validate (0 <= top, 1 <= h, top + h <= Ha, likewise
 * left / w / Wa); every tap is clamped to the frame, so an invalid box reads nothing outside it.  frames_hwc may have any
 * alignment. */
int xp_lfvila_frames_patchify_u8(const uint8_t* frames_hwc, const int32_t* params, void* patches_bf16, int32_t clips,
                                 int32_t N, int32_t H, int32_t W, int32_t Ha, int32_t Wa, int32_t Ho, int32_t Wo,
                                 int32_t patch, const float* mean3, const float* std3, void* stream);
/* CLIP_ViP.py:170-176,183-195: table[t*L+l] = interp(temporal_embedding)[t] + position_embedding[1+l] (bf16,
 * [T*L, C]) and the M = 1 + add_cls_num global rows x[b, m] = (class_embedding | added_cls[m-1]) + position_embedding[0]
 * written into x_bf16 [B, M+T*L, C].  temporal may be NULL (if_use_temporal_embed = 0); added is read only when M > 1.
 * Overwrites all of table_bf16 and ONLY the M global rows of each sequence of x_bf16 (its patch rows are left to the patch
 * GEMM).  Each element is one fp32 sum then one bf16 rounding; the interpolation taps are those of F.interpolate(
 * mode="linear", align_corners=False), the weight computed in fp32.  No alignment needs (scalar accesses). */
int xp_vip_embed_tables(const float* pos, const float* temporal, const float* cls, const float* added,
                        void* table_bf16, void* x_bf16, int32_t B, int32_t T, int32_t L, int32_t M, int32_t C,
                        int32_t temporal_size, void* stream);
/* Backward of the above: d_patch bf16 [B, T*L, C] and d_global bf16 [B, M, C] (the two compact halves of
 * d_embeddings) ACCUMULATED (+=, fp32 atomics) into the parameter gradients: d_pos is required; d_temporal, d_cls and
 * d_added are optional (NULL = not wanted).  The atomics make the result bits depend on scheduling: not bitwise
 * repeatable.  C % 8 == 0 and C <= 1024; d_patch_bf16 / d_global_bf16 16-byte aligned (16-byte loads).  Refusals happen
 * before any launch. */
int xp_vip_embed_bwd(const void* d_patch_bf16, const void* d_global_bf16, float* d_pos, float* d_temporal, float* d_cls,
                     float* d_added, int32_t B, int32_t T, int32_t L, int32_t M, int32_t C, int32_t temporal_size,
                     void* stream);
/* CLIPTextEmbeddings.forward (CLIP_ViP.py:222-225): x[r] = token_embedding[ids[r]] + position_embedding[r % Lt].
 * ids are int64 and indexed bit-exactly; *err_flag is set to 1 if any id is outside [0, vocab) (that row then uses id 0).
 * Overwrites the rows x C block of x_bf16; each element is one fp32 sum then one bf16 rounding.  C % 4 == 0; tok and pos
 * 16-byte aligned (float4 loads), x_bf16 8-byte aligned (8-byte stores).
 * xp_text_embed_bwd ACCUMULATES (+=, fp32 atomics, not bitwise repeatable) dx into d_tok[ids[r]] and d_pos[r % Lt] (either
 * may be NULL); rows with an out-of-range id are skipped.  Scalar accesses, no alignment needs. */
int xp_text_embed_fwd(const int64_t* ids, const float* tok, const float* pos, void* x_bf16, int32_t rows, int32_t Lt,
                      int32_t C, int32_t vocab, int32_t* err_flag, void* stream);
int xp_text_embed_bwd(const int64_t* ids, const void* dx_bf16, float* d_tok, float* d_pos, int32_t rows, int32_t Lt,
                      int32_t C, int32_t vocab, void* stream);
/* EOS pooling row (CLIP_ViP.py:776): offsets[b] = (b*Lt + first argmax_s ids[b,s]) * C; index[b] optional.  Overwrites
 * B entries of each; exact. */
int xp_eos_offsets(const int64_t* ids, int64_t* offsets, int32_t* index, int32_t B, int32_t Lt, int32_t C,
                   void* stream);

/* ------------------------------------------------------------ ViP attention --
 * CLIPAttention.forward2 (CLIP_ViP.py:332-381) between the QKV projection and out_proj.
 *   qkv  bf16 [B*S, 3C]  columns [q | k | v], head h at [h*64, h*64+64), q already scaled by 64**-0.5
 *   out  bf16 [B*S, C]   (the tensor out_proj consumes; rows ordered [M global, frame0 L, frame1 L, ...])
 *   lse  f32  [B, H, S]  log-sum-exp of every query row (saved for backward)
 * S = M + T*L, head_dim 64, 1 <= M <= 8, any L >= 1: M + L <= 208 stages a whole frame per CTA, longer frames (ViT-L/14:
 * L = 256 at 224 px, 576 at 336 px) stream 64-row blocks.  workspace: xp_vip_attention_workspace_bytes() bytes for both.
 * No float atomics: out, lse and dqkv are bit-identical across calls. */
int64_t xp_vip_attention_workspace_bytes(int32_t B, int32_t H, int32_t T, int32_t M);
int xp_vip_attention_fwd(const void* qkv, void* out, float* lse, float* workspace, int32_t B, int32_t H, int32_t T,
                         int32_t L, int32_t M, int32_t C, void* stream);
/* dqkv bf16 [B*S, 3C] = gradient w.r.t. the (un-scaled-q) projection outputs, i.e. the dq part already carries
 * q_scale (CLIP_ViP.py:341), so the QKV dgrad/wgrad GEMMs treat the three thirds uniformly. */
int xp_vip_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                         float* workspace, int32_t B, int32_t H, int32_t T, int32_t L, int32_t M, int32_t C,
                         float q_scale, void* stream);

/* ------------------------------------------------------- text-tower attention --
 * CLIPAttention.forward (CLIP_ViP.py:266-330) between the QKV projection and out_proj, with the causal mask
 * (CLIP_ViP.py:788-797) and the padding mask built from attention_mask int64 [B, Lt] (CLIP_ViP.py:50-61).
 * qkv bf16 [B*Lt, 3C] (q pre-scaled), out bf16 [B*Lt, C], probs f32 [B, H, Lt, Lt] (saved for backward). Lt <= 96. */
int xp_text_attention_fwd(const void* qkv, const int64_t* mask, void* out, float* probs, int32_t B, int32_t H,
                          int32_t Lt, int32_t C, void* stream);
int xp_text_attention_bwd(const void* qkv, const void* dout, const float* probs, void* dqkv, int32_t B, int32_t H,
                          int32_t Lt, int32_t C, float q_scale, void* stream);

/* ------------------------------------------------------------------ InfoNCE --
 * NCELearnableTempLoss.forward (loss.py:134-141) on the gathered [N, d] fp32 embeddings: xp_nce_gather_fused below, or,
 * for global batches beyond it, the logits GEMM through xp_gemm on the split operands and xp_nce_terms with the table
 * ((rows, A), (columns, A)); the two gradient GEMMs run through xp_gemm.
 *   xp_nce_split:        x f32 [rows, d] -> x3 bf16 [rows, 3d] = [hi|hi|lo] (pattern 0) or [hi|lo|hi] (pattern 1),
 *                        so that x3_a . x3_b^T = hi*hi + hi*lo + lo*hi (fp32-grade logits on bf16 tensor cores);
 *                        hi_bf16 (optional) receives the plain bf16 copy used by the gradient GEMMs. */
int xp_nce_split(const float* x, void* x3_bf16, void* hi_bf16, int32_t rows, int32_t d, int32_t pattern, void* stream);
/* Fused exchange + loss: replaces `hvd.allgather(vis)`, `hvd.allgather(txt)` (CLIP-ViP/src/pretrain/run_pretrain.py:344-345;
 * rank-major concat, semantics pinned by LF-VILA/src/utils/dist.py:21-41) AND NCELearnableTempLoss.forward (loss.py:134-141)
 * with ONE cooperative kernel (csrc/nce_fused.cu): device-side flag barrier over peer-mapped exchange buffers, logits tiles
 * on wgmma whose operand rows are loaded straight from the owning peer's memory over NVLink (hi/lo split in the producer),
 * row/column log-sum-exps, loss (overwritten), d logit_scale (overwritten), g_scaled bf16 [N, ld_g] = exp(logit_scale)*dL/dZ,
 * and the bf16 copies vis_hi / txt_hi [N, d] that the local gradient GEMMs use.  N = world * b <= 1536.  It writes
 * exactly the N x N block of g_scaled (columns N..ld_g untouched) and all of vis_hi / txt_hi; loss, d_logit_scale, g_scaled
 * and the copies are bit-identical across calls and, in mode 0, on every rank.  vis_local / txt_local and the rows
 * behind peer_bufs are read with 16-byte vector loads: every row pointer must be 16-byte aligned.
 *   mode 0: peer_bufs = device array of `world` exchange-buffer base pointers (own buffer at [rank]); every buffer is
 *           xp_nce_gather_exchange_bytes() large, zero-initialised once, and mapped by all ranks (symmetric memory);
 *           vis_local / txt_local fp32 [b, d] are published by the kernel; `epoch` must increase by 1 per call (from 1).
 *   mode 1: no exchange: peer_bufs = device array of 2*world pointers, [r] = rank r's vis rows, [world + r] = its txt rows
 *           (fp32 [b, d]) in local memory (single process, or rows pre-gathered by another transport).
 * workspace: xp_nce_gather_workspace_bytes(N) bytes: per-tile partials, which need no initialisation, followed by three
 * barrier counters, which must be zero before the first call; every call leaves them zero. */
typedef struct XpNceGather {
  const float* vis_local;
  const float* txt_local;
  void* const* peer_bufs;
  const float* logit_scale;
  void* g_scaled;
  void* vis_hi;
  void* txt_hi;
  float* loss;
  float* d_logit_scale;
  float* workspace;
  int32_t rank, world, b, d;
  uint32_t epoch;
  int32_t mode;
  int64_t ld_g;
} XpNceGather;
int64_t xp_nce_gather_exchange_bytes(int32_t b, int32_t d, int32_t world);
int64_t xp_nce_gather_workspace_bytes(int32_t N);
int xp_nce_gather_fused(const XpNceGather* args, void* stream);
/* The contrastive losses of CLIP-ViP/src/optimization/loss.py as one table: NCEContrastiveLoss (:67-83, fixed temperature),
 * VidImgDivideNCELearnableTempLoss (:162-183), NCELearnableTempLoss_vs_vc (:204-225), _vs_vc_fc (:227-254), _vsc (:256-286)
 * and _vsc_fc (:288-324).  z[m] is matrix m's UNSCALED logits, fp32 [n[m], n[m]] with row pitch ld[m] (>= n[m], a multiple
 * of 4, 16-byte aligned), scaled by s = exp(*logit_scale) or, when logit_scale is NULL, by the host constant `scale`.
 * A term is one cross-entropy averaged over its n rows (axis 0) or columns (axis 1): for index i,
 *   LSE over the union of row / column i of every member matrix (bit m of `members`), without the diagonal entry of the
 *   members in `excl_diag`, minus s * z[target][i, i].
 * The members of a term share one n; the target is a member and keeps its diagonal.  Outputs: loss = sum of the terms
 * (overwritten); d_logit_scale = dL/d logit_scale (overwritten; only with a device logit_scale, may be NULL otherwise);
 * g[m] = s * dL/d(s z[m]) as bf16 [n[m], ld[m]] (8-byte aligned; columns n..ceil4(n) written as 0, the rest of the pitch
 * untouched), which is what the two gradient GEMMs dX = g Y, dY = g^T X per matrix consume.  workspace:
 * xp_nce_terms_workspace_bytes(args) bytes, no initialisation needed.  Four launches; loss, d_logit_scale and g are
 * bit-identical across calls (fixed-order reductions, no float atomics). */
typedef struct XpNceTerm {
  int32_t axis;       /* 0 = rows, 1 = columns */
  int32_t members;    /* bit m: matrix m is part of the union */
  int32_t excl_diag;  /* bit m: matrix m enters without its diagonal entry */
  int32_t target;     /* matrix whose diagonal entry is the label */
} XpNceTerm;
typedef struct XpNceTerms {
  const float* z[3];
  void* g[3];
  int64_t ld[3];
  int32_t n[3];
  int32_t n_mats, n_terms;
  XpNceTerm term[6];
  const float* logit_scale;
  float scale;
  float* loss;
  float* d_logit_scale;
  float* workspace;
} XpNceTerms;
int64_t xp_nce_terms_workspace_bytes(const XpNceTerms* args);
int xp_nce_terms(const XpNceTerms* args, void* stream);
/* NCELearnableTempDSLLoss.forward, CLIP-ViP/src/optimization/loss.py:185-202 (the training-time dual softmax): with
 * Z = exp(*logit_scale) * z, Pc / Pr its column / row softmax, A' = Z Pc and B' = Z Pr,
 *   loss = mean_i(LSE_j A'_ij - A'_ii) + mean_j(LSE_i B'_ij - B'_jj)       (overwritten)
 * and, the re-weighting not being detached, G_Z = Pc (GA (1 + Z) - u_j) + Pr (GB (1 + Z) - w_i) with GA, GB the two
 * cross-entropy gradients, u_j = sum_i GA Z Pc, w_i = sum_j GB Z Pr.  g_bf16 = s * G_Z, bf16 [n, ld]; d_logit_scale =
 * sum G_Z Z (overwritten).  z, ld, alignment as for xp_nce_terms; workspace: xp_nce_dsl_workspace_bytes(n) bytes.
 * Eight launches, bit-identical across calls. */
int64_t xp_nce_dsl_workspace_bytes(int32_t n);
int xp_nce_dsl(const float* z, int64_t ld, int32_t n, const float* logit_scale, void* g_bf16, float* loss,
               float* d_logit_scale, float* workspace, void* stream);

/* ---- BASELINE.json config #4: HD-VILA TimeSformer (divided space-time attention), hd-vila/src/modeling/timesformer.py
 *
 * xp_seg_attention_{fwd,bwd}: multi-head attention (head_dim 64) over strided "sequences" of a token-major fused
 * [n_rows, ld_qkv] bf16 buffer (columns [q|k|v], head h at h*64; q pre-scaled by head_dim**-0.5).  Replaces
 * Attention.forward (timesformer.py:156-173) TOGETHER WITH the einops rearranges around it (Block.forward :210-219):
 *   sequence s starts at row (s / inner) * outer_stride + (s % inner) * inner_stride, its tokens are tok_stride rows
 *   apart, it has min(seq_len, rows that fit) tokens, and token i attends to token j iff i / seg_len == j / seg_len
 *   (seg_len >= seq_len: dense).
 *   temporal ('(b h w) t m'):  G = 64 / T groups per sequence: seq_len = G*T, seg_len = T, inner = 1,
 *                              outer_stride = G*T, tok_stride = 1, n_seq = ceil(n_rows / (G*T))
 *   spatial  ('(b t) (h w) m'): seq_len = seg_len = H*W, inner = T, outer_stride = H*W*T, inner_stride = 1,
 *                              tok_stride = T, n_seq = B*T
 * out: [n_rows, ld_out] bf16 (same row order as qkv); lse, delta: [heads, n_rows] fp32 (delta is scratch written by bwd);
 * dqkv: [n_rows, ld_qkv] bf16, every (row, head) slice covered by a sequence is overwritten; dq is multiplied by q_scale. */
typedef struct XpSegAttn {
  int64_t n_rows;
  int64_t ld_qkv, ld_out;
  int64_t outer_stride, inner_stride, tok_stride;
  int32_t heads, n_seq, seq_len, seg_len, inner, reserved;
  /* Window-attention extensions — LF-VILA WindowAttention3D.forward, LF-VILA/src/models/video_encoder.py:135-164, together
   * with the pad / roll / window_partition / window_reverse / crop around it (:214-243).  All optional (NULL / 0):
   *   row_index    int32 [n_seq, seq_len]: token row of every window position (replaces the stride pattern; dense sequences).
   *                Built once per feature-map shape by applying the reference's own pad/roll/partition to an index tensor;
   *                zero-padded positions point at extra all-zero input rows, whose k, v are the qkv bias exactly as in the
   *                reference.
   *   bias         fp32 [bias_windows, heads, seq_len, seq_len] added to the logits before the softmax: relative-position
   *                bias (+ the 0 / -100 shift mask of window type s % bias_windows)
   *   ds_out       (bwd) bf16 [n_seq, heads, seq_len, seq_len]: dL/dlogits, whose sum over windows is the bias gradient
   *   head_dim     64 (or 0) or 32 */
  const int32_t* row_index;
  const float* bias;
  void* ds_out;
  int32_t bias_windows;
  int32_t head_dim;
} XpSegAttn;
int xp_seg_attention_fwd(const void* qkv, void* out, float* lse, const XpSegAttn* desc, void* stream);
int xp_seg_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta, void* dqkv,
                         const XpSegAttn* desc, float q_scale, void* stream);

/* xp_dense_attention_{fwd,bwd}: non-causal, unmasked multi-head attention (head_dim 64) over n_seq sequences of seq_len
 * CONSECUTIVE rows of a token-major fused [n_rows, ld_qkv] bf16 buffer (columns [q|k|v], head h at h*64, q pre-scaled by
 * head_dim**-0.5): sequence s is rows [s*seq_len, (s+1)*seq_len).  Replaces Attention.forward (timesformer.py:156-173)
 * for attention_type 'joint_space_time' (one sequence per clip of H*W*T rows, :202-205) and 'space_only' (one per frame).
 *   n_rows >= n_seq * seq_len; seq_len >= 1 (any length: the 64-row tiles are masked at the end of each sequence, and
 *   rows of the next sequence never enter); n_seq <= 65535; heads * (n_seq * seq_len) < 2^31.
 *   ld_qkv >= 3*heads*64 and ld_out >= heads*64, both multiples of 8; qkv, dout 16-byte aligned (TMA).
 * out: [n_rows, ld_out] bf16, columns [0, 64*heads) of the sequences' rows overwritten, nothing else written;
 * lse: [heads, n_rows] fp32 (natural log).  bwd: delta [heads, n_rows] fp32 scratch (rowsum(dO * O), written first);
 * dqkv [n_rows, ld_qkv] bf16, columns [0, 3*64*heads) of the sequences' rows overwritten; dq is multiplied by q_scale.
 * TMA + wgmma, warp-specialised; no float atomics, so results are bitwise repeatable. */
typedef struct XpDenseAttn {
  int64_t n_rows;
  int64_t ld_qkv, ld_out;
  int32_t heads, n_seq, seq_len, reserved;
} XpDenseAttn;
int xp_dense_attention_fwd(const void* qkv, void* out, float* lse, const XpDenseAttn* desc, void* stream);
int xp_dense_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta,
                           void* dqkv, const XpDenseAttn* desc, float q_scale, void* stream);

/* Token assembly, TimeSformer.forward timesformer.py:481-509: x [B,T,C,H*W] (XP_DTYPE_*) -> tokens bf16 [(b, p, t), C]
 * (rows in the reference's (h w t) order) = x[b,t,:,p] + pos[p,:] + time[t,:]; pos [H*W, C] / time [T, C] fp32 are the
 * (already interpolated) tables, NULL = no table (plain tokenisation, used for the output gradient).
 * xp_tsf_untokenize is the inverse layout change (tokens -> [B,T,C,H*W]): the module output (:523) and d(x).
 * Both overwrite exactly their B*T*C*HW output elements.  Forward: (x + pos) + time in fp32, one bf16 rounding; untokenize:
 * one conversion bf16 -> x_dtype (exact for fp32).  Scalar accesses, no alignment needs; B*T <= 65535 (grid z), refused
 * before any launch otherwise. */
int xp_tsf_embed_fwd(const void* x, int32_t x_dtype, const float* pos, const float* time, void* tokens_bf16, int32_t B,
                     int32_t T, int32_t C, int32_t HW, void* stream);
int xp_tsf_untokenize(const void* tokens_bf16, void* x, int32_t x_dtype, int32_t B, int32_t T, int32_t C, int32_t HW,
                      void* stream);
/* Stochastic depth on a residual branch (DropPath, timesformer.py:98-121, as Block.forward applies it :212,:218,:225):
 * out[r,:] = (residual ? residual[r,:] : 0) + scale[r] * x[r,:], all [rows, C] bf16 contiguous, scale fp32 per row
 * (0 or 1/keep_prob of the row's sample/group).  out may alias x.  x, residual and out must be 16-byte aligned. */
int xp_rowscale_bf16(const void* x, const float* scale, const void* residual, void* out, int64_t rows, int32_t C,
                     void* stream);

/* ---- BASELINE.json config #5 helpers (LF-VILA Swin-3D, LF-VILA/src/models/video_encoder.py)
 * xp_layernorm_wide_*: nn.LayerNorm over 1024 < C <= 4096 contiguous columns — PatchMerging.norm (4C = 2048, :281,:304).
 * xp_gather_rows_bf16 / xp_scatter_rows_bf16: out[i, :] = src[index[i], :] (zeros for index < 0) and its inverse
 * dst[index[i], :] = in[i, :] — the 2x2 neighbour concatenation of PatchMerging.forward (:292-301; out viewed as
 * [n/4... , 4C]) with its odd-size zero padding, and its backward.
 * Every bf16 row operand of these four (x, y, dy, dx, src, out, in, dst) must be 16-byte aligned. */
int xp_layernorm_wide_fwd(const void* x, void* y, const float* gamma, const float* beta, float* mean, float* rstd,
                          int64_t rows, int32_t C, float eps, void* stream);
int xp_layernorm_wide_bwd(const void* dy, const void* x, const float* gamma, const float* mean, const float* rstd, void* dx,
                          float* dgamma, float* dbeta, int64_t rows, int32_t C, void* stream);
int xp_gather_rows_bf16(const void* src, const int32_t* index, void* out, int64_t n_items, int32_t C, void* stream);
int xp_scatter_rows_bf16(const void* in, const int32_t* index, void* dst, int64_t n_items, int32_t C, void* stream);

/* ---- SURVEY.md §8(f).3: retrieval evaluation.  Replaces the numpy calls of validate() (CLIP-ViP/src/pretrain/
 * run_pretrain.py:173-176, tasks/run_video_retrieval.py:155-172) on CLIP-ViP/src/utils/metrics.py:
 *   xp_sim_f32      cal_cossim (:3-5): out[Na, Nb] (row pitch ld) = a[Na, d] b[Nb, d]^T, fp32 FFMA accumulation
 *   xp_dsl_reweight sim *= softmax(theta * sim, axis=0) in place (np_softmax :7-39 as used at run_video_retrieval.py:169-170);
 *                   col_scratch: 2*cols floats
 *   xp_rank_counts  compute_metrics' rank search (:41-48) without the sort: greater[i] / equal[i] = number of entries of row i
 *                   (transpose != 0: column i) strictly larger than / equal to sim[i, i]; the reference's rank list is
 *                   {greater[i] + t : 0 <= t < equal[i]} (ties counted once per tied entry, as np.where(ind == 0) does).
 *                   A NaN or +-inf diagonal gives equal[i] = 0: the reference's sort(-x) - diag(-x) is NaN or inf there,
 *                   never 0, so that query leaves its rank list. */
int xp_sim_f32(const float* a, const float* b, float* out, int32_t Na, int32_t Nb, int32_t d, int64_t ld, void* stream);
int xp_dsl_reweight(float* sim, int32_t rows, int32_t cols, int64_t ld, float theta, float* col_scratch, void* stream);
int xp_rank_counts(const float* sim, int32_t N, int64_t ld, int32_t transpose, int32_t* greater, int32_t* equal, void* stream);

/* ---- SURVEY.md §8(f).1: the optimizer step.  Replaces AdamW.step (CLIP-ViP/src/optimization/adamw.py:40-103) and
 * torch.nn.utils.clip_grad_norm_ as called at pretrain/run_pretrain.py:408-411,422 — one table-driven launch over all
 * parameters instead of ~10 elementwise launches per parameter.
 *
 * table_dev:     device array of XpOptTensor, one per parameter (all fp32, contiguous).  step_size =
 *                lr * sqrt(1 - beta2^t) / (1 - beta1^t) (or lr when correct_bias is off) and decay = lr * weight_decay are
 *                computed by the host per parameter group; p_bf16 (optional) receives the bf16 copy of the updated p.
 * block_map_dev: device array of n_blocks {tensor index, chunk index} int32 pairs; chunk c of a tensor covers elements
 *                [c * xp_opt_chunk_elems(), ...).  Built once per parameter set by the host.
 * xp_opt_grad_norm:  norm_out_dev[0] = 2-norm over every g in the table, norm_out_dev[1] = min(1, max_norm/(norm+1e-6))
 *                    (1 if max_norm <= 0); partial_dev is n_blocks floats of scratch.  Deterministic for a given
 *                    table and block map: fixed-order fp32 sums per block, the block partials summed in double in
 *                    block-map order.  Reads g only.
 * xp_opt_scale_grads: g *= norm_dev[1] in place (clip_grad_norm_ used on its own); leaves g untouched when the
 *                    coefficient is >= 1.
 * xp_opt_adamw_step:  the fused update; norm_dev (optional) = the pair above, its coefficient is applied to g on the fly.
 *                    Overwrites the n elements of p, m, v (and p_bf16 when set) of every row, nothing else; reads g.
 * Alignment: none required.  Each chunk uses 16-byte vectors when all of its row's pointers allow it (p_bf16: 8 bytes)
 * and a scalar loop otherwise; the step, the scaling and the cast compute the same bits on both paths (the norm's fp32
 * summation order differs between them, within its rounding bound).  Refused before any launch: an empty block map, betas
 * outside [0, 1), eps < 0. */
typedef struct XpOptTensor {
  void* p;
  const void* g;
  void* m;
  void* v;
  void* p_bf16;
  int64_t n;
  float step_size;
  float decay;
  int32_t reserved[2];
} XpOptTensor;
int32_t xp_opt_chunk_elems(void);
int xp_opt_grad_norm(const XpOptTensor* table_dev, const int32_t* block_map_dev, int32_t n_blocks, float* partial_dev,
                     float max_norm, float* norm_out_dev, void* stream);
int xp_opt_scale_grads(const XpOptTensor* table_dev, const int32_t* block_map_dev, int32_t n_blocks, const float* norm_dev,
                       void* stream);
int xp_opt_adamw_step(const XpOptTensor* table_dev, const int32_t* block_map_dev, int32_t n_blocks, const float* norm_dev,
                      float beta1, float beta2, float eps, void* stream);
/* Multi-tensor refresh of the bf16 compute copies (replaces the reference's implicit "the module reads its own fp32
 * parameters", CLIP_ViP.py:445-460): per row, g = fp32 source, p_bf16 = bf16 destination, or if that is null p = fp32
 * destination (plain copy); n elements.  One launch for all weights of a tower, run on every forward.  Overwrites exactly
 * the n destination elements per row; bit-exact (round to nearest even, or a copy).  No alignment needs. */
int xp_cast_table(const XpOptTensor* table_dev, const int32_t* block_map_dev, int32_t n_blocks, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* XPRETRAIN_B200_H */
