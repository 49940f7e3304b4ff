// Standalone (no torch) correctness + timing harness for xp_gemm, run on the GPU box:
//   tools/gemm_selftest [quick]
// Compares against a naive fp32-accumulate CUDA-core GEMM on the same bf16 inputs.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../include/xpretrain_b200.h"

extern "C" void xp_debug_gemm_mn_desc(int lbo, int sbo);

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e = (x);                                                           \
    if (e != cudaSuccess) {                                                        \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(2);                                                                     \
    }                                                                              \
  } while (0)

__global__ void fill_bf16(__nv_bfloat16* p, size_t n, uint32_t seed, float scale) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t x = (uint32_t)i * 2654435761u + seed;
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  float f = ((x & 0xFFFF) / 65536.f - 0.5f) * 2.f * scale;
  p[i] = __float2bfloat16(f);
}
__global__ void fill_f32(float* p, size_t n, uint32_t seed, float scale) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t x = (uint32_t)i * 2654435761u + seed;
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  p[i] = ((x & 0xFFFF) / 65536.f - 0.5f) * 2.f * scale;
}

__device__ float qgelu(float x) { return x / (1.f + expf(-1.702f * x)); }
__device__ float qgelu_grad(float x) {
  float s = 1.f / (1.f + expf(-1.702f * x));
  return s * (1.f + 1.702f * x * (1.f - s));
}

// naive reference: one thread per output
__global__ void ref_gemm(const __nv_bfloat16* A, const __nv_bfloat16* B, float* C, float* AUX, int M, int N, int K,
                         long lda, long ldb, int a_layout, int b_layout, const float* bias,
                         const __nv_bfloat16* residual, long ldr, const __nv_bfloat16* aux_in, long ld_aux, int act,
                         int scale_cols, float alpha, float col_scale) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  int m = blockIdx.y;
  if (n >= N || m >= M) return;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) {
    float a = __bfloat162float(a_layout == 0 ? A[(long)m * lda + k] : A[(long)k * lda + m]);
    float b = __bfloat162float(b_layout == 0 ? B[(long)n * ldb + k] : B[(long)k * ldb + n]);
    acc += a * b;
  }
  float v = acc * alpha;
  if (bias) v += bias[n];
  if (n < scale_cols) v *= col_scale;
  if (act == XP_ACT_QUICK_GELU) {
    if (AUX) AUX[(long)m * N + n] = v;
    v = qgelu(v);
  } else if (act == XP_ACT_DQUICK_GELU) {
    v *= qgelu_grad(__bfloat162float(aux_in[(long)m * ld_aux + n]));
  }
  if (residual) v += __bfloat162float(residual[(long)m * ldr + n]);
  C[(long)m * N + n] = v;
}

struct Case {
  const char* name;
  int M, N, K, a_layout, b_layout, act, out, splits, bn;
  bool bias, residual, qscale;
};

static int run_case(const Case& c, bool timing) {
  size_t a_elems = (size_t)c.M * c.K, b_elems = (size_t)c.N * c.K;
  long lda = c.a_layout == 0 ? c.K : c.M;
  long ldb = c.b_layout == 0 ? c.K : c.N;
  __nv_bfloat16 *A, *B, *R = nullptr, *AUX = nullptr, *Cb = nullptr;
  float *Cf = nullptr, *Cref, *AUXref = nullptr, *bias = nullptr;
  CK(cudaMalloc(&A, a_elems * 2));
  CK(cudaMalloc(&B, b_elems * 2));
  fill_bf16<<<(a_elems + 255) / 256, 256>>>(A, a_elems, 1234u, 1.0f);
  fill_bf16<<<(b_elems + 255) / 256, 256>>>(B, b_elems, 987u, 1.0f);
  size_t c_elems = (size_t)c.M * c.N;
  CK(cudaMalloc(&Cref, c_elems * 4));
  if (c.out == XP_OUT_BF16) {
    CK(cudaMalloc(&Cb, c_elems * 2));
    CK(cudaMemset(Cb, 0xFF, c_elems * 2));
  } else {
    CK(cudaMalloc(&Cf, c_elems * 4));
    CK(cudaMemset(Cf, 0, c_elems * 4));
  }
  if (c.bias) {
    CK(cudaMalloc(&bias, c.N * 4));
    fill_f32<<<(c.N + 255) / 256, 256>>>(bias, c.N, 55u, 2.0f);
  }
  if (c.residual) {
    CK(cudaMalloc(&R, c_elems * 2));
    fill_bf16<<<(c_elems + 255) / 256, 256>>>(R, c_elems, 777u, 4.0f);
  }
  if (c.act == XP_ACT_QUICK_GELU || c.act == XP_ACT_DQUICK_GELU) {
    CK(cudaMalloc(&AUX, c_elems * 2));
    if (c.act == XP_ACT_DQUICK_GELU) fill_bf16<<<(c_elems + 255) / 256, 256>>>(AUX, c_elems, 4242u, 3.0f);
    else CK(cudaMemset(AUX, 0xFF, c_elems * 2));
    CK(cudaMalloc(&AUXref, c_elems * 4));
  }
  float alpha = 1.0f / sqrtf((float)c.K);  // keep outputs O(1)
  XpGemm g;
  memset(&g, 0, sizeof(g));
  g.a = A; g.b = B; g.c = c.out == XP_OUT_BF16 ? (void*)Cb : (void*)Cf;
  g.bias = bias; g.residual = R; g.aux = AUX;
  g.M = c.M; g.N = c.N; g.K = c.K;
  g.lda = lda; g.ldb = ldb; g.ldc = c.N; g.ldr = c.N; g.ld_aux = c.N;
  g.a_layout = c.a_layout; g.b_layout = c.b_layout;
  g.act = c.act; g.out = c.out; g.splits = c.splits;
  g.scale_cols = c.qscale ? (c.N / 3 / 8 * 8) : 0;
  g.alpha = alpha; g.col_scale = 0.125f;
  g.block_n = c.bn;
  g.cta_pair = 0;
  int rc = xp_gemm(&g, nullptr);
  if (rc) {
    printf("[%s] xp_gemm error: %s\n", c.name, xp_last_error());
    return 1;
  }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    printf("[%s] kernel failed: %s\n", c.name, cudaGetErrorString(e));
    exit(3);
  }
  dim3 rg((c.N + 127) / 128, c.M);
  ref_gemm<<<rg, 128>>>(A, B, Cref, c.act == XP_ACT_QUICK_GELU ? AUXref : nullptr, c.M, c.N, c.K, lda, ldb,
                        c.a_layout, c.b_layout, bias, R, c.N, AUX, c.N, c.act, g.scale_cols, alpha, 0.125f);
  CK(cudaDeviceSynchronize());
  std::vector<float> ref(c_elems), got(c_elems);
  CK(cudaMemcpy(ref.data(), Cref, c_elems * 4, cudaMemcpyDeviceToHost));
  if (c.out == XP_OUT_BF16) {
    std::vector<__nv_bfloat16> tmp(c_elems);
    CK(cudaMemcpy(tmp.data(), Cb, c_elems * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < c_elems; ++i) got[i] = __bfloat162float(tmp[i]);
  } else {
    CK(cudaMemcpy(got.data(), Cf, c_elems * 4, cudaMemcpyDeviceToHost));
  }
  double max_err = 0, max_ref = 0;
  size_t bad = 0, first_bad = (size_t)-1;
  for (size_t i = 0; i < c_elems; ++i) {
    double d = fabs((double)got[i] - (double)ref[i]);
    double tol = (c.out == XP_OUT_BF16 ? 1.0e-2 : 2e-3) * fmax(1.0, fabs((double)ref[i]));
    if (!(d <= tol)) {
      if (first_bad == (size_t)-1) first_bad = i;
      ++bad;
    }
    if (d > max_err || d != d) max_err = d;
    if (fabs(ref[i]) > max_ref) max_ref = fabs(ref[i]);
  }
  size_t aux_bad = 0;
  if (c.act == XP_ACT_QUICK_GELU) {
    std::vector<float> aref(c_elems);
    std::vector<__nv_bfloat16> agot(c_elems);
    CK(cudaMemcpy(aref.data(), AUXref, c_elems * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(agot.data(), AUX, c_elems * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < c_elems; ++i) {
      double d = fabs((double)__bfloat162float(agot[i]) - (double)aref[i]);
      if (!(d <= 1e-2 * fmax(1.0, fabs((double)aref[i])))) ++aux_bad;
    }
  }
  bool ok = bad == 0 && aux_bad == 0;
  printf("[%s] M=%d N=%d K=%d layout=(%d,%d) act=%d out=%d splits=%d bn=%d : %s max_err=%.4g max_ref=%.3g bad=%zu aux_bad=%zu\n",
         c.name, c.M, c.N, c.K, c.a_layout, c.b_layout, c.act, c.out, c.splits, c.bn, ok ? "PASS" : "FAIL", max_err,
         max_ref, bad, aux_bad);
  if (!ok && first_bad != (size_t)-1) {
    // print an error map: which (row block of 8, col block of 8) are wrong, for the top-left 128x128
    int R8 = c.M < 128 ? (c.M + 7) / 8 : 16, C8 = c.N < 128 ? (c.N + 7) / 8 : 16;
    printf("  first bad at (m=%zu, n=%zu): got %.5f ref %.5f; 8x8-block error map of the top-left tile:\n",
           first_bad / c.N, first_bad % c.N, got[first_bad], ref[first_bad]);
    for (int rb = 0; rb < R8; ++rb) {
      printf("  ");
      for (int cb = 0; cb < C8; ++cb) {
        int nb = 0;
        for (int i = 0; i < 8; ++i)
          for (int j = 0; j < 8; ++j) {
            size_t m = rb * 8 + i, n = cb * 8 + j;
            if (m < (size_t)c.M && n < (size_t)c.N) {
              size_t idx = m * c.N + n;
              if (!(fabs((double)got[idx] - ref[idx]) <= 1e-2 * fmax(1.0, fabs((double)ref[idx])))) ++nb;
            }
          }
        printf("%c", nb == 0 ? '.' : (nb == 64 ? '#' : 'x'));
      }
      printf("\n");
    }
  }
  if (timing && ok) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (int i = 0; i < 3; ++i) xp_gemm(&g, nullptr);
    const int iters = 20;
    CK(cudaEventRecord(e0));
    for (int i = 0; i < iters; ++i) xp_gemm(&g, nullptr);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    ms /= iters;
    double tf = 2.0 * c.M * c.N * (double)c.K / (ms * 1e-3) / 1e12;
    printf("  timing: %.3f ms  %.1f TFLOP/s\n", ms, tf);
  }
  cudaFree(A); cudaFree(B); cudaFree(Cref);
  if (Cb) cudaFree(Cb);
  if (Cf) cudaFree(Cf);
  if (bias) cudaFree(bias);
  if (R) cudaFree(R);
  if (AUX) cudaFree(AUX);
  if (AUXref) cudaFree(AUXref);
  return ok ? 0 : 1;
}

int main(int argc, char** argv) {
  int fails = 0;
  const Case basic[] = {
      {"kk_small_bn128", 128, 128, 64, 0, 0, 0, XP_OUT_F32, 1, 128, false, false, false},
      {"kk_k256_bn128", 128, 128, 256, 0, 0, 0, XP_OUT_F32, 1, 128, false, false, false},
      {"kk_small_bn256", 256, 256, 128, 0, 0, 0, XP_OUT_F32, 1, 256, false, false, false},
      {"kk_multi_tile", 1024, 768, 768, 0, 0, 0, XP_OUT_BF16, 1, 256, false, false, false},
      {"kk_persistent", 4096, 3072, 768, 0, 0, 0, XP_OUT_BF16, 1, 256, true, false, false},
      {"kk_ragged", 200, 136, 72, 0, 0, 0, XP_OUT_F32, 1, 128, true, false, false},
      {"kk_m64", 64, 512, 768, 0, 0, 0, XP_OUT_F32, 1, 0, false, false, false},
      {"kmn_dgrad_small", 128, 128, 64, 0, 1, 0, XP_OUT_F32, 1, 128, false, false, false},
      {"kmn_dgrad", 1024, 768, 3072, 0, 1, 0, XP_OUT_BF16, 1, 256, false, false, false},
      {"mnmn_wgrad_small", 128, 128, 64, 1, 1, 0, XP_OUT_F32, 1, 128, false, false, false},
      {"mnmn_wgrad", 768, 768, 4096, 1, 1, 0, XP_OUT_F32_ATOMIC, 4, 128, false, false, false},
      {"mnmn_wgrad_bn256", 3072, 768, 2048, 1, 1, 0, XP_OUT_F32_ATOMIC, 3, 256, false, false, false},
      {"mnk", 256, 256, 256, 1, 0, 0, XP_OUT_F32, 1, 128, false, false, false},
      {"epi_qkv", 512, 2304, 768, 0, 0, 0, XP_OUT_BF16, 1, 256, true, false, true},
      {"epi_gelu", 512, 3072, 768, 0, 0, XP_ACT_QUICK_GELU, XP_OUT_BF16, 1, 256, true, false, false},
      {"epi_dgelu", 512, 3072, 768, 0, 1, XP_ACT_DQUICK_GELU, XP_OUT_BF16, 1, 256, false, false, false},
      {"epi_residual", 512, 768, 3072, 0, 0, 0, XP_OUT_BF16, 1, 128, true, true, false},
  };
  const char* only = (argc > 2 && !strcmp(argv[1], "only")) ? argv[2] : nullptr;
  if (!only)
    for (const Case& c : basic) fails += run_case(c, false);

  if (argc > 1 && !strcmp(argv[1], "mnsweep")) {
    // If MN-major failed above, try the alternative LBO/SBO reading.
    const int alts[][2] = {{1024, 8192}, {8192, 128}, {128, 8192}};
    for (auto& a : alts) {
      printf("--- MN-major descriptor alt: LBO=%d SBO=%d\n", a[0], a[1]);
      xp_debug_gemm_mn_desc(a[0], a[1]);
      run_case(basic[7], false);
      run_case(basic[9], false);
    }
    xp_debug_gemm_mn_desc(0, 0);
  }

  // timing at the shapes of one ViP block at B=16 (M = 16*2356 = 37696 rows)
  const Case perf[] = {
      {"perf_qkv", 37696, 2304, 768, 0, 0, 0, XP_OUT_BF16, 1, 256, true, false, true},
      {"perf_outproj", 37696, 768, 768, 0, 0, 0, XP_OUT_BF16, 1, 256, true, true, false},
      {"perf_outproj_bn128", 37696, 768, 768, 0, 0, 0, XP_OUT_BF16, 1, 128, true, true, false},
      {"perf_fc1", 37696, 3072, 768, 0, 0, XP_ACT_QUICK_GELU, XP_OUT_BF16, 1, 256, true, false, false},
      {"perf_fc1_bn128", 37696, 3072, 768, 0, 0, XP_ACT_QUICK_GELU, XP_OUT_BF16, 1, 128, true, false, false},
      {"perf_fc2", 37696, 768, 3072, 0, 0, 0, XP_OUT_BF16, 1, 256, true, true, false},
      {"perf_dgrad_fc2", 37696, 3072, 768, 0, 1, XP_ACT_DQUICK_GELU, XP_OUT_BF16, 1, 256, false, false, false},
      {"perf_dgrad_fc1", 37696, 768, 3072, 0, 1, 0, XP_OUT_BF16, 1, 256, false, false, false},
      {"perf_wgrad_fc1", 3072, 768, 37696, 1, 1, 0, XP_OUT_F32_ATOMIC, 1, 128, false, false, false},
      {"perf_wgrad_fc1_s2", 3072, 768, 37696, 1, 1, 0, XP_OUT_F32_ATOMIC, 2, 256, false, false, false},
      {"perf_wgrad_fc2", 768, 3072, 37696, 1, 1, 0, XP_OUT_F32_ATOMIC, 1, 128, false, false, false},
      {"perf_wgrad_out", 768, 768, 37696, 1, 1, 0, XP_OUT_F32_ATOMIC, 4, 128, false, false, false},
      {"perf_square", 8192, 8192, 8192, 0, 0, 0, XP_OUT_BF16, 1, 256, false, false, false},
  };
  if (!(argc > 1 && !strcmp(argv[1], "quick")))
    for (const Case& c : perf)
      if (!only || !strcmp(only, c.name)) fails += run_case(c, true);
  printf("gemm_selftest: %d failing case(s)\n", fails);
  return fails ? 1 : 0;
}
