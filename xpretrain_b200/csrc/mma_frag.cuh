// Warp-level mma.sync.m16n8k16 (bf16 -> fp32) building blocks of the segment / window attention (seg_attention.cu):
// swizzled [rows][64] bf16 shared-memory tiles, cp.async staging, ldmatrix fragment loads.  vip_attention.cu shares the
// head-dim / exp2 constants and the zero-row store.
#pragma once
#include <cstdint>

#include "ptx.cuh"

namespace xp {

constexpr int HD = 64;          // head dim
constexpr float LOG2E = 1.4426950408889634f;

// ---- shared memory tile [ROWS][64] bf16, 128-byte rows, 16-byte chunks XOR-swizzled by (row & 7)
__device__ __forceinline__ uint32_t tile_addr(uint32_t base, int row, int chunk) {
  return base + row * 128 + ((chunk ^ (row & 7)) << 4);
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// wait until at most N committed cp.async groups of this thread are still in flight
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void st_shared_zero16(uint32_t dst) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(dst), "r"(0) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// A fragments (16 rows x 64 k) of rows [row0, row0+16) of a tile: 4 k-steps x 4 regs.
__device__ __forceinline__ void load_a_frags(uint32_t tile, int row0, int lane, uint32_t (&a)[4][4]) {
  const int r = row0 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) ldsm_x4(tile_addr(tile, r, ks * 2 + (lane >> 4)), a[ks]);
}
// B fragments for two n8 tiles (16 "n" rows starting at n0) at k-step ks from a [n][k] tile (k contiguous).
__device__ __forceinline__ void load_b_nk(uint32_t tile, int n0, int ks, int lane, uint32_t (&b)[4]) {
  const int r = n0 + (lane & 7) + (lane >> 4) * 8;
  ldsm_x4(tile_addr(tile, r, ks * 2 + ((lane >> 3) & 1)), b);  // {b0,b1} of n-tile 0, {b0,b1} of n-tile 1
}
// B fragments for two n8 tiles (columns [dp*16, dp*16+16)) over 16 k rows starting at k0 from a [k][n] tile.
__device__ __forceinline__ void load_b_kn(uint32_t tile, int k0, int dp, int lane, uint32_t (&b)[4]) {
  const int r = k0 + (lane & 7) + ((lane >> 3) & 1) * 8;
  ldsm_x4_t(tile_addr(tile, r, dp * 2 + (lane >> 4)), b);
}

}  // namespace xp
