// metamorph_b200 — helpers shared by the wgmma attention kernels (attention_tc.cu forward, attention_bwd_tc.cu
// backward): SW128 operand descriptors for the [128 x 64] TMA boxes, accumulator -> A-fragment packing, row tensor maps.
#pragma once
#include "wgmma.cuh"
#include <mutex>

namespace mm_attn_tc {

constexpr float kLog2e = 1.4426950408889634f;

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// K-major SW128 operand tile stored as two [rows x 64 elem] TMA boxes of 128 rows (16 KB each): k16-th 16-wide slice
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t tile, int k16) {
  return wgmma_desc(tile + (uint32_t)(k16 >> 2) * 16384u + (uint32_t)(k16 & 3) * 32u, 16);
}
// MN-major SW128 operand tile: two [128 k-rows x 64 mn-elem] boxes; LBO = 16 KB between MN chunks
__device__ __forceinline__ uint64_t desc_mnmajor(uint32_t tile, int k16) {
  return wgmma_desc(tile + (uint32_t)k16 * 2048u, 16384);
}
// fp32 accumulator columns [16k, 16k + 16) of a wgmma D fragment -> the bf16 A fragment of k-slice k
template <int NA>
__device__ __forceinline__ void acc_to_a(const float (&d)[NA], int k, uint32_t (&a)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) a[i] = pack_bf16x2(d[8 * k + 2 * i], d[8 * k + 2 * i + 1]);
}
// Release a shared-memory stage: one arrive per warp of the consumer warpgroups (barrier count 8).
__device__ __forceinline__ void consumer_release(uint32_t bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

}  // namespace mm_attn_tc

// One tensor map per operand: rows = tokens, box = [box_rows x 64 bf16] (128-byte swizzle). Defined in attention_tc.cu.
int mm_attn_make_tmap_rows(CUtensorMap* tm, const void* base, long long width, long long rows, long long ld,
                           int box_rows = 128);
// fp32 statistics rows [rows, width] (lse*log2e and delta of the backward): box = 128 values of one row.
int mm_attn_make_tmap_stats(CUtensorMap* tm, const float* base, long long width, long long rows);
