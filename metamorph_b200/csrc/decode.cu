// metamorph_b200 — KV-cached autoregressive decode step (SURVEY.md K20, row A9).
//
// The reference re-runs the whole prefix every step with no cache (metamorph_llama.py:510,526-535);
// the mathematically equivalent cached step is HBM-bound: every weight byte is streamed once per
// step for <= 128 sequences (33..128 through skinny_gemm_wide, decode_wide.cu). Kernels:
//   skinny_gemm   y[m<=32, N] = x[m, K] * W[N, K]^T : weight-streaming with mma.sync m16n8k16 where
//                 the 16-row operand is a slab of W (rows = output features) and the 8-wide operand
//                 is the batch (1, 2 or 4 n8 tiles). Weight slab and activation slice travel together
//                 through a TMA ring, 4 consumer warps split K, fp32 cross-warp reduction in smem, fused
//                 bias / residual / GELU / SwiGLU epilogue.
//   decode_attn   per (sequence, kv head): RoPE on the new q (4 GQA heads) and k, append k/v to the
//                 cache, single-query attention over the cache, all in one launch.
//   decode_state  the per-sequence text/image mode state machine of greedy_decode
//                 (metamorph_llama.py:547-582) on the device: no .item() host syncs.
#include "common.cuh"
#include "fp8.cuh"
#include <mutex>
#include <type_traits>
#include <stdlib.h>

typedef CUresult (*PFN_encodeTiledSk)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                      const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                      CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                      CUtensorMapFloatOOBfill);

namespace {

enum SkEpi : int { SK_STORE = 0, SK_BIAS = 1, SK_RESID = 2, SK_BIAS_GELU = 3, SK_SWIGLU = 4 };

// ---------------------------------------------------------------------------------------------
// skinny GEMM v2: the weight slab is streamed by TMA into an 8-deep ring of 128B-swizzled tiles
// ([ROWS rows x 256 k] per stage), so every CTA keeps 64-128 KB of HBM reads in flight without spending
// registers on them; one producer lane + four consumer warps (2 k32-chunks each per stage, same
// weight-slab-as-A-operand mma.sync trick as v1). Small-N projections (o_proj, down_proj) no longer pay
// the load-wait-compute round trips of the register-staged kernel.
constexpr int SK2_STAGES = 8;      // default ring depth (16-row slabs: 8 x 8 KB per CTA)
constexpr int SK2_KT = 256;      // k elements per stage
constexpr int SK2_THREADS = 160; // warp 0 = TMA producer, warps 1..4 = consumers

// FP8 (skinny_gemm_fp8_kernel): the weight slab is E4M3 bytes with one power-of-two fp32 scale per 128 k of a row
// (fp8_quant_row_warp); a stage holds 2 uint8 boxes [ROWS x 128 k] (one 128-byte swizzled row = 128 k) instead of 4 bf16
// boxes [ROWS x 64 k]. Each lane loads the 8 bytes of exactly the 8 k its bf16 counterpart loads, turns them into
// float(q) * scale (exact, a bf16 value) in the same four bf16x2 registers, and the same mma.sync sequence follows: on
// weights W-hat = float(q) * scale the output bits are skinny_gemm_tma_kernel's.
template <int ROWS, int NST, int NB, bool FP8>
__device__ __forceinline__ void
skinny_gemm_body(const CUtensorMap& tmap_w, const CUtensorMap& tmap_x, void* __restrict__ y, long long ldy,
                 const bf16* __restrict__ bias, const bf16* __restrict__ resid, long long ldr, int m, int N, int K, int epi,
                 int out_f32, const float* __restrict__ wsc, long long lds) {
  constexpr int G = ROWS >= 16 ? ROWS / 16 : 1;
  constexpr bool HALF = ROWS == 8;             // 8-row slab: rows 8..15 of the MMA operand are zero
  constexpr int MB = 8 * NB;                   // batch rows served: NB n8 tiles of the MMA's B operand
  constexpr int BOX = ROWS * 128;              // bytes of one weight box: [ROWS x 64 k] bf16 or [ROWS x 128 k] E4M3
  constexpr int NBOX = FP8 ? 2 : 4;            // weight boxes per stage of 256 k
  constexpr int XBOX = MB * 128;               // bytes of one [MB batch rows x 64 k] activation box
  constexpr int STAGE_W = NBOX * BOX;          // 256 k of the weight slab
  constexpr int STAGE = STAGE_W + 4 * XBOX;    // + the same 256 k of the activations (rows >= m zero-filled by TMA)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  constexpr int BARB = (2 * NST * 8 + 127) & ~127;      // bytes of the full/empty barrier block
  const uint32_t bar = base + NST * STAGE;
  float* red = reinterpret_cast<float*>(base_ptr + NST * STAGE + BARB);   // [4][ROWS][MB]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * ROWS;
  const int n_kt = (K + SK2_KT - 1) / SK2_KT;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_w);
    prefetch_tmap(&tmap_x);
    for (int s = 0; s < NST; ++s) {
      mbar_init(bar + 8 * s, 1);              // full
      mbar_init(bar + 8 * (NST + s), 4);      // empty: one arrive per consumer warp
    }
    fence_barrier_init();
  }
  griddep_launch();
  __syncthreads();
  if (warp == 0) {
    if (lane == 0) {
      // The activation slice of a stage travels WITH its weights: one transaction, NST stages of look-ahead. (Round 1
      // fetched each lane's x fragments through a private 2-deep cp.async ring: every stage then waited an L2 round trip
      // for fragments requested two stages earlier, which capped a CTA at ~30 GB/s whatever the ring depth —
      // profiles/r02_decode_skinny_fit_before.txt.) The weights of the first NST stages are requested BEFORE waiting for the
      // previous kernel (they never change during a step); x, which that kernel produces, follows after the wait.
      const int n_pre = n_kt < NST ? n_kt : NST;
      for (int kt = 0; kt < n_pre; ++kt) {
        mbar_arrive_expect_tx(bar + 8 * kt, STAGE);
#pragma unroll
        for (int bx = 0; bx < NBOX; ++bx)
          tma_load_2d(base + kt * STAGE + bx * BOX, &tmap_w, bar + 8 * kt, kt * SK2_KT + bx * (FP8 ? 128 : 64), n0);
      }
      griddep_wait();
      for (int kt = 0; kt < n_pre; ++kt) {
#pragma unroll
        for (int bx = 0; bx < 4; ++bx)
          tma_load_2d(base + kt * STAGE + STAGE_W + bx * XBOX, &tmap_x, bar + 8 * kt, kt * SK2_KT + bx * 64, 0);
      }
      for (int kt = n_pre; kt < n_kt; ++kt) {
        const int s = kt % NST;
        const uint32_t ph = (uint32_t)((kt / NST) & 1);
        mbar_wait(bar + 8 * (NST + s), ph ^ 1);
        mbar_arrive_expect_tx(bar + 8 * s, STAGE);
#pragma unroll
        for (int bx = 0; bx < NBOX; ++bx)
          tma_load_2d(base + s * STAGE + bx * BOX, &tmap_w, bar + 8 * s, kt * SK2_KT + bx * (FP8 ? 128 : 64), n0);
#pragma unroll
        for (int bx = 0; bx < 4; ++bx)
          tma_load_2d(base + s * STAGE + STAGE_W + bx * XBOX, &tmap_x, bar + 8 * s, kt * SK2_KT + bx * 64, 0);
      }
    }
  } else {
    const int cw = warp - 1;                 // consumer index 0..3
    const int g = lane >> 2, t = lane & 3;
    float acc[G][NB][4];
#pragma unroll
    for (int i = 0; i < G; ++i)
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][nb][j] = 0.f;
    for (int kt = 0; kt < n_kt; ++kt) {
      const int s = kt % NST;
      const uint32_t ph = (uint32_t)((kt / NST) & 1);
      // FP8: the scales of this warp's 64 k (group 2 kt + cw / 2) for its rows r0 / r1 of every 16-row group, requested
      // before the stage wait; rows past N and the group past K (zero-filled bytes) take 1
      float sc0[G], sc1[G];
      if constexpr (FP8) {
        const int grp = 2 * kt + (cw >> 1);
#pragma unroll
        for (int i = 0; i < G; ++i) {
          const int n = n0 + i * 16 + g;
          const bool gok = grp * 128 < K;
          sc0[i] = gok && n < N ? __ldg(wsc + (long long)n * lds + grp) : 1.f;
          sc1[i] = gok && !HALF && n + 8 < N ? __ldg(wsc + (long long)(n + 8) * lds + grp) : 1.f;
        }
      }
      mbar_wait(bar + 8 * s, ph);
      const uint8_t* st = base_ptr + s * STAGE;
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int cc = 2 * cw + u;             // k32 chunk of this stage: box cc/2, half cc%2
        const uint8_t* bx = st + (cc >> 1) * BOX;
        const int chunk = (cc & 1) * 4 + t;    // 16-byte chunk index inside the 128-byte row
        // FP8: the same 8 k sit at byte 64 (cw & 1) + 8 chunk of a row of box cw / 2
        const uint8_t* bx8 = st + (cw >> 1) * BOX;
        const int c8 = 4 * (cw & 1) + (chunk >> 1), h8 = (chunk & 1) * 8;
        // B fragments: batch rows g + 8 nb, the same 8 k values (128-byte swizzled [MB x 64] box; the swizzle repeats
        // every 8 rows, so row g + 8 nb uses the same chunk permutation as row g)
        int4 xb[NB];
#pragma unroll
        for (int nb = 0; nb < NB; ++nb)
          xb[nb] = *reinterpret_cast<const int4*>(st + STAGE_W + (cc >> 1) * XBOX + (nb * 8 + g) * 128 + ((chunk ^ g) << 4));
#pragma unroll
        for (int i = 0; i < G; ++i) {
          const int r0 = i * 16 + g, r1 = r0 + 8;
          int4 w0, w1;
          if constexpr (FP8) {
            const uint2 q0 = *reinterpret_cast<const uint2*>(bx8 + r0 * 128 + ((c8 ^ (r0 & 7)) << 4) + h8);
            const uint2 a0 = fp8x4_to_bf16x4(q0.x, sc0[i]), b0 = fp8x4_to_bf16x4(q0.y, sc0[i]);
            w0 = make_int4((int)a0.x, (int)a0.y, (int)b0.x, (int)b0.y);
            if (HALF) {
              w1 = make_int4(0, 0, 0, 0);
            } else {
              const uint2 q1 = *reinterpret_cast<const uint2*>(bx8 + r1 * 128 + ((c8 ^ (r1 & 7)) << 4) + h8);
              const uint2 a1 = fp8x4_to_bf16x4(q1.x, sc1[i]), b1 = fp8x4_to_bf16x4(q1.y, sc1[i]);
              w1 = make_int4((int)a1.x, (int)a1.y, (int)b1.x, (int)b1.y);
            }
          } else {
            w0 = *reinterpret_cast<const int4*>(bx + r0 * 128 + ((chunk ^ (r0 & 7)) << 4));
            w1 = HALF ? make_int4(0, 0, 0, 0)
                      : *reinterpret_cast<const int4*>(bx + r1 * 128 + ((chunk ^ (r1 & 7)) << 4));
          }
          const uint32_t a1[4] = {(uint32_t)w0.x, (uint32_t)w1.x, (uint32_t)w0.y, (uint32_t)w1.y};
          const uint32_t a2[4] = {(uint32_t)w0.z, (uint32_t)w1.z, (uint32_t)w0.w, (uint32_t)w1.w};
#pragma unroll
          for (int nb = 0; nb < NB; ++nb) {
            mma_bf16_16816(acc[i][nb], a1, (uint32_t)xb[nb].x, (uint32_t)xb[nb].y);
            mma_bf16_16816(acc[i][nb], a2, (uint32_t)xb[nb].z, (uint32_t)xb[nb].w);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar + 8 * (NST + s));
    }
#pragma unroll
    for (int i = 0; i < G; ++i)
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) {
        float* rr = red + (cw * ROWS + i * 16 + g) * MB + nb * 8 + 2 * t;
        rr[0] = acc[i][nb][0];
        rr[1] = acc[i][nb][1];
        if (!HALF) {
          rr[8 * MB] = acc[i][nb][2];
          rr[8 * MB + 1] = acc[i][nb][3];
        }
      }
  }
  griddep_wait();
  __syncthreads();
  if (epi == SK_SWIGLU) {
    if (ROWS >= 32) {
      // rows of the slab: [16 gate | 16 up] per group of 32 (engine/packing.py interleave_gate_up)
      for (int idx = threadIdx.x; idx < (ROWS / 2) * MB; idx += SK2_THREADS) {
        const int r = idx / MB, b = idx % MB;
        const int gr = (r >> 4) * 32 + (r & 15);
        float gsum = 0.f, usum = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          gsum += red[(w * ROWS + gr) * MB + b];
          usum += red[(w * ROWS + gr + 16) * MB + b];
        }
        const int col = (n0 >> 1) + r;
        if (b < m && n0 + gr < N)
          reinterpret_cast<bf16*>(y)[(long long)b * ldy + col] = __float2bfloat16(silu(gsum) * usum);
      }
    }
    return;
  }
  for (int idx = threadIdx.x; idx < ROWS * MB; idx += SK2_THREADS) {
    const int r = idx / MB, b = idx % MB;
    const int n = n0 + r;
    if (b >= m || n >= N) continue;
    float sacc = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) sacc += red[(w * ROWS + r) * MB + b];
    if (epi == SK_BIAS || epi == SK_BIAS_GELU) sacc += __bfloat162float(bias[n]);
    if (epi == SK_BIAS_GELU) sacc = gelu_erf(sacc);
    if (epi == SK_RESID) sacc += __bfloat162float(resid[(long long)b * ldr + n]);
    if (out_f32) reinterpret_cast<float*>(y)[(long long)b * ldy + n] = sacc;
    else reinterpret_cast<bf16*>(y)[(long long)b * ldy + n] = __float2bfloat16(sacc);
  }
}

template <int ROWS, int NST = SK2_STAGES, int NB = 1>
__global__ void __launch_bounds__(SK2_THREADS)
skinny_gemm_tma_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                       void* __restrict__ y, long long ldy, const bf16* __restrict__ bias,
                       const bf16* __restrict__ resid, long long ldr, int m, int N, int K, int epi, int out_f32) {
  skinny_gemm_body<ROWS, NST, NB, false>(tmap_w, tmap_x, y, ldy, bias, resid, ldr, m, N, K, epi, out_f32, nullptr, 0);
}

// wsc: the fp32 scale of row n, k group j (k in [128 j, 128 j + 128)) at wsc[n * lds + j]
template <int ROWS, int NST, int NB>
__global__ void __launch_bounds__(SK2_THREADS)
skinny_gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                       void* __restrict__ y, long long ldy, const bf16* __restrict__ bias,
                       const bf16* __restrict__ resid, long long ldr, int m, int N, int K, int epi, int out_f32,
                       const float* __restrict__ wsc, long long lds) {
  skinny_gemm_body<ROWS, NST, NB, true>(tmap_w, tmap_x, y, ldy, bias, resid, ldr, m, N, K, epi, out_f32, wsc, lds);
}

// FP8 weights: W [N, K] bf16 -> E4M3 bytes q [N, K] (row stride ldq) and scales [N, K / 128] (row stride lds), one warp
// per 128-value group under fp8_quant_row_warp (lane l: k 4l .. 4l + 3 of the group); and back, W-hat = float(q) * scale.
__global__ void weight_quant_fp8_kernel(const bf16* __restrict__ w, long long ldw, uint8_t* __restrict__ q,
                                        long long ldq, float* __restrict__ sc, long long lds, int N, int K) {
  const int lane = threadIdx.x & 31, ng = K / 128;
  const long long total = (long long)N * ng, stride = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long gi = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; gi < total; gi += stride) {
    const long long n = gi / ng;
    const int j = (int)(gi % ng);
    const uint2 raw = *reinterpret_cast<const uint2*>(w + n * ldw + j * 128 + 4 * lane);
    const float2 f0 = unpack_bf16x2(raw.x), f1 = unpack_bf16x2(raw.y);
    float x[4] = {f0.x, f0.y, f1.x, f1.y};
    uint16_t q01, q23;
    const float s = fp8_quant_row_warp(x, q01, q23);
    *reinterpret_cast<uint32_t*>(q + n * ldq + j * 128 + 4 * lane) = (uint32_t)q01 | ((uint32_t)q23 << 16);
    if (lane == 0) sc[n * lds + j] = s;
  }
}

__global__ void weight_dequant_fp8_kernel(const uint8_t* __restrict__ q, long long ldq, const float* __restrict__ sc,
                                          long long lds, bf16* __restrict__ w, long long ldw, int N, int K) {
  const int lane = threadIdx.x & 31, ng = K / 128;
  const long long total = (long long)N * ng, stride = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long gi = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; gi < total; gi += stride) {
    const long long n = gi / ng;
    const int j = (int)(gi % ng);
    const uint32_t u = *reinterpret_cast<const uint32_t*>(q + n * ldq + j * 128 + 4 * lane);
    *reinterpret_cast<uint2*>(w + n * ldw + j * 128 + 4 * lane) = fp8x4_to_bf16x4(u, sc[n * lds + j]);
  }
}

// ---------------------------------------------------------------------------------------------
// decode attention (split-context). qkv: [B, (Hq+2Hkv)*128] (pre-RoPE); cache K/V: [B, Hkv, Tmax, 128].
// grid (Hkv, B, S): every CTA handles 1/S of the cached positions of one (sequence, kv head) for the G
// query heads of the group and writes partial (max, sum, unnormalised output); decode_attn_combine merges
// the S partials. pos[b] = index of the new token; the CTA owning that position applies RoPE to the new k,
// appends k/v to the cache and uses its on-chip copies (no cross-CTA read-after-write).
// PAGED: kc / vc are block pools [num_blocks, Hkv, 1 << bs_shift, 128] and logical position p of sequence b lives in
// block table[b * max_blocks + (p >> bs_shift)] at row p & (block_size - 1); Tmax = max_blocks << bs_shift. Only the
// address of a K/V row changes: the split, the walk order and the arithmetic are the dense kernel's, so both give the
// same bits on the same logical cache. The table row is read through the read-only path (one entry per position, L1
// resident), which leaves the shared-memory footprint of the dense kernel unchanged.
// FP8: K/V rows are E4M3 bytes with one fp32 power-of-two scale per (position, kv head) row (fp8_quant_row_warp); the
// scale arrays are addressed like the rows ([B, Hkv, Tmax] dense, [num_blocks, Hkv, block_size] paged). Every cached
// element is dequantised to float(q) * 2^e, an exact bf16 value, and then meets the bf16 kernel's arithmetic unchanged,
// so the output bits are the bf16 kernel's on a bf16 cache holding those values. The owner of pos quantises the new
// k / v, appends them and scores pos from the dequantised copies.
constexpr int DA_THREADS = 256;
constexpr int DA_D = 128;

// The E4M3 row rule (fp8_quant_row_warp, fp8x4_dequant) lives in fp8.cuh, shared with the FP8 weights.

template <int G, bool PAGED, bool FP8 = false>
__global__ void __launch_bounds__(DA_THREADS)
decode_attn_kernel(const bf16* __restrict__ qkv, long long ldqkv,
                   std::conditional_t<FP8, uint8_t, bf16>* __restrict__ kc,
                   std::conditional_t<FP8, uint8_t, bf16>* __restrict__ vc, const int* __restrict__ pos_arr,
                   const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                   float* __restrict__ part, int Hq, int Hkv, int Tmax, int S, float scale,
                   const int* __restrict__ table, int max_blocks, int bs_shift, float* __restrict__ ksc,
                   float* __restrict__ vsc) {
  using KVT = std::conditional_t<FP8, uint8_t, bf16>;
  extern __shared__ float sm[];
  float* sq = sm;                          // [G][128] rotated, scaled q
  float* sknew = sq + G * DA_D;            // [128] rotated new k
  float* svnew = sknew + DA_D;             // [128] new v
  float* sred = svnew + DA_D;              // [8 warps][G][128] partial outputs
  float* sscore = sred + 8 * G * DA_D;     // [G][chunk_pad]
  const int hk = blockIdx.x, b = blockIdx.y, sp = blockIdx.z;
  griddep_launch();
  griddep_wait();
  const int pos = pos_arr[b];
  const int n_ctx = pos + 1;
  const int chunk = (n_ctx + S - 1) / S;
  const int p0 = sp * chunk, p1 = min(n_ctx, p0 + chunk);
  const int cpad = ((Tmax + S - 1) / S + 4) & ~3;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bf16* row = qkv + (long long)b * ldqkv;
  KVT* kcb = kc + (PAGED ? 0ll : ((long long)b * Hkv + hk) * Tmax * DA_D);
  KVT* vcb = vc + (PAGED ? 0ll : ((long long)b * Hkv + hk) * Tmax * DA_D);
  const int* trow = PAGED ? table + (long long)b * max_blocks : nullptr;
  // element offset of the K/V row of logical position p, relative to kcb / vcb
  auto row_off = [&](int p) -> long long {
    if constexpr (PAGED) {
      const long long blk = __ldg(trow + (p >> bs_shift));
      return (((blk * Hkv + hk) << bs_shift) + (p & ((1 << bs_shift) - 1))) * DA_D;
    } else {
      return (long long)p * DA_D;
    }
  };
  // FP8: index of the row of p (row_off(p) / 128) in the scale arrays, relative to kscb / vscb
  auto row_idx = [&](int p) -> long long {
    if constexpr (PAGED) {
      const long long blk = __ldg(trow + (p >> bs_shift));
      return ((blk * Hkv + hk) << bs_shift) + (p & ((1 << bs_shift) - 1));
    } else {
      return (long long)p;
    }
  };
  float* kscb = FP8 ? ksc + (PAGED ? 0ll : ((long long)b * Hkv + hk) * Tmax) : nullptr;
  float* vscb = FP8 ? vsc + (PAGED ? 0ll : ((long long)b * Hkv + hk) * Tmax) : nullptr;
  const float* cp = cos_t + (long long)pos * (DA_D / 2);
  const float* sp_ = sin_t + (long long)pos * (DA_D / 2);
  const bool owns_new = (pos >= p0 && pos < p1);
  for (int i = tid; i < G * (DA_D / 2); i += DA_THREADS) {
    const int h = i / (DA_D / 2), j = i % (DA_D / 2);
    const bf16* qh = row + (long long)(hk * G + h) * DA_D;
    const float a = __bfloat162float(qh[j]), c = __bfloat162float(qh[j + DA_D / 2]);
    // bf16 rounding of the rotated q mirrors the training kernel (rope_ writes bf16)
    sq[h * DA_D + j] = __bfloat162float(__float2bfloat16(rope_lo(a, c, cp[j], sp_[j]))) * scale;
    sq[h * DA_D + j + DA_D / 2] = __bfloat162float(__float2bfloat16(rope_hi(a, c, cp[j], sp_[j]))) * scale;
  }
  if constexpr (FP8) {
    // warp 0 quantises the rotated new k (lane: dims 2l, 2l+1, 2l+64, 2l+65), warp 1 the new v (dims 4l .. 4l+3)
    if (owns_new && warp < 2) {
      const long long ri = row_idx(pos);
      float x[4];
      if (warp == 0) {
        const bf16* kh = row + (long long)(Hq + hk) * DA_D;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j = 2 * lane + u;
          const float a = __bfloat162float(kh[j]), c = __bfloat162float(kh[j + DA_D / 2]);
          x[u] = __bfloat162float(__float2bfloat16(rope_lo(a, c, cp[j], sp_[j])));
          x[2 + u] = __bfloat162float(__float2bfloat16(rope_hi(a, c, cp[j], sp_[j])));
        }
        uint16_t q01, q23;
        const float sc = fp8_quant_row_warp(x, q01, q23);
        *reinterpret_cast<uint16_t*>(kcb + ri * DA_D + 2 * lane) = q01;
        *reinterpret_cast<uint16_t*>(kcb + ri * DA_D + DA_D / 2 + 2 * lane) = q23;
        if (lane == 0) kscb[ri] = sc;
        sknew[2 * lane] = x[0];
        sknew[2 * lane + 1] = x[1];
        sknew[DA_D / 2 + 2 * lane] = x[2];
        sknew[DA_D / 2 + 2 * lane + 1] = x[3];
      } else {
        const uint2 raw = *reinterpret_cast<const uint2*>(row + (long long)(Hq + Hkv + hk) * DA_D + 4 * lane);
        const float2 f0 = unpack_bf16x2(raw.x), f1 = unpack_bf16x2(raw.y);
        x[0] = f0.x; x[1] = f0.y; x[2] = f1.x; x[3] = f1.y;
        uint16_t q01, q23;
        const float sc = fp8_quant_row_warp(x, q01, q23);
        *reinterpret_cast<uint32_t*>(vcb + ri * DA_D + 4 * lane) = (uint32_t)q01 | ((uint32_t)q23 << 16);
        if (lane == 0) vscb[ri] = sc;
#pragma unroll
        for (int j = 0; j < 4; ++j) svnew[4 * lane + j] = x[j];
      }
    }
  } else if (owns_new && tid < DA_D / 2) {
    const bf16* kh = row + (long long)(Hq + hk) * DA_D;
    const bf16* vh = row + (long long)(Hq + Hkv + hk) * DA_D;
    const float a = __bfloat162float(kh[tid]), c = __bfloat162float(kh[tid + DA_D / 2]);
    const bf16 k0 = __float2bfloat16(rope_lo(a, c, cp[tid], sp_[tid]));   // the bits rope_ + kv_prefill would store
    const bf16 k1 = __float2bfloat16(rope_hi(a, c, cp[tid], sp_[tid]));
    const long long ro = row_off(pos);
    kcb[ro + tid] = k0;
    kcb[ro + tid + DA_D / 2] = k1;
    sknew[tid] = __bfloat162float(k0);
    sknew[tid + DA_D / 2] = __bfloat162float(k1);
    const bf16 v0 = vh[2 * tid], v1 = vh[2 * tid + 1];
    vcb[ro + 2 * tid] = v0;
    vcb[ro + 2 * tid + 1] = v1;
    svnew[2 * tid] = __bfloat162float(v0);
    svnew[2 * tid + 1] = __bfloat162float(v1);
  }
  __syncthreads();
  // ---- scores: one thread per cached position of this split
  for (int p = p0 + tid; p < p1; p += DA_THREADS) {
    float s[G];
#pragma unroll
    for (int h = 0; h < G; ++h) s[h] = 0.f;
    if (p == pos) {
      for (int d = 0; d < DA_D; ++d) {
        const float kf = sknew[d];
#pragma unroll
        for (int h = 0; h < G; ++h) s[h] += sq[h * DA_D + d] * kf;
      }
    } else if constexpr (FP8) {
      // the whole 128 B row is requested at once (8 x 16 B); each 16 B feeds two of the bf16 kernel's 8-value
      // groups, in the same order
      const long long ri = row_idx(p);
      const int4* kp = reinterpret_cast<const int4*>(kcb + ri * DA_D);
      const float ks = kscb[ri];
      int4 rawk[DA_D / 16];
#pragma unroll
      for (int v2 = 0; v2 < DA_D / 16; ++v2) rawk[v2] = kp[v2];
#pragma unroll
      for (int v2 = 0; v2 < DA_D / 16; ++v2) {
        const int4 raw = rawk[v2];
        const uint32_t u[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int v = 2 * v2 + half;
          float kf[8];
          fp8x4_dequant(u[2 * half], ks, kf);
          fp8x4_dequant(u[2 * half + 1], ks, kf + 4);
#pragma unroll
          for (int h = 0; h < G; ++h) {
            const float4 q0 = *reinterpret_cast<const float4*>(sq + h * DA_D + v * 8);
            const float4 q1 = *reinterpret_cast<const float4*>(sq + h * DA_D + v * 8 + 4);
            s[h] += q0.x * kf[0] + q0.y * kf[1] + q0.z * kf[2] + q0.w * kf[3] + q1.x * kf[4] + q1.y * kf[5] +
                    q1.z * kf[6] + q1.w * kf[7];
          }
        }
      }
    } else {
      const int4* kp = reinterpret_cast<const int4*>(kcb + row_off(p));
#pragma unroll 4
      for (int v = 0; v < DA_D / 8; ++v) {
        const int4 raw = kp[v];
        const uint32_t u[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
        float kf[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(u[j]);
          kf[2 * j] = f.x;
          kf[2 * j + 1] = f.y;
        }
#pragma unroll
        for (int h = 0; h < G; ++h) {
          const float4 q0 = *reinterpret_cast<const float4*>(sq + h * DA_D + v * 8);
          const float4 q1 = *reinterpret_cast<const float4*>(sq + h * DA_D + v * 8 + 4);
          s[h] += q0.x * kf[0] + q0.y * kf[1] + q0.z * kf[2] + q0.w * kf[3] + q1.x * kf[4] + q1.y * kf[5] +
                  q1.z * kf[6] + q1.w * kf[7];
        }
      }
    }
#pragma unroll
    for (int h = 0; h < G; ++h) sscore[h * cpad + (p - p0)] = s[h];
  }
  __syncthreads();
  // ---- local softmax statistics per head (warp h handles heads h, h+8, ...)
  __shared__ float s_m[8], s_l[8];
  const int n_loc = max(p1 - p0, 0);
  for (int h = warp; h < G; h += DA_THREADS / 32) {
    float mx = -INFINITY;
    for (int i = lane; i < n_loc; i += 32) mx = fmaxf(mx, sscore[h * cpad + i]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int i = lane; i < n_loc; i += 32) {
      const float e = __expf(sscore[h * cpad + i] - mx);
      sscore[h * cpad + i] = e;
      sum += e;
    }
    sum = warp_sum(sum);
    if (lane == 0) { s_m[h] = mx; s_l[h] = sum; }
  }
  __syncthreads();
  // ---- O_partial = P V: lane owns 4 dims, warp w takes positions p0+w, p0+w+8, ... (4 loads in flight)
  float o[G][4];
#pragma unroll
  for (int h = 0; h < G; ++h)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[h][j] = 0.f;
  for (int i0 = warp; i0 < n_loc; i0 += 4 * (DA_THREADS / 32)) {
    float vf[4][4];
    int idx[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      idx[u] = i0 + u * (DA_THREADS / 32);
      const int p = p0 + idx[u];
      if (idx[u] < n_loc) {
        if (p == pos) {
#pragma unroll
          for (int j = 0; j < 4; ++j) vf[u][j] = svnew[lane * 4 + j];
        } else if constexpr (FP8) {
          const long long ri = row_idx(p);
          fp8x4_dequant(*reinterpret_cast<const uint32_t*>(vcb + ri * DA_D + lane * 4), vscb[ri], vf[u]);
        } else {
          const uint2 raw = *reinterpret_cast<const uint2*>(vcb + row_off(p) + lane * 4);
          const float2 f0 = unpack_bf16x2(raw.x), f1 = unpack_bf16x2(raw.y);
          vf[u][0] = f0.x; vf[u][1] = f0.y; vf[u][2] = f1.x; vf[u][3] = f1.y;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) vf[u][j] = 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (idx[u] < n_loc) {
#pragma unroll
        for (int h = 0; h < G; ++h) {
          const float pr = sscore[h * cpad + idx[u]];
#pragma unroll
          for (int j = 0; j < 4; ++j) o[h][j] += pr * vf[u][j];
        }
      }
    }
  }
#pragma unroll
  for (int h = 0; h < G; ++h)
#pragma unroll
    for (int j = 0; j < 4; ++j) sred[(warp * G + h) * DA_D + lane * 4 + j] = o[h][j];
  __syncthreads();
  // partial layout: [B, Hkv, S, G, 2 + 128]
  float* pout = part + (((long long)b * Hkv + hk) * S + sp) * G * (2 + DA_D);
  for (int i = tid; i < G * DA_D; i += DA_THREADS) {
    const int h = i / DA_D, dcol = i % DA_D;
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < DA_THREADS / 32; ++w) acc += sred[(w * G + h) * DA_D + dcol];
    pout[h * (2 + DA_D) + 2 + dcol] = acc;
  }
  if (tid < G) {
    pout[tid * (2 + DA_D)] = n_loc > 0 ? s_m[tid] : -INFINITY;
    pout[tid * (2 + DA_D) + 1] = n_loc > 0 ? s_l[tid] : 0.f;
  }
}

// out[b, (hk*G+h)*128 + d] = sum_s o_s e^{m_s - M} / sum_s l_s e^{m_s - M}
__global__ void decode_attn_combine_kernel(const float* __restrict__ part, bf16* __restrict__ out,
                                           long long ldo, int Hkv, int G, int S) {
  const int hk = blockIdx.x, b = blockIdx.y;
  griddep_launch();
  griddep_wait();
  const float* pin = part + (((long long)b * Hkv + hk) * S) * G * (2 + DA_D);
  for (int i = threadIdx.x; i < G * DA_D; i += blockDim.x) {
    const int h = i / DA_D, dcol = i % DA_D;
    float M = -INFINITY;
    for (int s = 0; s < S; ++s) M = fmaxf(M, pin[(s * G + h) * (2 + DA_D)]);
    float L = 0.f, acc = 0.f;
    for (int s = 0; s < S; ++s) {
      const float* ps = pin + (s * G + h) * (2 + DA_D);
      const float w = (ps[0] == -INFINITY) ? 0.f : __expf(ps[0] - M);
      L += ps[1] * w;
      acc += ps[2 + dcol] * w;
    }
    out[(long long)b * ldo + (long long)(hk * G + h) * DA_D + dcol] = __float2bfloat16(acc / L);
  }
}

// copy post-RoPE K/V of a prefill pass (qkv rows [B*T, ld]) into the cache
__global__ void kv_prefill_kernel(const bf16* __restrict__ qkv, long long ld, bf16* __restrict__ kc,
                                  bf16* __restrict__ vc, int B, int T, int Hq, int Hkv, int Tmax) {
  const long long total = (long long)B * T * Hkv * (DA_D / 8);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % (DA_D / 8));
    long long r = i / (DA_D / 8);
    const int hk = (int)(r % Hkv);
    r /= Hkv;
    const int t = (int)(r % T), b = (int)(r / T);
    const bf16* src = qkv + ((long long)b * T + t) * ld;
    const long long dst = (((long long)b * Hkv + hk) * Tmax + t) * DA_D + v * 8;
    *reinterpret_cast<int4*>(kc + dst) = *reinterpret_cast<const int4*>(src + (long long)(Hq + hk) * DA_D + v * 8);
    *reinterpret_cast<int4*>(vc + dst) = *reinterpret_cast<const int4*>(src + (long long)(Hq + Hkv + hk) * DA_D + v * 8);
  }
}

// the same copy for one sequence into the blocks of its table row (pools [num_blocks, Hkv, 1 << bs_shift, 128])
__global__ void kv_prefill_paged_kernel(const bf16* __restrict__ qkv, long long ld, bf16* __restrict__ kc,
                                        bf16* __restrict__ vc, const int* __restrict__ trow, int T, int Hq, int Hkv,
                                        int bs_shift) {
  const long long total = (long long)T * Hkv * (DA_D / 8);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % (DA_D / 8));
    const long long r = i / (DA_D / 8);
    const int hk = (int)(r % Hkv), t = (int)(r / Hkv);
    const bf16* src = qkv + (long long)t * ld;
    const long long blk = __ldg(trow + (t >> bs_shift));
    const long long dst = (((blk * Hkv + hk) << bs_shift) + (t & ((1 << bs_shift) - 1))) * DA_D + v * 8;
    *reinterpret_cast<int4*>(kc + dst) = *reinterpret_cast<const int4*>(src + (long long)(Hq + hk) * DA_D + v * 8);
    *reinterpret_cast<int4*>(vc + dst) = *reinterpret_cast<const int4*>(src + (long long)(Hq + Hkv + hk) * DA_D + v * 8);
  }
}

// FP8 prefill: quantise the post-RoPE K and V rows of qkv rows [B*T, ld] (one warp per row, fp8_quant_row_warp) into the
// cache, and overwrite qkv's K / V columns with the dequantised rows, so that the prefill's attention reads exactly the
// values the cache holds. Dense: bytes [B, Hkv, Tmax, 128], scales [B, Hkv, Tmax]. PAGED (one sequence, B = 1): pools
// [num_blocks, Hkv, 1 << bs_shift, 128] and scales [num_blocks, Hkv, 1 << bs_shift] through the table row trow.
template <bool PAGED>
__global__ void kv_quant_prefill_kernel(bf16* __restrict__ qkv, long long ld, uint8_t* __restrict__ kc,
                                        uint8_t* __restrict__ vc, float* __restrict__ ks, float* __restrict__ vs,
                                        const int* __restrict__ trow, int B, int T, int Hq, int Hkv, int Tmax,
                                        int bs_shift) {
  const int lane = threadIdx.x & 31;
  const long long total = (long long)B * T * Hkv * 2;
  const long long stride = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < total; w += stride) {
    const int kind = (int)(w & 1);          // 0: K, 1: V
    long long r = w >> 1;
    const int hk = (int)(r % Hkv);
    r /= Hkv;
    const int t = (int)(r % T), b = (int)(r / T);
    bf16* src = qkv + ((long long)b * T + t) * ld + (long long)(Hq + kind * Hkv + hk) * DA_D + 4 * lane;
    long long ri;
    if constexpr (PAGED) {
      const long long blk = __ldg(trow + (t >> bs_shift));
      ri = ((blk * Hkv + hk) << bs_shift) + (t & ((1 << bs_shift) - 1));
    } else {
      ri = ((long long)b * Hkv + hk) * Tmax + t;
    }
    const uint2 raw = *reinterpret_cast<const uint2*>(src);
    const float2 f0 = unpack_bf16x2(raw.x), f1 = unpack_bf16x2(raw.y);
    float x[4] = {f0.x, f0.y, f1.x, f1.y};
    uint16_t q01, q23;
    const float sc = fp8_quant_row_warp(x, q01, q23);
    *reinterpret_cast<uint32_t*>((kind ? vc : kc) + ri * DA_D + 4 * lane) = (uint32_t)q01 | ((uint32_t)q23 << 16);
    if (lane == 0) (kind ? vs : ks)[ri] = sc;
    const __nv_bfloat162 h01 = __floats2bfloat162_rn(x[0], x[1]), h23 = __floats2bfloat162_rn(x[2], x[3]);
    uint2 out;
    out.x = *reinterpret_cast<const uint32_t*>(&h01);
    out.y = *reinterpret_cast<const uint32_t*>(&h23);
    *reinterpret_cast<uint2*>(src) = out;
  }
}

// bf16 staging copy of an FP8 pool: staging block i <- float(q) * 2^e of pool block trow[i], i < n_blocks (K and V)
__global__ void kv_dequant_paged_kernel(const uint8_t* __restrict__ kp, const uint8_t* __restrict__ vp,
                                        const float* __restrict__ ks, const float* __restrict__ vs,
                                        const int* __restrict__ trow, int n_blocks, int Hkv, int bs_shift,
                                        bf16* __restrict__ kst, bf16* __restrict__ vst) {
  const long long per_blk = (long long)Hkv << bs_shift;   // rows of one block
  const long long rows = n_blocks * per_blk;
  const long long total = rows * (DA_D / 16) * 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % (DA_D / 16));
    const long long r = (i / (DA_D / 16)) % rows;
    const int kind = (int)(i / ((DA_D / 16) * rows));
    const long long src_row = (long long)__ldg(trow + r / per_blk) * per_blk + r % per_blk;
    const int4 raw = reinterpret_cast<const int4*>((kind ? vp : kp) + src_row * DA_D)[c];
    const float sc = (kind ? vs : ks)[src_row];
    const uint32_t u[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
    uint32_t o[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float f[4];
      fp8x4_dequant(u[j], sc, f);
      const __nv_bfloat162 a = __floats2bfloat162_rn(f[0], f[1]), b = __floats2bfloat162_rn(f[2], f[3]);
      o[2 * j] = *reinterpret_cast<const uint32_t*>(&a);
      o[2 * j + 1] = *reinterpret_cast<const uint32_t*>(&b);
    }
    int4* dst = reinterpret_cast<int4*>((kind ? vst : kst) + r * DA_D + c * 16);
    dst[0] = make_int4((int)o[0], (int)o[1], (int)o[2], (int)o[3]);
    dst[1] = make_int4((int)o[4], (int)o[5], (int)o[6], (int)o[7]);
  }
}

// ---------------------------------------------------------------------------------------------
// greedy_decode state machine (metamorph_llama.py:547-582), one thread per sequence.
struct DecodeState {
  int* in_image_mode;      // [B]
  int* total_image_tokens; // [B]
  int* total_output;       // [B]
  int* finished;           // [B]
  int* pos;                // [B] next cache position
  int* n_ids;              // [B]
  int* n_img;              // [B]
  int* ids_out;            // [B, max_ids]
  int* append_kind;        // [B] out: 0 = token embedding, 1 = predicted visual embedding, -1 = none
  int* next_token;         // [B] out: token whose embedding is appended (when kind 0)
};

__global__ void decode_state_kernel(DecodeState st, const int* __restrict__ argmax_tok,
                                    const int* __restrict__ forced, int forced_ld, int step, int B,
                                    int num_image_tokens, int max_new_tokens, int max_ids,
                                    int start_id, int end_id, int eos0, int eos1,
                                    const bf16* __restrict__ pred_z, bf16* __restrict__ img_out,
                                    int max_img, int C, const int* __restrict__ max_new_slot) {
  const int b = blockIdx.x;
  __shared__ int s_store_img;
  __shared__ int s_slot;
  if (threadIdx.x == 0) {
    s_store_img = 0;
    int kind = -1;
    if (!st.finished[b]) {
      // forced schedule is indexed by this sequence's own step count (device-resident -> graph replayable)
      const int fidx = st.total_output[b];
      // a negative entry in the forced schedule means "free running" for that position (continuous batching mixes
      // teacher-forced and free sequences in one batch), and so does every position past the schedule's last column:
      // a schedule shorter than the run ends, it does not repeat its last token
      const int ftok = (forced && fidx < forced_ld) ? forced[(long long)b * forced_ld + fidx] : -1;
      const int tok = ftok >= 0 ? ftok : argmax_tok[b];
      const int max_new = max_new_slot ? max_new_slot[b] : max_new_tokens;
      const int mode = st.in_image_mode[b];
      if (!mode && tok == start_id) {
        st.in_image_mode[b] = 1;
        if (st.n_ids[b] < max_ids) st.ids_out[(long long)b * max_ids + st.n_ids[b]] = tok;
        st.n_ids[b]++;
        kind = 0;
      } else if (mode && st.total_image_tokens[b] < num_image_tokens) {
        st.total_image_tokens[b]++;
        s_store_img = 1;
        s_slot = st.n_img[b];
        st.n_img[b]++;
        kind = 1;
        if (st.total_image_tokens[b] == num_image_tokens) st.in_image_mode[b] = 0;
      } else if (tok == end_id) {
        st.in_image_mode[b] = 0;
        st.total_image_tokens[b] = 0;
        if (st.n_ids[b] < max_ids) st.ids_out[(long long)b * max_ids + st.n_ids[b]] = tok;
        st.n_ids[b]++;
        kind = 0;
      } else {
        if (st.n_ids[b] < max_ids) st.ids_out[(long long)b * max_ids + st.n_ids[b]] = tok;
        st.n_ids[b]++;
        kind = 0;
      }
      st.total_output[b]++;
      st.next_token[b] = tok;
      if (tok == eos0 || tok == eos1) st.finished[b] = 1;
      else if (st.total_output[b] > max_new) st.finished[b] = 1;
      st.pos[b]++;
    }
    st.append_kind[b] = kind;
  }
  __syncthreads();
  if (s_store_img && s_slot < max_img) {
    for (int c = threadIdx.x; c < C; c += blockDim.x)
      img_out[((long long)b * max_img + s_slot) * C + c] = pred_z[(long long)b * C + c];
  }
}

// next input embedding: kind 0 -> embed_tokens[next_token], kind 1 -> prediction row, else keep
__global__ void decode_next_input_kernel(const int* __restrict__ kind, const int* __restrict__ tok,
                                         const bf16* __restrict__ embed, const bf16* __restrict__ pred,
                                         bf16* __restrict__ x, int H) {
  const int b = blockIdx.x;
  const int k = kind[b];
  if (k < 0) return;
  const bf16* src = k == 0 ? embed + (long long)tok[b] * H : pred + (long long)b * H;
  for (int v = threadIdx.x; v < H / 8; v += blockDim.x)
    reinterpret_cast<int4*>(x + (long long)b * H)[v] = reinterpret_cast<const int4*>(src)[v];
}

// hidden_eff[b] = in_image_mode[b] ? prediction[b] : hidden[b]   (metamorph_llama.py:377)
__global__ void decode_select_hidden_kernel(const int* __restrict__ mode, const bf16* __restrict__ hidden,
                                            const bf16* __restrict__ pred, bf16* __restrict__ out, int H) {
  const int b = blockIdx.x;
  const bf16* src = mode[b] ? pred + (long long)b * H : hidden + (long long)b * H;
  for (int v = threadIdx.x; v < H / 8; v += blockDim.x)
    reinterpret_cast<int4*>(out + (long long)b * H)[v] = reinterpret_cast<const int4*>(src)[v];
}

}  // namespace

namespace {

template <int ROWS, int NST, int NB, bool FP8>
int launch_skinny_tma(const CUtensorMap& tw, const CUtensorMap& tx, void* y, long long ldy, const void* bias,
                      const void* resid, long long ldr, int m, int N, int K, int epilogue, int out_f32,
                      const float* wsc, long long lds, cudaStream_t stream) {
  constexpr int smem = NST * ((FP8 ? 2 : 4) * ROWS * 128 + 4 * 8 * NB * 128) + ((2 * NST * 8 + 127) & ~127) +
                       4 * ROWS * 8 * NB * 4 + 1024;
  static_assert(smem <= 227 * 1024, "skinny GEMM ring does not fit in shared memory");
  static std::once_flag once;
  static cudaError_t err = cudaSuccess;
  if constexpr (FP8) {
    std::call_once(once, [&] {
      err = cudaFuncSetAttribute(skinny_gemm_fp8_kernel<ROWS, NST, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    });
    MM_CHECK_CUDA(err);
    MM_CHECK_CUDA(launch_pdl(skinny_gemm_fp8_kernel<ROWS, NST, NB>, dim3((N + ROWS - 1) / ROWS), dim3(SK2_THREADS), smem,
                             stream, tw, tx, y, ldy, (const bf16*)bias, (const bf16*)resid, ldr, m, N, K, epilogue,
                             out_f32, wsc, lds));
  } else {
    std::call_once(once, [&] {
      err = cudaFuncSetAttribute(skinny_gemm_tma_kernel<ROWS, NST, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    });
    MM_CHECK_CUDA(err);
    MM_CHECK_CUDA(launch_pdl(skinny_gemm_tma_kernel<ROWS, NST, NB>, dim3((N + ROWS - 1) / ROWS), dim3(SK2_THREADS), smem,
                             stream, tw, tx, y, ldy, (const bf16*)bias, (const bf16*)resid, ldr, m, N, K, epilogue,
                             out_f32));
  }
  MM_CHECK_LAUNCH();
  return MM_OK;
}

// mm_skinny_gemm and mm_skinny_gemm_fp8: argument checks, tensor maps and the slab / batch-tile dispatch; `name` prefixes
// the error messages. FP8: W holds E4M3 bytes (ldw in bytes) and wsc the scales.
template <bool FP8>
int skinny_gemm_launch(const char* name, const void* x, const void* W, const float* wsc, void* y, const void* bias,
                       const void* resid, long long ldx, long long ldw, long long lds, long long ldy, long long ldr,
                       int m, int N, int K, int epilogue, int out_f32, cudaStream_t stream) {
  MM_CHECK_ARG(m >= 1 && m <= 32, "%s: batch must be in [1,32] (m=%d)", name, m);
  if constexpr (FP8) {
    MM_CHECK_ARG(K >= 128 && K % 128 == 0 && ldx % 8 == 0 && ldw % 16 == 0 && ldw >= K,
                 "%s: need K%%128==0, ldx%%8==0, ldw%%16==0 and ldw>=K", name);
    MM_CHECK_ARG(wsc != nullptr && lds >= K / 128, "%s: scales missing or lds < K/128", name);
    MM_CHECK_ARG(((uintptr_t)wsc & 3) == 0, "%s: scales must be 4-byte aligned", name);
  } else {
    MM_CHECK_ARG(K % 32 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "%s: need K%%32==0, ldx/ldw%%8==0", name);
  }
  MM_CHECK_ARG(((uintptr_t)W & 15) == 0 && ((uintptr_t)x & 15) == 0, "%s: x / W must be 16-byte aligned", name);
  MM_CHECK_ARG(epilogue >= SK_STORE && epilogue <= SK_SWIGLU, "%s: bad epilogue", name);
  MM_CHECK_ARG((epilogue != SK_BIAS && epilogue != SK_BIAS_GELU) || bias, "%s: bias missing", name);
  MM_CHECK_ARG(epilogue != SK_RESID || resid, "%s: residual missing", name);
  // The batch is the n dimension of the MMA: 1, 2 or 4 n8 tiles (8 / 16 / 32 sequences) share every weight fragment.
  const int nb = m <= 8 ? 1 : (m <= 16 ? 2 : 4);
  // 32-row slabs where the epilogue needs them (SwiGLU: 16 gate + 16 up rows of the same channels), for very large N
  // (lm_head: fewer, longer-lived CTAs) and for 32 sequences (each CTA re-reads the whole activation block from L2: the
  // taller slab halves that traffic); 16-row slabs otherwise
  const bool rows32 = (epilogue == SK_SWIGLU) || (N >= 32 * 4 * mm_num_sms()) || nb == 4;
  // 32 sequences, wide outputs (gate/up, lm_head): 64-row slabs halve the L2 -> SM activation traffic again, which at this
  // batch equals the weight stream and caps the kernel (measured 4.1 TB/s of weights + as much of x with 32-row slabs)
  const bool rows64 = nb == 4 && N >= 64 * 2 * mm_num_sms() && (epilogue != SK_SWIGLU || N % 64 == 0);
  if (epilogue == SK_SWIGLU) MM_CHECK_ARG(N % 32 == 0 && !out_f32, "%s: SWIGLU needs N%%32==0", name);
  static PFN_encodeTiledSk enc = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      enc = reinterpret_cast<PFN_encodeTiledSk>(fn);
  });
  MM_CHECK_ARG(enc != nullptr, "%s: cuTensorMapEncodeTiled unavailable", name);
  CUtensorMap tw, tx;
  cuuint32_t estr[2] = {1, 1};
  {
    // bf16: [rows x 64 k] boxes; FP8: [rows x 128 k] uint8 boxes. Either way one 128-byte swizzled row per weight row.
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
    cuuint64_t strides[1] = {(cuuint64_t)ldw * (FP8 ? 1 : 2)};
    cuuint32_t box[2] = {FP8 ? 128u : 64u, (cuuint32_t)(rows64 ? 64 : (rows32 ? 32 : 16))};
    CUresult r = enc(&tw, FP8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(W),
                     dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MM_CHECK_ARG(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled(W) failed (%d)", name, (int)r);
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)m};            // rows >= m of the box are zero-filled
    cuuint64_t strides[1] = {(cuuint64_t)ldx * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)(8 * nb)};
    CUresult r = enc(&tx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(x), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MM_CHECK_ARG(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled(x) failed (%d)", name, (int)r);
  }
  // Ring depths: as deep as keeps two CTAs per SM (profiles/r02_decode_skinny_ring_sweep.txt: deeper rings bought nothing);
  // 32 sequences: 32 KB (32-row slabs) or 48 KB (64-row slabs) stages, one CTA per SM. An FP8 stage carries half the
  // weight bytes of a bf16 one, so its ring is deeper in the same shared memory.
#define MM_SK(R, S, B) \
  return launch_skinny_tma<R, S, B, FP8>(tw, tx, y, ldy, bias, resid, ldr, m, N, K, epilogue, out_f32, wsc, lds, stream)
  if constexpr (FP8) {
    if (rows64) MM_SK(64, 6, 4);
    if (nb == 4) MM_SK(32, 6, 4);
    if (nb == 2) {
      if (rows32) MM_SK(32, 6, 2);
      MM_SK(16, 8, 2);
    }
    if (rows32) MM_SK(32, 8, 1);
    MM_SK(16, 12, 1);
  } else {
    if (rows64) MM_SK(64, 4, 4);
    if (nb == 4) MM_SK(32, 5, 4);
    if (nb == 2) {
      if (rows32) MM_SK(32, 4, 2);
      MM_SK(16, 6, 2);
    }
    if (rows32) MM_SK(32, 5, 1);
    MM_SK(16, 8, 1);
  }
#undef MM_SK
}

}  // namespace

MM_API int mm_skinny_gemm(const void* x, const void* W, void* y, const void* bias, const void* resid,
                          long long ldx, long long ldw, long long ldy, long long ldr, int m, int N,
                          int K, int epilogue, int out_f32, cudaStream_t stream) {
  return skinny_gemm_launch<false>("mm_skinny_gemm", x, W, nullptr, y, bias, resid, ldx, ldw, 0, ldy, ldr, m, N, K,
                                   epilogue, out_f32, stream);
}

MM_API int mm_skinny_gemm_fp8(const void* x, const void* Wq, const float* wscale, void* y, const void* bias,
                              const void* resid, long long ldx, long long ldw, long long lds, long long ldy,
                              long long ldr, int m, int N, int K, int epilogue, int out_f32, cudaStream_t stream) {
  return skinny_gemm_launch<true>("mm_skinny_gemm_fp8", x, Wq, wscale, y, bias, resid, ldx, ldw, lds, ldy, ldr, m, N, K,
                                  epilogue, out_f32, stream);
}

namespace {

int weight_fp8_check(const char* name, const void* a, const void* b, const void* sc, long long lda, long long ldb,
                     long long lds, int N, int K) {
  MM_CHECK_ARG(a != nullptr && b != nullptr && sc != nullptr, "%s: null pointer", name);
  MM_CHECK_ARG(N >= 1 && K >= 128 && K % 128 == 0, "%s: need N>=1 and K a positive multiple of 128 (N=%d K=%d)", name,
               N, K);
  MM_CHECK_ARG(lda >= K && ldb >= K && lds >= K / 128 && lda % 4 == 0 && ldb % 4 == 0,
               "%s: need row strides >= K (multiples of 4) and lds >= K/128", name);
  MM_CHECK_ARG((((uintptr_t)a | (uintptr_t)b) & 7) == 0 && ((uintptr_t)sc & 3) == 0, "%s: misaligned operand", name);
  return MM_OK;
}

}  // namespace

MM_API int mm_weight_quant_fp8(const void* W, long long ldw, void* q, long long ldq, float* scale, long long lds, int N,
                               int K, cudaStream_t stream) {
  const int rc = weight_fp8_check("mm_weight_quant_fp8", W, q, scale, ldw, ldq, lds, N, K);
  if (rc != MM_OK) return rc;
  long long blocks = ceil_div64((long long)N * (K / 128) * 32, 256);
  if (blocks > (long long)mm_num_sms() * 16) blocks = (long long)mm_num_sms() * 16;
  weight_quant_fp8_kernel<<<(int)blocks, 256, 0, stream>>>((const bf16*)W, ldw, (uint8_t*)q, ldq, scale, lds, N, K);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_weight_dequant_fp8(const void* q, long long ldq, const float* scale, long long lds, void* W,
                                 long long ldw, int N, int K, cudaStream_t stream) {
  const int rc = weight_fp8_check("mm_weight_dequant_fp8", q, W, scale, ldq, ldw, lds, N, K);
  if (rc != MM_OK) return rc;
  long long blocks = ceil_div64((long long)N * (K / 128) * 32, 256);
  if (blocks > (long long)mm_num_sms() * 16) blocks = (long long)mm_num_sms() * 16;
  weight_dequant_fp8_kernel<<<(int)blocks, 256, 0, stream>>>((const uint8_t*)q, ldq, scale, lds, (bf16*)W, ldw, N, K);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API long long mm_decode_attn_workspace_bytes(int B, int Hq, int Hkv, int splits) {
  return (long long)B * Hkv * splits * (Hq / Hkv) * (2 + DA_D) * 4;
}

namespace {

// shared by the dense and the paged entry points; `name` prefixes the error messages. Dense: table == nullptr.
template <bool PAGED, bool FP8 = false>
int decode_attn_launch(const char* name, const void* qkv, long long ldqkv, void* kcache, void* vcache, const int* pos,
                       const float* cos_t, const float* sin_t, void* out, long long ldo, int B, int Hq, int Hkv,
                       int head_dim, int Tmax, float scale, void* workspace, long long workspace_bytes, int splits,
                       const int* table, int max_blocks, int bs_shift, cudaStream_t stream, float* kscale = nullptr,
                       float* vscale = nullptr) {
  using KVT = std::conditional_t<FP8, uint8_t, bf16>;
  MM_CHECK_ARG(!FP8 || (kscale != nullptr && vscale != nullptr), "%s: scale arrays missing", name);
  MM_CHECK_ARG(head_dim == DA_D && Hq % Hkv == 0, "%s: need head_dim 128", name);
  const int G = Hq / Hkv;
  MM_CHECK_ARG(G == 1 || G == 2 || G == 4 || G == 8, "%s: GQA group must be 1, 2, 4 or 8", name);
  MM_CHECK_ARG(splits >= 1 && splits <= 64, "%s: splits in [1,64]", name);
  MM_CHECK_ARG(workspace != nullptr && workspace_bytes >= mm_decode_attn_workspace_bytes(B, Hq, Hkv, splits),
               "%s: workspace too small", name);
  const int cpad = ((Tmax + splits - 1) / splits + 4) & ~3;
  const size_t smem = (size_t)(G * DA_D + 2 * DA_D + 8 * G * DA_D + G * cpad) * sizeof(float);
  MM_CHECK_ARG(smem <= 200 * 1024, "%s: Tmax/splits = %d positions per CTA is too large", name, cpad);
  dim3 grid(Hkv, B, splits);
#define MM_DA_LAUNCH(GG)                                                                                     \
  do {                                                                                                       \
    if (smem > 48 * 1024)                                                                                    \
      MM_CHECK_CUDA(cudaFuncSetAttribute(decode_attn_kernel<GG, PAGED, FP8>,                                 \
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));           \
    MM_CHECK_CUDA(launch_pdl(decode_attn_kernel<GG, PAGED, FP8>, grid, dim3(DA_THREADS), smem, stream,       \
                             (const bf16*)qkv, ldqkv, (KVT*)kcache, (KVT*)vcache, pos, cos_t, sin_t,         \
                             (float*)workspace, Hq, Hkv, Tmax, splits, scale, table, max_blocks, bs_shift,   \
                             kscale, vscale));                                                               \
  } while (0)
  if (G == 1) MM_DA_LAUNCH(1);
  else if (G == 2) MM_DA_LAUNCH(2);
  else if (G == 4) MM_DA_LAUNCH(4);
  else MM_DA_LAUNCH(8);
#undef MM_DA_LAUNCH
  MM_CHECK_LAUNCH();
  MM_CHECK_CUDA(launch_pdl(decode_attn_combine_kernel, dim3(Hkv, B), dim3(128), 0, stream, (const float*)workspace,
                           (bf16*)out, ldo, Hkv, G, splits));
  MM_CHECK_LAUNCH();
  return MM_OK;
}

// log2 of a block size in [16, 256], or -1
int paged_block_shift(int block_size) {
  if (block_size < 16 || block_size > 256 || (block_size & (block_size - 1))) return -1;
  return __builtin_ctz((unsigned)block_size);
}

}  // namespace

MM_API int mm_decode_attn(const void* qkv, long long ldqkv, void* kcache, void* vcache, const int* pos,
                          const float* cos_t, const float* sin_t, void* out, long long ldo, int B,
                          int Hq, int Hkv, int head_dim, int Tmax, float scale, void* workspace,
                          long long workspace_bytes, int splits, cudaStream_t stream) {
  return decode_attn_launch<false>("mm_decode_attn", qkv, ldqkv, kcache, vcache, pos, cos_t, sin_t, out, ldo, B, Hq,
                                   Hkv, head_dim, Tmax, scale, workspace, workspace_bytes, splits, nullptr, 0, 0,
                                   stream);
}

MM_API int mm_decode_attn_paged(const void* qkv, long long ldqkv, void* kpool, void* vpool, const int* block_table,
                                int max_blocks, int block_size, const int* pos, const float* cos_t,
                                const float* sin_t, void* out, long long ldo, int B, int Hq, int Hkv, int head_dim,
                                float scale, void* workspace, long long workspace_bytes, int splits,
                                cudaStream_t stream) {
  const int shift = paged_block_shift(block_size);
  MM_CHECK_ARG(shift >= 0, "mm_decode_attn_paged: block_size must be a power of two in [16,256] (got %d)", block_size);
  MM_CHECK_ARG(max_blocks >= 1, "mm_decode_attn_paged: max_blocks must be >= 1 (got %d)", max_blocks);
  MM_CHECK_ARG(block_table != nullptr, "mm_decode_attn_paged: block table missing");
  MM_CHECK_ARG(Hkv >= 1, "mm_decode_attn_paged: need Hkv >= 1");
  MM_CHECK_ARG((long long)max_blocks * block_size <= (1 << 30), "mm_decode_attn_paged: max_blocks too large");
  return decode_attn_launch<true>("mm_decode_attn_paged", qkv, ldqkv, kpool, vpool, pos, cos_t, sin_t, out, ldo, B,
                                  Hq, Hkv, head_dim, max_blocks * block_size, scale, workspace, workspace_bytes,
                                  splits, block_table, max_blocks, shift, stream);
}

MM_API int mm_decode_attn_fp8(const void* qkv, long long ldqkv, void* kcache, void* vcache, float* kscale,
                              float* vscale, const int* pos, const float* cos_t, const float* sin_t, void* out,
                              long long ldo, int B, int Hq, int Hkv, int head_dim, int Tmax, float scale,
                              void* workspace, long long workspace_bytes, int splits, cudaStream_t stream) {
  return decode_attn_launch<false, true>("mm_decode_attn_fp8", qkv, ldqkv, kcache, vcache, pos, cos_t, sin_t, out, ldo,
                                         B, Hq, Hkv, head_dim, Tmax, scale, workspace, workspace_bytes, splits, nullptr,
                                         0, 0, stream, kscale, vscale);
}

MM_API int mm_decode_attn_paged_fp8(const void* qkv, long long ldqkv, void* kpool, void* vpool, float* kscale,
                                    float* vscale, const int* block_table, int max_blocks, int block_size,
                                    const int* pos, const float* cos_t, const float* sin_t, void* out, long long ldo,
                                    int B, int Hq, int Hkv, int head_dim, float scale, void* workspace,
                                    long long workspace_bytes, int splits, cudaStream_t stream) {
  const int shift = paged_block_shift(block_size);
  MM_CHECK_ARG(shift >= 0, "mm_decode_attn_paged_fp8: block_size must be a power of two in [16,256] (got %d)",
               block_size);
  MM_CHECK_ARG(max_blocks >= 1, "mm_decode_attn_paged_fp8: max_blocks must be >= 1 (got %d)", max_blocks);
  MM_CHECK_ARG(block_table != nullptr, "mm_decode_attn_paged_fp8: block table missing");
  MM_CHECK_ARG(Hkv >= 1, "mm_decode_attn_paged_fp8: need Hkv >= 1");
  MM_CHECK_ARG((long long)max_blocks * block_size <= (1 << 30), "mm_decode_attn_paged_fp8: max_blocks too large");
  return decode_attn_launch<true, true>("mm_decode_attn_paged_fp8", qkv, ldqkv, kpool, vpool, pos, cos_t, sin_t, out,
                                        ldo, B, Hq, Hkv, head_dim, max_blocks * block_size, scale, workspace,
                                        workspace_bytes, splits, block_table, max_blocks, shift, stream, kscale, vscale);
}

namespace {

int kv_quant_prefill_launch(const char* name, void* qkv, long long ld, void* kc, void* vc, float* ks, float* vs,
                            const int* trow, int B, int T, int Hq, int Hkv, int head_dim, int Tmax, int shift,
                            cudaStream_t stream) {
  MM_CHECK_ARG(ks != nullptr && vs != nullptr, "%s: scale arrays missing", name);
  MM_CHECK_ARG(head_dim == DA_D && Hkv >= 1 && B >= 1 && T >= 0, "%s: need head_dim 128, Hkv >= 1, B >= 1, T >= 0",
               name);
  MM_CHECK_ARG(ld % 4 == 0 && ((uintptr_t)qkv & 7) == 0, "%s: qkv rows must be 8-byte aligned", name);
  if (T == 0) return MM_OK;
  const long long total = (long long)B * T * Hkv * 2 * 32;
  long long blocks = ceil_div64(total, 256);
  if (blocks > (long long)mm_num_sms() * 16) blocks = (long long)mm_num_sms() * 16;
  if (trow)
    kv_quant_prefill_kernel<true><<<(int)blocks, 256, 0, stream>>>((bf16*)qkv, ld, (uint8_t*)kc, (uint8_t*)vc, ks, vs,
                                                                   trow, B, T, Hq, Hkv, Tmax, shift);
  else
    kv_quant_prefill_kernel<false><<<(int)blocks, 256, 0, stream>>>((bf16*)qkv, ld, (uint8_t*)kc, (uint8_t*)vc, ks, vs,
                                                                    nullptr, B, T, Hq, Hkv, Tmax, 0);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

}  // namespace

MM_API int mm_kv_quant_prefill(void* qkv, long long ld, void* kcache, void* vcache, float* kscale, float* vscale, int B,
                               int T, int Hq, int Hkv, int head_dim, int Tmax, cudaStream_t stream) {
  MM_CHECK_ARG(T <= Tmax, "mm_kv_quant_prefill: need T <= Tmax");
  return kv_quant_prefill_launch("mm_kv_quant_prefill", qkv, ld, kcache, vcache, kscale, vscale, nullptr, B, T, Hq, Hkv,
                                 head_dim, Tmax, 0, stream);
}

MM_API int mm_kv_quant_prefill_paged(void* qkv, long long ld, void* kpool, void* vpool, float* kscale, float* vscale,
                                     const int* block_table_row, int max_blocks, int block_size, int T, int Hq,
                                     int Hkv, int head_dim, cudaStream_t stream) {
  const int shift = paged_block_shift(block_size);
  MM_CHECK_ARG(shift >= 0, "mm_kv_quant_prefill_paged: block_size must be a power of two in [16,256] (got %d)",
               block_size);
  MM_CHECK_ARG(max_blocks >= 1, "mm_kv_quant_prefill_paged: max_blocks must be >= 1 (got %d)", max_blocks);
  MM_CHECK_ARG(block_table_row != nullptr, "mm_kv_quant_prefill_paged: block table missing");
  MM_CHECK_ARG((long long)T <= (long long)max_blocks * block_size, "mm_kv_quant_prefill_paged: need T <= max_blocks * block_size");
  return kv_quant_prefill_launch("mm_kv_quant_prefill_paged", qkv, ld, kpool, vpool, kscale, vscale, block_table_row, 1,
                                 T, Hq, Hkv, head_dim, 0, shift, stream);
}

MM_API int mm_kv_dequant_paged(const void* kpool, const void* vpool, const float* kscale, const float* vscale,
                               const int* block_table_row, int max_blocks, int block_size, int n_blocks, int Hkv,
                               int head_dim, void* kstage, void* vstage, cudaStream_t stream) {
  const int shift = paged_block_shift(block_size);
  MM_CHECK_ARG(shift >= 0, "mm_kv_dequant_paged: block_size must be a power of two in [16,256] (got %d)", block_size);
  MM_CHECK_ARG(block_table_row != nullptr, "mm_kv_dequant_paged: block table missing");
  MM_CHECK_ARG(kscale != nullptr && vscale != nullptr, "mm_kv_dequant_paged: scale arrays missing");
  MM_CHECK_ARG(head_dim == DA_D && Hkv >= 1 && n_blocks >= 0 && n_blocks <= max_blocks,
               "mm_kv_dequant_paged: need head_dim 128, Hkv >= 1 and 0 <= n_blocks <= max_blocks");
  if (n_blocks == 0) return MM_OK;
  const long long total = ((long long)n_blocks * Hkv * block_size) * (DA_D / 16) * 2;
  long long blocks = ceil_div64(total, 256);
  if (blocks > (long long)mm_num_sms() * 16) blocks = (long long)mm_num_sms() * 16;
  kv_dequant_paged_kernel<<<(int)blocks, 256, 0, stream>>>((const uint8_t*)kpool, (const uint8_t*)vpool, kscale,
                                                           vscale, block_table_row, n_blocks, Hkv, shift,
                                                           (bf16*)kstage, (bf16*)vstage);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_kv_prefill_paged(const void* qkv, long long ld, void* kpool, void* vpool, const int* block_table_row,
                               int max_blocks, int block_size, int T, int Hq, int Hkv, int head_dim,
                               cudaStream_t stream) {
  const int shift = paged_block_shift(block_size);
  MM_CHECK_ARG(shift >= 0, "mm_kv_prefill_paged: block_size must be a power of two in [16,256] (got %d)", block_size);
  MM_CHECK_ARG(max_blocks >= 1, "mm_kv_prefill_paged: max_blocks must be >= 1 (got %d)", max_blocks);
  MM_CHECK_ARG(block_table_row != nullptr, "mm_kv_prefill_paged: block table missing");
  MM_CHECK_ARG(head_dim == DA_D && Hkv >= 1 && T >= 0 && (long long)T <= (long long)max_blocks * block_size,
               "mm_kv_prefill_paged: need head_dim 128 and 0<=T<=max_blocks*block_size");
  if (T == 0) return MM_OK;
  const long long total = (long long)T * Hkv * (DA_D / 8);
  long long blocks = ceil_div64(total, 256);
  if (blocks > (long long)mm_num_sms() * 16) blocks = (long long)mm_num_sms() * 16;
  kv_prefill_paged_kernel<<<(int)blocks, 256, 0, stream>>>((const bf16*)qkv, ld, (bf16*)kpool, (bf16*)vpool,
                                                           block_table_row, T, Hq, Hkv, shift);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_kv_prefill(const void* qkv, long long ld, void* kcache, void* vcache, int B, int T, int Hq,
                         int Hkv, int head_dim, int Tmax, cudaStream_t stream) {
  MM_CHECK_ARG(head_dim == DA_D && T <= Tmax, "mm_kv_prefill: need head_dim 128 and T<=Tmax");
  const long long total = (long long)B * T * Hkv * (DA_D / 8);
  long long blocks = ceil_div64(total, 256);
  if (blocks > (long long)mm_num_sms() * 16) blocks = (long long)mm_num_sms() * 16;
  kv_prefill_kernel<<<(int)blocks, 256, 0, stream>>>((const bf16*)qkv, ld, (bf16*)kcache, (bf16*)vcache, B,
                                                     T, Hq, Hkv, Tmax);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_decode_state_step(int* in_image_mode, int* total_image_tokens, int* total_output,
                                int* finished, int* pos, int* n_ids, int* n_img, int* ids_out,
                                int* append_kind, int* next_token, const int* argmax_tok,
                                const int* forced, int forced_ld, int step, int B, int num_image_tokens,
                                int max_new_tokens, int max_ids, int start_id, int end_id, int eos0,
                                int eos1, const void* pred_z, void* img_out, int max_img, int C,
                                cudaStream_t stream) {
  DecodeState st{in_image_mode, total_image_tokens, total_output, finished, pos,
                 n_ids, n_img, ids_out, append_kind, next_token};
  decode_state_kernel<<<B, 128, 0, stream>>>(st, argmax_tok, forced, forced_ld, step, B, num_image_tokens,
                                             max_new_tokens, max_ids, start_id, end_id, eos0, eos1,
                                             (const bf16*)pred_z, (bf16*)img_out, max_img, C, nullptr);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

// Same state machine with a per-slot output limit (max_new_slot[b], device) — continuous batching (SURVEY 8f N4):
// every slot of the batch serves a different request.
MM_API int mm_decode_state_step_slots(int* in_image_mode, int* total_image_tokens, int* total_output,
                                      int* finished, int* pos, int* n_ids, int* n_img, int* ids_out,
                                      int* append_kind, int* next_token, const int* argmax_tok,
                                      const int* forced, int forced_ld, const int* max_new_slot, int B,
                                      int num_image_tokens, int max_ids, int start_id, int end_id, int eos0,
                                      int eos1, const void* pred_z, void* img_out, int max_img, int C,
                                      cudaStream_t stream) {
  MM_CHECK_ARG(max_new_slot != nullptr, "mm_decode_state_step_slots: per-slot limits missing");
  DecodeState st{in_image_mode, total_image_tokens, total_output, finished, pos,
                 n_ids, n_img, ids_out, append_kind, next_token};
  decode_state_kernel<<<B, 128, 0, stream>>>(st, argmax_tok, forced, forced_ld, 0, B, num_image_tokens, 0, max_ids,
                                             start_id, end_id, eos0, eos1, (const bf16*)pred_z, (bf16*)img_out,
                                             max_img, C, max_new_slot);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_decode_next_input(const int* kind, const int* tok, const void* embed, const void* pred,
                                void* x, int B, int H, cudaStream_t stream) {
  MM_CHECK_ARG(H % 8 == 0, "mm_decode_next_input: H%%8");
  decode_next_input_kernel<<<B, 128, 0, stream>>>(kind, tok, (const bf16*)embed, (const bf16*)pred,
                                                  (bf16*)x, H);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_decode_select_hidden(const int* mode, const void* hidden, const void* pred, void* out,
                                   int B, int H, cudaStream_t stream) {
  MM_CHECK_ARG(H % 8 == 0, "mm_decode_select_hidden: H%%8");
  decode_select_hidden_kernel<<<B, 128, 0, stream>>>(mode, (const bf16*)hidden, (const bf16*)pred,
                                                     (bf16*)out, H);
  MM_CHECK_LAUNCH();
  return MM_OK;
}
