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
#include <mutex>
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

template <int ROWS, int NST = SK2_STAGES, int NB = 1>
__global__ void __launch_bounds__(SK2_THREADS)
skinny_gemm_tma_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                       void* __restrict__ y, long long ldy, const bf16* __restrict__ bias,
                       const bf16* __restrict__ resid, long long ldr, int m, int N, int K, int epi, int out_f32,
                       int pdl) {
  constexpr int G = ROWS >= 16 ? ROWS / 16 : 1;
  constexpr bool HALF = ROWS == 8;             // 8-row slab: rows 8..15 of the MMA operand are zero
  constexpr int MB = 8 * NB;                   // batch rows served: NB n8 tiles of the MMA's B operand
  constexpr int BOX = ROWS * 128;              // bytes of one [ROWS x 64 k] weight box
  constexpr int XBOX = MB * 128;               // bytes of one [MB batch rows x 64 k] activation box
  constexpr int STAGE_W = 4 * BOX;             // 4 boxes = 256 k of the weight slab
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
  if (!(pdl & 8)) griddep_launch();
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
        for (int bx = 0; bx < 4; ++bx)
          tma_load_2d(base + kt * STAGE + bx * BOX, &tmap_w, bar + 8 * kt, kt * SK2_KT + bx * 64, n0);
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
        for (int bx = 0; bx < 4; ++bx)
          tma_load_2d(base + s * STAGE + bx * BOX, &tmap_w, bar + 8 * s, kt * SK2_KT + bx * 64, n0);
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
      mbar_wait(bar + 8 * s, ph);
      const uint8_t* st = base_ptr + s * STAGE;
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int cc = 2 * cw + u;             // k32 chunk of this stage: box cc/2, half cc%2
        const uint8_t* bx = st + (cc >> 1) * BOX;
        const int chunk = (cc & 1) * 4 + t;    // 16-byte chunk index inside the 128-byte row
        // B fragments: batch rows g + 8 nb, the same 8 k values (128-byte swizzled [MB x 64] box; the swizzle repeats
        // every 8 rows, so row g + 8 nb uses the same chunk permutation as row g)
        int4 xb[NB];
#pragma unroll
        for (int nb = 0; nb < NB; ++nb)
          xb[nb] = *reinterpret_cast<const int4*>(st + STAGE_W + (cc >> 1) * XBOX + (nb * 8 + g) * 128 + ((chunk ^ g) << 4));
#pragma unroll
        for (int i = 0; i < G; ++i) {
          const int r0 = i * 16 + g, r1 = r0 + 8;
          const int4 w0 = *reinterpret_cast<const int4*>(bx + r0 * 128 + ((chunk ^ (r0 & 7)) << 4));
          const int4 w1 = HALF ? make_int4(0, 0, 0, 0)
                               : *reinterpret_cast<const int4*>(bx + r1 * 128 + ((chunk ^ (r1 & 7)) << 4));
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
  if (pdl & 8) griddep_launch();
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
constexpr int DA_THREADS = 256;
constexpr int DA_D = 128;

template <int G, bool PAGED>
__global__ void __launch_bounds__(DA_THREADS)
decode_attn_kernel(const bf16* __restrict__ qkv, long long ldqkv, bf16* __restrict__ kc,
                   bf16* __restrict__ vc, const int* __restrict__ pos_arr,
                   const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                   float* __restrict__ part, int Hq, int Hkv, int Tmax, int S, float scale,
                   const int* __restrict__ table, int max_blocks, int bs_shift) {
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
  bf16* kcb = kc + (PAGED ? 0ll : ((long long)b * Hkv + hk) * Tmax * DA_D);
  bf16* vcb = vc + (PAGED ? 0ll : ((long long)b * Hkv + hk) * Tmax * DA_D);
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
  if (owns_new && tid < DA_D / 2) {
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

template <int ROWS, int NST, int NB>
int launch_skinny_tma(const CUtensorMap& tw, const CUtensorMap& tx, void* y, long long ldy, const void* bias,
                      const void* resid, long long ldr, int m, int N, int K, int epilogue, int out_f32, int pm,
                      cudaStream_t stream) {
  constexpr int smem = NST * (4 * ROWS * 128 + 4 * 8 * NB * 128) + ((2 * NST * 8 + 127) & ~127) + 4 * ROWS * 8 * NB * 4 + 1024;
  static_assert(smem <= 227 * 1024, "skinny GEMM ring does not fit in shared memory");
  static std::once_flag once;
  static cudaError_t err = cudaSuccess;
  std::call_once(once, [&] {
    err = cudaFuncSetAttribute(skinny_gemm_tma_kernel<ROWS, NST, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  });
  MM_CHECK_CUDA(err);
  MM_CHECK_CUDA(launch_pdl(pm & 1, skinny_gemm_tma_kernel<ROWS, NST, NB>, dim3((N + ROWS - 1) / ROWS), dim3(SK2_THREADS),
                           smem, stream, tw, tx, y, ldy, (const bf16*)bias, (const bf16*)resid, ldr, m, N, K, epilogue,
                           out_f32, pm));
  MM_CHECK_LAUNCH();
  return MM_OK;
}

}  // namespace

MM_API int mm_skinny_gemm(const void* x, const void* W, void* y, const void* bias, const void* resid,
                          long long ldx, long long ldw, long long ldy, long long ldr, int m, int N,
                          int K, int epilogue, int out_f32, cudaStream_t stream) {
  MM_CHECK_ARG(m >= 1 && m <= 32, "mm_skinny_gemm: batch must be in [1,32] (m=%d)", m);
  MM_CHECK_ARG(K % 32 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "mm_skinny_gemm: need K%%32==0, ldx/ldw%%8==0");
  MM_CHECK_ARG(((uintptr_t)W & 15) == 0 && ((uintptr_t)x & 15) == 0, "mm_skinny_gemm: x / W must be 16-byte aligned");
  MM_CHECK_ARG(epilogue >= SK_STORE && epilogue <= SK_SWIGLU, "mm_skinny_gemm: bad epilogue");
  MM_CHECK_ARG((epilogue != SK_BIAS && epilogue != SK_BIAS_GELU) || bias, "mm_skinny_gemm: bias missing");
  MM_CHECK_ARG(epilogue != SK_RESID || resid, "mm_skinny_gemm: residual missing");
  const int pm = mm_pdl_mode();
  // The batch is the n dimension of the MMA: 1, 2 or 4 n8 tiles (8 / 16 / 32 sequences) share every weight fragment.
  const int nb = m <= 8 ? 1 : (m <= 16 ? 2 : 4);
  // 32-row slabs where the epilogue needs them (SwiGLU: 16 gate + 16 up rows of the same channels), for very large N
  // (lm_head: fewer, longer-lived CTAs) and for 32 sequences (each CTA re-reads the whole activation block from L2: the
  // taller slab halves that traffic); 16-row slabs otherwise
  const bool rows32 = (epilogue == SK_SWIGLU) || (N >= 32 * 4 * mm_num_sms()) || nb == 4;
  // 32 sequences, wide outputs (gate/up, lm_head): 64-row slabs halve the L2 -> SM activation traffic again, which at this
  // batch equals the weight stream and caps the kernel (measured 4.1 TB/s of weights + as much of x with 32-row slabs)
  const bool rows64 = nb == 4 && N >= 64 * 2 * mm_num_sms() && (epilogue != SK_SWIGLU || N % 64 == 0);
  if (epilogue == SK_SWIGLU) MM_CHECK_ARG(N % 32 == 0 && !out_f32, "mm_skinny_gemm: SWIGLU needs N%%32==0");
  static PFN_encodeTiledSk enc = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      enc = reinterpret_cast<PFN_encodeTiledSk>(fn);
  });
  MM_CHECK_ARG(enc != nullptr, "mm_skinny_gemm: cuTensorMapEncodeTiled unavailable");
  CUtensorMap tw, tx;
  cuuint32_t estr[2] = {1, 1};
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
    cuuint64_t strides[1] = {(cuuint64_t)ldw * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)(rows64 ? 64 : (rows32 ? 32 : 16))};
    CUresult r = enc(&tw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(W), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MM_CHECK_ARG(r == CUDA_SUCCESS, "mm_skinny_gemm: cuTensorMapEncodeTiled(W) failed (%d)", (int)r);
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)m};            // rows >= m of the box are zero-filled
    cuuint64_t strides[1] = {(cuuint64_t)ldx * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)(8 * nb)};
    CUresult r = enc(&tx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(x), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MM_CHECK_ARG(r == CUDA_SUCCESS, "mm_skinny_gemm: cuTensorMapEncodeTiled(x) failed (%d)", (int)r);
  }
  // Ring depths: as deep as keeps two CTAs per SM (profiles/r02_decode_skinny_ring_sweep.txt: deeper rings bought nothing);
  // 32 sequences: 32 KB (32-row slabs) or 48 KB (64-row slabs) stages, one CTA per SM.
#define MM_SK(R, S, B) return launch_skinny_tma<R, S, B>(tw, tx, y, ldy, bias, resid, ldr, m, N, K, epilogue, out_f32, pm, stream)
  if (rows64) MM_SK(64, 4, 4);
  if (nb == 4) MM_SK(32, 5, 4);
  if (nb == 2) {
    if (rows32) MM_SK(32, 4, 2);
    MM_SK(16, 6, 2);
  }
  if (rows32) MM_SK(32, 5, 1);
  MM_SK(16, 8, 1);
#undef MM_SK
}

MM_API long long mm_decode_attn_workspace_bytes(int B, int Hq, int Hkv, int splits) {
  return (long long)B * Hkv * splits * (Hq / Hkv) * (2 + DA_D) * 4;
}

namespace {

// shared by the dense and the paged entry points; `name` prefixes the error messages. Dense: table == nullptr.
template <bool PAGED>
int decode_attn_launch(const char* name, const void* qkv, long long ldqkv, void* kcache, void* vcache, const int* pos,
                       const float* cos_t, const float* sin_t, void* out, long long ldo, int B, int Hq, int Hkv,
                       int head_dim, int Tmax, float scale, void* workspace, long long workspace_bytes, int splits,
                       const int* table, int max_blocks, int bs_shift, cudaStream_t stream) {
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
      MM_CHECK_CUDA(cudaFuncSetAttribute(decode_attn_kernel<GG, PAGED>,                                      \
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));           \
    MM_CHECK_CUDA(launch_pdl(mm_pdl_mode() & 2, decode_attn_kernel<GG, PAGED>, grid, dim3(DA_THREADS), smem, stream, \
                             (const bf16*)qkv, ldqkv, (bf16*)kcache, (bf16*)vcache, pos, cos_t, sin_t,       \
                             (float*)workspace, Hq, Hkv, Tmax, splits, scale, table, max_blocks, bs_shift));  \
  } while (0)
  if (G == 1) MM_DA_LAUNCH(1);
  else if (G == 2) MM_DA_LAUNCH(2);
  else if (G == 4) MM_DA_LAUNCH(4);
  else MM_DA_LAUNCH(8);
#undef MM_DA_LAUNCH
  MM_CHECK_LAUNCH();
  MM_CHECK_CUDA(launch_pdl(mm_pdl_mode() & 2, decode_attn_combine_kernel, dim3(Hkv, B), dim3(128), 0, stream, (const float*)workspace,
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
