// metamorph_b200 — fused attention (SURVEY.md K12: LLaMA causal GQA d=128 fwd+bwd; K4: SigLIP
// non-causal MHA d=72 fwd).  Flash-style: scores never leave the SM, softmax statistics in fp32
// registers (exp2 domain, warp-shuffle row reductions), O(T) memory.
//
// Round-1 implementation uses the legacy warp-level tensor path (ldmatrix + mma.sync m16n8k16,
// SASS HMMA) with cp.async double-buffered K/V tiles; the product path runs the wgmma kernels of
// attention_tc.cu / attention_bwd_tc.cu; these stay as the tests' comparison kernels.  The backward accumulates dQ with the TMA
// engine's bulk reduce-add (cp.reduce.async.bulk ... .add.f32, smem -> global fp32) instead of
// per-lane atomics, and keeps dK/dV in registers across the query heads of a GQA group.
//
// Layouts: Q/K/V are addressed as [token_row, head*dh + c] with independent row pitches, so the
// fused QKV GEMM output [B*T, (Hq+2Hkv)*dh] is consumed in place (no head transpose copies).
#include "common.cuh"
#include <mutex>

namespace {

constexpr float kLog2e = 1.4426950408889634f;

template <int LDS>
__device__ __forceinline__ uint32_t addr_A(uint32_t base, int row0, int col0, int lane) {
  return base + (uint32_t)(((row0 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + col0 + (lane >> 4) * 8) * 2);
}
template <int LDS>
__device__ __forceinline__ uint32_t addr_Bn(uint32_t base, int n0, int k0, int lane) {
  return base + (uint32_t)(((n0 + (lane & 7) + (lane >> 4) * 8) * LDS + k0 + ((lane >> 3) & 1) * 8) * 2);
}
template <int LDS>
__device__ __forceinline__ uint32_t addr_Bt(uint32_t base, int k0, int n0, int lane) {
  return base + (uint32_t)(((k0 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + n0 + (lane >> 4) * 8) * 2);
}
template <int LDS>
__device__ __forceinline__ uint32_t addr_At(uint32_t base, int k0, int m0, int lane) {
  return base + (uint32_t)(((k0 + (lane & 7) + (lane >> 4) * 8) * LDS + m0 + ((lane >> 3) & 1) * 8) * 2);
}

// Load `rows` x (dh/8) 16-byte chunks of a [*, ld] global matrix into a padded smem tile.
// Rows >= row_limit are zero-filled. All threads of the CTA participate.
template <int LDS>
__device__ __forceinline__ void load_tile_async(uint32_t smem_tile, const bf16* g, long long ld,
                                                int row0, int rows, int row_limit, int dh,
                                                int nthreads) {
  const int cpr = dh >> 3;
  for (int i = threadIdx.x; i < rows * cpr; i += nthreads) {
    const int r = i / cpr, c = i - r * cpr;
    const int gr = row0 + r;
    const bool ok = gr < row_limit;
    const bf16* src = g + (long long)(ok ? gr : (row_limit > 0 ? row_limit - 1 : 0)) * ld + c * 8;
    cp_async16(smem_tile + (uint32_t)((r * LDS + c * 8) * 2), src, ok);
  }
}

// ================================================================================== forward
constexpr int FWD_BR = 128, FWD_BC = 64, FWD_THREADS = 256;

struct FwdParams {
  const bf16 *q, *k, *v;
  bf16* o;
  float* lse;  // [B, Hq, T] natural-log LSE of the scaled scores (may be null)
  const int* seqlens;  // [B] valid length (right padding); null => T
  long long ldq, ldk, ldv, ldo;
  int B, T, Hq, Hkv, dh;
  float scale;
};

template <int D, bool CAUSAL>
__global__ void __launch_bounds__(FWD_THREADS)
flash_fwd_kernel(FwdParams p) {
  constexpr int LDS = D + 8;
  extern __shared__ __align__(16) uint8_t smem[];
  bf16* sQ = reinterpret_cast<bf16*>(smem);
  bf16* sK = sQ + FWD_BR * LDS;
  bf16* sV = sK + 2 * FWD_BC * LDS;
  const uint32_t uQ = smem_u32(sQ), uK = smem_u32(sK), uV = smem_u32(sV);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int hk = h / (p.Hq / p.Hkv);
  const int q0 = qt * FWD_BR;
  const int kv_len = p.seqlens ? p.seqlens[b] : p.T;
  const long long tok0 = (long long)b * p.T;
  const bf16* gq = p.q + tok0 * p.ldq + (long long)h * p.dh;
  const bf16* gk = p.k + tok0 * p.ldk + (long long)hk * p.dh;
  const bf16* gv = p.v + tok0 * p.ldv + (long long)hk * p.dh;

  int kv_end = kv_len;
  if (CAUSAL) kv_end = min(kv_end, q0 + FWD_BR);
  const int n_tiles = (kv_end + FWD_BC - 1) / FWD_BC;

  // zero the padding columns [dh, D+8) of every tile once (cp.async never touches them)
  if (p.dh < LDS) {
    const int padc = LDS - p.dh;
    const int total_rows = FWD_BR + 4 * FWD_BC;
    for (int i = threadIdx.x; i < total_rows * padc; i += FWD_THREADS) {
      const int r = i / padc, c = p.dh + (i - r * padc);
      sQ[r * LDS + c] = __float2bfloat16(0.f);
    }
  }
  __syncthreads();

  load_tile_async<LDS>(uQ, gq, p.ldq, q0, FWD_BR, p.T, p.dh, FWD_THREADS);
  if (n_tiles > 0) {
    load_tile_async<LDS>(uK, gk, p.ldk, 0, FWD_BC, kv_len, p.dh, FWD_THREADS);
    load_tile_async<LDS>(uV, gv, p.ldv, 0, FWD_BC, kv_len, p.dh, FWD_THREADS);
  }
  cp_async_commit();

  float o_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o_acc[i][j] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  uint32_t qf[D / 16][4];
  const float sl2 = p.scale * kLog2e;
  const int r_lo = q0 + warp * 16 + (lane >> 2);  // global q row of c0,c1 ; +8 for c2,c3

  for (int j = 0; j < n_tiles; ++j) {
    const int buf = j & 1;
    if (j + 1 < n_tiles) {
      const uint32_t nK = uK + (uint32_t)((buf ^ 1) * FWD_BC * LDS * 2);
      const uint32_t nV = uV + (uint32_t)((buf ^ 1) * FWD_BC * LDS * 2);
      load_tile_async<LDS>(nK, gk, p.ldk, (j + 1) * FWD_BC, FWD_BC, kv_len, p.dh, FWD_THREADS);
      load_tile_async<LDS>(nV, gv, p.ldv, (j + 1) * FWD_BC, FWD_BC, kv_len, p.dh, FWD_THREADS);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (j == 0) {
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk)
        ldsm_x4(addr_A<LDS>(uQ, warp * 16, kk * 16, lane), qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);
    }
    const uint32_t cK = uK + (uint32_t)(buf * FWD_BC * LDS * 2);
    const uint32_t cV = uV + (uint32_t)(buf * FWD_BC * LDS * 2);

    float s[FWD_BC / 8][4];
#pragma unroll
    for (int i = 0; i < FWD_BC / 8; ++i)
#pragma unroll
      for (int t = 0; t < 4; ++t) s[i][t] = 0.f;
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
      for (int np = 0; np < FWD_BC / 16; ++np) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4(addr_Bn<LDS>(cK, np * 16, kk * 16, lane), b0, b1, b2, b3);
        mma_bf16_16816(s[2 * np], qf[kk], b0, b1);
        mma_bf16_16816(s[2 * np + 1], qf[kk], b2, b3);
      }
    }
    // mask + online softmax (exp2 domain)
    const int kv0 = j * FWD_BC;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < FWD_BC / 8; ++i) {
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int col = kv0 + i * 8 + (lane & 3) * 2 + (t & 1);
        const int row = r_lo + (t >> 1) * 8;
        const bool ok = (col < kv_len) && (!CAUSAL || col <= row);
        const float val = ok ? s[i][t] * sl2 : -INFINITY;
        s[i][t] = val;
        mx[t >> 1] = fmaxf(mx[t >> 1], val);
      }
    }
    float corr[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      m_use[r] = (m_new == -INFINITY) ? 0.f : m_new;
      corr[r] = exp2f(m_run[r] - m_use[r]);  // m_run=-inf -> 0
      m_run[r] = m_new;
      l_run[r] *= corr[r];
    }
    uint32_t pf[FWD_BC / 16][4];
#pragma unroll
    for (int i = 0; i < FWD_BC / 8; ++i) {
      const float p0 = exp2f(s[i][0] - m_use[0]), p1 = exp2f(s[i][1] - m_use[0]);
      const float p2 = exp2f(s[i][2] - m_use[1]), p3 = exp2f(s[i][3] - m_use[1]);
      l_run[0] += p0 + p1;
      l_run[1] += p2 + p3;
      pf[i >> 1][(i & 1) * 2] = pack_bf16x2(p0, p1);
      pf[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      o_acc[i][0] *= corr[0];
      o_acc[i][1] *= corr[0];
      o_acc[i][2] *= corr[1];
      o_acc[i][3] *= corr[1];
    }
#pragma unroll
    for (int kk = 0; kk < FWD_BC / 16; ++kk) {
#pragma unroll
      for (int np = 0; np < D / 16; ++np) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(addr_Bt<LDS>(cV, kk * 16, np * 16, lane), b0, b1, b2, b3);
        mma_bf16_16816(o_acc[2 * np], pf[kk], b0, b1);
        mma_bf16_16816(o_acc[2 * np + 1], pf[kk], b2, b3);
      }
    }
    __syncthreads();  // everyone done with buf before iteration j+1 refills it (as buffer j+2)
  }
  if (n_tiles == 0) {
    cp_async_wait<0>();
    __syncthreads();
  }

  // finalize: O /= l, LSE, stage O through this warp's rows of sQ for coalesced stores
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const float inv0 = l_run[0] > 0.f ? 1.f / l_run[0] : 0.f;
  const float inv1 = l_run[1] > 0.f ? 1.f / l_run[1] : 0.f;
  if (p.lse != nullptr && (lane & 3) == 0) {
    float* lp = p.lse + ((long long)b * p.Hq + h) * p.T;
    if (r_lo < p.T)
      lp[r_lo] = l_run[0] > 0.f ? (m_run[0] + log2f(l_run[0])) / kLog2e : -INFINITY;
    if (r_lo + 8 < p.T)
      lp[r_lo + 8] = l_run[1] > 0.f ? (m_run[1] + log2f(l_run[1])) / kLog2e : -INFINITY;
  }
  __syncwarp();
  {
    bf16* wq = sQ + (warp * 16) * LDS;
    const int rr = lane >> 2, cc = (lane & 3) * 2;
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      *reinterpret_cast<uint32_t*>(wq + rr * LDS + i * 8 + cc) =
          pack_bf16x2(o_acc[i][0] * inv0, o_acc[i][1] * inv0);
      *reinterpret_cast<uint32_t*>(wq + (rr + 8) * LDS + i * 8 + cc) =
          pack_bf16x2(o_acc[i][2] * inv1, o_acc[i][3] * inv1);
    }
    __syncwarp();
    const int cpr = p.dh >> 3;
    bf16* go = p.o + tok0 * p.ldo + (long long)h * p.dh;
    for (int i = lane; i < 16 * cpr; i += 32) {
      const int r = i / cpr, c = i - r * cpr;
      const int grow = q0 + warp * 16 + r;
      if (grow < p.T)
        *reinterpret_cast<int4*>(go + (long long)grow * p.ldo + c * 8) =
            *reinterpret_cast<const int4*>(wq + r * LDS + c * 8);
    }
  }
}

// ================================================================================== backward
// delta[b,h,t] = sum_c dO[t,h,c] * O[t,h,c]; one warp per (token,head)
__global__ void attn_delta_kernel(const bf16* __restrict__ o, const bf16* __restrict__ dout,
                                  float* __restrict__ delta, long long ldo, long long lddo, int B,
                                  int T, int Hq, int dh) {
  const int warps_per_block = blockDim.x >> 5, lane = threadIdx.x & 31;
  const long long total = (long long)B * T * Hq;
  for (long long w = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); w < total;
       w += (long long)gridDim.x * warps_per_block) {
    const int h = (int)(w % Hq);
    const long long tok = w / Hq;
    const bf16* po = o + tok * ldo + (long long)h * dh;
    const bf16* pd = dout + tok * lddo + (long long)h * dh;
    float s = 0.f;
    for (int c = lane * 8; c < dh; c += 256) {
      const int4 a = *reinterpret_cast<const int4*>(po + c);
      const int4 g = *reinterpret_cast<const int4*>(pd + c);
      const uint32_t ua[4] = {(uint32_t)a.x, (uint32_t)a.y, (uint32_t)a.z, (uint32_t)a.w};
      const uint32_t ug[4] = {(uint32_t)g.x, (uint32_t)g.y, (uint32_t)g.z, (uint32_t)g.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 x = unpack_bf16x2(ua[j]);
        const float2 y = unpack_bf16x2(ug[j]);
        s += x.x * y.x + x.y * y.y;
      }
    }
    s = warp_sum(s);
    if (lane == 0) {
      const int b = (int)(tok / T), t = (int)(tok % T);
      delta[((long long)b * Hq + h) * T + t] = s;
    }
  }
}

constexpr int BWD_BQ = 64, BWD_BC = 64, BWD_THREADS = 256, BWD_D = 128;
constexpr int BWD_LDS = BWD_D + 8;   // bf16 elements
constexpr int BWD_LDP = BWD_BC + 8;  // bf16 elements (P / dS tiles)

struct BwdParams {
  const bf16 *q, *k, *v, *dout;
  const float *lse, *delta;  // [B,Hq,T]
  float* dq_accum;           // [B*T, Hq*128] fp32, zero-initialised
  bf16 *dk, *dv;             // written in place of the K/V layout (row pitch lddk/lddv)
  const int* seqlens;
  long long ldq, ldk, ldv, lddo, lddk, lddv;
  int B, T, Hq, Hkv;
  float scale;
};

constexpr int BWD_SMEM = (2 * BWD_BC * BWD_LDS + 4 * BWD_BQ * BWD_LDS + 2 * BWD_BQ * BWD_LDP) * 2 +
                         2 * BWD_BQ * BWD_D * 4 + 4 * BWD_BQ * 4;

__global__ void __launch_bounds__(BWD_THREADS, 1)
flash_bwd_kernel(BwdParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  bf16* sK = reinterpret_cast<bf16*>(smem);
  bf16* sV = sK + BWD_BC * BWD_LDS;
  bf16* sQ = sV + BWD_BC * BWD_LDS;        // [2][BQ][LDS]
  bf16* sdO = sQ + 2 * BWD_BQ * BWD_LDS;   // [2][BQ][LDS]
  bf16* sP = sdO + 2 * BWD_BQ * BWD_LDS;   // [BQ][LDP]
  bf16* sdS = sP + BWD_BQ * BWD_LDP;       // [BQ][LDP]
  float* sdQ = reinterpret_cast<float*>(sdS + BWD_BQ * BWD_LDP);  // [2][BQ][128] fp32 staging
  float* sLse = sdQ + 2 * BWD_BQ * BWD_D;                         // [2][BQ]
  float* sDelta = sLse + 2 * BWD_BQ;                              // [2][BQ]
  const uint32_t uK = smem_u32(sK), uV = smem_u32(sV), uQ = smem_u32(sQ), udO = smem_u32(sdO),
                 uP = smem_u32(sP), udS = smem_u32(sdS);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = warp & 3, wn = warp >> 2;
  const int jt = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int G = p.Hq / p.Hkv;
  const int kv0 = jt * BWD_BC;
  const int kv_len = p.seqlens ? p.seqlens[b] : p.T;
  const long long tok0 = (long long)b * p.T;
  const float sl2 = p.scale * kLog2e;

  // zero padding columns of the bf16 tiles
  {
    const int total_rows = 2 * BWD_BC + 4 * BWD_BQ;
    for (int i = threadIdx.x; i < total_rows * 8; i += BWD_THREADS)
      sK[(i >> 3) * BWD_LDS + BWD_D + (i & 7)] = __float2bfloat16(0.f);
  }
  const bf16* gk = p.k + tok0 * p.ldk + (long long)hk * BWD_D;
  const bf16* gv = p.v + tok0 * p.ldv + (long long)hk * BWD_D;
  load_tile_async<BWD_LDS>(uK, gk, p.ldk, kv0, BWD_BC, kv_len, BWD_D, BWD_THREADS);
  load_tile_async<BWD_LDS>(uV, gv, p.ldv, kv0, BWD_BC, kv_len, BWD_D, BWD_THREADS);

  const int qt_begin = kv0 / BWD_BQ;  // causal: query tiles at or after this KV tile
  const int qt_end = (p.T + BWD_BQ - 1) / BWD_BQ;
  const int n_qt = qt_end - qt_begin;
  const int n_it = n_qt * G;

  auto issue_loads = [&](int it) {
    const int hq = hk * G + it / n_qt;
    const int q0 = (qt_begin + it % n_qt) * BWD_BQ;
    const int buf = it & 1;
    const bf16* gq = p.q + tok0 * p.ldq + (long long)hq * BWD_D;
    const bf16* gdo = p.dout + tok0 * p.lddo + (long long)hq * BWD_D;
    load_tile_async<BWD_LDS>(uQ + (uint32_t)(buf * BWD_BQ * BWD_LDS * 2), gq, p.ldq, q0, BWD_BQ, p.T,
                             BWD_D, BWD_THREADS);
    load_tile_async<BWD_LDS>(udO + (uint32_t)(buf * BWD_BQ * BWD_LDS * 2), gdo, p.lddo, q0, BWD_BQ,
                             p.T, BWD_D, BWD_THREADS);
    if (threadIdx.x < BWD_BQ) {
      const int r = q0 + threadIdx.x;
      const long long off = ((long long)b * p.Hq + hq) * p.T + (r < p.T ? r : 0);
      sLse[buf * BWD_BQ + threadIdx.x] = (r < p.T) ? p.lse[off] : INFINITY;
      sDelta[buf * BWD_BQ + threadIdx.x] = (r < p.T) ? p.delta[off] : 0.f;
    }
  };

  float dk_acc[8][4], dv_acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int t = 0; t < 4; ++t) dk_acc[i][t] = dv_acc[i][t] = 0.f;

  if (n_it > 0) issue_loads(0);
  cp_async_commit();

  for (int it = 0; it < n_it; ++it) {
    const int buf = it & 1;
    const int hq = hk * G + it / n_qt;
    const int q0 = (qt_begin + it % n_qt) * BWD_BQ;
    cp_async_wait<0>();
    if (threadIdx.x < BWD_BQ)  // staging buffer `buf` was last read by the bulk reduce of it-2
      asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
    __syncthreads();  // (A)
    if (it + 1 < n_it) issue_loads(it + 1);
    cp_async_commit();

    const uint32_t cQ = uQ + (uint32_t)(buf * BWD_BQ * BWD_LDS * 2);
    const uint32_t cdO = udO + (uint32_t)(buf * BWD_BQ * BWD_LDS * 2);

    // ---- S = Q K^T, dP = dO V^T   (warp: 16 q rows x 32 kv cols)
    float s[4][4], dp[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int t = 0; t < 4; ++t) s[i][t] = dp[i][t] = 0.f;
#pragma unroll
    for (int kk = 0; kk < BWD_D / 16; ++kk) {
      uint32_t aq[4], ado[4];
      ldsm_x4(addr_A<BWD_LDS>(cQ, wm * 16, kk * 16, lane), aq[0], aq[1], aq[2], aq[3]);
      ldsm_x4(addr_A<BWD_LDS>(cdO, wm * 16, kk * 16, lane), ado[0], ado[1], ado[2], ado[3]);
#pragma unroll
      for (int np = 0; np < 2; ++np) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4(addr_Bn<BWD_LDS>(uK, wn * 32 + np * 16, kk * 16, lane), b0, b1, b2, b3);
        mma_bf16_16816(s[2 * np], aq, b0, b1);
        mma_bf16_16816(s[2 * np + 1], aq, b2, b3);
        ldsm_x4(addr_Bn<BWD_LDS>(uV, wn * 32 + np * 16, kk * 16, lane), b0, b1, b2, b3);
        mma_bf16_16816(dp[2 * np], ado, b0, b1);
        mma_bf16_16816(dp[2 * np + 1], ado, b2, b3);
      }
    }
    // ---- P = exp(S*scale - lse), dS = P * (dP - delta)  -> smem (bf16)
    {
      const int rl = wm * 16 + (lane >> 2);
      const float lse0 = sLse[buf * BWD_BQ + rl] * kLog2e, lse1 = sLse[buf * BWD_BQ + rl + 8] * kLog2e;
      const float dl0 = sDelta[buf * BWD_BQ + rl], dl1 = sDelta[buf * BWD_BQ + rl + 8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float pv[4], dsv[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int col = kv0 + wn * 32 + i * 8 + (lane & 3) * 2 + (t & 1);
          const int row = q0 + rl + (t >> 1) * 8;
          const bool ok = (col < kv_len) && (col <= row) && (row < p.T);
          const float e = ok ? exp2f(s[i][t] * sl2 - ((t >> 1) ? lse1 : lse0)) : 0.f;
          pv[t] = e;
          dsv[t] = e * (dp[i][t] - ((t >> 1) ? dl1 : dl0));
        }
        const int cc = wn * 32 + i * 8 + (lane & 3) * 2;
        *reinterpret_cast<uint32_t*>(sP + rl * BWD_LDP + cc) = pack_bf16x2(pv[0], pv[1]);
        *reinterpret_cast<uint32_t*>(sP + (rl + 8) * BWD_LDP + cc) = pack_bf16x2(pv[2], pv[3]);
        *reinterpret_cast<uint32_t*>(sdS + rl * BWD_LDP + cc) = pack_bf16x2(dsv[0], dsv[1]);
        *reinterpret_cast<uint32_t*>(sdS + (rl + 8) * BWD_LDP + cc) = pack_bf16x2(dsv[2], dsv[3]);
      }
    }
    __syncthreads();  // (B)

    // ---- dV += P^T dO ; dK += dS^T Q     (warp: 16 kv rows x 64 d cols)
#pragma unroll
    for (int kk = 0; kk < BWD_BQ / 16; ++kk) {
      uint32_t ap[4], ads[4];
      ldsm_x4_t(addr_At<BWD_LDP>(uP, kk * 16, wm * 16, lane), ap[0], ap[1], ap[2], ap[3]);
      ldsm_x4_t(addr_At<BWD_LDP>(udS, kk * 16, wm * 16, lane), ads[0], ads[1], ads[2], ads[3]);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(addr_Bt<BWD_LDS>(cdO, kk * 16, wn * 64 + np * 16, lane), b0, b1, b2, b3);
        mma_bf16_16816(dv_acc[2 * np], ap, b0, b1);
        mma_bf16_16816(dv_acc[2 * np + 1], ap, b2, b3);
        ldsm_x4_t(addr_Bt<BWD_LDS>(cQ, kk * 16, wn * 64 + np * 16, lane), b0, b1, b2, b3);
        mma_bf16_16816(dk_acc[2 * np], ads, b0, b1);
        mma_bf16_16816(dk_acc[2 * np + 1], ads, b2, b3);
      }
    }
    // ---- dQ tile = dS K   (warp: 16 q rows x 64 d cols) -> fp32 staging -> TMA bulk reduce-add
    {
      float dq[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int t = 0; t < 4; ++t) dq[i][t] = 0.f;
#pragma unroll
      for (int kk = 0; kk < BWD_BC / 16; ++kk) {
        uint32_t a[4];
        ldsm_x4(addr_A<BWD_LDP>(udS, wm * 16, kk * 16, lane), a[0], a[1], a[2], a[3]);
#pragma unroll
        for (int np = 0; np < 4; ++np) {
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(addr_Bt<BWD_LDS>(uK, kk * 16, wn * 64 + np * 16, lane), b0, b1, b2, b3);
          mma_bf16_16816(dq[2 * np], a, b0, b1);
          mma_bf16_16816(dq[2 * np + 1], a, b2, b3);
        }
      }
      float* st = sdQ + buf * BWD_BQ * BWD_D;
      const int rl = wm * 16 + (lane >> 2);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int cc = wn * 64 + i * 8 + (lane & 3) * 2;
        *reinterpret_cast<float2*>(st + rl * BWD_D + cc) = make_float2(dq[i][0] * p.scale, dq[i][1] * p.scale);
        *reinterpret_cast<float2*>(st + (rl + 8) * BWD_D + cc) = make_float2(dq[i][2] * p.scale, dq[i][3] * p.scale);
      }
    }
    fence_proxy_async_smem();
    __syncthreads();  // (C)
    if (threadIdx.x < BWD_BQ) {
      const int r = q0 + threadIdx.x;
      if (r < p.T) {
        float* dst = p.dq_accum + (tok0 + r) * ((long long)p.Hq * BWD_D) + (long long)hq * BWD_D;
        const uint32_t src = smem_u32(sdQ + buf * BWD_BQ * BWD_D + threadIdx.x * BWD_D);
        asm volatile(
            "cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(dst),
            "r"(src), "r"(BWD_D * 4)
            : "memory");
      }
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  cp_async_wait<0>();
  if (threadIdx.x < BWD_BQ) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");

  // ---- write dK (scaled) and dV as bf16
  {
    const int rl = wm * 16 + (lane >> 2);
    bf16* gdk = p.dk + tok0 * p.lddk + (long long)hk * BWD_D;
    bf16* gdv = p.dv + tok0 * p.lddv + (long long)hk * BWD_D;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int cc = wn * 64 + i * 8 + (lane & 3) * 2;
      const int r0 = kv0 + rl, r1 = kv0 + rl + 8;
      if (r0 < p.T) {
        *reinterpret_cast<uint32_t*>(gdk + (long long)r0 * p.lddk + cc) =
            pack_bf16x2(dk_acc[i][0] * p.scale, dk_acc[i][1] * p.scale);
        *reinterpret_cast<uint32_t*>(gdv + (long long)r0 * p.lddv + cc) =
            pack_bf16x2(dv_acc[i][0], dv_acc[i][1]);
      }
      if (r1 < p.T) {
        *reinterpret_cast<uint32_t*>(gdk + (long long)r1 * p.lddk + cc) =
            pack_bf16x2(dk_acc[i][2] * p.scale, dk_acc[i][3] * p.scale);
        *reinterpret_cast<uint32_t*>(gdv + (long long)r1 * p.lddv + cc) =
            pack_bf16x2(dv_acc[i][2], dv_acc[i][3]);
      }
    }
  }
}

// fp32 [R, C] (pitch C) -> bf16 [R, ld_out] columns [0, C)
__global__ void f32_to_bf16_rows_kernel(const float* __restrict__ x, bf16* __restrict__ y,
                                        long long R, int C, long long ld_out) {
  const int c8 = C >> 3;
  const long long total = R * c8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / c8;
    const int c = (int)(i % c8) * 8;
    const float4 a = *reinterpret_cast<const float4*>(x + r * C + c);
    const float4 b = *reinterpret_cast<const float4*>(x + r * C + c + 4);
    *reinterpret_cast<int4*>(y + r * ld_out + c) =
        make_int4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(b.x, b.y),
                  pack_bf16x2(b.z, b.w));
  }
}

template <int D, bool CAUSAL>
int launch_fwd(const FwdParams& p, cudaStream_t stream) {
  constexpr int LDS = D + 8;
  constexpr int smem = (FWD_BR + 4 * FWD_BC) * LDS * 2;
  auto kern = flash_fwd_kernel<D, CAUSAL>;
  static std::once_flag once;
  static cudaError_t err = cudaSuccess;
  std::call_once(once, [&] {
    err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  });
  MM_CHECK_CUDA(err);
  dim3 grid((p.T + FWD_BR - 1) / FWD_BR, p.Hq, p.B);
  kern<<<grid, FWD_THREADS, smem, stream>>>(p);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

}  // namespace

// Shared by the mma.sync and wgmma backward paths (declared in common.cuh).
MM_API int mm_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse,
                       const int* seqlens, long long ldq, long long ldk, long long ldv,
                       long long ldo, int B, int T, int Hq, int Hkv, int head_dim, int causal,
                       float scale, cudaStream_t stream) {
  MM_CHECK_ARG(B > 0 && T > 0 && Hq > 0 && Hkv > 0 && Hq % Hkv == 0, "mm_attn_fwd: bad head counts");
  MM_CHECK_ARG(head_dim % 8 == 0 && ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0,
               "mm_attn_fwd: head_dim and pitches must be multiples of 8");
  FwdParams p;
  p.q = (const bf16*)q; p.k = (const bf16*)k; p.v = (const bf16*)v; p.o = (bf16*)o;
  p.lse = lse; p.seqlens = seqlens;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
  p.B = B; p.T = T; p.Hq = Hq; p.Hkv = Hkv; p.dh = head_dim; p.scale = scale;
  if (head_dim == 128) return causal ? launch_fwd<128, true>(p, stream) : launch_fwd<128, false>(p, stream);
  if (head_dim == 64) return causal ? launch_fwd<64, true>(p, stream) : launch_fwd<64, false>(p, stream);
  if (head_dim == 72 || head_dim == 80)
    return causal ? launch_fwd<80, true>(p, stream) : launch_fwd<80, false>(p, stream);
  mm_set_error("mm_attn_fwd: unsupported head_dim %d (supported: 64, 72, 80, 128)", head_dim);
  return MM_ERR_ARG;
}

// Workspace of the mma.sync backward (test-only comparison kernel): delta [B*Hq*T] fp32 + dq_accum [B*T*Hq*128] fp32.
MM_API long long mm_attn_bwd_workspace_bytes(int B, int T, int Hq) {
  const long long delta = ((long long)B * Hq * T * 4 + 255) / 256 * 256;
  return delta + (long long)B * T * Hq * 128 * 4;
}

MM_API int mm_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout,
                       const float* lse, void* dq, void* dk, void* dv, const int* seqlens,
                       long long ldq, long long ldk, long long ldv, long long ldo, long long lddo,
                       long long lddq, long long lddk, long long lddv, int B, int T, int Hq, int Hkv,
                       int head_dim, float scale, void* workspace, long long workspace_bytes,
                       cudaStream_t stream) {
  MM_CHECK_ARG(head_dim == 128, "mm_attn_bwd: only head_dim 128 (LLaMA) is implemented");
  MM_CHECK_ARG(B > 0 && T > 0 && Hq % Hkv == 0, "mm_attn_bwd: bad shape");
  MM_CHECK_ARG(workspace != nullptr && workspace_bytes >= mm_attn_bwd_workspace_bytes(B, T, Hq),
               "mm_attn_bwd: workspace too small");
  MM_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 &&
                   lddq % 8 == 0 && lddk % 8 == 0 && lddv % 8 == 0, "mm_attn_bwd: pitches %% 8");
  float* delta = reinterpret_cast<float*>(workspace);
  const long long delta_bytes = ((long long)B * Hq * T * 4 + 255) / 256 * 256;
  float* dq_accum = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + delta_bytes);
  MM_CHECK_CUDA(cudaMemsetAsync(dq_accum, 0, (size_t)B * T * Hq * 128 * 4, stream));
  {
    const long long total = (long long)B * T * Hq;
    long long blocks = ceil_div64(total, 8);
    if (blocks > (long long)mm_num_sms() * 16) blocks = (long long)mm_num_sms() * 16;
    attn_delta_kernel<<<(int)blocks, 256, 0, stream>>>((const bf16*)o, (const bf16*)dout, delta, ldo,
                                                       lddo, B, T, Hq, head_dim);
    MM_CHECK_LAUNCH();
  }
  BwdParams p;
  p.q = (const bf16*)q; p.k = (const bf16*)k; p.v = (const bf16*)v; p.dout = (const bf16*)dout;
  p.lse = lse; p.delta = delta; p.dq_accum = dq_accum;
  p.dk = (bf16*)dk; p.dv = (bf16*)dv; p.seqlens = seqlens;
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.lddo = lddo; p.lddk = lddk; p.lddv = lddv;
  p.B = B; p.T = T; p.Hq = Hq; p.Hkv = Hkv; p.scale = scale;
  static std::once_flag once;
  static cudaError_t err = cudaSuccess;
  std::call_once(once, [&] {
    err = cudaFuncSetAttribute(flash_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM);
  });
  MM_CHECK_CUDA(err);
  dim3 grid((T + BWD_BC - 1) / BWD_BC, Hkv, B);
  flash_bwd_kernel<<<grid, BWD_THREADS, BWD_SMEM, stream>>>(p);
  MM_CHECK_LAUNCH();
  {
    const long long R = (long long)B * T;
    const int C = Hq * 128;
    long long blocks = ceil_div64(R * (C / 8), 256);
    if (blocks > (long long)mm_num_sms() * 16) blocks = (long long)mm_num_sms() * 16;
    f32_to_bf16_rows_kernel<<<(int)blocks, 256, 0, stream>>>(dq_accum, (bf16*)dq, R, C, lddq);
    MM_CHECK_LAUNCH();
  }
  return MM_OK;
}
