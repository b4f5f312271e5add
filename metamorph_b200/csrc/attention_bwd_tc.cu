// metamorph_b200 — flash attention BACKWARD on Hopper tensor cores (wgmma + TMA + mbarrier; head_dim 128, causal,
// GQA): two kernels. (Backward of SURVEY.md K12: HF modeling_llama.py:199-220 / SDPA under autograd; reference call
// site metamorph_llama.py:349-359 via loss.backward().)
//
//   kernel 1  flash_bwd_dq_kernel   query-stationary: one CTA = 128 queries of one (batch, q-head); two consumer
//             warpgroups own 64 queries each. Per 128-key tile, in two halves of 64 keys:
//             delta = rowsum(dO o O) (preamble, from the TMA tiles)   -> also written for kernel 2, with lse*log2(e)
//             S  = Q  K^T,  dP = dO V^T      (wgmma, operands K-major in shared memory, results in registers)
//             dS = P o (dP - delta) * scale   elementwise on the accumulator fragments, packed to bf16 A fragments
//             dQ += dS K                      (A = dS from registers, B = K MN-major from the same TMA tile)
//   kernel 2  flash_bwd_dkv_kernel  key-stationary: one CTA = 128 keys of one (batch, kv-head); loops over the G query
//             heads of the group and the query tiles at/after the key tile, in the TRANSPOSED orientation:
//             S^T = K Q^T,  dP^T = V dO^T;  P^T, dS^T elementwise (lse / delta per column, from shared memory);
//             dV += P^T dO,  dK += dS^T Q   (B = dO / Q MN-major); dK, dV stay in registers for the whole CTA.
// Nothing is reduced through global memory, so the backward is bit-reproducible.
//
// Rows beyond a sample's length (seqlens[b] <= row < T, right padding) are not part of the sequence: they receive zero
// dQ/dK/dV and contribute nothing, exactly as the reference's masked positions carry no gradient (their q/k/v/dO values
// only have to be finite: a masked probability is an exact 0 that multiplies them inside the MMAs).
#include "attention_tc.cuh"

using namespace mm_attn_tc;

namespace {

constexpr int BW_THREADS = 384;  // producer warpgroup + 2 consumer warpgroups
constexpr int BW_TILE = 32768;   // 128 x 128 bf16
constexpr int BW_SMEM = 6 * BW_TILE + 2048 /*stats / reduction scratch*/ + 256 /*barriers*/ + 1024 /*alignment*/;

struct BwdTcParams {
  const float* lse;    // forward log-sum-exp [B,Hq,T] (natural log)
  float* lse2;         // lse * log2(e)            [B,Hq,Tp]   written by kernel 1, read by kernel 2
  float* delta;        // rowsum(dO o O) * scale   [B,Hq,Tp]   written by kernel 1, read by kernel 2
  bf16* dq;
  bf16* dk;
  bf16* dv;
  const int* seqlens;     // valid length per sequence (nullptr: T)
  const int* seg_start;   // packed layout: first row of every sequence (nullptr: b*T)
  const int2* work_q;     // packed layout: (sequence, query tile) per CTA of kernel 1, heaviest first
  const int2* work_k;     // packed layout: (sequence, key tile) per CTA of kernel 2, heaviest first
  long long lddq, lddk, lddv;
  int B, T, Tp, Hq, Hkv;  // T = row pitch of lse and the largest sequence length, Tp = T rounded up to 128
  float scale;
};

// rows g and g + 8 of a 64 x 128 fp32 accumulator fragment -> bf16 (zero when !ok), 16 x bf16x2 stores per row
__device__ __forceinline__ void store_acc_rows(bf16* dst0, bf16* dst1, bool w0, bool w1, bool ok0, bool ok1,
                                               const float (&a)[64], int q2) {
#pragma unroll
  for (int t = 0; t < 16; ++t) {
    if (w0) *reinterpret_cast<uint32_t*>(dst0 + 8 * t + q2) = ok0 ? pack_bf16x2(a[4 * t], a[4 * t + 1]) : 0u;
    if (w1) *reinterpret_cast<uint32_t*>(dst1 + 8 * t + q2) = ok1 ? pack_bf16x2(a[4 * t + 2], a[4 * t + 3]) : 0u;
  }
}

// ======================================================================================================= kernel 1: dQ
__global__ void __launch_bounds__(BW_THREADS, 1)
flash_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                    const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do,
                    const __grid_constant__ CUtensorMap tmap_o, BwdTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int qt = p.work_q ? p.work_q[blockIdx.x].y : (int)gridDim.x - 1 - (int)blockIdx.x;   // heavy (late) tiles first
  const int h = blockIdx.y, b = p.work_q ? p.work_q[blockIdx.x].x : (int)blockIdx.z;
  const int hk = h / (p.Hq / p.Hkv);
  const int q0 = qt * 128;
  const int kv_len = p.seqlens ? min(p.seqlens[b], p.T) : p.T;
  const int tok0 = p.seg_start ? p.seg_start[b] : b * p.T;
  const int row_limit = p.seg_start ? kv_len : p.T;      // packed: rows past the sequence belong to the next one
  const long long stat0 = ((long long)b * p.Hq + h) * p.Tp + q0;

  if (q0 >= kv_len) {
    // the whole tile is padding: zero dQ, neutral statistics (kernel 2 skips these query tiles)
    for (int i = threadIdx.x; i < 128 * 16; i += BW_THREADS) {
      const int r = i >> 4, c = (i & 15) * 8;
      if (q0 + r < row_limit)
        *reinterpret_cast<int4*>(p.dq + (long long)(tok0 + q0 + r) * p.lddq + (long long)h * 128 + c) = make_int4(0, 0, 0, 0);
    }
    if (threadIdx.x < 128) {
      p.lse2[stat0 + threadIdx.x] = 0.f;
      p.delta[stat0 + threadIdx.x] = 0.f;
    }
    return;
  }
  const int n_tiles = (min(kv_len, q0 + 128) + 127) / 128;   // causal: key tiles 0 .. qt

  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t sQ = base, sdO = base + BW_TILE;
  const uint32_t sK[2] = {base + 2 * BW_TILE, base + 4 * BW_TILE};
  const uint32_t sV[2] = {base + 3 * BW_TILE, base + 5 * BW_TILE};
  float* sRed = reinterpret_cast<float*>(base_ptr + 6 * BW_TILE);            // [2][128]
  const uint32_t bar = base + 6 * BW_TILE + 2048;
  const uint32_t q_full = bar, k_full0 = bar + 8, k_full1 = bar + 16, k_empty0 = bar + 24, k_empty1 = bar + 32,
                 v_full0 = bar + 40, v_full1 = bar + 48, v_empty0 = bar + 56, v_empty1 = bar + 64, o_used = bar + 72;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_q);
    prefetch_tmap(&tmap_k);
    prefetch_tmap(&tmap_v);
    prefetch_tmap(&tmap_do);
    prefetch_tmap(&tmap_o);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(k_full0 + 8 * i, 1);
      mbar_init(v_full0 + 8 * i, 1);
      mbar_init(k_empty0 + 8 * i, 8);   // one arrive per consumer warp
      mbar_init(v_empty0 + 8 * i, 8);
    }
    mbar_init(o_used, 8);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ---------------------------------------------------------------- TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, 3 * BW_TILE);
      tma_load_2d(sQ, &tmap_q, q_full, h * 128, tok0 + q0);
      tma_load_2d(sQ + 16384, &tmap_q, q_full, h * 128 + 64, tok0 + q0);
      tma_load_2d(sdO, &tmap_do, q_full, h * 128, tok0 + q0);
      tma_load_2d(sdO + 16384, &tmap_do, q_full, h * 128 + 64, tok0 + q0);
      tma_load_2d(sV[1], &tmap_o, q_full, h * 128, tok0 + q0);            // O parks in V stage 1 until delta is done
      tma_load_2d(sV[1] + 16384, &tmap_o, q_full, h * 128 + 64, tok0 + q0);
      for (int j = 0; j < n_tiles; ++j) {
        const int bf = j & 1;
        const uint32_t ph = (uint32_t)((j >> 1) & 1);
        mbar_wait(bf ? k_empty1 : k_empty0, ph ^ 1);
        mbar_arrive_expect_tx(bf ? k_full1 : k_full0, BW_TILE);
        tma_load_2d(sK[bf], &tmap_k, bf ? k_full1 : k_full0, hk * 128, tok0 + j * 128);
        tma_load_2d(sK[bf] + 16384, &tmap_k, bf ? k_full1 : k_full0, hk * 128 + 64, tok0 + j * 128);
        mbar_wait(bf ? v_empty1 : v_empty0, ph ^ 1);
        if (j == 1) mbar_wait(o_used, 0);
        mbar_arrive_expect_tx(bf ? v_full1 : v_full0, BW_TILE);
        tma_load_2d(sV[bf], &tmap_v, bf ? v_full1 : v_full0, hk * 128, tok0 + j * 128);
        tma_load_2d(sV[bf] + 16384, &tmap_v, bf ? v_full1 : v_full0, hk * 128 + 64, tok0 + j * 128);
      }
    }
    return;
  }

  setmaxnreg_inc<232>();
  const int c = wg - 1, ct = threadIdx.x - 128;
  // ---- preamble: delta = rowsum(dO o O) from the swizzled TMA tiles (two [128 x 64] boxes, 16-byte chunks XOR row%8)
  mbar_wait(q_full, 0);
  {
    const int r = ct & 127, hh = ct >> 7;
    float part = 0.f;
    const uint32_t off = (uint32_t)hh * 16384u + (uint32_t)r * 128u;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint32_t slot = (uint32_t)((i ^ (r & 7)) << 4);
      const int4 a = *reinterpret_cast<const int4*>(base_ptr + BW_TILE + off + slot);          // dO
      const int4 o = *reinterpret_cast<const int4*>(base_ptr + 5 * BW_TILE + off + slot);      // O (V stage 1)
      const uint32_t ua[4] = {(uint32_t)a.x, (uint32_t)a.y, (uint32_t)a.z, (uint32_t)a.w};
      const uint32_t uo[4] = {(uint32_t)o.x, (uint32_t)o.y, (uint32_t)o.z, (uint32_t)o.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 x = unpack_bf16x2(ua[t]);
        const float2 y = unpack_bf16x2(uo[t]);
        part = fmaf(x.x, y.x, fmaf(x.y, y.y, part));
      }
    }
    sRed[hh * 128 + r] = part;
  }
  consumer_release(o_used);                                  // this warp no longer reads the O tile
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (ct < 128) {
    const bool ok = q0 + ct < kv_len;
    p.delta[stat0 + ct] = ok ? (sRed[ct] + sRed[128 + ct]) * p.scale : 0.f;
    p.lse2[stat0 + ct] = ok ? p.lse[((long long)b * p.Hq + h) * p.T + q0 + ct] * kLog2e : 0.f;
  }
  const int g = ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2), q2 = (lane & 3) * 2;
  int q_idx[2];
  bool q_ok[2];
  float delta[2], lse2[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = c * 64 + g + 8 * i;
    q_idx[i] = q0 + r;
    q_ok[i] = q_idx[i] < kv_len;
    delta[i] = q_ok[i] ? (sRed[r] + sRed[128 + r]) * p.scale : 0.f;
    lse2[i] = q_ok[i] ? p.lse[((long long)b * p.Hq + h) * p.T + q_idx[i]] * kLog2e : 0.f;
  }
  const float sl2 = p.scale * kLog2e;
  const uint32_t sQc = sQ + (uint32_t)c * 8192u, sdOc = sdO + (uint32_t)c * 8192u;
  float dq[64];
  for (int j = 0; j < n_tiles; ++j) {
    const int bf = j & 1;
    const uint32_t ph = (uint32_t)((j >> 1) & 1);
    mbar_wait(bf ? k_full1 : k_full0, ph);
    mbar_wait(bf ? v_full1 : v_full0, ph);
#pragma unroll 1
    for (int hf = 0; hf < 2; ++hf) {               // 64 keys at a time
      float s[32], dp[32];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        wgmma_m64n64_ss<0, 0>(s, desc_kmajor(sQc, k), desc_kmajor(sK[bf] + hf * 8192u, k), k != 0 ? 1u : 0u);
        wgmma_m64n64_ss<0, 0>(dp, desc_kmajor(sdOc, k), desc_kmajor(sV[bf] + hf * 8192u, k), k != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // P = exp2(S * scale*log2e - lse2);  dS = P o (dP*scale - delta)
      const int k0 = j * 128 + hf * 64;
#pragma unroll
      for (int t = 0; t < 32; ++t) {
        const int i = (t >> 1) & 1;
        const int col = k0 + (t >> 2) * 8 + q2 + (t & 1);
        const bool ok = q_ok[i] && col <= q_idx[i] && col < kv_len;
        const float pv = ok ? fast_exp2(fmaf(s[t], sl2, -lse2[i])) : 0.f;
        s[t] = pv * fmaf(dp[t], p.scale, -delta[i]);
      }
      uint32_t da[4][4];
#pragma unroll
      for (int k = 0; k < 4; ++k) acc_to_a(s, k, da[k]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_m64n128_rs<1>(dq, da[k], desc_mnmajor(sK[bf], hf * 4 + k), (j | hf | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
    }
    consumer_release(bf ? k_empty1 : k_empty0);
    consumer_release(bf ? v_empty1 : v_empty0);
  }
  // ---- epilogue: dQ (already scaled through dS) -> bf16
  bf16* d0 = p.dq + (long long)(tok0 + q_idx[0]) * p.lddq + (long long)h * 128;
  bf16* d1 = p.dq + (long long)(tok0 + q_idx[1]) * p.lddq + (long long)h * 128;
  store_acc_rows(d0, d1, q_idx[0] < row_limit, q_idx[1] < row_limit, q_ok[0], q_ok[1], dq, q2);
}

// =================================================================================================== kernel 2: dK, dV
// One CTA = 64 keys. Warpgroup 1 accumulates dV, warpgroup 2 dK (both compute S^T and dP^T): the two 64 x 128 fp32
// accumulators of one warpgroup would not fit its register budget next to the S^T / dP^T fragments.
__global__ void __launch_bounds__(BW_THREADS, 1)
flash_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                     const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do,
                     const __grid_constant__ CUtensorMap tmap_stat, BwdTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  // grid = (Hkv*B, 64-key tiles): CTAs are dispatched x-fastest, so ALL (head, batch) instances of the heaviest key tile
  // (tile 0 sees every query tile) start first and the light tiles fill the tail (LPT-style schedule)
  // (packed sequences: grid = (2 x key-tile work list, kv heads); the list names 128-key tiles)
  const int jt = p.work_k ? 2 * p.work_k[blockIdx.x >> 1].y + (int)(blockIdx.x & 1) : (int)blockIdx.y;
  const int hk = p.work_k ? (int)blockIdx.y : (int)(blockIdx.x % p.Hkv);
  const int b = p.work_k ? p.work_k[blockIdx.x >> 1].x : (int)(blockIdx.x / p.Hkv);
  const int G = p.Hq / p.Hkv;
  const int kv0 = jt * 64;
  const int kv_len = p.seqlens ? min(p.seqlens[b], p.T) : p.T;
  const int tok0 = p.seg_start ? p.seg_start[b] : b * p.T;
  const int row_limit = p.seg_start ? kv_len : p.T;

  if (kv0 >= kv_len) {   // the whole key tile is padding
    for (int i = threadIdx.x; i < 64 * 16; i += BW_THREADS) {
      const int r = i >> 4, c = (i & 15) * 8;
      if (kv0 + r < row_limit) {
        *reinterpret_cast<int4*>(p.dk + (long long)(tok0 + kv0 + r) * p.lddk + (long long)hk * 128 + c) = make_int4(0, 0, 0, 0);
        *reinterpret_cast<int4*>(p.dv + (long long)(tok0 + kv0 + r) * p.lddv + (long long)hk * 128 + c) = make_int4(0, 0, 0, 0);
      }
    }
    return;
  }
  const int qt_begin = kv0 / 128;                            // causal: query tiles of 128 at or after this key tile ...
  const int n_qt = (kv_len + 127) / 128 - qt_begin;          // ... that contain at least one real query
  const int n_it = n_qt * G;

  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t sK = base, sV = base + BW_TILE;             // [64 keys x 64] boxes at +0 / +16 KB (the K-major layout)
  const uint32_t sQ[2] = {base + 2 * BW_TILE, base + 4 * BW_TILE};
  const uint32_t sdO[2] = {base + 3 * BW_TILE, base + 5 * BW_TILE};
  const float* sStat = reinterpret_cast<const float*>(base_ptr + 6 * BW_TILE);   // [2 buffers][lse2 128 | delta 128]
  const uint32_t uStat = base + 6 * BW_TILE;
  const uint32_t bar = base + 6 * BW_TILE + 2048;
  const uint32_t kv_full = bar, qdo_full0 = bar + 8, qdo_full1 = bar + 16, qdo_empty0 = bar + 24, qdo_empty1 = bar + 32;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_q);
    prefetch_tmap(&tmap_k);
    prefetch_tmap(&tmap_v);
    prefetch_tmap(&tmap_do);
    prefetch_tmap(&tmap_stat);
    mbar_init(kv_full, 1);
    mbar_init(qdo_full0, 1);
    mbar_init(qdo_full1, 1);
    mbar_init(qdo_empty0, 8);   // one arrive per consumer warp: Q, dO and the statistics rows of the buffer are read
    mbar_init(qdo_empty1, 8);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ---------------------------------------------------------------- TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(kv_full, 4 * 64 * 128);
      tma_load_2d(sK, &tmap_k, kv_full, hk * 128, tok0 + kv0);
      tma_load_2d(sK + 16384, &tmap_k, kv_full, hk * 128 + 64, tok0 + kv0);
      tma_load_2d(sV, &tmap_v, kv_full, hk * 128, tok0 + kv0);
      tma_load_2d(sV + 16384, &tmap_v, kv_full, hk * 128 + 64, tok0 + kv0);
      for (int it = 0; it < n_it; ++it) {
        const int buf = it & 1, use = it >> 1;
        const int hq = hk * G + it / n_qt;
        const int q0 = (qt_begin + it % n_qt) * 128;
        const uint32_t full = buf ? qdo_full1 : qdo_full0, empty = buf ? qdo_empty1 : qdo_empty0;
        mbar_wait(empty, (uint32_t)((use & 1) ^ 1));
        mbar_arrive_expect_tx(full, 2 * BW_TILE + 1024);
        tma_load_2d(sQ[buf], &tmap_q, full, hq * 128, tok0 + q0);
        tma_load_2d(sQ[buf] + 16384, &tmap_q, full, hq * 128 + 64, tok0 + q0);
        tma_load_2d(sdO[buf], &tmap_do, full, hq * 128, tok0 + q0);
        tma_load_2d(sdO[buf] + 16384, &tmap_do, full, hq * 128 + 64, tok0 + q0);
        // statistics rows of the workspace: [lse2 rows of all (b, head) | delta rows of all (b, head)], 128 values each
        tma_load_2d(uStat + buf * 1024, &tmap_stat, full, q0, b * p.Hq + hq);
        tma_load_2d(uStat + buf * 1024 + 512, &tmap_stat, full, q0, (p.B + b) * p.Hq + hq);
      }
    }
    return;
  }

  setmaxnreg_inc<232>();
  const bool is_dk = wg == 2;
  const int g = ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2), q2 = (lane & 3) * 2;
  int key_idx[2];
  bool key_ok[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    key_idx[i] = kv0 + g + 8 * i;
    key_ok[i] = key_idx[i] < kv_len;
  }
  const float sl2 = p.scale * kLog2e;
  float acc[64];                                   // dV (warpgroup 1) or dK (warpgroup 2)
  mbar_wait(kv_full, 0);
  for (int it = 0; it < n_it; ++it) {
    const int buf = it & 1;
    const int q0 = (qt_begin + it % n_qt) * 128;
    mbar_wait(buf ? qdo_full1 : qdo_full0, (uint32_t)((it >> 1) & 1));
    const float* sLse = sStat + buf * 256;
    const float* sDelta = sLse + 128;
#pragma unroll 1
    for (int hf = 0; hf < 2; ++hf) {               // 64 queries at a time
      float s[32], dp[32];
      uint32_t fa[4][4];
      // both warpgroups issue the same products (dP^T is only used by the dK one): wgmma in a warpgroup-divergent branch
      // would make ptxas serialise every wgmma of the kernel, and the dK warpgroup sets the pace either way
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        wgmma_m64n64_ss<0, 0>(s, desc_kmajor(sK, k), desc_kmajor(sQ[buf] + hf * 8192u, k), k != 0 ? 1u : 0u);
        wgmma_m64n64_ss<0, 0>(dp, desc_kmajor(sV, k), desc_kmajor(sdO[buf] + hf * 8192u, k), k != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // P^T = exp2(S^T * scale*log2e - lse2[q]);  dK warpgroup: dS^T = P^T o (dP^T*scale - delta[q])
#pragma unroll
      for (int t = 0; t < 32; ++t) {
        const int i = (t >> 1) & 1;
        const int ql = hf * 64 + (t >> 2) * 8 + q2 + (t & 1);   // query column within the 128-query tile
        const bool ok = key_ok[i] && (q0 + ql < kv_len) && (key_idx[i] <= q0 + ql);
        const float pv = ok ? fast_exp2(fmaf(s[t], sl2, -sLse[ql])) : 0.f;
        s[t] = is_dk ? pv * fmaf(dp[t], p.scale, -sDelta[ql]) : pv;
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) acc_to_a(s, k, fa[k]);
      // dV += P^T dO  /  dK += dS^T Q   (B MN-major: query rows of the tile are the contraction)
      const uint32_t sB = is_dk ? sQ[buf] : sdO[buf];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_m64n128_rs<1>(acc, fa[k], desc_mnmajor(sB, hf * 4 + k), (it | hf | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
    }
    consumer_release(buf ? qdo_empty1 : qdo_empty0);
  }
  // ---- final: dK (already scaled through dS) or dV
  bf16* dst = is_dk ? p.dk : p.dv;
  const long long ld = is_dk ? p.lddk : p.lddv;
  store_acc_rows(dst + (long long)(tok0 + key_idx[0]) * ld + (long long)hk * 128,
                 dst + (long long)(tok0 + key_idx[1]) * ld + (long long)hk * 128, key_idx[0] < row_limit,
                 key_idx[1] < row_limit, key_ok[0], key_ok[1], acc, q2);
}

}  // namespace

// Workspace of the backward: lse*log2e and delta, [B, Hq, Tp] fp32 each (Tp = T rounded up to 128).
MM_API long long mm_attn_bwd_tc_workspace_bytes(int B, int T, int Hq) {
  const long long Tp = ((long long)T + 127) / 128 * 128;
  return 2 * (((long long)B * Hq * Tp * 4 + 255) / 256 * 256);
}

namespace {

int launch_bwd_tc(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse, void* dq,
                  void* dk, void* dv, const int* seqlens, const int* seg_start, const int* work_q, int n_work_q,
                  const int* work_k, int n_work_k, long long total_rows, long long ldq, long long ldk, long long ldv,
                  long long ldo, long long lddo, long long lddq, long long lddk, long long lddv, int B, int T, int Hq,
                  int Hkv, float scale, void* workspace, long long workspace_bytes, cudaStream_t stream) {
  MM_CHECK_ARG(B > 0 && T > 0 && Hq > 0 && Hkv > 0 && Hq % Hkv == 0, "mm_attn_bwd_tc: bad shape");
  MM_CHECK_ARG(workspace != nullptr && workspace_bytes >= mm_attn_bwd_tc_workspace_bytes(B, T, Hq),
               "mm_attn_bwd_tc: workspace too small (use mm_attn_bwd_tc_workspace_bytes)");
  MM_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 &&
                   lddk % 8 == 0 && lddv % 8 == 0, "mm_attn_bwd_tc: pitches %% 8");
  MM_CHECK_ARG(((uintptr_t)q & 15) == 0 && ((uintptr_t)k & 15) == 0 && ((uintptr_t)v & 15) == 0 &&
                   ((uintptr_t)o & 15) == 0 && ((uintptr_t)dout & 15) == 0 && ((uintptr_t)dq & 15) == 0 &&
                   ((uintptr_t)dk & 15) == 0 && ((uintptr_t)dv & 15) == 0 && ((uintptr_t)workspace & 15) == 0,
               "mm_attn_bwd_tc: 16-byte alignment required");
  const int Tp = (T + 127) / 128 * 128;
  const long long stat_bytes = ((long long)B * Hq * Tp * 4 + 255) / 256 * 256;
  CUtensorMap tq, tk, tv, tdo, to, tstat, tk64, tv64;
  int rc;
  MM_CHECK_ARG(stat_bytes == (long long)B * Hq * Tp * 4, "mm_attn_bwd_tc: statistics rows must be contiguous");
  if ((rc = mm_attn_make_tmap_stats(&tstat, reinterpret_cast<const float*>(workspace), Tp, 2LL * B * Hq))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&tq, q, (long long)Hq * 128, total_rows, ldq))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&tk, k, (long long)Hkv * 128, total_rows, ldk))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&tv, v, (long long)Hkv * 128, total_rows, ldv))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&tdo, dout, (long long)Hq * 128, total_rows, lddo))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&to, o, (long long)Hq * 128, total_rows, ldo))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&tk64, k, (long long)Hkv * 128, total_rows, ldk, 64))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&tv64, v, (long long)Hkv * 128, total_rows, ldv, 64))) return rc;
  static std::once_flag once;
  static cudaError_t err = cudaSuccess;
  std::call_once(once, [&] {
    err = cudaFuncSetAttribute(flash_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BW_SMEM);
    if (err == cudaSuccess)
      err = cudaFuncSetAttribute(flash_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BW_SMEM);
  });
  MM_CHECK_CUDA(err);
  BwdTcParams p;
  p.lse = lse;
  p.lse2 = reinterpret_cast<float*>(workspace);
  p.delta = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + stat_bytes);
  p.dq = (bf16*)dq; p.dk = (bf16*)dk; p.dv = (bf16*)dv; p.seqlens = seqlens; p.seg_start = seg_start;
  p.work_q = reinterpret_cast<const int2*>(work_q); p.work_k = reinterpret_cast<const int2*>(work_k);
  p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
  p.B = B; p.T = T; p.Tp = Tp; p.Hq = Hq; p.Hkv = Hkv; p.scale = scale;
  const int n_tiles = (T + 127) / 128;
  const dim3 grid_q = work_q ? dim3(n_work_q, Hq, 1) : dim3(n_tiles, Hq, B);
  const dim3 grid_k = work_k ? dim3(2 * n_work_k, Hkv, 1) : dim3(Hkv * B, 2 * n_tiles, 1);
  flash_bwd_dq_kernel<<<grid_q, BW_THREADS, BW_SMEM, stream>>>(tq, tk, tv, tdo, to, p);
  MM_CHECK_LAUNCH();
  flash_bwd_dkv_kernel<<<grid_k, BW_THREADS, BW_SMEM, stream>>>(tq, tk64, tv64, tdo, tstat, p);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

}  // namespace

// wgmma flash-attention backward (workspace from mm_attn_bwd_tc_workspace_bytes). See include/metamorph_b200.h for the
// contract.
MM_API int mm_attn_bwd_tc(const void* q, const void* k, const void* v, const void* o, const void* dout,
                          const float* lse, void* dq, void* dk, void* dv, const int* seqlens, long long ldq,
                          long long ldk, long long ldv, long long ldo, long long lddo, long long lddq,
                          long long lddk, long long lddv, int B, int T, int Hq, int Hkv, int head_dim,
                          float scale, void* workspace, long long workspace_bytes, cudaStream_t stream) {
  MM_CHECK_ARG(head_dim == 128, "mm_attn_bwd_tc: head_dim must be 128");
  return launch_bwd_tc(q, k, v, o, dout, lse, dq, dk, dv, seqlens, nullptr, nullptr, 0, nullptr, 0, (long long)B * T, ldq,
                       ldk, ldv, ldo, lddo, lddq, lddk, lddv, B, T, Hq, Hkv, scale, workspace, workspace_bytes, stream);
}

// Packed sequences: the backward of mm_attn_fwd_tc_varlen (same segment tables; work_q lists (sequence, query tile)
// pairs, work_k (sequence, key tile) pairs, both heaviest first; workspace from mm_attn_bwd_tc_workspace_bytes(n_seg,
// max_len, Hq)). Rows that belong to no sequence are not written.
MM_API int mm_attn_bwd_tc_varlen(const void* q, const void* k, const void* v, const void* o, const void* dout,
                                 const float* lse, void* dq, void* dk, void* dv, const int* seg_start,
                                 const int* seg_len, int n_seg, int max_len, const int* work_q, int n_work_q,
                                 const int* work_k, int n_work_k, long long total_rows, long long ldq, long long ldk,
                                 long long ldv, long long ldo, long long lddo, long long lddq, long long lddk,
                                 long long lddv, int Hq, int Hkv, int head_dim, float scale, void* workspace,
                                 long long workspace_bytes, cudaStream_t stream) {
  MM_CHECK_ARG(head_dim == 128, "mm_attn_bwd_tc_varlen: head_dim must be 128");
  MM_CHECK_ARG(seg_start != nullptr && seg_len != nullptr && work_q != nullptr && work_k != nullptr && n_work_q > 0 &&
                   n_work_k > 0 && n_seg > 0 && max_len > 0, "mm_attn_bwd_tc_varlen: segment tables missing");
  return launch_bwd_tc(q, k, v, o, dout, lse, dq, dk, dv, seg_len, seg_start, work_q, n_work_q, work_k, n_work_k,
                       total_rows, ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv, n_seg, max_len, Hq, Hkv, scale, workspace,
                       workspace_bytes, stream);
}
