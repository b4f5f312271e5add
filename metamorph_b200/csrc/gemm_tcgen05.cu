// metamorph_b200 — bf16 GEMM on Hopper tensor cores (wgmma.mma_async, fp32 accumulators in registers, operands
// staged by TMA into 128B-swizzled shared memory), persistent + warp-specialised, fused epilogues.
// (This file keeps its historical name; nothing in it uses tcgen05.)
//
// One kernel family serves every dense contraction on the hot path (SURVEY.md §2.1 K1,K3,K5,K6,K8,
// K11,K13,K14,K15,K16 and their dgrad/wgrad):
//     C[M,N] = A[M,K] * B[N,K]^T           (nn.Linear forward;   A K-major,  B K-major)
//     C[M,N] = A[M,K] * B[K,N]             (dgrad  dX = dY * W;  A K-major,  B MN-major)
//     C[M,N] = A[K,M]^T * B[K,N]           (wgrad  dW = dY^T X;  A MN-major, B MN-major)
// "K-major" = the contraction index is the contiguous one in memory. MN-major operands are fed to
// the tensor core directly through the wgmma transpose bits of the shared-memory descriptors (no transpose pass).
//
// CTA layout (384 threads, 1 CTA/SM, grid = min(#tiles, #SMs), static persistent schedule, tile BM=128 x BN):
//   warpgroup 0, one thread : TMA producer (global -> smem ring, kStages deep, mbarrier tx-count); it keeps loading
//                             the next tile while the consumers run the epilogue of the current one
//   warpgroups 1, 2         : consumers, 64 rows each: wgmma m64nBNk16 per 16-wide k-slice, then the fused epilogue
//                             (accumulators -> padded smem staging, 64 columns at a time -> one row x 32 columns per
//                             thread -> epilogue_chunk -> global)
#include "wgmma.cuh"
#include <mutex>
#include <stdlib.h>

namespace {

constexpr int BM = 128;
constexpr int BK = 64;       // 64 bf16 = 128 bytes = one swizzle-128B row
constexpr int kThreads = 384;
constexpr int kStageLd = 68;  // fp32 pitch of the epilogue staging rows (64 + 4: conflict-free float4 row reads)

enum Epilogue : int {
  EPI_STORE = 0,           // C = acc
  EPI_BIAS = 1,            // C = acc + bias[n]
  EPI_BIAS_GELU_ERF = 2,   // C = gelu_erf(acc + bias[n])        (mm_projector / vision_head)
  EPI_BIAS_GELU_TANH = 3,  // C = gelu_tanh(acc + bias[n])       (SigLIP fc1)
  EPI_RESID = 4,           // C = acc + R[m,n]                   (o_proj / down_proj + residual)
  EPI_BIAS_RESID = 5,      // C = acc + bias[n] + R[m,n]         (SigLIP out_proj / fc2)
  EPI_SWIGLU = 6,          // columns interleaved [16 gate | 16 up]: C[m, n/2] = silu(g) * u
  EPI_SWIGLU_BWD = 7,      // acc = d(act)[m, n]; aux holds (gate|up)[m, 2n] interleaved and is overwritten
                           // with d(gate|up); C[m, n] = silu(g) * u (recomputed activation for the wgrad)
};

struct EpiParams {
  void* C;
  long long ldc;
  const bf16* bias;
  const bf16* resid;
  long long ldr;
  bf16* aux;  // EPI_SWIGLU: optional raw (gate|up interleaved) copy [M, N]
  long long ld_aux;
  int epi;
  int out_f32;     // 1: C is fp32, 0: bf16
  int accumulate;  // 1: C += result (C read in its own dtype)
  float alpha;     // result scale applied to acc before everything else
};

template <int BN>
struct Cfg {
  static constexpr int kStages = (BN == 256) ? 3 : 5;
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiBytes = 2 * 64 * kStageLd * 4;   // one [64 x 64] fp32 staging tile per consumer warpgroup
  static constexpr int kSmemBytes = kStages * kStageBytes + kEpiBytes + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory budget of one H100 CTA");
};

// Fused epilogue for one 32-column accumulator chunk held by one thread (one output row).
__device__ __forceinline__ void epilogue_chunk(const EpiParams& ep, float (&v)[32], int row, bool row_ok,
                                               int col0, int N) {
    const bool full_chunk = (col0 + 32 <= N);

    if (ep.epi == EPI_SWIGLU_BWD) {
      // LlamaMLP backward fused into the down_proj dgrad: this thread owns d(act) for 32 intermediate
      // channels of one token = two [16 gate | 16 up] blocks of the interleaved gate/up buffer.
      if (row_ok) {
        bf16* gp = ep.aux + (long long)row * ep.ld_aux + 2 * col0;
        bf16* cp = reinterpret_cast<bf16*>(ep.C) + (long long)row * ep.ldc + col0;
#pragma unroll
        for (int blk = 0; blk < 2; ++blk) {
          uint32_t og[8], ou[8], oa[8];
#pragma unroll
          for (int hv = 0; hv < 2; ++hv) {
            const int4 graw = *reinterpret_cast<const int4*>(gp + blk * 32 + hv * 8);
            const int4 uraw = *reinterpret_cast<const int4*>(gp + blk * 32 + 16 + hv * 8);
            const uint32_t ug[4] = {(uint32_t)graw.x, (uint32_t)graw.y, (uint32_t)graw.z, (uint32_t)graw.w};
            const uint32_t uu[4] = {(uint32_t)uraw.x, (uint32_t)uraw.y, (uint32_t)uraw.z, (uint32_t)uraw.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float2 g = unpack_bf16x2(ug[j]);
              const float2 u = unpack_bf16x2(uu[j]);
              const float d0 = v[blk * 16 + hv * 8 + 2 * j], d1 = v[blk * 16 + hv * 8 + 2 * j + 1];
              const float s0 = 1.f / (1.f + __expf(-g.x)), s1 = 1.f / (1.f + __expf(-g.y));
              const float a0 = g.x * s0, a1 = g.y * s1;
              oa[hv * 4 + j] = pack_bf16x2(a0 * u.x, a1 * u.y);
              og[hv * 4 + j] = pack_bf16x2(d0 * u.x * (s0 + a0 * (1.f - s0)), d1 * u.y * (s1 + a1 * (1.f - s1)));
              ou[hv * 4 + j] = pack_bf16x2(d0 * a0, d1 * a1);
            }
          }
          *reinterpret_cast<int4*>(gp + blk * 32) = make_int4(og[0], og[1], og[2], og[3]);
          *reinterpret_cast<int4*>(gp + blk * 32 + 8) = make_int4(og[4], og[5], og[6], og[7]);
          *reinterpret_cast<int4*>(gp + blk * 32 + 16) = make_int4(ou[0], ou[1], ou[2], ou[3]);
          *reinterpret_cast<int4*>(gp + blk * 32 + 24) = make_int4(ou[4], ou[5], ou[6], ou[7]);
          *reinterpret_cast<int4*>(cp + blk * 16) = make_int4(oa[0], oa[1], oa[2], oa[3]);
          *reinterpret_cast<int4*>(cp + blk * 16 + 8) = make_int4(oa[4], oa[5], oa[6], oa[7]);
        }
      }
      return;
    }
    if (ep.epi == EPI_SWIGLU) {
      // chunk = 16 gate columns followed by their 16 up columns
      if (row_ok) {
        if (ep.aux != nullptr) {
          bf16* ap = ep.aux + (long long)row * ep.ld_aux + col0;
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            int4 o;
            o.x = pack_bf16x2(v[j], v[j + 1]);
            o.y = pack_bf16x2(v[j + 2], v[j + 3]);
            o.z = pack_bf16x2(v[j + 4], v[j + 5]);
            o.w = pack_bf16x2(v[j + 6], v[j + 7]);
            *reinterpret_cast<int4*>(ap + j) = o;
          }
        }
        float o16[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) o16[j] = silu(v[j]) * v[16 + j];
        bf16* cp = reinterpret_cast<bf16*>(ep.C) + (long long)row * ep.ldc + (col0 >> 1);
#pragma unroll
        for (int j = 0; j < 16; j += 8) {
          int4 o;
          o.x = pack_bf16x2(o16[j], o16[j + 1]);
          o.y = pack_bf16x2(o16[j + 2], o16[j + 3]);
          o.z = pack_bf16x2(o16[j + 4], o16[j + 5]);
          o.w = pack_bf16x2(o16[j + 6], o16[j + 7]);
          *reinterpret_cast<int4*>(cp + j) = o;
        }
      }
      return;
    }

    if (ep.epi == EPI_BIAS || ep.epi == EPI_BIAS_GELU_ERF || ep.epi == EPI_BIAS_GELU_TANH ||
        ep.epi == EPI_BIAS_RESID) {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (full_chunk || col0 + j < N) v[j] += __bfloat162float(__ldg(ep.bias + col0 + j));
    }
    if (ep.epi == EPI_BIAS_GELU_ERF) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
    } else if (ep.epi == EPI_BIAS_GELU_TANH) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = gelu_tanh(v[j]);
    }
    if (!row_ok) return;
    if (ep.epi == EPI_RESID || ep.epi == EPI_BIAS_RESID) {
      const bf16* rp = ep.resid + (long long)row * ep.ldr + col0;
      if (full_chunk) {
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          const int4 rr = *reinterpret_cast<const int4*>(rp + j);
          float2 f;
          f = unpack_bf16x2(rr.x); v[j] += f.x; v[j + 1] += f.y;
          f = unpack_bf16x2(rr.y); v[j + 2] += f.x; v[j + 3] += f.y;
          f = unpack_bf16x2(rr.z); v[j + 4] += f.x; v[j + 5] += f.y;
          f = unpack_bf16x2(rr.w); v[j + 6] += f.x; v[j + 7] += f.y;
        }
      } else {
        for (int j = 0; j < 32; ++j)
          if (col0 + j < N) v[j] += __bfloat162float(rp[j]);
      }
    }
    if (ep.out_f32) {
      float* cp = reinterpret_cast<float*>(ep.C) + (long long)row * ep.ldc + col0;
      if (full_chunk) {
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          float4 o = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
          if (ep.accumulate) {
            const float4 old = *reinterpret_cast<const float4*>(cp + j);
            o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w;
          }
          *reinterpret_cast<float4*>(cp + j) = o;
        }
      } else {
        for (int j = 0; j < 32; ++j)
          if (col0 + j < N) cp[j] = ep.accumulate ? cp[j] + v[j] : v[j];
      }
    } else {
      bf16* cp = reinterpret_cast<bf16*>(ep.C) + (long long)row * ep.ldc + col0;
      if (full_chunk) {
#pragma unroll
        for (int j = 0; j < 32; j += 8) {
          if (ep.accumulate) {
            const int4 old = *reinterpret_cast<const int4*>(cp + j);
            float2 f;
            f = unpack_bf16x2(old.x); v[j] += f.x; v[j + 1] += f.y;
            f = unpack_bf16x2(old.y); v[j + 2] += f.x; v[j + 3] += f.y;
            f = unpack_bf16x2(old.z); v[j + 4] += f.x; v[j + 5] += f.y;
            f = unpack_bf16x2(old.w); v[j + 6] += f.x; v[j + 7] += f.y;
          }
          int4 o;
          o.x = pack_bf16x2(v[j], v[j + 1]);
          o.y = pack_bf16x2(v[j + 2], v[j + 3]);
          o.z = pack_bf16x2(v[j + 4], v[j + 5]);
          o.w = pack_bf16x2(v[j + 6], v[j + 7]);
          *reinterpret_cast<int4*>(cp + j) = o;
        }
      } else {
        for (int j = 0; j < 32; ++j)
          if (col0 + j < N) {
            float x = v[j];
            if (ep.accumulate) x += __bfloat162float(cp[j]);
            cp[j] = __float2bfloat16(x);
          }
      }
    }
}

// D[64 x BN] (+)= A * B for one 16-wide k-slice; the transpose bits are template arguments of the instruction
template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_k16(float (&d)[BN / 2], uint64_t da, uint64_t db, uint32_t acc) {
  if constexpr (BN == 256) wgmma_m64n256_ss<TA, TB>(d, da, db, acc);
  else wgmma_m64n128_ss<TA, TB>(d, da, db, acc);
}

template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int M, int N,
                  int K, int group_m, EpiParams ep) {
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t epi_base = smem_base + C::kStages * C::kStageBytes;
  const uint32_t bar_base = epi_base + C::kEpiBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::kStages + s); };

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int num_m = (M + BM - 1) / BM, num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    for (int s = 0; s < C::kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  auto tile_coords = [&](int t, int& m_blk, int& n_blk) {
    // rasterisation: a group of `group_m` row-blocks (its A panel sized to stay L2-resident) sweeps all
    // column-blocks, so A is read from HBM once and B once per group
    const int per_group = group_m * num_n;
    const int g = t / per_group;
    const int first_m = g * group_m;
    const int gsz = min(group_m, num_m - first_m);
    const int r = t - g * per_group;
    m_blk = first_m + (r % gsz);
    n_blk = r / gsz;
  };

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int s = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int m_blk, n_blk;
        tile_coords(t, m_blk, n_blk);
        const int m0 = m_blk * BM, n0 = n_blk * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(empty_bar(s), phase ^ 1);
          const uint32_t sa = smem_base + s * C::kStageBytes;
          const uint32_t sb = sa + C::kABytes;
          mbar_arrive_expect_tx(full_bar(s), C::kStageBytes);
          const int k0 = kb * BK;
          if constexpr (!A_MN) {
            tma_load_2d(sa, &tmap_a, full_bar(s), k0, m0);
          } else {
#pragma unroll
            for (int j = 0; j < BM / 64; ++j) tma_load_2d(sa + j * (BK * 128), &tmap_a, full_bar(s), m0 + 64 * j, k0);
          }
          if constexpr (!B_MN) {
            tma_load_2d(sb, &tmap_b, full_bar(s), k0, n0);
          } else {
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * (BK * 128), &tmap_b, full_bar(s), n0 + 64 * j, k0);
          }
          if (++s == C::kStages) { s = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: rows [64 c, 64 c + 64) of the tile
    setmaxnreg_inc<232>();
    const int c = wg - 1;
    const int tid = threadIdx.x & 127, warp_in_wg = tid >> 5;
    // both layouts place the 64-row half c at +8 KB: K-major = 64 rows x 128 B, MN-major = the c-th 64-wide M chunk
    constexpr uint32_t a_kstep = A_MN ? (16 * 128) : 32, b_kstep = B_MN ? (16 * 128) : 32;
    constexpr uint32_t a_lbo = A_MN ? (BK * 128) : 16, b_lbo = B_MN ? (BK * 128) : 16;
    float* stage = reinterpret_cast<float*>(smem_raw + (epi_base - smem_u32(smem_raw))) + c * 64 * kStageLd;
    const int er = tid & 63, ehalf = tid >> 6;   // epilogue: this thread's row of the 64 and 32-column half of a chunk
    int s = 0;
    uint32_t phase = 0;
    float d[BN / 2];
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      int m_blk, n_blk;
      tile_coords(t, m_blk, n_blk);
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(full_bar(s), phase);
        const uint32_t sa = smem_base + s * C::kStageBytes + c * (64 * 128);
        const uint32_t sb = smem_base + s * C::kStageBytes + C::kABytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_k16<BN, A_MN, B_MN>(d, wgmma_desc(sa + k * a_kstep, a_lbo), wgmma_desc(sb + k * b_kstep, b_lbo),
                                    (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(s));   // this warp's share of the stage has been read
        if (++s == C::kStages) { s = 0; phase ^= 1; }
      }
      // ---------------------------------------------------------------- epilogue, 64 columns at a time
      const int row = m_blk * BM + c * 64 + er;
      const bool row_ok = row < M;
      const int g = warp_in_wg * 16 + (lane >> 2), q2 = (lane & 3) * 2;
#pragma unroll
      for (int cc = 0; cc < BN / 64; ++cc) {
        const int colc = n_blk * BN + cc * 64;
        if (colc >= N) break;                                 // warpgroup-uniform
        asm volatile("bar.sync %0, 128;" ::"r"(1 + c) : "memory");   // the previous chunk has been read
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float* src = d + 4 * (cc * 8 + j);
          *reinterpret_cast<float2*>(stage + g * kStageLd + j * 8 + q2) = make_float2(src[0], src[1]);
          *reinterpret_cast<float2*>(stage + (g + 8) * kStageLd + j * 8 + q2) = make_float2(src[2], src[3]);
        }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + c) : "memory");
        const int col0 = colc + ehalf * 32;
        if (col0 < N) {
          float v[32];
          const float* rp = stage + er * kStageLd + ehalf * 32;
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 x = *reinterpret_cast<const float4*>(rp + j);
            v[j] = x.x * ep.alpha; v[j + 1] = x.y * ep.alpha; v[j + 2] = x.z * ep.alpha; v[j + 3] = x.w * ep.alpha;
          }
          epilogue_chunk(ep, v, row, row_ok, col0, N);
        }
      }
    }
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

// 2-D bf16 tensor: inner (contiguous) extent `inner`, outer extent `outer`, row pitch `ld` elements.
int make_tmap(CUtensorMap* tm, const void* base, long long inner, long long outer, long long ld,
              int box_inner, int box_outer) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) {
    mm_set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return MM_ERR_CUDA;
  }
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    mm_set_error("cuTensorMapEncodeTiled failed (%d): base=%p inner=%lld outer=%lld ld=%lld", (int)r,
                 base, inner, outer, ld);
    return MM_ERR_CUDA;
  }
  return MM_OK;
}

int env_group_m() {   // MM_GEMM_GM: rasterisation group size override (experiments; read once per process)
  static const int v = [] { const char* e = getenv("MM_GEMM_GM"); return e ? atoi(e) : 0; }();
  return v;
}

template <int BN, bool A_MN, bool B_MN>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, int M, int N, int K, const EpiParams& ep,
           cudaStream_t stream) {
  auto kern = gemm_wgmma_kernel<BN, A_MN, B_MN>;
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [&] {
    attr_err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::kSmemBytes);
  });
  MM_CHECK_CUDA(attr_err);
  const int num_tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
  const int grid = num_tiles < mm_num_sms() ? num_tiles : mm_num_sms();
  // Rasterisation group (row-blocks per group):
  //  * a wave of concurrently running tiles should be about square in bytes so that every k-slab fetched from HBM
  //    is shared by as many tiles as possible through L2: 132 SMs -> about 11 x 12 tiles;
  //  * when K is short the A panel of a group (gm * BM * K * 2 bytes) can stay L2-resident across the whole sweep
  //    over N, so B is streamed once per group: up to 16 MB, a third of the H100's 50 MB L2.
  long long gm = (16ll << 20) / ((long long)BM * K * 2);
  if (gm < 11) gm = 11;
  if (gm > 64) gm = 64;
  if (env_group_m() > 0) gm = env_group_m();
  kern<<<grid, kThreads, Cfg<BN>::kSmemBytes, stream>>>(ta, tb, M, N, K, (int)gm, ep);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

}  // namespace

// See include/metamorph_b200.h for the contract.
MM_API int mm_gemm_bf16(const void* A, const void* B, void* C, const void* bias,
                            const void* resid, void* aux, long long M, long long N, long long K,
                            long long lda, long long ldb, long long ldc, long long ldr,
                            long long ld_aux, int a_mn_major, int b_mn_major, int epilogue,
                            int out_f32, int accumulate, float alpha, int force_bn,
                            cudaStream_t stream) {
  MM_CHECK_ARG(M > 0 && N > 0 && K > 0, "mm_gemm_bf16: empty problem M=%lld N=%lld K=%lld", M, N, K);
  MM_CHECK_ARG(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31), "mm_gemm_bf16: dims too large");
  MM_CHECK_ARG(epilogue >= EPI_STORE && epilogue <= EPI_SWIGLU_BWD, "mm_gemm_bf16: bad epilogue %d",
               epilogue);
  if (epilogue == EPI_SWIGLU_BWD)
    MM_CHECK_ARG(N % 32 == 0 && !out_f32 && !accumulate && aux != nullptr && ld_aux % 8 == 0 &&
                     ((uintptr_t)aux & 15) == 0,
                 "mm_gemm_bf16: SWIGLU_BWD epilogue needs N%%32==0, bf16 out and a 16B-aligned gate|up buffer");
  MM_CHECK_ARG(((uintptr_t)A & 15) == 0 && ((uintptr_t)B & 15) == 0 && ((uintptr_t)C & 15) == 0,
               "mm_gemm_bf16: A/B/C must be 16-byte aligned");
  MM_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "mm_gemm_bf16: lda/ldb must be multiples of 8 elements");
  MM_CHECK_ARG(out_f32 ? (ldc % 4 == 0) : (ldc % 8 == 0), "mm_gemm_bf16: ldc alignment (ldc=%lld)", ldc);
  const bool needs_bias = epilogue == EPI_BIAS || epilogue == EPI_BIAS_GELU_ERF ||
                          epilogue == EPI_BIAS_GELU_TANH || epilogue == EPI_BIAS_RESID;
  const bool needs_res = epilogue == EPI_RESID || epilogue == EPI_BIAS_RESID;
  MM_CHECK_ARG(!needs_bias || bias != nullptr, "mm_gemm_bf16: epilogue %d needs bias", epilogue);
  MM_CHECK_ARG(!needs_res || (resid != nullptr && ldr % 8 == 0 && ((uintptr_t)resid & 15) == 0),
               "mm_gemm_bf16: epilogue %d needs 16B-aligned residual with ldr%%8==0", epilogue);
  if (epilogue == EPI_SWIGLU) {
    MM_CHECK_ARG(N % 32 == 0 && !out_f32 && !accumulate && !a_mn_major && !b_mn_major,
                 "mm_gemm_bf16: SWIGLU epilogue needs N%%32==0, bf16 out, K-major operands");
    MM_CHECK_ARG(aux == nullptr || (ld_aux % 8 == 0 && ((uintptr_t)aux & 15) == 0),
                 "mm_gemm_bf16: SWIGLU aux alignment");
  }
  MM_CHECK_ARG(!(a_mn_major && !b_mn_major), "mm_gemm_bf16: (A MN-major, B K-major) not instantiated");
  MM_CHECK_ARG(force_bn == 0 || force_bn == 128 || force_bn == 256, "mm_gemm_bf16: force_bn must be 0, 128 or 256 (got %d)",
               force_bn);

  // BN = 256 halves the B-operand traffic per flop; it needs a full wave of tiles to keep every SM busy.
  int bn = 256;
  if (force_bn == 128 || force_bn == 256) {
    bn = force_bn;
  } else {
    const long long tiles256 = ceil_div64(M, BM) * ceil_div64(N, 256);
    if (tiles256 < mm_num_sms() || N <= 128) bn = 128;
  }

  CUtensorMap ta, tb;
  int rc;
  if (!a_mn_major) rc = make_tmap(&ta, A, K, M, lda, BK, BM);       // A[M,K], K contiguous
  else             rc = make_tmap(&ta, A, M, K, lda, 64, BK);       // A stored [K,M], M contiguous
  if (rc) return rc;
  if (!b_mn_major) rc = make_tmap(&tb, B, K, N, ldb, BK, bn);       // B[N,K], K contiguous
  else             rc = make_tmap(&tb, B, N, K, ldb, 64, BK);       // B stored [K,N], N contiguous
  if (rc) return rc;

  EpiParams ep;
  ep.C = C; ep.ldc = ldc;
  ep.bias = reinterpret_cast<const bf16*>(bias);
  ep.resid = reinterpret_cast<const bf16*>(resid); ep.ldr = ldr;
  ep.aux = reinterpret_cast<bf16*>(aux); ep.ld_aux = ld_aux;
  ep.epi = epilogue; ep.out_f32 = out_f32; ep.accumulate = accumulate; ep.alpha = alpha;

  const int m = (int)M, n = (int)N, k = (int)K;
  if (bn == 256) {
    if (!a_mn_major && !b_mn_major) return launch<256, false, false>(ta, tb, m, n, k, ep, stream);
    if (!a_mn_major && b_mn_major) return launch<256, false, true>(ta, tb, m, n, k, ep, stream);
    return launch<256, true, true>(ta, tb, m, n, k, ep, stream);
  } else {
    if (!a_mn_major && !b_mn_major) return launch<128, false, false>(ta, tb, m, n, k, ep, stream);
    if (!a_mn_major && b_mn_major) return launch<128, false, true>(ta, tb, m, n, k, ep, stream);
    return launch<128, true, true>(ta, tb, m, n, k, ep, stream);
  }
}
