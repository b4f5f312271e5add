// metamorph_b200 — weight-streaming GEMM of the decode step for 33..128 sequences (row A9).
//
//   skinny_gemm_wide  y[m<=128, N] = x[m, K] * W[N, K]^T with the epilogues of skinny_gemm (decode.cu). Swap-AB on
//                     wgmma: the M=64 operand is a slab of W (rows = output features), the N=128 operand is the batch,
//                     both K-major, 128B-swizzled and delivered by TMA (batch rows >= m are zero-filled). One TMA producer
//                     warp feeds a 3-deep ring of [128 weight rows + 128 batch rows] x 64 k stages to two consumer
//                     warpgroups (64 weight rows each) that share the activation stage. K is split over a cluster of S
//                     CTAs; their fp32 partial tiles are added through distributed shared memory in rank order, with no
//                     float atomics. S depends only on (N, K, #SMs), and the batch operand is always 128 wide, so a row's
//                     bits do not depend on m.
#include <cooperative_groups.h>
#include <mutex>

#include "common.cuh"
#include "fp8.cuh"
#include "wgmma.cuh"

namespace cg = cooperative_groups;

typedef CUresult (*PFN_encodeTiledWide)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                        CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                        CUtensorMapFloatOOBfill);

namespace {

enum WideEpi : int { SK_STORE = 0, SK_BIAS = 1, SK_RESID = 2, SK_BIAS_GELU = 3, SK_SWIGLU = 4 };

constexpr int kRows = 128;                      // weight rows per CTA: two consumer warpgroups x 64
constexpr int kMB = 128;                        // batch rows of the activation operand (the wgmma N)
constexpr int kBK = 64;                         // k per stage (one 128-byte swizzle row)
constexpr int kStages = 3;
constexpr int kWBytes = kRows * kBK * 2;        // 16 KB weight box
constexpr int kXBytes = kMB * kBK * 2;          // 16 KB activation box
constexpr int kStageBytes = kWBytes + kXBytes;
constexpr int kThreads = 288;                   // warps 0..7 = consumer warpgroups 0 and 1, warp 8 = TMA producer
constexpr int kPLd = kRows + 4;                 // partial tile [batch][weight row] fp32 pitch (conflict-free stores)
constexpr int kBarOff = kStages * kStageBytes;
constexpr int kSmem = kBarOff + 128 + 1024;     // ring + barriers + alignment slack
constexpr int kMaxSplits = 8;                   // portable cluster size
static_assert(kMB * kPLd * 4 <= kStages * kStageBytes, "the partial tile reuses the ring");
// FP8 weights (skinny_gemm_wide_fp8_kernel): a stage holds the [128 rows x 64 k] E4M3 box (64 bytes a row, unswizzled) and
// the same activation box; each consumer warpgroup expands its 64 rows into a 128B-swizzled bf16 tile, the layout the
// bf16 kernel's TMA writes, in one of two tiles it alternates between.
constexpr int kWBytes8 = kRows * kBK;           // 8 KB E4M3 weight box
constexpr int kStageBytes8 = kWBytes8 + kXBytes;
constexpr int kExpOff8 = kStages * kStageBytes8;                 // 2 tiles x [128 rows x 64 k] bf16
constexpr int kBarOff8 = kExpOff8 + 2 * kWBytes;
constexpr int kSmem8 = kBarOff8 + 128 + 1024;
static_assert(kMB * kPLd * 4 <= kStages * kStageBytes8, "the partial tile reuses the FP8 ring");
static_assert(kXBytes % 1024 == 0 && kWBytes8 % 1024 == 0, "128B-swizzled tiles need 1024-byte alignment");

template <bool FP8>
__device__ __forceinline__ void
skinny_gemm_wide_body(const CUtensorMap& tmap_w, const CUtensorMap& tmap_x, void* __restrict__ y, long long ldy,
                      const bf16* __restrict__ bias, const bf16* __restrict__ resid, long long ldr, int m, int N, int K,
                      int epi, int out_f32, const float* __restrict__ wsc, long long lds) {
  constexpr int kSB = FP8 ? kStageBytes8 : kStageBytes;   // bytes of one ring stage
  constexpr int kWB = FP8 ? kWBytes8 : kWBytes;           // of which weights
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t bar = base + (FP8 ? kBarOff8 : kBarOff);   // full[s] = bar + 8 s, empty[s] = bar + 8 (kStages + s)
  cg::cluster_group cluster = cg::this_cluster();
  const int S = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int n0 = (blockIdx.x / S) * kRows;
  const int nk = (K + kBK - 1) / kBK;
  const int kt0 = (int)((long long)nk * rank / S);              // this CTA's k stages [kt0, kt1), never empty (S <= nk)
  const int n_kt = (int)((long long)nk * (rank + 1) / S) - kt0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_w);
    prefetch_tmap(&tmap_x);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(bar + 8 * s, 1);                 // full: the producer's expect_tx
      mbar_init(bar + 8 * (kStages + s), 8);     // empty: one arrive per consumer warp
    }
    fence_barrier_init();
  }
  griddep_launch();
  __syncthreads();
  float d[64];
  if (warp == 8) {
    if (lane == 0) {
      // Weights never change during a step: the first stages' weights are requested before waiting for the previous
      // kernel; the activations, which that kernel produces, follow after the wait.
      const int n_pre = n_kt < kStages ? n_kt : kStages;
      for (int i = 0; i < n_pre; ++i) {
        mbar_arrive_expect_tx(bar + 8 * i, kSB);
        tma_load_2d(base + i * kSB, &tmap_w, bar + 8 * i, (kt0 + i) * kBK, n0);
      }
      griddep_wait();
      for (int i = 0; i < n_pre; ++i)
        tma_load_2d(base + i * kSB + kWB, &tmap_x, bar + 8 * i, (kt0 + i) * kBK, 0);
      for (int i = n_pre; i < n_kt; ++i) {
        const int s = i % kStages;
        mbar_wait(bar + 8 * (kStages + s), (uint32_t)(((i / kStages) & 1) ^ 1));
        mbar_arrive_expect_tx(bar + 8 * s, kSB);
        tma_load_2d(base + s * kSB, &tmap_w, bar + 8 * s, (kt0 + i) * kBK, n0);
        tma_load_2d(base + s * kSB + kWB, &tmap_x, bar + 8 * s, (kt0 + i) * kBK, 0);
      }
    }
  } else {
    const int wg = warp >> 2;
#pragma unroll
    for (int j = 0; j < 64; ++j) d[j] = 0.f;
    if constexpr (FP8) {
      // Thread tw of the warpgroup expands rows 16 j + tw / 8 (j < 4) of its 64, 16-byte bf16 chunk tw % 8 (8 k), of
      // stage i into tile i & 1. Stage i + 1 is expanded while the wgmmas of stage i run; tile (i + 1) & 1 was last read
      // by the wgmmas of stage i - 1, which every warp of the warpgroup has waited for before the barrier ending i - 1.
      const int tw = threadIdx.x & 127, c = tw & 7;
      auto expand = [&](int i) {
        const int s = i % kStages, grp = (kt0 + i) >> 1;
        float sc[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {                  // requested before the stage wait
          const int n = n0 + wg * 64 + 16 * j + (tw >> 3);
          sc[j] = n < N ? __ldg(wsc + (long long)n * lds + grp) : 1.f;
        }
        mbar_wait(bar + 8 * s, (uint32_t)((i / kStages) & 1));
        const uint8_t* src = base_ptr + s * kSB + wg * (64 * kBK);
        uint8_t* dst = base_ptr + kExpOff8 + (i & 1) * kWBytes + wg * (64 * 128);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int r = 16 * j + (tw >> 3);
          const uint2 q = *reinterpret_cast<const uint2*>(src + r * kBK + c * 8);
          const uint2 lo = fp8x4_to_bf16x4(q.x, sc[j]), hi = fp8x4_to_bf16x4(q.y, sc[j]);
          *reinterpret_cast<uint4*>(dst + r * 128 + ((c ^ (r & 7)) << 4)) = make_uint4(lo.x, lo.y, hi.x, hi.y);
        }
        fence_proxy_async_smem();                      // the generic-proxy stores, before wgmma reads them
      };
      expand(0);
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
      for (int i = 0; i < n_kt; ++i) {
        const int s = i % kStages;
        const uint32_t sa = base + kExpOff8 + (i & 1) * kWBytes + wg * (64 * 128);
        const uint32_t sb = base + s * kSB + kWB;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)
          wgmma_m64n128_ss<0, 0>(d, wgmma_desc(sa + k * 32, 16), wgmma_desc(sb + k * 32, 16), 1u);
        wgmma_commit();
        if (i + 1 < n_kt) expand(i + 1);
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar + 8 * (kStages + s));   // stage s (E4M3 box and activations) is consumed
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
      }
    } else {
      for (int i = 0; i < n_kt; ++i) {
        const int s = i % kStages;
        mbar_wait(bar + 8 * s, (uint32_t)((i / kStages) & 1));
        const uint32_t sa = base + s * kSB + wg * (64 * 128);   // this warpgroup's 64 weight rows
        const uint32_t sb = base + s * kSB + kWB;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)
          wgmma_m64n128_ss<0, 0>(d, wgmma_desc(sa + k * 32, 16), wgmma_desc(sb + k * 32, 16), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar + 8 * (kStages + s));
      }
    }
  }
  __syncthreads();                               // every stage has been consumed: the ring holds the partial tile now
  float* part = reinterpret_cast<float*>(base_ptr);   // [kMB batch rows][kPLd] fp32, weight row fastest
  if (warp < 8) {
    // accumulator of warp w of warpgroup wg: d[4j + 0..1] = weight row 16w + g, batch 8j + 2t + {0,1}; d[4j + 2..3] = row + 8
    const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2), t = lane & 3;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int b = 8 * j + 2 * t;
      part[b * kPLd + r0] = d[4 * j];
      part[(b + 1) * kPLd + r0] = d[4 * j + 1];
      part[b * kPLd + r0 + 8] = d[4 * j + 2];
      part[(b + 1) * kPLd + r0 + 8] = d[4 * j + 3];
    }
  }
  griddep_wait();                                // resid and y belong to the kernels before this one
  cluster.sync();                                // every CTA's partial tile is complete
  // Each output element is the sum of the S partial tiles in rank order, whichever CTA finishes it (they are spread over
  // the cluster, consecutive weight rows on consecutive threads so that stores run along n).
  // A thread finishes kU elements per pass and issues all their loads of one rank before adding them, so the distributed
  // shared memory latency is paid once per rank and pass rather than once per element.
  constexpr int kU = 4;
  const int stride = S * kThreads;
  const bool swiglu = epi == SK_SWIGLU;
  const int per_b = swiglu ? kRows / 2 : kRows;  // outputs per batch row of the slab
  const int total = m * per_b;
  for (int e0 = rank * kThreads + threadIdx.x; e0 < total; e0 += kU * stride) {
    int off[kU], b[kU], c[kU];
    bool ok[kU];
    float acc[kU], up[kU], add[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int e = e0 + u * stride;
      b[u] = e / per_b;
      c[u] = e % per_b;
      // SwiGLU: rows of the slab are [16 gate | 16 up] per group of 32 (engine/packing.py interleave_gate_up)
      const int r = swiglu ? (c[u] >> 4) * 32 + (c[u] & 15) : c[u];
      ok[u] = e < total && n0 + r < N;
      off[u] = b[u] * kPLd + r;
      add[u] = 0.f;
      if (ok[u] && (epi == SK_BIAS || epi == SK_BIAS_GELU)) add[u] = __bfloat162float(bias[n0 + r]);
      if (ok[u] && epi == SK_RESID) add[u] = __bfloat162float(resid[(long long)b[u] * ldr + n0 + r]);
      acc[u] = up[u] = 0.f;
    }
    for (int q = 0; q < S; ++q) {                // rank order: the same sum for every element whatever m is
      const float* pq = cluster.map_shared_rank(part, q);
      float v[kU], w[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        v[u] = ok[u] ? pq[off[u]] : 0.f;
        w[u] = ok[u] && swiglu ? pq[off[u] + 16] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        acc[u] = q == 0 ? v[u] : acc[u] + v[u];
        up[u] = q == 0 ? w[u] : up[u] + w[u];
      }
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      if (!ok[u]) continue;
      if (swiglu) {
        reinterpret_cast<bf16*>(y)[(long long)b[u] * ldy + (n0 >> 1) + c[u]] = __float2bfloat16(silu(acc[u]) * up[u]);
        continue;
      }
      float sacc = acc[u];
      if (epi == SK_BIAS || epi == SK_BIAS_GELU || epi == SK_RESID) sacc += add[u];
      if (epi == SK_BIAS_GELU) sacc = gelu_erf(sacc);
      const long long o = (long long)b[u] * ldy + n0 + c[u];
      if (out_f32) reinterpret_cast<float*>(y)[o] = sacc;
      else reinterpret_cast<bf16*>(y)[o] = __float2bfloat16(sacc);
    }
  }
  cluster.sync();                                // keep this CTA's partial tile alive until the cluster has read it
}

__global__ void __launch_bounds__(kThreads, 2)
skinny_gemm_wide_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                        void* __restrict__ y, long long ldy, const bf16* __restrict__ bias,
                        const bf16* __restrict__ resid, long long ldr, int m, int N, int K, int epi, int out_f32) {
  skinny_gemm_wide_body<false>(tmap_w, tmap_x, y, ldy, bias, resid, ldr, m, N, K, epi, out_f32, nullptr, 0);
}

// wsc: the fp32 scale of row n, k group j (k in [128 j, 128 j + 128)) at wsc[n * lds + j]. On W-hat = float(q) * scale the
// output bits are skinny_gemm_wide_kernel's: the expanded tile is the one its TMA writes, and the wgmma sequence, the
// split and the reduction are unchanged.
__global__ void __launch_bounds__(kThreads, 2)
skinny_gemm_wide_fp8_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                            void* __restrict__ y, long long ldy, const bf16* __restrict__ bias,
                            const bf16* __restrict__ resid, long long ldr, int m, int N, int K, int epi, int out_f32,
                            const float* __restrict__ wsc, long long lds) {
  skinny_gemm_wide_body<true>(tmap_w, tmap_x, y, ldy, bias, resid, ldr, m, N, K, epi, out_f32, wsc, lds);
}

// Split-K factor: grow the cluster until the CTAs cover ~90 % of the SMs, keeping at least two k stages per CTA. A function
// of (N, K, #SMs) only, so the summation order of a row never depends on the batch.
int wide_splits(int N, int K) {
  const int slabs = (N + kRows - 1) / kRows, nk = (K + kBK - 1) / kBK, sms = mm_num_sms();
  int s = 1;
  while (s < kMaxSplits && 10 * slabs * s < 9 * sms && 2 * (s + 1) <= nk) ++s;
  return s;
}

}  // namespace

namespace {

// mm_skinny_gemm_wide and mm_skinny_gemm_wide_fp8; `name` prefixes the error messages. FP8: W holds E4M3 bytes (ldw in
// bytes) and wsc the scales.
template <bool FP8>
int skinny_gemm_wide_launch(const char* name, const void* x, const void* W, const float* wsc, void* y, const void* bias,
                            const void* resid, long long ldx, long long ldw, long long lds, long long ldy, long long ldr,
                            int m, int N, int K, int epilogue, int out_f32, cudaStream_t stream) {
  MM_CHECK_ARG(m >= 1 && m <= 128, "%s: batch must be in [1,128] (m=%d)", name, m);
  MM_CHECK_ARG(N >= 1 && K >= 32, "%s: need N>=1, K>=32", name);
  if constexpr (FP8) {
    MM_CHECK_ARG(K % 128 == 0 && ldx % 8 == 0 && ldw % 16 == 0 && ldw >= K,
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
  if (epilogue == SK_SWIGLU) MM_CHECK_ARG(N % 32 == 0 && !out_f32, "%s: SWIGLU needs N%%32==0", name);
  static PFN_encodeTiledWide enc = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      enc = reinterpret_cast<PFN_encodeTiledWide>(fn);
  });
  MM_CHECK_ARG(enc != nullptr, "%s: cuTensorMapEncodeTiled unavailable", name);
  CUtensorMap tw, tx;
  cuuint32_t estr[2] = {1, 1};
  {
    // bf16: 128B-swizzled [128 rows x 64 k] box; FP8: the same rows and k as an unswizzled 64-byte-wide uint8 box
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
    cuuint64_t strides[1] = {(cuuint64_t)ldw * (FP8 ? 1 : 2)};
    cuuint32_t box[2] = {kBK, kRows};
    CUresult r = enc(&tw, FP8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(W),
                     dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     FP8 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MM_CHECK_ARG(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled(W) failed (%d)", name, (int)r);
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)m};            // batch rows >= m of the box are zero-filled
    cuuint64_t strides[1] = {(cuuint64_t)ldx * 2};
    cuuint32_t box[2] = {kBK, kMB};
    CUresult r = enc(&tx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(x), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MM_CHECK_ARG(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled(x) failed (%d)", name, (int)r);
  }
  constexpr int smem = FP8 ? kSmem8 : kSmem;
  static std::once_flag attr_once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once, [] {
    if constexpr (FP8)
      attr_err = cudaFuncSetAttribute(skinny_gemm_wide_fp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    else
      attr_err = cudaFuncSetAttribute(skinny_gemm_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  });
  MM_CHECK_CUDA(attr_err);
  const int S = wide_splits(N, K);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(((N + kRows - 1) / kRows) * S));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)S;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 2;
  if constexpr (FP8)
    MM_CHECK_CUDA(cudaLaunchKernelEx(&cfg, skinny_gemm_wide_fp8_kernel, tw, tx, y, ldy, (const bf16*)bias,
                                     (const bf16*)resid, ldr, m, N, K, epilogue, out_f32, wsc, lds));
  else
    MM_CHECK_CUDA(cudaLaunchKernelEx(&cfg, skinny_gemm_wide_kernel, tw, tx, y, ldy, (const bf16*)bias,
                                     (const bf16*)resid, ldr, m, N, K, epilogue, out_f32));
  MM_CHECK_LAUNCH();
  return MM_OK;
}

}  // namespace

MM_API int mm_skinny_gemm_wide(const void* x, const void* W, void* y, const void* bias, const void* resid,
                               long long ldx, long long ldw, long long ldy, long long ldr, int m, int N, int K,
                               int epilogue, int out_f32, cudaStream_t stream) {
  return skinny_gemm_wide_launch<false>("mm_skinny_gemm_wide", x, W, nullptr, y, bias, resid, ldx, ldw, 0, ldy, ldr, m,
                                        N, K, epilogue, out_f32, stream);
}

MM_API int mm_skinny_gemm_wide_fp8(const void* x, const void* Wq, const float* wscale, void* y, const void* bias,
                                   const void* resid, long long ldx, long long ldw, long long lds, long long ldy,
                                   long long ldr, int m, int N, int K, int epilogue, int out_f32, cudaStream_t stream) {
  return skinny_gemm_wide_launch<true>("mm_skinny_gemm_wide_fp8", x, Wq, wscale, y, bias, resid, ldx, ldw, lds, ldy, ldr,
                                       m, N, K, epilogue, out_f32, stream);
}
