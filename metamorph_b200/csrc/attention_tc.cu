// metamorph_b200 — flash attention FORWARD on Hopper tensor cores (wgmma + TMA + mbarrier), head_dim 128.
// (SURVEY.md K12: LLaMA causal GQA attention, HF modeling_llama.py:199-220 / SDPA in 4.45.)
//
// One CTA = 128 query rows of one (batch, q-head), 1 CTA/SM; K/V tiles of 128 keys stream through a double-buffered
// TMA ring.
//   warpgroup 0, one thread : TMA producer
//   warpgroups 1, 2         : 64 query rows each. S_j = Q K_j^T (wgmma, both operands K-major in shared memory) lands
//                             in registers; the online softmax runs on the accumulator fragments (a row's 128 scores
//                             are spread over the 4 lanes of a quad); P_j is packed to bf16 in place and is the
//                             register A operand of O += P_j V_j (V MN-major from the same TMA tile).
// The backward lives in attention_bwd_tc.cu.
//
// PAGED (mm_attn_fwd_tc_paged): the same kernel for ONE sequence whose keys / values sit in a paged KV pool
// [num_blocks, Hkv, block_size, 128] addressed through a block-table row, and whose queries are the rows of positions
// q_start .. q_start + n_q - 1 only. Query tiles stay aligned to absolute multiples of 128, so a row meets the key tiles,
// mask decisions and consumer code of the dense kernel at T = q_start + n_q; the producer fills a 128-key tile with one
// TMA box per block (the 128B swizzle repeats every 8 rows, so boxes of >= 16 rows land where one box would); V rows at or
// past kv_len hold another request's data and are zeroed in shared memory, as the dense kernel's TMA zero fill would.
#include "attention_tc.cuh"

using namespace mm_attn_tc;

namespace {

constexpr int TC_BR = 128, TC_BC = 128, TC_D = 128;
constexpr int TC_TILE_BYTES = 128 * 128 * 2;  // 32 KB

struct TcFwdParams {
  bf16* o;
  float* lse;
  const int* seqlens;     // valid length per sequence (nullptr: T)
  const int* seg_start;   // packed layout: first row of every sequence in the [rows, width] operands (nullptr: b*T)
  const int2* work;       // packed layout: (sequence, query tile) of every CTA, heaviest first (nullptr: the grid itself)
  long long ldo;
  int B, T, Hq, Hkv;      // T = row pitch of lse and the largest sequence length
  float scale;
  int causal;
};

// paged addressing (PAGED only): tmap_k / tmap_v cover the pool as [num_blocks * Hkv * block_size, 128] rows with
// boxes of min(block_size, 128) rows; tmap_q covers the n_q query rows
struct TcPagedParams {
  const int* table;       // the sequence's block-table row
  int q_start;            // absolute position of query row 0; kv_len = p.T = q_start + n_q
  int bs_shift;           // log2(block_size)
};

constexpr int TC_THREADS = 384;
constexpr int TC_SMEM = 5 * TC_TILE_BYTES + 256 + 1024;

template <bool PAGED>
__global__ void __launch_bounds__(TC_THREADS, 1)
flash_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                       const __grid_constant__ CUtensorMap tmap_v, TcFwdParams p, TcPagedParams pg) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base;
  const uint32_t sK[2] = {base + TC_TILE_BYTES, base + 2 * TC_TILE_BYTES};
  const uint32_t sV[2] = {base + 3 * TC_TILE_BYTES, base + 4 * TC_TILE_BYTES};
  const uint32_t bar = base + 5 * TC_TILE_BYTES;
  const uint32_t q_full = bar, k_full0 = bar + 8, k_full1 = bar + 16, k_empty0 = bar + 24, k_empty1 = bar + 32,
                 v_full0 = bar + 40, v_full1 = bar + 48, v_empty0 = bar + 56, v_empty1 = bar + 64;

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  // padded batch: grid = (query tiles, heads, sequences), heavy (late) tiles first; packed sequences (SURVEY 8f N2):
  // grid.x walks a host-built list of the (sequence, query tile) pairs that exist, one launch for all segments
  int qt = p.work ? p.work[blockIdx.x].y : (int)gridDim.x - 1 - (int)blockIdx.x;
  if constexpr (PAGED) qt += pg.q_start / TC_BR;        // absolute tiles from the one holding q_start
  const int h = blockIdx.y, b = p.work ? p.work[blockIdx.x].x : (int)blockIdx.z;
  const int hk = h / (p.Hq / p.Hkv);
  const int q0 = qt * TC_BR;
  const int kv_len = p.seqlens ? min(p.seqlens[b], p.T) : p.T;
  int kv_end = kv_len;
  if (p.causal) kv_end = min(kv_end, q0 + TC_BR);
  const int n_tiles = (kv_end + TC_BC - 1) / TC_BC;
  const int tok0 = p.seg_start ? p.seg_start[b] : b * p.T;
  const int row_limit = p.seg_start ? kv_len : p.T;   // packed: rows past the sequence belong to the next one

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_q);
    prefetch_tmap(&tmap_k);
    prefetch_tmap(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(k_full0 + 8 * i, 1);
      mbar_init(v_full0 + 8 * i, 1);
      mbar_init(k_empty0 + 8 * i, 8);   // one arrive per consumer warp
      mbar_init(v_empty0 + 8 * i, 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      if (n_tiles > 0) {
        // paged: the operand holds rows q_start.. only; rows before it (negative coordinates) arrive as zero fill
        const int qrow = PAGED ? q0 - pg.q_start : tok0 + q0;
        mbar_arrive_expect_tx(q_full, TC_TILE_BYTES);
        tma_load_2d(sQ, &tmap_q, q_full, h * TC_D, qrow);
        tma_load_2d(sQ + 16384, &tmap_q, q_full, h * TC_D + 64, qrow);
      }
      for (int j = 0; j < n_tiles; ++j) {
        const int bf = j & 1;
        const uint32_t ph = (uint32_t)((j >> 1) & 1);
        if constexpr (PAGED) {
          // one box of sb rows per block; boxes starting at or past kv_len are not loaded (their keys are masked and
          // their values zeroed by the consumers)
          const int sb = min(TC_BC, 1 << pg.bs_shift), kv0 = j * TC_BC;
          const int nbox = (min(TC_BC, kv_len - kv0) + sb - 1) / sb;
          const uint32_t bytes = (uint32_t)(nbox * sb * 256);
          int prow[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if (i < nbox) {
              const int pos = kv0 + i * sb;
              const int blk = __ldg(pg.table + (pos >> pg.bs_shift));
              prow[i] = ((blk * p.Hkv + hk) << pg.bs_shift) + (pos & ((1 << pg.bs_shift) - 1));
            }
          }
          mbar_wait(bf ? k_empty1 : k_empty0, ph ^ 1);
          mbar_arrive_expect_tx(bf ? k_full1 : k_full0, bytes);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if (i < nbox) {
              const uint32_t off = (uint32_t)(i * sb * 128);
              tma_load_2d(sK[bf] + off, &tmap_k, bf ? k_full1 : k_full0, 0, prow[i]);
              tma_load_2d(sK[bf] + 16384 + off, &tmap_k, bf ? k_full1 : k_full0, 64, prow[i]);
            }
          }
          mbar_wait(bf ? v_empty1 : v_empty0, ph ^ 1);
          mbar_arrive_expect_tx(bf ? v_full1 : v_full0, bytes);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if (i < nbox) {
              const uint32_t off = (uint32_t)(i * sb * 128);
              tma_load_2d(sV[bf] + off, &tmap_v, bf ? v_full1 : v_full0, 0, prow[i]);
              tma_load_2d(sV[bf] + 16384 + off, &tmap_v, bf ? v_full1 : v_full0, 64, prow[i]);
            }
          }
          continue;
        }
        mbar_wait(bf ? k_empty1 : k_empty0, ph ^ 1);
        mbar_arrive_expect_tx(bf ? k_full1 : k_full0, TC_TILE_BYTES);
        tma_load_2d(sK[bf], &tmap_k, bf ? k_full1 : k_full0, hk * TC_D, tok0 + j * TC_BC);
        tma_load_2d(sK[bf] + 16384, &tmap_k, bf ? k_full1 : k_full0, hk * TC_D + 64, tok0 + j * TC_BC);
        mbar_wait(bf ? v_empty1 : v_empty0, ph ^ 1);
        mbar_arrive_expect_tx(bf ? v_full1 : v_full0, TC_TILE_BYTES);
        tma_load_2d(sV[bf], &tmap_v, bf ? v_full1 : v_full0, hk * TC_D, tok0 + j * TC_BC);
        tma_load_2d(sV[bf] + 16384, &tmap_v, bf ? v_full1 : v_full0, hk * TC_D + 64, tok0 + j * TC_BC);
      }
    }
    return;
  }

  setmaxnreg_inc<232>();
  const int c = wg - 1;
  const int g = ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2), q2 = (lane & 3) * 2;
  const int rows[2] = {q0 + c * 64 + g, q0 + c * 64 + g + 8};   // the two query rows of this thread
  const float sl2 = p.scale * kLog2e;
  const uint32_t sQc = sQ + (uint32_t)c * 8192u;                  // this warpgroup's 64 rows of the Q tile
  float o[64], sacc[64];
  float m_run[2] = {-INFINITY, -INFINITY}, l_part[2] = {0.f, 0.f};
  if (n_tiles > 0) mbar_wait(q_full, 0);
  for (int j = 0; j < n_tiles; ++j) {
    const int bf = j & 1;
    const uint32_t ph = (uint32_t)((j >> 1) & 1);
    mbar_wait(bf ? k_full1 : k_full0, ph);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TC_D / 16; ++k)
      wgmma_m64n128_ss<0, 0>(sacc, desc_kmajor(sQc, k), desc_kmajor(sK[bf], k), k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    consumer_release(bf ? k_empty1 : k_empty0);
    const bool need_mask = (j * TC_BC + TC_BC > kv_len) || (p.causal && j * TC_BC + TC_BC - 1 > q0);
    if (need_mask) {
#pragma unroll
      for (int t = 0; t < 64; ++t) {
        const int col = j * TC_BC + (t >> 2) * 8 + q2 + (t & 1);
        const int row = rows[(t >> 1) & 1];
        if (!((col < kv_len) && (!p.causal || col <= row))) sacc[t] = -INFINITY;
      }
    }
    float f[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int t = 0; t < 16; ++t) mx = fmaxf(mx, fmaxf(sacc[4 * t + 2 * i], sacc[4 * t + 2 * i + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[i], mx * sl2);
      f[i] = (m_new == -INFINITY) ? 1.f : fast_exp2(m_run[i] - m_new);
      m_run[i] = m_new;
      l_part[i] *= f[i];
      const float m_eff = (m_new == -INFINITY) ? 0.f : m_new;
#pragma unroll
      for (int t = 0; t < 16; ++t) {
        const float e0 = fast_exp2(fmaf(sacc[4 * t + 2 * i], sl2, -m_eff));   // masked: exp2(-inf) = 0
        const float e1 = fast_exp2(fmaf(sacc[4 * t + 2 * i + 1], sl2, -m_eff));
        l_part[i] += e0 + e1;
        sacc[4 * t + 2 * i] = e0;
        sacc[4 * t + 2 * i + 1] = e1;
      }
    }
    if (j > 0) {
#pragma unroll
      for (int t = 0; t < 64; ++t) o[t] *= f[(t >> 1) & 1];
    }
    uint32_t pa[TC_BC / 16][4];
#pragma unroll
    for (int k = 0; k < TC_BC / 16; ++k) acc_to_a(sacc, k, pa[k]);
    mbar_wait(bf ? v_full1 : v_full0, ph);
    if constexpr (PAGED) {
      // The tile straddling kv_len (the CTA's last, at most once): pool rows past kv_len are stale, possibly NaN, and
      // 0 * NaN would poison O. Zero them in both 64-column halves, as the dense kernel's TMA zero fill leaves them, then
      // make the generic-proxy stores visible to wgmma and wait for both consumer warpgroups.
      const int valid = kv_len - j * TC_BC;
      if (valid < TC_BC) {
        for (int idx = (int)threadIdx.x - 128; idx < (TC_BC - valid) * 16; idx += 256) {
          const uint32_t a = sV[bf] + (uint32_t)(idx & 8) * 2048u + (uint32_t)(valid + (idx >> 4)) * 128u +
                             (uint32_t)(idx & 7) * 16u;
          asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(a), "r"(0u) : "memory");
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
    }
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TC_BC / 16; ++k) wgmma_m64n128_rs<1>(o, pa[k], desc_mnmajor(sV[bf], k), (j | k) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    consumer_release(bf ? v_empty1 : v_empty0);
  }
  // epilogue: combine the quad's partial row sums, normalise, store
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_part[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = (n_tiles > 0 && l > 0.f) ? 1.f / l : 0.f;
    const int row = rows[i];
    bool keep = row < row_limit;
    if constexpr (PAGED) keep = keep && row >= pg.q_start;   // zero-filled query rows before q_start are never stored
    if (keep) {
      bf16* orow = p.o + (long long)(tok0 + row - (PAGED ? pg.q_start : 0)) * p.ldo + (long long)h * TC_D + q2;
#pragma unroll
      for (int t = 0; t < 16; ++t) {
        const float x0 = n_tiles > 0 ? o[4 * t + 2 * i] * inv : 0.f, x1 = n_tiles > 0 ? o[4 * t + 2 * i + 1] * inv : 0.f;
        *reinterpret_cast<uint32_t*>(orow + 8 * t) = pack_bf16x2(x0, x1);
      }
      if ((lane & 3) == 0 && p.lse != nullptr)
        p.lse[((long long)b * p.Hq + h) * p.T + row] = l > 0.f ? (m_run[i] + log2f(l)) / kLog2e : -INFINITY;
    }
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);

}  // namespace

static PFN_encodeTiled tmap_encoder() {
  static PFN_encodeTiled enc = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      enc = reinterpret_cast<PFN_encodeTiled>(fn);
  });
  if (!enc) mm_set_error("cuTensorMapEncodeTiled unavailable");
  return enc;
}

// fp32 statistics rows ([rows, width] contiguous, width % 128 == 0): box = 128 consecutive values of one row, no swizzle.
int mm_attn_make_tmap_stats(CUtensorMap* tm, const float* base, long long width, long long rows) {
  PFN_encodeTiled enc = tmap_encoder();
  if (!enc) return MM_ERR_CUDA;
  cuuint64_t dims[2] = {(cuuint64_t)width, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)width * 4};
  cuuint32_t box[2] = {128, 1};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    mm_set_error("cuTensorMapEncodeTiled failed (%d) for the attention statistics rows", (int)r);
    return MM_ERR_CUDA;
  }
  return MM_OK;
}

int mm_attn_make_tmap_rows(CUtensorMap* tm, const void* base, long long width, long long rows, long long ld,
                           int box_rows) {
  PFN_encodeTiled enc = tmap_encoder();
  if (!enc) return MM_ERR_CUDA;
  cuuint64_t dims[2] = {(cuuint64_t)width, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    mm_set_error("cuTensorMapEncodeTiled failed (%d) for attention operand", (int)r);
    return MM_ERR_CUDA;
  }
  return MM_OK;
}


namespace {

int launch_fwd_tc(const void* q, const void* k, const void* v, void* o, float* lse, const int* seqlens,
                  const int* seg_start, const int* work, int n_work, long long total_rows, long long ldq, long long ldk,
                  long long ldv, long long ldo, int B, int T, int Hq, int Hkv, int causal, float scale,
                  cudaStream_t stream) {
  MM_CHECK_ARG(B > 0 && T > 0 && Hq > 0 && Hkv > 0 && Hq % Hkv == 0, "mm_attn_fwd_tc: bad head counts");
  MM_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 &&
                   ((uintptr_t)q & 15) == 0 && ((uintptr_t)k & 15) == 0 && ((uintptr_t)v & 15) == 0 &&
                   ((uintptr_t)o & 15) == 0, "mm_attn_fwd_tc: 16-byte alignment / pitch %% 8 required");
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = mm_attn_make_tmap_rows(&tq, q, (long long)Hq * 128, total_rows, ldq))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&tk, k, (long long)Hkv * 128, total_rows, ldk))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&tv, v, (long long)Hkv * 128, total_rows, ldv))) return rc;
  TcFwdParams p;
  p.o = (bf16*)o; p.lse = lse; p.seqlens = seqlens; p.seg_start = seg_start;
  p.work = reinterpret_cast<const int2*>(work); p.ldo = ldo;
  p.B = B; p.T = T; p.Hq = Hq; p.Hkv = Hkv; p.scale = scale; p.causal = causal;
  const dim3 grid = work ? dim3(n_work, Hq, 1) : dim3((T + TC_BR - 1) / TC_BR, Hq, B);
  static std::once_flag once;
  static cudaError_t err = cudaSuccess;
  std::call_once(once, [&] {
    err = cudaFuncSetAttribute(flash_fwd_wgmma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM);
  });
  MM_CHECK_CUDA(err);
  flash_fwd_wgmma_kernel<false><<<grid, TC_THREADS, TC_SMEM, stream>>>(tq, tk, tv, p, TcPagedParams{});
  MM_CHECK_LAUNCH();
  return MM_OK;
}

// log2 of a block size in [16, 256], or -1 (the block sizes of mm_decode_attn_paged)
int paged_block_shift(int block_size) {
  if (block_size < 16 || block_size > 256 || (block_size & (block_size - 1))) return -1;
  return __builtin_ctz((unsigned)block_size);
}

}  // namespace

// wgmma flash-attention forward, head_dim 128. See include/metamorph_b200.h for the contract.
MM_API int mm_attn_fwd_tc(const void* q, const void* k, const void* v, void* o, float* lse,
                          const int* seqlens, long long ldq, long long ldk, long long ldv, long long ldo,
                          int B, int T, int Hq, int Hkv, int head_dim, int causal, float scale,
                          cudaStream_t stream) {
  MM_CHECK_ARG(head_dim == 128, "mm_attn_fwd_tc: head_dim must be 128");
  return launch_fwd_tc(q, k, v, o, lse, seqlens, nullptr, nullptr, 0, (long long)B * T, ldq, ldk, ldv, ldo, B, T, Hq, Hkv,
                       causal, scale, stream);
}

// Packed sequences (block-diagonal causal attention, one launch for all segments): sequence s occupies rows
// [seg_start[s], seg_start[s] + seg_len[s]) of the [total_rows, width] operands; lse is [n_seg, Hq, max_len];
// work = n_work (sequence, query tile) int pairs covering every tile with tile*128 < seg_len, heaviest first.
MM_API int mm_attn_fwd_tc_varlen(const void* q, const void* k, const void* v, void* o, float* lse,
                                 const int* seg_start, const int* seg_len, int n_seg, int max_len, const int* work,
                                 int n_work, long long total_rows, long long ldq, long long ldk, long long ldv,
                                 long long ldo, int Hq, int Hkv, int head_dim, float scale, cudaStream_t stream) {
  MM_CHECK_ARG(head_dim == 128, "mm_attn_fwd_tc_varlen: head_dim must be 128");
  MM_CHECK_ARG(seg_start != nullptr && seg_len != nullptr && work != nullptr && n_work > 0 && n_seg > 0 && max_len > 0,
               "mm_attn_fwd_tc_varlen: segment tables missing");
  return launch_fwd_tc(q, k, v, o, lse, seg_len, seg_start, work, n_work, total_rows, ldq, ldk, ldv, ldo, n_seg, max_len,
                       Hq, Hkv, 1, scale, stream);
}

// Causal attention of query rows at positions q_start .. q_start + n_q - 1 of ONE sequence (q: [n_q, ldq]) over keys
// and values 0 .. q_start + n_q - 1 in a paged pool (kpool / vpool [num_blocks, Hkv, block_size, 128], positions mapped
// by block_table_row as in mm_decode_attn_paged). o: [n_q, ldo]. No lse.
MM_API int mm_attn_fwd_tc_paged(const void* q, long long ldq, const void* kpool, const void* vpool, int num_blocks,
                                const int* block_table_row, int max_blocks, int block_size, void* o, long long ldo,
                                int q_start, int n_q, int Hq, int Hkv, int head_dim, float scale, cudaStream_t stream) {
  const int shift = paged_block_shift(block_size);
  MM_CHECK_ARG(shift >= 0, "mm_attn_fwd_tc_paged: block_size must be a power of two in [16,256] (got %d)", block_size);
  MM_CHECK_ARG(max_blocks >= 1, "mm_attn_fwd_tc_paged: max_blocks must be >= 1 (got %d)", max_blocks);
  MM_CHECK_ARG(block_table_row != nullptr, "mm_attn_fwd_tc_paged: block table missing");
  MM_CHECK_ARG(head_dim == 128, "mm_attn_fwd_tc_paged: head_dim must be 128");
  MM_CHECK_ARG(Hq > 0 && Hkv > 0 && Hq % Hkv == 0, "mm_attn_fwd_tc_paged: bad head counts");
  MM_CHECK_ARG(num_blocks >= 1 && (long long)num_blocks * Hkv * block_size < (1ll << 31),
               "mm_attn_fwd_tc_paged: num_blocks * Hkv * block_size must be in [1, 2^31)");
  MM_CHECK_ARG(q_start >= 0 && n_q >= 1, "mm_attn_fwd_tc_paged: need q_start >= 0 and n_q >= 1 (got %d, %d)", q_start,
               n_q);
  MM_CHECK_ARG((long long)q_start + n_q <= (long long)max_blocks * block_size,
               "mm_attn_fwd_tc_paged: q_start + n_q = %lld exceeds max_blocks * block_size = %lld",
               (long long)q_start + n_q, (long long)max_blocks * block_size);
  MM_CHECK_ARG(ldq % 8 == 0 && ldo % 8 == 0 && ((uintptr_t)q & 15) == 0 && ((uintptr_t)kpool & 15) == 0 &&
                   ((uintptr_t)vpool & 15) == 0 && ((uintptr_t)o & 15) == 0,
               "mm_attn_fwd_tc_paged: 16-byte alignment / pitch %% 8 required");
  const int sb = block_size < TC_BC ? block_size : TC_BC;
  const long long pool_rows = (long long)num_blocks * Hkv * block_size;
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = mm_attn_make_tmap_rows(&tq, q, (long long)Hq * 128, n_q, ldq))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&tk, kpool, 128, pool_rows, 128, sb))) return rc;
  if ((rc = mm_attn_make_tmap_rows(&tv, vpool, 128, pool_rows, 128, sb))) return rc;
  TcFwdParams p;
  p.o = (bf16*)o; p.lse = nullptr; p.seqlens = nullptr; p.seg_start = nullptr; p.work = nullptr; p.ldo = ldo;
  p.B = 1; p.T = q_start + n_q; p.Hq = Hq; p.Hkv = Hkv; p.scale = scale; p.causal = 1;
  TcPagedParams pg;
  pg.table = block_table_row; pg.q_start = q_start; pg.bs_shift = shift;
  const int qt0 = q_start / TC_BR, qt1 = (q_start + n_q - 1) / TC_BR;
  static std::once_flag once;
  static cudaError_t err = cudaSuccess;
  std::call_once(once, [&] {
    err = cudaFuncSetAttribute(flash_fwd_wgmma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM);
  });
  MM_CHECK_CUDA(err);
  flash_fwd_wgmma_kernel<true><<<dim3(qt1 - qt0 + 1, Hq, 1), TC_THREADS, TC_SMEM, stream>>>(tq, tk, tv, p, pg);
  MM_CHECK_LAUNCH();
  return MM_OK;
}
