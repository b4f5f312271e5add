// metamorph_b200 — loss kernels of the train step.
//   cross-entropy (SURVEY.md K15; metamorph_llama.py:402-413): shifted CE, mean over labels != -100.
//     The lm_head GEMM writes an fp32 logits chunk [R, V]; this kernel makes one online-softmax pass
//     (running max + sum, warp-shuffle + smem reduction) and one write pass that emits the gradient
//     d logits = (softmax - onehot) * grad_scale as bf16, ready to be the A operand of the dgrad /
//     wgrad GEMMs. Logits are never normalised in place and no [B,T,V] log-softmax is materialised.
//   visual-embedding regression (K16; metamorph_llama.py:433-453): L2-normalise the vision_head
//     output, -mean cosine similarity against the target SigLIP embedding, fused with its gradient.
//   argmax over the vocabulary for greedy decode (metamorph_llama.py:542).
#include "common.cuh"

namespace {

constexpr int kCEThreads = 512;

// Loss sums are accumulated as fixed-point integers (integer addition is exact, so the total does not depend on the
// order in which blocks finish); the last block of the launch converts the total and adds it to *loss_sum once.
// Non-finite terms are not lost: NaN (or +Inf together with -Inf) makes the sum NaN, +/-Inf makes it +/-Inf, as a float
// sum would. A finite term too large for the fixed-point range (`limit`, set so that no launch can overflow it) goes to
// an fp64 side sum. The accumulator lives in per-stream scratch (mm_stream_scratch) and is reset by the last block.
struct LossAcc {
  unsigned long long fixed;
  double big;
  unsigned int blocks;
  unsigned int flags;   // 1 NaN, 2 +Inf, 4 -Inf
};

__device__ __forceinline__ void loss_add(LossAcc* a, float v, double scale, float limit) {
  if (isnan(v)) atomicOr(&a->flags, 1u);
  else if (isinf(v)) atomicOr(&a->flags, v > 0.f ? 2u : 4u);
  else if (fabsf(v) < limit) atomicAdd(&a->fixed, (unsigned long long)llrint((double)v * scale));
  else atomicAdd(&a->big, (double)v);
}
// one thread per block, after every loss_add of the block
__device__ __forceinline__ void loss_block_done(LossAcc* a, double scale, float* loss_sum) {
  __threadfence();
  if (atomicAdd(&a->blocks, 1u) == gridDim.x - 1) {
    __threadfence();
    const long long fixed = (long long)atomicExch(&a->fixed, 0ull);
    const double big = __longlong_as_double((long long)atomicExch(reinterpret_cast<unsigned long long*>(&a->big), 0ull));
    const unsigned int f = atomicExch(&a->flags, 0u);
    a->blocks = 0;
    float tot;
    if ((f & 1u) || (f & 6u) == 6u) tot = NAN;
    else if (f & 2u) tot = INFINITY;
    else if (f & 4u) tot = -INFINITY;
    else tot = (float)((double)fixed / scale + big);
    *loss_sum += tot;
  }
}

// fixed-point scales of the two sums; limit = 2^62 / (scale * rows) keeps every launch inside int64
constexpr double kCEScale = 4294967296.0;            // 2^32: CE terms are O(10)
constexpr double kCosScale = 1099511627776.0;        // 2^40: cosine terms are -cos/R, at most 1 in magnitude
inline float loss_limit(double scale, long long rows) { return (float)(4611686018427387904.0 / (scale * (double)(rows > 0 ? rows : 1))); }

__global__ void __launch_bounds__(kCEThreads)
ce_fwd_bwd_kernel(const float* __restrict__ logits, long long ld, const int* __restrict__ labels,
                  bf16* __restrict__ dlogits, long long ld_d, float* __restrict__ loss_sum, LossAcc* __restrict__ acc,
                  float limit, float* __restrict__ lse_out, int V, float grad_scale, int ignore_index) {
  __shared__ float red[32];
  const long long row = blockIdx.x;
  const float* x = logits + row * ld;
  const int label = labels[row];
  const bool valid = (label != ignore_index);
  bf16* dx = dlogits ? dlogits + row * ld_d : nullptr;
  if (!valid && lse_out == nullptr) {
    if (dx != nullptr) {
      for (long long j = threadIdx.x * 8; j < ld_d; j += kCEThreads * 8)
        *reinterpret_cast<int4*>(dx + j) = make_int4(0, 0, 0, 0);
    }
    if (threadIdx.x == 0 && loss_sum != nullptr) loss_block_done(acc, kCEScale, loss_sum);
    return;
  }
  // pass 1: online max / sum(exp)
  float m = -INFINITY, s = 0.f;
  const int V4 = V & ~3;
  for (int j = threadIdx.x * 4; j < V4; j += kCEThreads * 4) {
    const float4 v = *reinterpret_cast<const float4*>(x + j);
    const float mx = fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w));
    if (mx > m) {
      s *= __expf(m - mx);
      m = mx;
    }
    s += __expf(v.x - m) + __expf(v.y - m) + __expf(v.z - m) + __expf(v.w - m);
  }
  for (int j = V4 + threadIdx.x; j < V; j += kCEThreads) {
    const float v = x[j];
    if (v > m) {
      s *= __expf(m - v);
      m = v;
    }
    s += __expf(v - m);
  }
  const float gm = block_max(m, red);
  s *= (m == -INFINITY) ? 0.f : __expf(m - gm);
  const float gs = block_sum(s, red);
  const float lse = gm + logf(gs);
  if (threadIdx.x == 0) {
    if (lse_out != nullptr) lse_out[row] = lse;
    if (loss_sum != nullptr) {
      if (valid) loss_add(acc, lse - x[label], kCEScale, limit);
      loss_block_done(acc, kCEScale, loss_sum);
    }
  }
  if (dx == nullptr) return;
  // pass 2: gradient
  const float sc = valid ? grad_scale : 0.f;
  const int V8 = V & ~7;
  for (int j = threadIdx.x * 8; j < V8; j += kCEThreads * 8) {
    const float4 a = *reinterpret_cast<const float4*>(x + j);
    const float4 b = *reinterpret_cast<const float4*>(x + j + 4);
    float p[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int t = 0; t < 8; ++t) p[t] = (__expf(p[t] - lse) - ((j + t) == label ? 1.f : 0.f)) * sc;
    *reinterpret_cast<int4*>(dx + j) = make_int4(pack_bf16x2(p[0], p[1]), pack_bf16x2(p[2], p[3]),
                                                 pack_bf16x2(p[4], p[5]), pack_bf16x2(p[6], p[7]));
  }
  for (long long j = V8 + threadIdx.x; j < ld_d; j += kCEThreads) {
    float g = 0.f;
    if (j < V) g = (__expf(x[j] - lse) - (j == label ? 1.f : 0.f)) * sc;
    dx[j] = __float2bfloat16(g);
  }
}

// one warp per row
__global__ void cosine_loss_kernel(const bf16* __restrict__ pred, const bf16* __restrict__ target,
                                   bf16* __restrict__ pred_norm, bf16* __restrict__ dpred,
                                   float* __restrict__ loss_sum, LossAcc* __restrict__ acc, float limit,
                                   long long R, int C, float grad_scale) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nvec = C >> 3;
  for (long long r = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < R;
       r += (long long)gridDim.x * warps_per_block) {
    const bf16* pr = pred + r * C;
    const bf16* tr = target ? target + r * C : nullptr;
    float pp = 0.f;
    for (int v = lane; v < nvec; v += 32) {
      const int4 a = *reinterpret_cast<const int4*>(pr + v * 8);
      const uint32_t u[4] = {(uint32_t)a.x, (uint32_t)a.y, (uint32_t)a.z, (uint32_t)a.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        pp += f.x * f.x + f.y * f.y;
      }
    }
    pp = warp_sum(pp);
    // F.normalize(pred): bf16 norm, clamp 1e-12, bf16 divide
    const float pn = fmaxf(__bfloat162float(__float2bfloat16(sqrtf(pp))), 1e-12f);
    float tp = 0.f, tt = 0.f, hh = 0.f;
    for (int v = lane; v < nvec; v += 32) {
      const int4 a = *reinterpret_cast<const int4*>(pr + v * 8);
      const uint32_t u[4] = {(uint32_t)a.x, (uint32_t)a.y, (uint32_t)a.z, (uint32_t)a.w};
      uint32_t tu[4] = {0, 0, 0, 0};
      if (tr != nullptr) {
        const int4 b = *reinterpret_cast<const int4*>(tr + v * 8);
        tu[0] = b.x; tu[1] = b.y; tu[2] = b.z; tu[3] = b.w;
      }
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        const float2 t = unpack_bf16x2(tu[j]);
        o[j] = pack_bf16x2(f.x / pn, f.y / pn);
        const float2 h = unpack_bf16x2(o[j]);
        tp += t.x * h.x + t.y * h.y;
        tt += t.x * t.x + t.y * t.y;
        hh += h.x * h.x + h.y * h.y;
      }
      if (pred_norm != nullptr)
        *reinterpret_cast<int4*>(pred_norm + r * C + v * 8) = make_int4(o[0], o[1], o[2], o[3]);
    }
    if (tr == nullptr) continue;
    tp = warp_sum(tp);
    tt = warp_sum(tt);
    hh = warp_sum(hh);
    const float tn = fmaxf(sqrtf(tt), 1e-8f), hn = fmaxf(sqrtf(hh), 1e-8f);
    const float cosv = tp / (tn * hn);
    if (lane == 0 && loss_sum != nullptr) loss_add(acc, -cosv / (float)R, kCosScale, limit);
    if (dpred != nullptr) {
      // d(-mean cos)/d pred = -(1/R) * (t_hat - cos * p_hat) / |pred|
      const float g = -grad_scale / ((float)R * pn);
      for (int v = lane; v < nvec; v += 32) {
        const int4 a = *reinterpret_cast<const int4*>(pr + v * 8);
        const int4 b = *reinterpret_cast<const int4*>(tr + v * 8);
        const uint32_t u[4] = {(uint32_t)a.x, (uint32_t)a.y, (uint32_t)a.z, (uint32_t)a.w};
        const uint32_t tu[4] = {(uint32_t)b.x, (uint32_t)b.y, (uint32_t)b.z, (uint32_t)b.w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(u[j]);
          const float2 t = unpack_bf16x2(tu[j]);
          o[j] = pack_bf16x2(g * (t.x / tn - cosv * f.x / pn), g * (t.y / tn - cosv * f.y / pn));
        }
        *reinterpret_cast<int4*>(dpred + r * C + v * 8) = make_int4(o[0], o[1], o[2], o[3]);
      }
    }
  }
  if (loss_sum != nullptr) {
    __syncthreads();
    if (threadIdx.x == 0) loss_block_done(acc, kCosScale, loss_sum);
  }
}

// argmax over V fp32 logits per row, two stages so that a handful of rows still fills the GPU:
// stage 1: grid (R, kArgmaxSplits) partial (value, index) per slice; stage 2: one warp per row.
// Ties resolve to the smallest index (deterministic). NaN never compares greater, so it is never chosen; a row with no
// value above -inf (all -inf, all NaN, or a mix of the two) gives 0, as the sampler does, so the token is always in [0, V).
constexpr int kArgmaxSplits = 64;

__device__ __forceinline__ void argmax_combine(float& best, int& bi, float ov, int oi) {
  if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
}

__global__ void __launch_bounds__(256)
argmax_partial_kernel(const float* __restrict__ logits, long long ld, int V, float* __restrict__ pval,
                      int* __restrict__ pidx) {
  __shared__ float sval[8];
  __shared__ int sidx[8];
  const int r = blockIdx.x, sp = blockIdx.y;
  const int per = (V + kArgmaxSplits - 1) / kArgmaxSplits;
  const int j0 = sp * per, j1 = min(V, j0 + per);
  const float* x = logits + (long long)r * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = j0 + threadIdx.x; j < j1; j += blockDim.x) {
    const float v = x[j];
    if (v > best) { best = v; bi = j; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    argmax_combine(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
  if ((threadIdx.x & 31) == 0) { sval[threadIdx.x >> 5] = best; sidx[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) argmax_combine(best, bi, sval[w], sidx[w]);
    pval[r * kArgmaxSplits + sp] = best;
    pidx[r * kArgmaxSplits + sp] = bi;
  }
}

__global__ void argmax_final_kernel(const float* __restrict__ pval, const int* __restrict__ pidx,
                                    int* __restrict__ out) {
  const int r = blockIdx.x, lane = threadIdx.x;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int s = lane; s < kArgmaxSplits; s += 32) argmax_combine(best, bi, pval[r * kArgmaxSplits + s], pidx[r * kArgmaxSplits + s]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    argmax_combine(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
  if (lane == 0) out[r] = bi != 0x7fffffff ? bi : 0;
}

}  // namespace

MM_API int mm_ce_fwd_bwd(const float* logits, long long ld, const int* labels, void* dlogits,
                         long long ld_d, float* loss_sum, float* lse_out, long long R, int V,
                         float grad_scale, int ignore_index, cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && V > 0 && ld >= V && ld % 4 == 0, "mm_ce_fwd_bwd: need ld>=V and ld%%4==0");
  MM_CHECK_ARG(dlogits == nullptr || (ld_d >= V && ld_d % 8 == 0), "mm_ce_fwd_bwd: need ld_d>=V, ld_d%%8==0");
  LossAcc* acc = nullptr;
  if (loss_sum != nullptr && (acc = static_cast<LossAcc*>(mm_stream_scratch(MM_SCRATCH_LOSS, sizeof(LossAcc), stream))) == nullptr)
    return MM_ERR_CUDA;
  ce_fwd_bwd_kernel<<<(unsigned)R, kCEThreads, 0, stream>>>(logits, ld, labels, (bf16*)dlogits, ld_d,
                                                            loss_sum, acc, loss_limit(kCEScale, R), lse_out, V,
                                                            grad_scale, ignore_index);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_cosine_loss(const void* pred, const void* target, void* pred_norm, void* dpred,
                          float* loss_sum, long long R, int C, float grad_scale,
                          cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && C % 8 == 0, "mm_cosine_loss: need C%%8==0");
  long long blocks = ceil_div64(R, 4);
  if (blocks > (long long)mm_num_sms() * 8) blocks = (long long)mm_num_sms() * 8;
  LossAcc* acc = nullptr;
  if (loss_sum != nullptr && (acc = static_cast<LossAcc*>(mm_stream_scratch(MM_SCRATCH_LOSS, sizeof(LossAcc), stream))) == nullptr)
    return MM_ERR_CUDA;
  cosine_loss_kernel<<<(int)blocks, 128, 0, stream>>>((const bf16*)pred, (const bf16*)target,
                                                      (bf16*)pred_norm, (bf16*)dpred, loss_sum, acc,
                                                      loss_limit(kCosScale, R), R, C, grad_scale);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

// workspace: R * 64 floats followed by R * 64 ints (mm_argmax_workspace_bytes)
MM_API long long mm_argmax_workspace_bytes(long long R) { return R * kArgmaxSplits * 8; }

MM_API int mm_argmax_rows(const float* logits, long long ld, long long R, int V, int* out, void* workspace,
                          long long workspace_bytes, cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && V > 0 && ld >= V, "mm_argmax_rows: bad shape");
  MM_CHECK_ARG(workspace != nullptr && workspace_bytes >= mm_argmax_workspace_bytes(R),
               "mm_argmax_rows: workspace too small");
  float* pval = reinterpret_cast<float*>(workspace);
  int* pidx = reinterpret_cast<int*>(pval + R * kArgmaxSplits);
  argmax_partial_kernel<<<dim3((unsigned)R, kArgmaxSplits), 256, 0, stream>>>(logits, ld, V, pval, pidx);
  MM_CHECK_LAUNCH();
  argmax_final_kernel<<<(unsigned)R, 32, 0, stream>>>(pval, pidx, out);
  MM_CHECK_LAUNCH();
  return MM_OK;
}
