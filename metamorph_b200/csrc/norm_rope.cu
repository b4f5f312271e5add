// metamorph_b200 — RMSNorm (fwd/bwd), LayerNorm (fwd) and rotary embedding kernels.
// HBM-bound: one pass over each tensor, 128-bit accesses, fp32 statistics via warp shuffles.
//   RMSNorm   : HF LlamaRMSNorm (modeling_llama.py:53-67)   y = w * bf16(x * rsqrt(mean(x^2)+eps))
//   LayerNorm : SigLIP pre-LN (modeling_siglip.py:348,357)  eps 1e-6, affine
//   RoPE      : HF apply_rotary_pos_emb (modeling_llama.py:146-168), rotate-half convention
#include "common.cuh"

namespace {

constexpr int kNormThreads = 256;
constexpr int kMaxVec = 4;  // 8-element vectors per thread => H <= 8192

// ---------------------------------------------------------------------------------- RMSNorm fwd
// Row r + gridDim.x is requested BEFORE the reduction of row r (as in the backward below): every block keeps a second row
// of HBM reads in flight across its barrier; the weight vector lives in registers (packed). One __syncthreads per row.
template <int VPT>   // 8-element vectors per thread (H <= 8 * 256 * VPT)
__global__ void __launch_bounds__(kNormThreads, (VPT <= 2 ? 4 : 1))
rmsnorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y,
                   int M, int H, float eps) {
  __shared__ float red[2][kNormThreads / 32];
  const int nvec = H >> 3;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int4 wp[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * kNormThreads;
    wp[i] = v < nvec ? *reinterpret_cast<const int4*>(w + v * 8) : make_int4(0, 0, 0, 0);   // weights: never written by a kernel
  }
  griddep_launch();
  griddep_wait();
  int4 nx[VPT];
  auto fetch = [&](int row) {
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * kNormThreads;
      nx[i] = (row < M && v < nvec) ? ld_nc_int4(x + (size_t)row * H + v * 8) : make_int4(0, 0, 0, 0);
    }
  };
  fetch(blockIdx.x);
  int par = 0;
  for (int row = blockIdx.x; row < M; row += gridDim.x, par ^= 1) {
    float xv[VPT][8];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const uint32_t u[4] = {(uint32_t)nx[i].x, (uint32_t)nx[i].y, (uint32_t)nx[i].z, (uint32_t)nx[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        xv[i][2 * j] = f.x;
        xv[i][2 * j + 1] = f.y;
        ss += f.x * f.x + f.y * f.y;
      }
    }
    fetch(row + gridDim.x);                  // in flight across the reduction below
    ss = warp_sum(ss);
    if (lane == 0) red[par][warp] = ss;
    __syncthreads();
    float tss = 0.f;
#pragma unroll
    for (int k = 0; k < kNormThreads / 32; ++k) tss += red[par][k];
    const float rstd = rsqrtf(tss / (float)H + eps);
    bf16* yr = y + (size_t)row * H;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * kNormThreads;
      if (v < nvec) {
        const uint32_t wu[4] = {(uint32_t)wp[i].x, (uint32_t)wp[i].y, (uint32_t)wp[i].z, (uint32_t)wp[i].w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 wf = unpack_bf16x2(wu[j]);
          // reference rounds the normalised activation to bf16 before the weight multiply
          const float n0 = __bfloat162float(__float2bfloat16(xv[i][2 * j] * rstd));
          const float n1 = __bfloat162float(__float2bfloat16(xv[i][2 * j + 1] * rstd));
          o[j] = pack_bf16x2(wf.x * n0, wf.y * n1);
        }
        *reinterpret_cast<int4*>(yr + v * 8) = make_int4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------- RMSNorm bwd
// dx = dres_in + rstd*dy*w - x * rstd^3 * sum(dy*w*x)/H ;  dw += sum_rows dy * x * rstd
// Every block stores its fp32 dw partial (the rows it owns) to a scratch row; rmsnorm_dw_reduce_kernel then adds the
// partials in block order, so the weight gradient is the same bits on every run (no float atomics).
// Both row statistics (sum x^2 and sum dy*w*x) come from ONE pass and ONE block reduction per row
// (double-buffered smem scratch -> a single __syncthreads per row).
// The loads of row r + gridDim.x (x, dy and the residual gradient: 6 of the 8 bytes per element the kernel moves) are
// issued BEFORE the reduction of row r, so every block keeps two rows of HBM traffic in flight across its barrier
// (round 1 loaded one row, reduced, and only then fetched the residual gradient: 41 % of the HBM peak).
template <int VPT>   // 8-element vectors per thread (H <= 8 * 256 * VPT): sized to H so registers stay low
__global__ void __launch_bounds__(kNormThreads, (VPT <= 2 ? 2 : 1))
rmsnorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                   const bf16* __restrict__ w, const bf16* __restrict__ dres_in,
                   bf16* __restrict__ dx, float* __restrict__ dw_part, int M, int H, float eps) {
  __shared__ float red[2][2][kNormThreads / 32];
  const int nvec = H >> 3;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float dwp[VPT][8];
  float wv[VPT][8];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int v = threadIdx.x + i * kNormThreads;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      dwp[i][j] = 0.f;
      wv[i][j] = (v < nvec) ? __bfloat162float(w[v * 8 + j]) : 0.f;
    }
  }
  int4 nx[VPT], ng[VPT], nr[VPT];          // the next row, still packed
  auto fetch = [&](int row) {
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * kNormThreads;
      if (row < M && v < nvec) {
        nx[i] = ld_nc_int4(x + (size_t)row * H + v * 8);
        ng[i] = ld_nc_int4(dy + (size_t)row * H + v * 8);
        nr[i] = dres_in != nullptr ? ld_nc_int4(dres_in + (size_t)row * H + v * 8) : make_int4(0, 0, 0, 0);
      } else {
        nx[i] = ng[i] = nr[i] = make_int4(0, 0, 0, 0);
      }
    }
  };
  fetch(blockIdx.x);
  int par = 0;
  for (int row = blockIdx.x; row < M; row += gridDim.x, par ^= 1) {
    float xv[VPT][8], gv[VPT][8];
    int4 rres[VPT];
    float ss = 0.f, gwx = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const uint32_t ux[4] = {(uint32_t)nx[i].x, (uint32_t)nx[i].y, (uint32_t)nx[i].z, (uint32_t)nx[i].w};
      const uint32_t ug[4] = {(uint32_t)ng[i].x, (uint32_t)ng[i].y, (uint32_t)ng[i].z, (uint32_t)ng[i].w};
      rres[i] = nr[i];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(ux[j]);
        const float2 g = unpack_bf16x2(ug[j]);
        xv[i][2 * j] = f.x; xv[i][2 * j + 1] = f.y;
        gv[i][2 * j] = g.x; gv[i][2 * j + 1] = g.y;
        ss += f.x * f.x + f.y * f.y;
        gwx += g.x * wv[i][2 * j] * f.x + g.y * wv[i][2 * j + 1] * f.y;
      }
    }
    fetch(row + gridDim.x);                  // in flight across the reduction below
    ss = warp_sum(ss);
    gwx = warp_sum(gwx);
    if (lane == 0) { red[par][0][warp] = ss; red[par][1][warp] = gwx; }
    __syncthreads();
    float tss = 0.f, tg = 0.f;
#pragma unroll
    for (int k = 0; k < kNormThreads / 32; ++k) { tss += red[par][0][k]; tg += red[par][1][k]; }
    const float rstd = rsqrtf(tss / (float)H + eps);
    const float coef = rstd * rstd * rstd * tg / (float)H;
    bf16* dxr = dx + (size_t)row * H;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * kNormThreads;
      if (v < nvec) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          o[j] = rstd * gv[i][j] * wv[i][j] - xv[i][j] * coef;
          dwp[i][j] += gv[i][j] * xv[i][j] * rstd;
        }
        if (dres_in != nullptr) {
          const uint32_t ur[4] = {(uint32_t)rres[i].x, (uint32_t)rres[i].y, (uint32_t)rres[i].z, (uint32_t)rres[i].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = unpack_bf16x2(ur[j]);
            o[2 * j] += f.x;
            o[2 * j + 1] += f.y;
          }
        }
        *reinterpret_cast<int4*>(dxr + v * 8) =
            make_int4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]),
                      pack_bf16x2(o[6], o[7]));
      }
    }
  }
  if (dw_part != nullptr) {
    float* part = dw_part + (size_t)blockIdx.x * H;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int v = threadIdx.x + i * kNormThreads;
      if (v < nvec) {
        *reinterpret_cast<float4*>(part + v * 8) = make_float4(dwp[i][0], dwp[i][1], dwp[i][2], dwp[i][3]);
        *reinterpret_cast<float4*>(part + v * 8 + 4) = make_float4(dwp[i][4], dwp[i][5], dwp[i][6], dwp[i][7]);
      }
    }
  }
}

// dw[c] += sum over the n_part block partials of column c, in block order
__global__ void rmsnorm_dw_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw, int n_part, int H) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  float s = 0.f;
  for (int b = 0; b < n_part; ++b) s += part[(size_t)b * H + c];
  dw[c] += s;
}


// ---------------------------------------------------------------------------------- LayerNorm fwd
__global__ void __launch_bounds__(kNormThreads)
layernorm_fwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                     const bf16* __restrict__ b, bf16* __restrict__ y, int M, int H, float eps) {
  __shared__ float red[32];
  const int nvec = H >> 3;
  for (int row = blockIdx.x; row < M; row += gridDim.x) {
    const bf16* xr = x + (size_t)row * H;
    float xv[kMaxVec][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int v = threadIdx.x + i * kNormThreads;
      if (v < nvec) {
        const int4 raw = *reinterpret_cast<const int4*>(xr + v * 8);
        const uint32_t u[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(u[j]);
          xv[i][2 * j] = f.x; xv[i][2 * j + 1] = f.y;
          s += f.x + f.y;
        }
      }
    }
    const float mean = block_sum(s, red) / (float)H;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int v = threadIdx.x + i * kNormThreads;
      if (v < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = xv[i][j] - mean;
          ss += d * d;
        }
      }
    }
    const float rstd = rsqrtf(block_sum(ss, red) / (float)H + eps);
    bf16* yr = y + (size_t)row * H;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int v = threadIdx.x + i * kNormThreads;
      if (v < nvec) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
          o[j] = (xv[i][j] - mean) * rstd * __bfloat162float(w[v * 8 + j]) +
                 __bfloat162float(b[v * 8 + j]);
        *reinterpret_cast<int4*>(yr + v * 8) =
            make_int4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]),
                      pack_bf16x2(o[6], o[7]));
      }
    }
  }
}

// ---------------------------------------------------------------------------------- RoPE
// In-place rotate-half on the first `n_rot_heads` heads of each row of a [M, ld] buffer.
// cos/sin: fp32 tables [n_pos, d/2]; pos[M] int32. `sign` = +1 forward, -1 backward (transpose).
__global__ void rope_kernel(bf16* __restrict__ qkv, const int* __restrict__ pos,
                            const float* __restrict__ cos_t, const float* __restrict__ sin_t, int M,
                            long long ld, int n_rot_heads, int d, float sign) {
  const int half = d >> 1;
  const int vec_per_head = half >> 3;
  const long long total = (long long)M * n_rot_heads * vec_per_head;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % vec_per_head);
    const long long t = idx / vec_per_head;
    const int head = (int)(t % n_rot_heads);
    const int row = (int)(t / n_rot_heads);
    bf16* p = qkv + (size_t)row * ld + head * d + v * 8;
    const int4 lo = *reinterpret_cast<const int4*>(p);
    const int4 hi = *reinterpret_cast<const int4*>(p + half);
    const float* cp = cos_t + (size_t)pos[row] * half + v * 8;
    const float* sp = sin_t + (size_t)pos[row] * half + v * 8;
    const uint32_t ul[4] = {(uint32_t)lo.x, (uint32_t)lo.y, (uint32_t)lo.z, (uint32_t)lo.w};
    const uint32_t uh[4] = {(uint32_t)hi.x, (uint32_t)hi.y, (uint32_t)hi.z, (uint32_t)hi.w};
    uint32_t ol[4], oh[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a = unpack_bf16x2(ul[j]);
      const float2 b = unpack_bf16x2(uh[j]);
      const float c0 = cp[2 * j], c1 = cp[2 * j + 1];
      const float s0 = sign * sp[2 * j], s1 = sign * sp[2 * j + 1];
      ol[j] = pack_bf16x2(rope_lo(a.x, b.x, c0, s0), rope_lo(a.y, b.y, c1, s1));
      oh[j] = pack_bf16x2(rope_hi(a.x, b.x, c0, s0), rope_hi(a.y, b.y, c1, s1));
    }
    *reinterpret_cast<int4*>(p) = make_int4(ol[0], ol[1], ol[2], ol[3]);
    *reinterpret_cast<int4*>(p + half) = make_int4(oh[0], oh[1], oh[2], oh[3]);
  }
}

int norm_grid(int M) {
  const int cap = mm_num_sms() * 8;
  return M < cap ? M : cap;
}

}  // namespace

MM_API int mm_rmsnorm_fwd(const void* x, const void* w, void* y, long long M, long long H, float eps,
                          cudaStream_t stream) {
  MM_CHECK_ARG(M > 0 && H > 0 && H % 8 == 0 && H <= 8 * kNormThreads * kMaxVec,
               "mm_rmsnorm_fwd: need H%%8==0 and H<=%d (H=%lld)", 8 * kNormThreads * kMaxVec, H);
  const int vpt = (int)((H / 8 + kNormThreads - 1) / kNormThreads);
  const int cap = mm_num_sms() * (vpt <= 2 ? 8 : 2);     // resident blocks per SM x 2 (tail balance)
  const dim3 grid(M < cap ? (int)M : cap);
#define MM_RMS_FWD(V)                                                                                                \
  MM_CHECK_CUDA(launch_pdl(mm_pdl_mode() & 2, rmsnorm_fwd_kernel<V>, grid, dim3(kNormThreads), 0, stream, (const bf16*)x, \
                           (const bf16*)w, (bf16*)y, (int)M, (int)H, eps))
  if (vpt <= 1) MM_RMS_FWD(1);
  else if (vpt == 2) MM_RMS_FWD(2);
  else MM_RMS_FWD(4);
#undef MM_RMS_FWD
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_rmsnorm_bwd(const void* dy, const void* x, const void* w, const void* dres_in, void* dx,
                          float* dw_accum, long long M, long long H, float eps, cudaStream_t stream) {
  MM_CHECK_ARG(M > 0 && H > 0 && H % 8 == 0 && H <= 8 * kNormThreads * kMaxVec,
               "mm_rmsnorm_bwd: need H%%8==0 and H<=%d (H=%lld)", 8 * kNormThreads * kMaxVec, H);
  const int cap = mm_num_sms() * 4;       // 2 resident blocks per SM x 2 (tail balance)
  const int grid = M < cap ? (int)M : cap;
  const int vpt = (int)((H / 8 + kNormThreads - 1) / kNormThreads);
  float* part = nullptr;
  if (dw_accum != nullptr) {
    part = static_cast<float*>(mm_stream_scratch(MM_SCRATCH_RMSNORM_DW, (size_t)grid * H * sizeof(float), stream));
    if (part == nullptr) return MM_ERR_CUDA;
  }
#define MM_RMS_BWD(V)                                                                                      \
  rmsnorm_bwd_kernel<V><<<grid, kNormThreads, 0, stream>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w, \
                                                           (const bf16*)dres_in, (bf16*)dx, part, (int)M, \
                                                           (int)H, eps)
  if (vpt <= 1) MM_RMS_BWD(1);
  else if (vpt == 2) MM_RMS_BWD(2);
  else MM_RMS_BWD(4);
#undef MM_RMS_BWD
  MM_CHECK_LAUNCH();
  if (dw_accum != nullptr) {
    rmsnorm_dw_reduce_kernel<<<(unsigned)((H + 255) / 256), 256, 0, stream>>>(part, dw_accum, grid, (int)H);
    MM_CHECK_LAUNCH();
  }
  return MM_OK;
}

MM_API int mm_layernorm_fwd(const void* x, const void* w, const void* b, void* y, long long M,
                            long long H, float eps, cudaStream_t stream) {
  MM_CHECK_ARG(M > 0 && H > 0 && H % 8 == 0 && H <= 8 * kNormThreads * kMaxVec,
               "mm_layernorm_fwd: need H%%8==0 and H<=%d (H=%lld)", 8 * kNormThreads * kMaxVec, H);
  layernorm_fwd_kernel<<<norm_grid((int)M), kNormThreads, 0, stream>>>(
      (const bf16*)x, (const bf16*)w, (const bf16*)b, (bf16*)y, (int)M, (int)H, eps);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_rope_inplace(void* qkv, const int* pos, const float* cos_t, const float* sin_t,
                           long long M, long long ld, int n_rot_heads, int head_dim, int backward,
                           cudaStream_t stream) {
  MM_CHECK_ARG(M > 0 && head_dim % 16 == 0 && ld % 8 == 0 && n_rot_heads > 0,
               "mm_rope_inplace: need head_dim%%16==0, ld%%8==0");
  const long long total = M * n_rot_heads * (head_dim / 16);
  const int threads = 256;
  long long blocks = ceil_div64(total, threads);
  const long long cap = (long long)mm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  rope_kernel<<<(int)blocks, threads, 0, stream>>>((bf16*)qkv, pos, cos_t, sin_t, (int)M, ld,
                                                   n_rot_heads, head_dim, backward ? -1.f : 1.f);
  MM_CHECK_LAUNCH();
  return MM_OK;
}
