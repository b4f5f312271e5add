// metamorph_b200 — HBM-bound elementwise kernels of the train step (128-bit accesses, grid-stride):
//   swiglu_bwd     : (gate|up interleaved, dact) -> act (recompute), d(gate|up)   [LlamaMLP bwd]
//   gelu fwd/bwd   : erf GELU of mm_projector / vision_head (projector builder.py:55-59)
//   colsum         : bias gradient (sum over rows)
//   im2col_patch14 : SigLIP patch-embed Conv2d(k=s=14) as GEMM operand (modeling_siglip.py:178-184)
//   add_pos_emb    : + learned position embedding
//   sumsq          : squared gradient norm for clipping (per-block partials added in a fixed order by a second launch)
#include "common.cuh"

namespace {

// gu: [M, 2I] with every 32-column chunk = [16 gate | 16 up]; dact/act: [M, I]
__global__ void swiglu_bwd_kernel(const bf16* __restrict__ gu, const bf16* __restrict__ dact,
                                  bf16* __restrict__ dgu, bf16* __restrict__ act, long long M,
                                  long long I) {
  const long long chunks_per_row = I / 16;
  const long long total = M * chunks_per_row * 2;  // one thread = 8 gate + 8 up columns
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int halfsel = (int)(idx & 1);
    const long long c = (idx >> 1) % chunks_per_row;
    const long long row = (idx >> 1) / chunks_per_row;
    const bf16* gp = gu + row * 2 * I + c * 32 + halfsel * 8;
    const int4 graw = *reinterpret_cast<const int4*>(gp);
    const int4 uraw = *reinterpret_cast<const int4*>(gp + 16);
    const long long acol = c * 16 + halfsel * 8;
    const int4 draw = *reinterpret_cast<const int4*>(dact + row * I + acol);
    const uint32_t ug[4] = {(uint32_t)graw.x, (uint32_t)graw.y, (uint32_t)graw.z, (uint32_t)graw.w};
    const uint32_t uu[4] = {(uint32_t)uraw.x, (uint32_t)uraw.y, (uint32_t)uraw.z, (uint32_t)uraw.w};
    const uint32_t ud[4] = {(uint32_t)draw.x, (uint32_t)draw.y, (uint32_t)draw.z, (uint32_t)draw.w};
    uint32_t og[4], ou[4], oa[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 g = unpack_bf16x2(ug[j]);
      const float2 u = unpack_bf16x2(uu[j]);
      const float2 d = unpack_bf16x2(ud[j]);
      const float s0 = 1.f / (1.f + __expf(-g.x)), s1 = 1.f / (1.f + __expf(-g.y));
      const float a0 = g.x * s0, a1 = g.y * s1;  // silu(g)
      oa[j] = pack_bf16x2(a0 * u.x, a1 * u.y);
      og[j] = pack_bf16x2(d.x * u.x * (s0 + a0 * (1.f - s0)), d.y * u.y * (s1 + a1 * (1.f - s1)));
      ou[j] = pack_bf16x2(d.x * a0, d.y * a1);
    }
    bf16* dgp = dgu + row * 2 * I + c * 32 + halfsel * 8;
    *reinterpret_cast<int4*>(dgp) = make_int4(og[0], og[1], og[2], og[3]);
    *reinterpret_cast<int4*>(dgp + 16) = make_int4(ou[0], ou[1], ou[2], ou[3]);
    if (act != nullptr)
      *reinterpret_cast<int4*>(act + row * I + acol) = make_int4(oa[0], oa[1], oa[2], oa[3]);
  }
}

__global__ void gelu_fwd_kernel(const bf16* __restrict__ z, bf16* __restrict__ a, long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const int4 raw = *reinterpret_cast<const int4*>(z + i * 8);
    const uint32_t u[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(u[j]);
      o[j] = pack_bf16x2(gelu_erf(f.x), gelu_erf(f.y));
    }
    *reinterpret_cast<int4*>(a + i * 8) = make_int4(o[0], o[1], o[2], o[3]);
  }
}

__global__ void gelu_bwd_kernel(const bf16* __restrict__ z, const bf16* __restrict__ da,
                                bf16* __restrict__ dz, long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const int4 raw = *reinterpret_cast<const int4*>(z + i * 8);
    const int4 graw = *reinterpret_cast<const int4*>(da + i * 8);
    const uint32_t u[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
    const uint32_t g[4] = {(uint32_t)graw.x, (uint32_t)graw.y, (uint32_t)graw.z, (uint32_t)graw.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(u[j]);
      const float2 d = unpack_bf16x2(g[j]);
      o[j] = pack_bf16x2(d.x * gelu_erf_grad(f.x), d.y * gelu_erf_grad(f.y));
    }
    *reinterpret_cast<int4*>(dz + i * 8) = make_int4(o[0], o[1], o[2], o[3]);
  }
}

// out[n] (+)= sum_r x[r, n]. One block owns 64 columns (32 column pairs x 8 row phases); each thread adds its rows in
// order and the 8 phases are combined in order, so the sum does not depend on scheduling (bias gradients are the same
// bits on every run).
__global__ void __launch_bounds__(256) colsum_kernel(const bf16* __restrict__ x, float* __restrict__ out, long long R,
                                                     long long N, long long ld) {
  __shared__ float2 part[8][32];
  const long long col = ((long long)blockIdx.x * 32 + threadIdx.x) * 2;
  float s0 = 0.f, s1 = 0.f;
  if (col < N) {
    for (long long r = threadIdx.y; r < R; r += 8) {
      const float2 f = __bfloat1622float2(*reinterpret_cast<const bf162*>(x + r * ld + col));
      s0 += f.x;
      s1 += f.y;
    }
  }
  part[threadIdx.y][threadIdx.x] = make_float2(s0, s1);
  __syncthreads();
  if (threadIdx.y != 0 || col >= N) return;
  for (int k = 1; k < 8; ++k) {
    s0 += part[k][threadIdx.x].x;
    s1 += part[k][threadIdx.x].y;
  }
  out[col] += s0;
  if (col + 1 < N) out[col + 1] += s1;
}

// images [N,3,S,S] (bf16, NCHW) -> patches [N*(S/14)^2, ldp]; column = c*196 + ky*14 + kx
// (matches Conv2d weight [O, 3, 14, 14] flattened); columns >= 588 are zero padding.
__global__ void im2col_patch14_kernel(const bf16* __restrict__ img, bf16* __restrict__ out, int N,
                                      int S, int ldp) {
  const int G = S / 14;
  const long long rows = (long long)N * G * G;
  const long long total = rows * ldp;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(idx % ldp);
    const long long row = idx / ldp;
    bf16 v = __float2bfloat16(0.f);
    if (col < 588) {
      const int c = col / 196, rem = col % 196, ky = rem / 14, kx = rem % 14;
      const int n = (int)(row / (G * G)), p = (int)(row % (G * G)), py = p / G, px = p % G;
      v = img[(((size_t)n * 3 + c) * S + (py * 14 + ky)) * S + (px * 14 + kx)];
    }
    out[idx] = v;
  }
}

// x[r, :] += pos[r % P, :]
__global__ void add_pos_emb_kernel(bf16* __restrict__ x, const bf16* __restrict__ pos, long long R,
                                   int P, int H) {
  const long long nvec = R * (H / 8);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / (H / 8);
    const int v = (int)(i % (H / 8));
    const int4 a = *reinterpret_cast<const int4*>(x + r * H + v * 8);
    const int4 b = *reinterpret_cast<const int4*>(pos + (size_t)(r % P) * H + v * 8);
    const uint32_t ua[4] = {(uint32_t)a.x, (uint32_t)a.y, (uint32_t)a.z, (uint32_t)a.w};
    const uint32_t ub[4] = {(uint32_t)b.x, (uint32_t)b.y, (uint32_t)b.z, (uint32_t)b.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(ua[j]);
      const float2 g = unpack_bf16x2(ub[j]);
      o[j] = pack_bf16x2(f.x + g.x, f.y + g.y);
    }
    *reinterpret_cast<int4*>(x + r * H + v * 8) = make_int4(o[0], o[1], o[2], o[3]);
  }
}

// part[b] = sum of x^2 over the elements block b owns (grid-stride). Each thread adds its elements in order and the block
// reduction has a fixed shape, so every partial is a function of (x, grid) only. No float atomics: sumsq_finish_kernel
// adds the partials in a fixed order, so the gradient norm (and the clip coefficient) is the same bits on every run.
__global__ void sumsq_bf16_kernel(const bf16* __restrict__ x, float* __restrict__ part, long long n8) {
  __shared__ float red[32];
  float s = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const int4 raw = ld_nc_int4(x + i * 8);
    const uint32_t u[4] = {(uint32_t)raw.x, (uint32_t)raw.y, (uint32_t)raw.z, (uint32_t)raw.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(u[j]);
      s += f.x * f.x + f.y * f.y;
    }
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// *out += sum of the n_part partials. One warp: lane l adds partials l, l+32, l+64, ... in block order (fp64), then lane
// 0 adds the 32 lane sums in lane order and rounds once to fp32.
__global__ void sumsq_finish_kernel(const float* __restrict__ part, float* __restrict__ out, int n_part) {
  __shared__ double lane_sum[32];
  double s = 0.0;
  for (int b = threadIdx.x; b < n_part; b += 32) s += (double)part[b];
  lane_sum[threadIdx.x] = s;
  __syncwarp();
  if (threadIdx.x != 0) return;
  double total = 0.0;
  for (int l = 0; l < 32; ++l) total += lane_sum[l];
  *out = (float)((double)*out + total);
}

int ew_grid(long long work_items, int threads) {
  long long b = ceil_div64(work_items, threads);
  const long long cap = (long long)mm_num_sms() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

MM_API int mm_swiglu_bwd(const void* gu, const void* dact, void* dgu, void* act, long long M,
                         long long I, cudaStream_t stream) {
  MM_CHECK_ARG(M > 0 && I > 0 && I % 16 == 0, "mm_swiglu_bwd: need I%%16==0 (I=%lld)", I);
  const long long total = M * (I / 16) * 2;
  swiglu_bwd_kernel<<<ew_grid(total, 256), 256, 0, stream>>>((const bf16*)gu, (const bf16*)dact,
                                                             (bf16*)dgu, (bf16*)act, M, I);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_gelu_fwd(const void* z, void* a, long long n, cudaStream_t stream) {
  MM_CHECK_ARG(n > 0 && n % 8 == 0, "mm_gelu_fwd: n%%8 != 0");
  gelu_fwd_kernel<<<ew_grid(n / 8, 256), 256, 0, stream>>>((const bf16*)z, (bf16*)a, n / 8);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_gelu_bwd(const void* z, const void* da, void* dz, long long n, cudaStream_t stream) {
  MM_CHECK_ARG(n > 0 && n % 8 == 0, "mm_gelu_bwd: n%%8 != 0");
  gelu_bwd_kernel<<<ew_grid(n / 8, 256), 256, 0, stream>>>((const bf16*)z, (const bf16*)da,
                                                           (bf16*)dz, n / 8);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_colsum_accum(const void* x, float* out, long long R, long long N, long long ld,
                           cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && N > 0 && N % 2 == 0 && ld % 2 == 0, "mm_colsum_accum: N, ld must be even");
  colsum_kernel<<<(unsigned)ceil_div64(N, 64), dim3(32, 8), 0, stream>>>((const bf16*)x, out, R, N, ld);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_im2col_patch14(const void* img, void* out, int n_img, int image_size, int ldp,
                             cudaStream_t stream) {
  // Conv2d(k=14, s=14, padding="valid"): floor(S/14) patches per side (384 -> 27, last 6 px unused)
  MM_CHECK_ARG(n_img > 0 && image_size >= 14 && ldp >= 588 && ldp % 8 == 0,
               "mm_im2col_patch14: need image_size>=14, ldp>=588, ldp%%8==0");
  const int G = image_size / 14;
  const long long total = (long long)n_img * G * G * ldp;
  im2col_patch14_kernel<<<ew_grid(total, 256), 256, 0, stream>>>((const bf16*)img, (bf16*)out, n_img,
                                                                 image_size, ldp);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_add_pos_emb(void* x, const void* pos, long long R, int P, int H, cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && P > 0 && H % 8 == 0, "mm_add_pos_emb: H%%8 != 0");
  add_pos_emb_kernel<<<ew_grid(R * (H / 8), 256), 256, 0, stream>>>((bf16*)x, (const bf16*)pos, R, P, H);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_sumsq_bf16_accum(const void* x, float* out, long long n, cudaStream_t stream) {
  MM_CHECK_ARG(n > 0 && n % 8 == 0, "mm_sumsq_bf16_accum: n%%8 != 0");
  const int grid = ew_grid(n / 8, 256);
  float* part = static_cast<float*>(mm_stream_scratch(MM_SCRATCH_SUMSQ, (size_t)grid * sizeof(float), stream));
  if (part == nullptr) return MM_ERR_CUDA;
  sumsq_bf16_kernel<<<grid, 256, 0, stream>>>((const bf16*)x, part, n / 8);
  MM_CHECK_LAUNCH();
  sumsq_finish_kernel<<<1, 32, 0, stream>>>(part, out, grid);
  MM_CHECK_LAUNCH();
  return MM_OK;
}
