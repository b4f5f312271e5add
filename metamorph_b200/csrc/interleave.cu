// metamorph_b200 — image/text token gather-interleave (SURVEY.md K9) and its backward.
//
// The reference builds `inputs_embeds` with a per-sample Python loop of embed_tokens() calls,
// torch.cat and zero-padding (metamorph_arch.py:272-399). Here the host computes, once per batch,
// an int32 row map with the same (bit-exact) index semantics, and ONE kernel materialises
// inputs_embeds[B*T, H]:
//     row_map[r] >= 0            -> embed_tokens.weight[row_map[r]]          (text token id)
//     row_map[r] <= -2           -> image_features[-(row_map[r]) - 2]        (projected visual token)
//     row_map[r] == -1           -> zeros                                    (padding)
// One warp moves one 8 KB row with coalesced 128-bit loads/stores (HBM-bound, 2*H bytes per row
// read + written).  Backward scatters d(inputs_embeds) into the embedding-table gradient and into d(image_features)
// (rows are unique: plain stores). Token ids repeat: the warp of a token's FIRST row sums all of that token's rows in
// row order in fp32 and stores once, so the embedding gradient is the same bits on every run (no atomics).
#include "common.cuh"

namespace {

constexpr int kScatterVec = 8;   // 16-byte vectors per lane held in fp32 while one token's rows are summed

__global__ void interleave_gather_kernel(const bf16* __restrict__ embed,
                                         const bf16* __restrict__ img,
                                         const int* __restrict__ row_map, bf16* __restrict__ out,
                                         long long R, int H) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nvec = H >> 3;
  for (long long r = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < R;
       r += (long long)gridDim.x * warps_per_block) {
    const int m = row_map[r];
    int4* dst = reinterpret_cast<int4*>(out + r * H);
    if (m == -1) {
      for (int v = lane; v < nvec; v += 32) st_na_int4(dst + v, make_int4(0, 0, 0, 0));
    } else {
      const bf16* srow = (m >= 0) ? embed + (size_t)m * H : img + (size_t)(-(m) - 2) * H;
      const int4* src = reinterpret_cast<const int4*>(srow);
      int v = lane;
      for (; v + 96 < nvec; v += 128) {  // 4 independent 128-bit loads in flight per lane
        const int4 a = ld_nc_int4(src + v), b = ld_nc_int4(src + v + 32),
                   c = ld_nc_int4(src + v + 64), d = ld_nc_int4(src + v + 96);
        st_na_int4(dst + v, a);
        st_na_int4(dst + v + 32, b);
        st_na_int4(dst + v + 64, c);
        st_na_int4(dst + v + 96, d);
      }
      for (; v < nvec; v += 32) st_na_int4(dst + v, ld_nc_int4(src + v));
    }
  }
}

__global__ void interleave_scatter_kernel(const bf16* __restrict__ dout,
                                          const int* __restrict__ row_map,
                                          bf16* __restrict__ dembed, bf16* __restrict__ dimg,
                                          long long R, int H) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nvec = H >> 3;
  for (long long r = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < R;
       r += (long long)gridDim.x * warps_per_block) {
    const int m = row_map[r];
    if (m == -1) continue;
    const int4* src = reinterpret_cast<const int4*>(dout + r * H);
    if (m <= -2) {
      if (dimg == nullptr) continue;
      int4* dst = reinterpret_cast<int4*>(dimg + (size_t)(-(m) - 2) * H);
      for (int v = lane; v < nvec; v += 32) dst[v] = ld_nc_int4(src + v);
    } else {
      if (dembed == nullptr) continue;
      // only the first row carrying token m writes its gradient row
      bool first = true;
      for (long long r0 = 0; r0 < r && first; r0 += 32) {
        const long long q = r0 + lane;
        first = !__any_sync(0xffffffffu, q < r && row_map[q] == m);
      }
      if (!first) continue;
      bf16* drow = dembed + (size_t)m * H;
      for (int c0 = 0; c0 < nvec; c0 += 32 * kScatterVec) {   // kScatterVec 16-byte vectors per lane at a time
        float acc[kScatterVec][8];
#pragma unroll
        for (int i = 0; i < kScatterVec; ++i) {
          const int v = c0 + i * 32 + lane;
          const int4 a = v < nvec ? reinterpret_cast<const int4*>(drow)[v] : make_int4(0, 0, 0, 0);
          const uint32_t u[4] = {(uint32_t)a.x, (uint32_t)a.y, (uint32_t)a.z, (uint32_t)a.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = unpack_bf16x2(u[j]);
            acc[i][2 * j] = f.x;
            acc[i][2 * j + 1] = f.y;
          }
        }
        for (long long r0 = r; r0 < R; r0 += 32) {
          const long long q = r0 + lane;
          unsigned hit = __ballot_sync(0xffffffffu, q < R && row_map[q] == m);
          while (hit) {
            const int b = __ffs(hit) - 1;
            hit &= hit - 1;
            const int4* g = reinterpret_cast<const int4*>(dout + (r0 + b) * H);
#pragma unroll
            for (int i = 0; i < kScatterVec; ++i) {
              const int v = c0 + i * 32 + lane;
              if (v < nvec) {
                const int4 t = ld_nc_int4(g + v);
                const uint32_t u[4] = {(uint32_t)t.x, (uint32_t)t.y, (uint32_t)t.z, (uint32_t)t.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const float2 f = unpack_bf16x2(u[j]);
                  acc[i][2 * j] += f.x;
                  acc[i][2 * j + 1] += f.y;
                }
              }
            }
          }
        }
#pragma unroll
        for (int i = 0; i < kScatterVec; ++i) {
          const int v = c0 + i * 32 + lane;
          if (v < nvec)
            reinterpret_cast<int4*>(drow)[v] =
                make_int4(pack_bf16x2(acc[i][0], acc[i][1]), pack_bf16x2(acc[i][2], acc[i][3]),
                          pack_bf16x2(acc[i][4], acc[i][5]), pack_bf16x2(acc[i][6], acc[i][7]));
        }
      }
    }
  }
}

// out[i, :] = x[idx[i], :]  (row gather used for the vision-head inputs, SURVEY.md K16)
__global__ void gather_rows_kernel(const bf16* __restrict__ x, const int* __restrict__ idx,
                                   bf16* __restrict__ out, long long R, int H) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nvec = H >> 3;
  for (long long r = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < R;
       r += (long long)gridDim.x * warps_per_block) {
    const int4* src = reinterpret_cast<const int4*>(x + (size_t)idx[r] * H);
    int4* dst = reinterpret_cast<int4*>(out + r * H);
    for (int v = lane; v < nvec; v += 32) dst[v] = src[v];
  }
}

// x[idx[i], :] += g[i, :]   (idx unique)
__global__ void scatter_add_rows_kernel(bf16* __restrict__ x, const int* __restrict__ idx,
                                        const bf16* __restrict__ g, long long R, int H) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nvec = H >> 3;
  for (long long r = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < R;
       r += (long long)gridDim.x * warps_per_block) {
    int4* dst = reinterpret_cast<int4*>(x + (size_t)idx[r] * H);
    const int4* src = reinterpret_cast<const int4*>(g + r * H);
    for (int v = lane; v < nvec; v += 32) {
      const int4 a = dst[v], b = src[v];
      const uint32_t ua[4] = {(uint32_t)a.x, (uint32_t)a.y, (uint32_t)a.z, (uint32_t)a.w};
      const uint32_t ub[4] = {(uint32_t)b.x, (uint32_t)b.y, (uint32_t)b.z, (uint32_t)b.w};
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(ua[j]);
        const float2 h = unpack_bf16x2(ub[j]);
        o[j] = pack_bf16x2(f.x + h.x, f.y + h.y);
      }
      dst[v] = make_int4(o[0], o[1], o[2], o[3]);
    }
  }
}

int row_grid(long long R, int warps_per_block) {
  long long b = ceil_div64(R, warps_per_block);
  const long long cap = (long long)mm_num_sms() * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

MM_API int mm_interleave_gather(const void* embed, const void* img, const int* row_map, void* out,
                                long long R, int H, cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && H > 0 && H % 8 == 0, "mm_interleave_gather: need H%%8==0");
  MM_CHECK_ARG(embed != nullptr && out != nullptr && row_map != nullptr, "mm_interleave_gather: null pointer");
  interleave_gather_kernel<<<row_grid(R, 8), 256, 0, stream>>>((const bf16*)embed, (const bf16*)img,
                                                               row_map, (bf16*)out, R, H);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_interleave_scatter(const void* dout, const int* row_map, void* dembed, void* dimg,
                                 long long R, int H, cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && H > 0 && H % 8 == 0, "mm_interleave_scatter: need H%%8==0");
  interleave_scatter_kernel<<<row_grid(R, 8), 256, 0, stream>>>((const bf16*)dout, row_map,
                                                                (bf16*)dembed, (bf16*)dimg, R, H);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_gather_rows(const void* x, const int* idx, void* out, long long R, int H,
                          cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && H % 8 == 0, "mm_gather_rows: need H%%8==0");
  gather_rows_kernel<<<row_grid(R, 8), 256, 0, stream>>>((const bf16*)x, idx, (bf16*)out, R, H);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_scatter_add_rows(void* x, const int* idx, const void* g, long long R, int H,
                               cudaStream_t stream) {
  MM_CHECK_ARG(R > 0 && H % 8 == 0, "mm_scatter_add_rows: need H%%8==0");
  scatter_add_rows_kernel<<<row_grid(R, 8), 256, 0, stream>>>((bf16*)x, idx, (const bf16*)g, R, H);
  MM_CHECK_LAUNCH();
  return MM_OK;
}
