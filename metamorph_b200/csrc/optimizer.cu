// metamorph_b200 — fused AdamW (SURVEY.md K18; reference: --optim adamw_torch, train.py:82).
// One pass over flat buffers: reads grad (bf16 or fp32), fp32 master weight, fp32 m and v; writes
// master, m, v and the bf16 compute copy. 16 + 2 (or 4) bytes read and 14 bytes written per
// parameter -> HBM-bound; 128-bit accesses, grid-stride. Update order follows torch.optim.AdamW:
//   p *= 1 - lr*wd;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
//   p -= (lr / (1-b1^t)) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
#include "common.cuh"

namespace {

// BCAST: the updated bf16 values are not stored locally but BROADCAST to every rank's replica of the parameter buffer in
// the same kernel (the all-gather of a sharded-optimizer step fused into the optimizer): one multimem.st through the
// NVSwitch multicast mapping of the symmetric buffer when the fabric offers it (NVLS), else one st.global per peer over
// NVLink P2P. The compute step (AdamW on this rank's slice) and its collective (all-gather of the slice) are ONE kernel.
// GRAD_MC (with BCAST): `grad` is the MULTICAST address of this rank's slice of the symmetric gradient buffers: one
// multimem.ld_reduce returns the SUM over all ranks' buffers, added inside the NVSwitch (NVLS) with fp32 accumulation — the
// reduce-scatter of the data-parallel step without a collective kernel. With both flags the whole
// [reduce-scatter -> AdamW -> all-gather] of a parameter bucket is this ONE kernel.
template <bool GRAD_F32, bool BCAST, bool GRAD_MC = false>
__global__ void adamw_kernel(bf16* __restrict__ p16, float* __restrict__ p32, float* __restrict__ m,
                             float* __restrict__ v, const void* __restrict__ grad, long long n4,
                             float lr, float b1, float b2, float eps, float wd, float c1,
                             float sqrt_c2, const float* __restrict__ grad_scale_ptr,
                             float grad_scale, bf16* const* __restrict__ peers, int n_peers) {
  float gs = grad_scale;
  if (grad_scale_ptr != nullptr) gs *= *grad_scale_ptr;
  const float step = lr / c1;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float g[4];
    if (GRAD_MC && GRAD_F32) {
      asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(g[0]), "=f"(g[1]), "=f"(g[2]), "=f"(g[3])
                   : "l"(reinterpret_cast<const float*>(grad) + i * 4)
                   : "memory");
    } else if (GRAD_MC) {
      uint32_t u0, u1;
      asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v2.bf16x2 {%0, %1}, [%2];"
                   : "=r"(u0), "=r"(u1)
                   : "l"(reinterpret_cast<const bf16*>(grad) + i * 4)
                   : "memory");
      const float2 a = unpack_bf16x2(u0), b = unpack_bf16x2(u1);
      g[0] = a.x; g[1] = a.y; g[2] = b.x; g[3] = b.y;
    } else if (GRAD_F32) {
      const float4 t = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(grad) + i * 4);
      g[0] = t.x; g[1] = t.y; g[2] = t.z; g[3] = t.w;
    } else {
      const uint2 t = *reinterpret_cast<const uint2*>(reinterpret_cast<const bf16*>(grad) + i * 4);
      const float2 a = unpack_bf16x2(t.x), b = unpack_bf16x2(t.y);
      g[0] = a.x; g[1] = a.y; g[2] = b.x; g[3] = b.y;
    }
    float4 pw = *reinterpret_cast<float4*>(p32 + i * 4);
    float4 mm = *reinterpret_cast<float4*>(m + i * 4);
    float4 vv = *reinterpret_cast<float4*>(v + i * 4);
    float* pp = reinterpret_cast<float*>(&pw);
    float* pm = reinterpret_cast<float*>(&mm);
    float* pv = reinterpret_cast<float*>(&vv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gj = g[j] * gs;
      pp[j] *= (1.f - lr * wd);
      pm[j] = b1 * pm[j] + (1.f - b1) * gj;
      pv[j] = b2 * pv[j] + (1.f - b2) * gj * gj;
      pp[j] -= step * pm[j] / (sqrtf(pv[j]) / sqrt_c2 + eps);
    }
    *reinterpret_cast<float4*>(p32 + i * 4) = pw;
    *reinterpret_cast<float4*>(m + i * 4) = mm;
    *reinterpret_cast<float4*>(v + i * 4) = vv;
    uint2 o;
    o.x = pack_bf16x2(pp[0], pp[1]);
    o.y = pack_bf16x2(pp[2], pp[3]);
    if (!BCAST) {
      *reinterpret_cast<uint2*>(p16 + i * 4) = o;
    } else if (peers == nullptr) {      // p16 = multicast address of this slice: one store, the switch replicates it
      asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(p16 + i * 4), "f"(__uint_as_float(o.x)),
                   "f"(__uint_as_float(o.y))
                   : "memory");
    } else {                            // p16 = OFFSET of the slice (in elements) inside every peer's buffer
      const long long off = reinterpret_cast<long long>(p16) / 2;
      for (int r = 0; r < n_peers; ++r) *reinterpret_cast<uint2*>(peers[r] + off + i * 4) = o;
    }
  }
}

// out = min(1, max_norm / (sqrt(sumsq) + 1e-6))  (torch.nn.utils.clip_grad_norm_)
// A NaN norm gives a NaN coefficient, as torch's clamp(max=1) does, so the update turns every parameter NaN instead of
// applying the finite gradients unclipped. (fminf would return 1 for a NaN operand.)
__global__ void clip_coef_kernel(const float* __restrict__ sumsq, float* __restrict__ out,
                                 float max_norm) {
  const float total = sqrtf(*sumsq);
  const float c = max_norm / (total + 1e-6f);
  out[0] = c >= 1.f ? 1.f : c;
  out[1] = total;
}

}  // namespace

MM_API int mm_adamw_step(void* p16, float* p32, float* m, float* v, const void* grad, int grad_f32,
                         long long n, float lr, float beta1, float beta2, float eps, float wd,
                         int step, const float* grad_scale_ptr, float grad_scale,
                         cudaStream_t stream) {
  MM_CHECK_ARG(n > 0 && n % 4 == 0, "mm_adamw_step: n must be a positive multiple of 4 (n=%lld)", n);
  MM_CHECK_ARG(step >= 1, "mm_adamw_step: step starts at 1");
  const float c1 = 1.f - powf(beta1, (float)step);
  const float sqrt_c2 = sqrtf(1.f - powf(beta2, (float)step));
  const long long n4 = n / 4;
  long long blocks = ceil_div64(n4, 256);
  const long long cap = (long long)mm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (grad_f32)
    adamw_kernel<true, false><<<(int)blocks, 256, 0, stream>>>((bf16*)p16, p32, m, v, grad, n4, lr, beta1, beta2, eps, wd,
                                                               c1, sqrt_c2, grad_scale_ptr, grad_scale, nullptr, 0);
  else
    adamw_kernel<false, false><<<(int)blocks, 256, 0, stream>>>((bf16*)p16, p32, m, v, grad, n4, lr, beta1, beta2, eps, wd,
                                                                c1, sqrt_c2, grad_scale_ptr, grad_scale, nullptr, 0);
  MM_CHECK_LAUNCH();
  return MM_OK;
}

// AdamW on this rank's slice + broadcast of the updated bf16 slice into every rank's parameter buffer (see adamw_kernel).
// multicast_p16 != NULL: the multicast (NVLS) address of the slice; else peers = DEVICE array of n_peers buffer base
// pointers and slice_offset = first element of the slice inside each of them.
MM_API int mm_adamw_step_bcast(void* multicast_p16, const void* const* peers, int n_peers, long long slice_offset,
                               float* p32, float* m, float* v, const void* grad, int grad_f32, int grad_multicast,
                               long long n, float lr, float beta1, float beta2, float eps, float wd, int step,
                               const float* grad_scale_ptr, float grad_scale, cudaStream_t stream) {
  MM_CHECK_ARG(!grad_multicast || multicast_p16 != nullptr,
               "mm_adamw_step_bcast: the in-switch gradient reduction needs the multicast parameter address as well");
  MM_CHECK_ARG(n > 0 && n % 4 == 0 && slice_offset % 4 == 0, "mm_adamw_step_bcast: n / offset must be multiples of 4");
  MM_CHECK_ARG(step >= 1, "mm_adamw_step_bcast: step starts at 1");
  MM_CHECK_ARG(multicast_p16 != nullptr || (peers != nullptr && n_peers > 0), "mm_adamw_step_bcast: no destination");
  const float c1 = 1.f - powf(beta1, (float)step);
  const float sqrt_c2 = sqrtf(1.f - powf(beta2, (float)step));
  const long long n4 = n / 4;
  long long blocks = ceil_div64(n4, 256);
  const long long cap = (long long)mm_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  bf16* dst = multicast_p16 ? (bf16*)multicast_p16 : reinterpret_cast<bf16*>(slice_offset * 2);   // address or byte offset
  bf16* const* pr = multicast_p16 ? nullptr : (bf16* const*)peers;
#define MM_ADAMW_B(F32, MC)                                                                                          \
  adamw_kernel<F32, true, MC><<<(int)blocks, 256, 0, stream>>>(dst, p32, m, v, grad, n4, lr, beta1, beta2, eps, wd, c1, \
                                                               sqrt_c2, grad_scale_ptr, grad_scale, pr, n_peers)
  if (grad_f32 && grad_multicast) MM_ADAMW_B(true, true);
  else if (grad_f32) MM_ADAMW_B(true, false);
  else if (grad_multicast) MM_ADAMW_B(false, true);
  else MM_ADAMW_B(false, false);
#undef MM_ADAMW_B
  MM_CHECK_LAUNCH();
  return MM_OK;
}

MM_API int mm_clip_coef(const float* sumsq, float* out2, float max_norm, cudaStream_t stream) {
  clip_coef_kernel<<<1, 1, 0, stream>>>(sumsq, out2, max_norm);
  MM_CHECK_LAUNCH();
  return MM_OK;
}
