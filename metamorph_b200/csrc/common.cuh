// metamorph_b200 — shared device/host helpers for the sm_90a kernels.
// Hand-written for Hopper (H100): mbarrier, TMA, cp.async / ldmatrix / mma.sync PTX wrappers,
// warp-shuffle reductions, 128-bit global access helpers and the C-ABI error plumbing (wgmma lives in wgmma.cuh).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

typedef __nv_bfloat16 bf16;
typedef __nv_bfloat162 bf162;

// ----------------------------------------------------------------------------------------------
// C-ABI error handling: every exported function returns 0 on success, negative on failure, and
// leaves a thread-local message readable through mm_last_error().
// ----------------------------------------------------------------------------------------------
#define MM_API extern "C" __attribute__((visibility("default")))
#define MM_OK 0
#define MM_ERR_ARG (-1)
#define MM_ERR_CUDA (-2)
#define MM_ERR_ARCH (-3)

void mm_set_error(const char* fmt, ...);

#define MM_CHECK_ARG(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      mm_set_error(__VA_ARGS__);           \
      return MM_ERR_ARG;                   \
    }                                      \
  } while (0)

#define MM_CHECK_CUDA(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      mm_set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, cudaGetErrorName(_e),  \
                   cudaGetErrorString(_e));                                              \
      return MM_ERR_CUDA;                                                                \
    }                                                                                    \
  } while (0)

#define MM_CHECK_LAUNCH() MM_CHECK_CUDA(cudaGetLastError())

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

int mm_num_sms();
// Zero-initialised device scratch private to (current device, stream, tag), grown on demand. Kernels that use it leave
// it as they found it (or overwrite it fully), so stream-ordered calls can reuse it; calls on different streams never
// share it. nullptr (with the error text set) when the allocation fails.
void* mm_stream_scratch(int tag, size_t bytes, cudaStream_t stream);
enum { MM_SCRATCH_LOSS = 0, MM_SCRATCH_RMSNORM_DW = 1, MM_SCRATCH_SUMSQ = 2 };
// programmatic dependent launch (PDL) for the decode chain: 1 unless MM_PDL=0 (api.cu)
int mm_pdl_enabled();
// MM_PDL_MODE bitmask (default 3): 1 = weight-streaming GEMMs launched with the PDL attribute, 2 = the small decode kernels
// too, 8 = trigger dependents after the main loop instead of at kernel entry. The early trigger lets the next kernel's
// producer fill its ring with weights while this one drains.
int mm_pdl_mode();

// ----------------------------------------------------------------------------------------------
// Device helpers
// ----------------------------------------------------------------------------------------------
#ifdef __CUDACC__

// Programmatic dependent launch. A kernel launched through launch_pdl may start while its stream predecessor is
// still running (as soon as every predecessor CTA has executed griddep_launch or exited): everything before
// griddep_wait() may only touch memory no earlier kernel writes (weights, tensor maps, barriers); griddep_wait()
// returns once the predecessor grid has completed and flushed. Every kernel launched this way MUST execute
// griddep_wait() (completion order along the chain is what makes buffer reuse two kernels back safe).
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(int allow, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                     cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = allow ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum; `red` is a shared float[32]. All threads get the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : 0.f;
  r = warp_sum(r);
  return r;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : -INFINITY;
  r = warp_max(r);
  return r;
}

// 128-bit vector of 8 bf16
struct __align__(16) bf16x8 {
  bf162 v[4];
};
__device__ __forceinline__ bf16x8 ld_bf16x8(const bf16* p) {
  return *reinterpret_cast<const bf16x8*>(p);
}
__device__ __forceinline__ void st_bf16x8(bf16* p, const bf16x8& x) {
  *reinterpret_cast<bf16x8*>(p) = x;
}
// streaming (no L1 allocate) 128-bit load/store for single-touch data
__device__ __forceinline__ int4 ld_nc_int4(const void* p) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_na_int4(void* p, const int4& v) {
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  bf162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  bf162 t = *reinterpret_cast<bf162*>(&u);
  return __bfloat1622float2(t);
}

__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float gelu_erf_grad(float x) {
  const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752440f));
  const float pdf = 0.39894228040143267794f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k = 0.7978845608028654f;
  return 0.5f * x * (1.f + tanhf(k * (x + 0.044715f * x * x * x)));
}
__device__ __forceinline__ float silu(float x) { return x / (1.f + __expf(-x)); }

// Rotate-half RoPE of the pair (a, b) = (x[j], x[j + d/2]): a c - b s and b c + a s. The rounded product and the fused
// multiply-add are spelled out so that every kernel that rotates (rope_kernel, decode_attn_kernel) gets the same bits
// whatever the compiler would contract: a prefilled K cache and a decoded one are identical.
__device__ __forceinline__ float rope_lo(float a, float b, float c, float s) { return __fmaf_rn(a, c, -__fmul_rn(b, s)); }
__device__ __forceinline__ float rope_hi(float a, float b, float c, float s) { return __fmaf_rn(b, c, __fmul_rn(a, s)); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (launch failure) instead of a hung GPU. The bound is in TIME (about
// two seconds of SM clock): one try_wait may itself block for a hardware-defined interval, so a spin count says little.
// No printf here: a call in a kernel that issues wgmma makes ptxas serialise every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3FFu) == 0 && clock64() - t0 > 4000000000ll) __trap();
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2-D tiled load global -> shared, completion on an mbarrier (tx bytes).
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void* tmap, uint32_t bar,
                                            int32_t c_inner, int32_t c_outer) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c_inner),
      "r"(c_outer)
      : "memory");
}

// ---------------------------------------------------------------- cp.async / ldmatrix / mma.sync
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gsrc, bool pred) {
  const int sz = pred ? 16 : 0;  // src-size 0 => zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc),
               "r"(sz)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                        uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1,
                                          uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
// D(16x8,f32) += A(16x16,bf16,row) * B(16x8,bf16,col)
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0,
                                               uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, "
      "{%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

#endif  // __CUDACC__
