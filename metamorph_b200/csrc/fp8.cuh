// metamorph_b200 — the E4M3 row rule shared by the FP8 KV cache (decode.cu) and the FP8 weights (decode.cu,
// decode_wide.cu): one power-of-two scale per 128 values, DESIGN.md §1.
#pragma once
#include <cuda_fp8.h>

#include "common.cuh"

// E4M3 row quantisation, one warp per 128-value row, 4 values per lane (any assignment of values to lanes). a = max |x|;
// e = the least integer with a <= 448 * 2^e, at least -124 (so every float(q) * 2^e is a bf16 value and 2^e an fp32
// normal); q = RNE_e4m3(x * 2^-e) (exact multiply, |x * 2^-e| <= 448: nothing saturates), except that at e = 120, the
// largest e a bf16 row reaches, an entry that rounds to 256 (|x| >= 1.9375 * 2^127) would dequantise to 2^128, past the
// bf16 and fp32 range: it stores 240 (0x77), the largest magnitude whose float(q) * 2^e is finite. A zero row stores
// zeros with e = 0; a row holding any Inf or NaN stores the E4M3 NaN 0x7f everywhere with e = 0. On return x holds
// float(q) * 2^e, q01 / q23 the bytes of (x[0], x[1]) and (x[2], x[3]) (first value in the low byte); returns 2^e.
__device__ __forceinline__ uint16_t fp8x2_cap_256(uint16_t q) {
  const uint16_t lo = (q & 0x7f) == 0x78 ? (q & 0x80) | 0x77 : q & 0xff;
  const uint16_t hi = ((q >> 8) & 0x7f) == 0x78 ? ((q >> 8) & 0x80) | 0x77 : q >> 8;
  return (uint16_t)(lo | (hi << 8));
}

__device__ __forceinline__ float fp8_quant_row_warp(float (&x)[4], uint16_t& q01, uint16_t& q23) {
  float a = 0.f;
  bool bad = false;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float m = fabsf(x[j]);
    bad |= !(m <= 3.402823466e38f);
    a = fmaxf(a, m);
  }
  a = warp_max(a);
  bad = __any_sync(0xffffffffu, bad);
  int e = 0;
  if (!bad && a > 0.f) {
    int E;
    const float f = frexpf(a, &E);          // a = f 2^E, f in [0.5, 1); 448 = 0.875 * 2^9
    e = max(f <= 0.875f ? E - 9 : E - 8, -124);
  }
  const float sc = __int_as_float((127 + e) << 23), inv = __int_as_float((127 - e) << 23);
  if (bad) {
    q01 = q23 = 0x7f7f;
  } else {
    q01 = __nv_cvt_float2_to_fp8x2(make_float2(x[0] * inv, x[1] * inv), __NV_SATFINITE, __NV_E4M3);
    q23 = __nv_cvt_float2_to_fp8x2(make_float2(x[2] * inv, x[3] * inv), __NV_SATFINITE, __NV_E4M3);
    if (e == 120) {
      q01 = fp8x2_cap_256(q01);
      q23 = fp8x2_cap_256(q23);
    }
  }
  const float2 d01 = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2(q01, __NV_E4M3)));
  const float2 d23 = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2(q23, __NV_E4M3)));
  x[0] = d01.x * sc; x[1] = d01.y * sc; x[2] = d23.x * sc; x[3] = d23.y * sc;
  return sc;
}

// four E4M3 values (first in the low byte) -> float(q) * sc
__device__ __forceinline__ void fp8x4_dequant(uint32_t u, float sc, float* f) {
  const float2 a = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(u & 0xffffu), __NV_E4M3)));
  const float2 b = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(u >> 16), __NV_E4M3)));
  f[0] = a.x * sc; f[1] = a.y * sc; f[2] = b.x * sc; f[3] = b.y * sc;
}

// four E4M3 values -> the two bf16x2 registers of float(q) * sc (exact when sc is a scale of the row rule)
__device__ __forceinline__ uint2 fp8x4_to_bf16x4(uint32_t u, float sc) {
  float f[4];
  fp8x4_dequant(u, sc, f);
  return make_uint2(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]));
}
