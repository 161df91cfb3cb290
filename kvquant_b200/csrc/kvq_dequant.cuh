// kvquant_b200 -- per-element dequantisation steps shared by every kernel that reads the cache back as fp16
// (kvq_dequant.cu writes it to HBM, kvq_chunk.cu feeds it to the tensor cores from shared memory).
//
// The fp16 K/V operand of a slot is defined by these functions alone, so two kernels that call them produce the same
// bits: LUT entry (K) or one fma of the affine centroid map (V), plus at most one non-zero fp32 outlier residual per
// (slot, channel), then for rotated K the rotate-half with the (cos, sin) of the slot's position, then one rounding
// to fp16.  The arithmetic is spelled with explicit-rounding intrinsics so that no caller's surroundings can change
// how the compiler contracts it.
#pragma once
#include <cuda_fp16.h>

#include "kvq_common.cuh"

namespace kvq {

constexpr int kMaxOutDq = 128;  // outlier row width bound (2 * n_each, n_each <= 64)

// 32 channels (one quarter of a head) of one token: w = the quarter's packed words (4 / 3 / 2 of them), channel l of
// the quarter at code_of<BITS>(w, l).  K: tab = the quarter's LUT rows, `pitch` floats apart; V: tab = the centroids
// and (sf, off) the token's affine map.  Writes dst[0..31] (16-byte aligned).
template <int BITS, bool IS_V>
__device__ __forceinline__ void dq_quarter(const uint32_t* w, const float* tab, int pitch, float sf, float off,
                                           float* dst) {
#pragma unroll
  for (int l = 0; l < 32; l += 4) {
    float x[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t code = code_of<BITS>(w, l + k);
      if constexpr (IS_V) x[k] = __fmaf_rn(tab[code], sf, off);
      else x[k] = tab[(l + k) * pitch + code];
    }
    *reinterpret_cast<float4*>(dst + l) = make_float4(x[0], x[1], x[2], x[3]);
  }
}

// outlier residual of one (slot, channel) added to its dequantised value (a V row may repeat channel 0 as a pad
// whose value is 0: skipped, so each element receives at most one non-zero residual and the order of adds is moot)
__device__ __forceinline__ void dq_add_outlier(float* x, float v) {
  if (v != 0.f) atomicAdd(x, v);
}

// rotate-half of channel c with its partner c ^ 64: cos*x - sin*partner (c < 64, sgn = -1), cos*x + sin*partner
// (c >= 64, sgn = +1)
__device__ __forceinline__ float dq_rotate(float x, float partner, float2 cs, float sgn) {
  return __fmaf_rn(cs.x, x, __fmul_rn(sgn, __fmul_rn(cs.y, partner)));
}

// 8 consecutive channels of one token, channel c0..c0+7 of the fp32 row `src`, as one 16-byte fp16 vector; rotated
// when `cs` (the 8 (cos, sin) pairs of channels (c0 & 63) + k at the token's position) is given
template <bool ROPE>
__device__ __forceinline__ uint4 dq_finish8(const float* src, int c0, const float2* cs) {
  const float4 a = *reinterpret_cast<const float4*>(src + c0);
  const float4 b = *reinterpret_cast<const float4*>(src + c0 + 4);
  float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  if constexpr (ROPE) {
    const float4 pa = *reinterpret_cast<const float4*>(src + (c0 ^ 64));
    const float4 pb = *reinterpret_cast<const float4*>(src + (c0 ^ 64) + 4);
    const float pv[8] = {pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w};
    const float sgn = c0 < 64 ? -1.f : 1.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = dq_rotate(v[k], pv[k], cs[k], sgn);
  }
  uint4 o;
  __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
  for (int k = 0; k < 4; ++k) oh[k] = __floats2half2_rn(v[2 * k], v[2 * k + 1]);
  return o;
}

}  // namespace kvq
