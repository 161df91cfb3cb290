// kvquant_b200 -- batch-1 fp16 GEMV of the LLaMA decode harness (kvquant_b200/decode.py) with the element-wise
// neighbours fused in.  NOT part of the reference's quant_cuda surface (the reference calls cuBLAS through
// nn.Linear, modeling_llama.py:1811-1813, 2004); it exists because at batch 1 the 13.2 GB of fp16 weights are a
// pure HBM stream, and the library GEMV comes with an RMSNorm / SwiGLU / cast launch in front of every call.
//
//   y[r] = (residual ? residual[r] : 0) + sum_k W[r,k] * f(x)[k]              W fp16 [N,K] row-major, fp32 accumulate
//   f = identity on an fp16 or f32 vector | RMSNorm(x, norm_w) (HF LlamaRMSNorm rounding) | silu(gate) * up
//
// Every CTA stages f(x) once as f32 in shared memory (K <= 14336), then its warps stream whole rows: 16-byte loads,
// 8 in flight per lane, two rows at a time; rows are dealt to CTAs in equal contiguous blocks (+-1 row).
#include "kvq_common.cuh"
#include <cuda_fp16.h>

namespace kvq {

constexpr int kGemvThreads = 512;
constexpr int kGemvMaxK = 14336;

__device__ __forceinline__ uint4 ld_w16(const uint4* p, uint64_t pol) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ float dot8(const uint4 w, const float4 a, const float4 b, float acc) {
  const float2 w0 = __half22float2(*reinterpret_cast<const __half2*>(&w.x));
  const float2 w1 = __half22float2(*reinterpret_cast<const __half2*>(&w.y));
  const float2 w2 = __half22float2(*reinterpret_cast<const __half2*>(&w.z));
  const float2 w3 = __half22float2(*reinterpret_cast<const __half2*>(&w.w));
  acc = fmaf(w0.x, a.x, acc); acc = fmaf(w0.y, a.y, acc); acc = fmaf(w1.x, a.z, acc); acc = fmaf(w1.y, a.w, acc);
  acc = fmaf(w2.x, b.x, acc); acc = fmaf(w2.y, b.y, acc); acc = fmaf(w3.x, b.z, acc); acc = fmaf(w3.y, b.w, acc);
  return acc;
}

// shared layout of f(x): the 8 floats lane l needs for 16-byte chunk c of a row are two float4 at [c][0][l] and
// [c][1][l] -> both LDS.128 of a warp are contiguous (conflict-free)
__device__ __forceinline__ int xperm(int i) {
  return (i & ~255) | ((i & 4) << 5) | ((i & 0xF8) >> 1) | (i & 3);
}

// XK: 0 = fp16 vector, 1 = f32 vector, 2 = fp16 [2K] gate|up -> silu(gate)*up, 3 = fp16 vector + RMSNorm(norm_w)
template <int XK>
__global__ void __launch_bounds__(kGemvThreads, 1) dec_gemv_kernel(
    const uint4* __restrict__ W, int N, int K, const void* __restrict__ x, const __half* __restrict__ norm_w, float eps,
    const __half* __restrict__ residual, void* __restrict__ y, int y_f32) {
  extern __shared__ float4 s_x4[];                  // f(x) as f32 [K]
  float* s_x = reinterpret_cast<float*>(s_x4);
  __shared__ float s_red[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if constexpr (XK == 0) {
    const __half* xh = static_cast<const __half*>(x);
    for (int i = tid; i < K; i += kGemvThreads) s_x[xperm(i)] = __half2float(xh[i]);
  } else if constexpr (XK == 1) {
    // the library GEMV consumed the fp16-rounded vector (decode.py cast o to fp16): keep that rounding
    const float* xf = static_cast<const float*>(x);
    for (int i = tid; i < K; i += kGemvThreads) s_x[xperm(i)] = __half2float(__float2half(xf[i]));
  } else if constexpr (XK == 2) {
    const __half* gu = static_cast<const __half*>(x);
    for (int i = tid; i < K; i += kGemvThreads) {
      const float g = __half2float(gu[i]);
      const __half s = __float2half(g / (1.f + __expf(-g)));
      s_x[xperm(i)] = __half2float(__hmul(s, gu[K + i]));
    }
  } else {
    const __half* xh = static_cast<const __half*>(x);
    float ss = 0.f;
    for (int i = tid; i < K; i += kGemvThreads) { const float v = __half2float(xh[i]); ss = fmaf(v, v, ss); }
    ss = warp_sum(ss);
    if (lane == 0) s_red[warp] = ss;
    __syncthreads();
    if (tid < 32) {
      float v = tid < (kGemvThreads >> 5) ? s_red[tid] : 0.f;
      v = warp_sum(v);
      if (tid == 0) s_red[0] = rsqrtf(v / (float)K + eps);
    }
    __syncthreads();
    const float r = s_red[0];
    for (int i = tid; i < K; i += kGemvThreads)
      s_x[xperm(i)] = __half2float(__hmul(__float2half(__half2float(xh[i]) * r), norm_w[i]));
  }
  __syncthreads();

  // this CTA's rows: equal contiguous blocks
  const int r_begin = (int)(((int64_t)N * blockIdx.x) / gridDim.x);
  const int r_end = (int)(((int64_t)N * (blockIdx.x + 1)) / gridDim.x);
  const uint64_t pol = policy_evict_first();
  const int kc = K >> 8;                            // 16-byte chunks per lane per row (K % 256 == 0)
  const int row_u4 = K >> 3;                        // uint4 per row
  constexpr int NW = kGemvThreads / 32;
  for (int r = r_begin + 2 * warp; r < r_end; r += 2 * NW) {
    const bool two = (r + 1) < r_end;
    const uint4* w0 = W + (int64_t)r * row_u4 + lane;
    const uint4* w1 = two ? w0 + row_u4 : w0;
    float a0 = 0.f, a1 = 0.f;
    int c = 0;
    for (; c + 4 <= kc; c += 4) {
      uint4 u0[4], u1[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { u0[i] = ld_w16(w0 + (c + i) * 32, pol); u1[i] = ld_w16(w1 + (c + i) * 32, pol); }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 xa = s_x4[(c + i) * 64 + lane], xb = s_x4[(c + i) * 64 + 32 + lane];
        a0 = dot8(u0[i], xa, xb, a0);
        a1 = dot8(u1[i], xa, xb, a1);
      }
    }
    for (; c < kc; ++c) {
      const uint4 u0 = ld_w16(w0 + c * 32, pol), u1 = ld_w16(w1 + c * 32, pol);
      const float4 xa = s_x4[c * 64 + lane], xb = s_x4[c * 64 + 32 + lane];
      a0 = dot8(u0, xa, xb, a0);
      a1 = dot8(u1, xa, xb, a1);
    }
    a0 = warp_sum(a0);
    a1 = warp_sum(a1);
    if (lane < 2 && (lane == 0 || two)) {
      const int rr = r + lane;
      float v = lane ? a1 : a0;
      if (residual != nullptr) v += __half2float(residual[rr]);
      if (y_f32) static_cast<float*>(y)[rr] = v;
      else static_cast<__half*>(y)[rr] = __float2half(v);
    }
  }
}

int num_sms_cached();

}  // namespace kvq

using namespace kvq;

extern "C" {

int kvq_dec_gemv(const void* w_f16, int N, int K, const void* x, int x_kind, const void* norm_w_f16, float eps,
                 const void* residual_f16, void* y, int y_f32, void* stream) {
  if (!w_f16 || !x || !y) return KVQ_E_NULL;
  if (N <= 0 || K <= 0 || (K & 255) != 0 || K > kGemvMaxK) return KVQ_E_SHAPE;
  if (x_kind < 0 || x_kind > 3 || (x_kind == 3 && !norm_w_f16)) return KVQ_E_SHAPE;
  if ((reinterpret_cast<uintptr_t>(w_f16) & 15) != 0) return KVQ_E_ALIGN;
  if (x == y) return KVQ_E_SHAPE;   // in place on the residual is fine; the input vector must not be the output
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    const int mx = kGemvMaxK * 4;
    cudaError_t e = cudaFuncSetAttribute(dec_gemv_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(dec_gemv_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(dec_gemv_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(dec_gemv_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  const int sms = num_sms_cached();
  const int grid = N < sms ? N : sms;
  const size_t smem = (size_t)K * 4;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint4* W = static_cast<const uint4*>(w_f16);
  const __half* nw = static_cast<const __half*>(norm_w_f16);
  const __half* res = static_cast<const __half*>(residual_f16);
  switch (x_kind) {
    case 0: dec_gemv_kernel<0><<<grid, kGemvThreads, smem, st>>>(W, N, K, x, nw, eps, res, y, y_f32); break;
    case 1: dec_gemv_kernel<1><<<grid, kGemvThreads, smem, st>>>(W, N, K, x, nw, eps, res, y, y_f32); break;
    case 2: dec_gemv_kernel<2><<<grid, kGemvThreads, smem, st>>>(W, N, K, x, nw, eps, res, y, y_f32); break;
    default: dec_gemv_kernel<3><<<grid, kGemvThreads, smem, st>>>(W, N, K, x, nw, eps, res, y, y_f32); break;
  }
  KVQ_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
