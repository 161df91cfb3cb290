// kvquant_b200 -- shared device helpers (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include "../../include/kvquant_b200.h"

#ifndef __CUDA_ARCH__
#else
#if __CUDA_ARCH__ != 900
#error "kvquant_b200 is written for sm_90a (H100) only"
#endif
#endif

namespace kvq {

constexpr int kHeadDim = 128;
constexpr int kHalf = 64;

extern unsigned long long g_launch_count;  // host-side counter (kvq_launch_count)

#define KVQ_LAUNCH_CHECK()                         \
  do {                                             \
    ++::kvq::g_launch_count;                       \
    cudaError_t e__ = cudaGetLastError();          \
    if (e__ != cudaSuccess) return (int)e__;       \
  } while (0)

// "done once per device" flag for cudaFuncSetAttribute & co.  Function attributes are per device, and the reference
// drives several GPUs from ONE process (LlamaModel.set_devices, modeling_llama.py:2428-2453), so a plain static bool
// would leave every device but the first without its shared-memory opt-in.
struct PerDeviceOnce {
  bool done[64] = {};
  bool& cur() {
    int d = 0;
    cudaGetDevice(&d);
    return done[d & 63];
  }
};

template <int BITS> struct Layout {
  static constexpr int kWords = kHeadDim * BITS / 32;  // int32 rows per head: 16 / 12 / 8
  static constexpr int kLevels = 1 << BITS;            // LUT entries
  static constexpr int kZeroPoint = (BITS == 4) ? 7 : (BITS == 3 ? 3 : 1);
};

// code of channel c (0..127, compile-time after unrolling) of one head given that head's packed words.
// Layout rules: reference quant_cuda_kernel.cu:1240-1243 (4b), 1395-1424 (3b), 1601-1604 (2b).
template <int BITS>
__device__ __forceinline__ uint32_t code_of(const uint32_t* __restrict__ w, int c) {
  if constexpr (BITS == 4) {
    return (w[c >> 3] >> ((c & 7) * 4)) & 0xFu;
  } else if constexpr (BITS == 2) {
    return (w[c >> 4] >> ((c & 15) * 2)) & 0x3u;
  } else {
    const int g = (c >> 5) * 3, l = c & 31;
    if (l < 10) return (w[g] >> (3 * l)) & 0x7u;
    if (l == 10) return ((w[g] >> 30) | (w[g + 1] << 2)) & 0x7u;
    if (l < 21) return (w[g + 1] >> ((3 * l) & 31)) & 0x7u;
    if (l == 21) return ((w[g + 1] >> 31) | (w[g + 2] << 1)) & 0x7u;
    return (w[g + 2] >> ((3 * l) & 31)) & 0x7u;
  }
}

// Where channel j (flat index within the hidden vector) lands: word row (relative to the whole [H*W] matrix),
// shift, and for the two 3-bit straddlers a second (row, right-shift).  Used by the packers.
template <int BITS>
__device__ __forceinline__ void pack_slot(int j, int& row, int& shift, int& row2, int& rshift2) {
  row2 = -1; rshift2 = 0;
  if constexpr (BITS == 4) { row = j >> 3; shift = (j & 7) * 4; }
  else if constexpr (BITS == 2) { row = j >> 4; shift = (j & 15) * 2; }
  else {
    const int g = (j >> 5) * 3, l = j & 31;
    if (l == 10) { row = g; shift = 30; row2 = g + 1; rshift2 = 2; }
    else if (l == 21) { row = g + 1; shift = 31; row2 = g + 2; rshift2 = 1; }
    else { row = g + l / 11; shift = (3 * l) & 31; }
  }
}

// nearest LUT entry, strict '<' scan from 0 (first minimum wins) -- reference quant_cuda_kernel.cu:1219-1235.
// `lut` points at this element's 2^BITS fp32 entries.  Written as the reference's linear scan on
// fabsf(lut[i]-x): a binary search would have to end in the same two-entry comparison to stay bit-exact
// under duplicated / fp32-collapsed entries, and at 16 entries the scan is not what bounds the append.
template <int BITS>
__device__ __forceinline__ uint32_t nearest_code(const float* __restrict__ lut, float x) {
  uint32_t best = 0;
  float bd = fabsf(lut[0] - x);
#pragma unroll
  for (int i = 1; i < Layout<BITS>::kLevels; ++i) {
    const float d = fabsf(lut[i] - x);
    if (d < bd) { bd = d; best = i; }
  }
  return best;
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

// float atomic max via integer ordering trick (works for all non-NaN floats)
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// L2 cache policies: a createpolicy descriptor passed through .L2::cache_hint
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// streaming loads: packed codes are read exactly once per decode step
__device__ __forceinline__ uint32_t ld_stream_u32(const uint32_t* p, uint64_t pol) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
// re-used data (rope table: shared by every head group and every layer)
__device__ __forceinline__ float2 ld_keep_f2(const float2* p, uint64_t pol) {
  float2 v;
  asm volatile("ld.global.nc.L2::cache_hint.v2.f32 {%0,%1}, [%2], %3;" : "=f"(v.x), "=f"(v.y) : "l"(p), "l"(pol));
  return v;
}

// ---- mbarrier / TMA (cp.async.bulk.tensor) wrappers -------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 2D tiled TMA load: coordinates (x = innermost = token, y = word row)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y) : "memory");
}
// 1D bulk copy global -> shared (bytes multiple of 16, both 16B aligned)
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// host: build a 2D tensor map over the packed cache viewed as uint32 [rows = H*W, cols = Lmax]
int make_cache_tensor_map(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                          uint32_t box_cols, uint32_t box_rows, int swizzle_bytes);

}  // namespace kvq
