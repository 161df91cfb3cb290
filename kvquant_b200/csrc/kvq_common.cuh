// kvquant_b200 -- shared device helpers (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <type_traits>
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

// Page table of a paged batch (kvq_append_kv_fused_paged, kvq_attend_paged; DESIGN.md section 4.11): sequence b's
// token t lives in page table[b * max_pages + t / P], column t % P, of a pool of n_pool pages, each page laid out as a
// single-sequence cache with Lmax = P.  Only the leading npages[b] entries of row b are mapped (and ever read).
// P % 160 == 0: every 80-token K box and 32-token V tile lies inside one page.  Passed by value as the trailing
// argument of the switched kernels; instantiations without the paged switch ignore it.
struct PageRef {
  const int32_t* table;    // int32 [B][max_pages] page ids (device)
  const int32_t* npages;   // int32 [B] mapped entries per row (device)
  int max_pages, P, n_pool;
};
constexpr int kPageQuantum = 160;   // lcm of the K box (80 tokens) and the V tile / length rounding (32 tokens)

// host: the page-geometry checks of the paged entry points (kvq_page.cu): P a positive multiple of 160, max_pages >= 1
// with max_pages * P < 2^30, n_pool >= 1 with n_pool * rows (packed-word rows of one page) < 2^31 (TMA row coordinate)
// and n_pool * P < 2^31 (32-bit pool rows)
int check_pages(int n_pool, int max_pages, int P, int64_t rows);

// sequence b's mapped token count (npages[b] * P, the row capped at max_pages)
__device__ __forceinline__ int64_t page_cap(const PageRef& pg, int b) {
  const int n = pg.npages[b];
  return (int64_t)(n < 0 ? 0 : (n < pg.max_pages ? n : pg.max_pages)) * pg.P;
}
// page of sequence b's token t (t below page_cap < 2^30: 32-bit division)
__device__ __forceinline__ int page_of(const PageRef& pg, int b, int t) {
  return pg.table[b * pg.max_pages + t / pg.P];
}
// One sequence's slot s (s < 2^30) when pg.table is that sequence's page-table row (the single-sequence paged entry
// points kvq_append_kv_fused_chunk_paged, kvq_dequant_kv_paged): its page and column, and its pool row page * P + column
struct PageCol {
  int page, col;
};
__device__ __forceinline__ PageCol page_col(const PageRef& pg, int s) {
  const int q = s / pg.P;
  return PageCol{pg.table[q], s - q * pg.P};
}
__device__ __forceinline__ int64_t page_row(const PageRef& pg, int s) {
  const PageCol pc = page_col(pg, s);
  return (int64_t)pc.page * pg.P + pc.col;
}

// Ragged calls (kvq_append_kv_fused_chunk_ragged*, kvq_attend_chunk_ragged*; DESIGN.md section 4.15): a host segment
// table segs int64 [n_seg][4] of (slot b, first slot s0, T, first row) packs several slots' chunks into one launch.
// The table travels to the kernels by value (as a __grid_constant__ parameter), so n_seg is bounded by the batch.
constexpr int kMaxSeg = 256;

// host: the segment checks of the ragged entry points (kvq_page.cu), in order: slots in [0, B) and distinct, s0 >= 0,
// T >= 0, rows packed in segment order (row0 = the earlier segments' T), s0 + T <= Lmax (the per-slot cap), and when
// n_mapped is given 0 <= n_mapped[i] <= max_pages with the slots the call touches mapped: s0 + T for a call that writes
// them (the append), s0 for one that reads the first s0 (the attend); N = the sum of T and N < 2^31 -> KVQ_E_SHAPE.
// *max_s0 (optional) receives the largest s0.
int check_segments(int B, int n_seg, const int64_t* segs, int64_t N, int64_t Lmax, const int32_t* n_mapped,
                   int max_pages, int P, bool writes, int64_t* max_s0);

// device: the last i < n with first[i] <= x (first[] non-decreasing, first[0] == 0), i.e. the segment owning block x of
// a ragged grid; a segment of no blocks shares its start with the next one and is never returned
__device__ __forceinline__ int find_segment(const int* first, int n, int x) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// host: build a 2D tensor map over the packed cache viewed as uint32 [rows = H*W, cols = Lmax]  (kvq_capi.cu)
int make_cache_tensor_map(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                          uint32_t box_cols, uint32_t box_rows, int swizzle_bytes);
// host: SM count of the current device, queried once per device  (kvq_capi.cu)
int num_sms_cached();

// host: the kernel flavour of a call as compile-time constants.  Calls f(GQA, BATCH, PAGED) with std::bool_constant
// arguments (GQA() is a constant expression, usable as a template argument) for exactly the six flavours that exist: a
// paged call is a batch, so there is no <BATCH = false, PAGED = true> instantiation.
template <class F>
inline auto with_flavour(bool gqa, bool batch, bool paged, F&& f) {
  auto g = [&](auto b, auto p) { return gqa ? f(std::true_type{}, b, p) : f(std::false_type{}, b, p); };
  return paged ? g(std::true_type{}, std::true_type{})
       : batch ? g(std::true_type{}, std::false_type{}) : g(std::false_type{}, std::false_type{});
}

}  // namespace kvq
