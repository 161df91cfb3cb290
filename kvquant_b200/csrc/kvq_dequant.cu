// kvquant_b200 -- dequantisation of a slot range of a layer cache to fp16 K (pre-RoPE or rotated) and V.
//
// One kernel per side, persistent CTAs: CTA (x, y) owns head group y (kGroup heads) and walks the token tiles
// x, x + gridDim.x, ...  Per tile of kTile tokens:
//   1. the group's packed words are read coalesced along the sequence axis into shared memory, token-major
//      (so code_of<BITS> reads one token's words contiguously); K also stages the tile's cos/sin, V its (sf, off);
//   2. one thread per (head, token, 32-channel group) dequantises into an fp32 tile [kGroup][kTile][128 + 4]: the group's
//      words in registers, code_of<BITS> at compile-time channel offsets (K: the group's LUT, staged once per CTA as
//      [channel][2^BITS + 1], so the 32 tokens of a warp, one channel, meet distinct codes in distinct banks; V:
//      v_cent[code]*sf + off as one fma); padded rows keep the warp's 16-byte tile stores conflict-free;
//   3. the tile's outlier entries that fall in the group are added (shared-memory atomics: a V row may repeat
//      channel 0 as a pad, whose value 0 is skipped);
//   4. each thread converts 8 consecutive channels of one token to fp16 and writes them as one 16-byte store --
//      for rotated K after combining with the partner channels c ^ 64, which step 3 has already completed.
// The per-element arithmetic of steps 2-4 is kvq_dequant.cuh's, which kvq_chunk.cu calls too.
#include <cuda_fp16.h>

#include "kvq_common.cuh"
#include "kvq_dequant.cuh"

namespace kvq {

constexpr int kTile = 32;       // tokens per tile
constexpr int kGroup = 2;       // heads per CTA (every accepted H but 1 is even; H = 1: dequant_one_kernel)
constexpr int kThreads = 256;
constexpr int kRopePitch = 65;  // float2 per staged cos/sin row (one token); odd pitch spreads the transposing writes
constexpr int kTP = kHeadDim + 4;  // fp32 tile row pitch (one token of one head)

struct DqParams {
  const int32_t* cache;
  const float* klut;        // K: [H*128, 2^BITS]
  const float* v_cent;      // V: [2^BITS]
  const float* v_aff;       // V: [Lmax, 2] = (sf, off)
  const float* outliers;    // [Lmax, n_out] or NULL
  const int32_t* outlier_idx;
  const float2* rope;       // K: [64, rope_npos] (cos, sin) or NULL
  int64_t rope_npos;
  int64_t pos_offset;
  __half* out;
  int64_t head_stride;
  int64_t Lmax, start, stop;
  int n_out;
};

template <int BITS, int NG = kGroup>   // NG: heads per CTA
struct DqLayout {
  static constexpr int W = Layout<BITS>::kWords;
  static constexpr int kWPitch = W + 1;  // odd pitch: the transposing word stores of a warp hit distinct banks
  static constexpr int kWordsSmem = NG * kTile * kWPitch;
  static constexpr int kTileSmem = NG * kTile * kTP;
  static constexpr int kLP = Layout<BITS>::kLevels + 1;   // K LUT pitch per channel
};

template <int BITS, int NG = kGroup>
__host__ __device__ constexpr size_t dq_smem_bytes(bool is_v, bool rope) {
  using D = DqLayout<BITS, NG>;
  return sizeof(float) * (D::kTileSmem + D::kWordsSmem) +
         (is_v ? sizeof(float) * (Layout<BITS>::kLevels + 2 * kTile)
               : sizeof(float) * D::kLP * NG * kHeadDim + (rope ? sizeof(float2) * kTile * kRopePitch : 0));
}

// IS_V: V side (affine centroids) else K side (per-channel LUT, optional rotation).
// PAGED (dequant_paged_kernel, DESIGN.md section 4.12): p's cache pointers are page pools ([n_pool, H, W, P] words, rows
// [n_pool*P, .]) and pg.table is one sequence's page-table row; slot s is read from page pg.table[s / P], column s % P.
// The tiles are the contiguous kernel's, and every read looks its token's page up (a 32-token tile starting at any
// `start` may straddle a page boundary); the arithmetic and the output offsets are those of logical slots.
template <int BITS, bool IS_V, bool ROPE, bool PAGED, int NG = kGroup>
__device__ __forceinline__ void dequant_body(const DqParams& p, const PageRef& pg) {
  using D = DqLayout<BITS, NG>;
  constexpr int W = D::W;
  constexpr int NL = Layout<BITS>::kLevels;
  extern __shared__ __align__(16) float smem[];
  float* tile = smem;                                                       // [NG][kTile][kTP]
  uint32_t* words = reinterpret_cast<uint32_t*>(tile + D::kTileSmem);       // [NG][kTile][kWPitch]
  float* tab = reinterpret_cast<float*>(words + D::kWordsSmem);             // K: LUT [NG*128][kLP]; V: cent[NL], aff[kTile][2]
  float2* cs = reinterpret_cast<float2*>(tab + D::kLP * NG * kHeadDim); // K + ROPE: [kTile][kRopePitch]
  float* aff = tab + NL;

  const int tid = threadIdx.x;
  const int h0 = blockIdx.y * NG;
  if constexpr (IS_V) {
    if (tid < NL) tab[tid] = p.v_cent[tid];
  } else {
    for (int i = tid; i < NG * kHeadDim * NL; i += kThreads)
      tab[(i / NL) * D::kLP + i % NL] = p.klut[(int64_t)h0 * kHeadDim * NL + i];
  }

  const int64_t n = p.stop - p.start;
  const int64_t n_tiles = (n + kTile - 1) / kTile;
  for (int64_t tl = blockIdx.x; tl < n_tiles; tl += gridDim.x) {
    const int64_t t0 = p.start + tl * kTile;                  // first slot of the tile
    const int nt = (int)min((int64_t)kTile, p.stop - t0);
    __syncthreads();                                          // previous tile fully written out
    if constexpr (PAGED) {
      static_assert(kThreads % kTile == 0, "a thread keeps one token of the tile through the word loads");
      const int t = tid % kTile;                              // = i % kTile for every i of this thread below
      int64_t base = 0;                                       // word row 0 of the group at token t's page column
      if (t < nt) {
        const PageCol pc = page_col(pg, (int)(t0 + t));
        base = ((int64_t)pc.page * gridDim.y * NG + h0) * W * pg.P + pc.col;
      }
      for (int i = tid; i < NG * W * kTile; i += kThreads) {
        const int r = i / kTile;
        uint32_t w = 0;
        if (t < nt) w = static_cast<uint32_t>(p.cache[base + (int64_t)r * pg.P]);
        words[((r / W) * kTile + t) * D::kWPitch + (r % W)] = w;
      }
    } else {
      for (int i = tid; i < NG * W * kTile; i += kThreads) {
        const int r = i / kTile, t = i % kTile;               // r: word row within the group, t fastest (coalesced)
        uint32_t w = 0;
        if (t < nt) w = static_cast<uint32_t>(p.cache[((int64_t)h0 * W + r) * p.Lmax + t0 + t]);
        words[((r / W) * kTile + t) * D::kWPitch + (r % W)] = w;
      }
    }
    if constexpr (IS_V) {
      if constexpr (PAGED) {
        if (tid < 2 * kTile) aff[tid] = tid < 2 * nt ? p.v_aff[2 * page_row(pg, (int)(t0 + tid / 2)) + (tid & 1)] : 0.f;
      } else {
        if (tid < 2 * kTile) aff[tid] = tid < 2 * nt ? p.v_aff[2 * t0 + tid] : 0.f;
      }
    } else if constexpr (ROPE) {
      for (int i = tid; i < 64 * kTile; i += kThreads) {
        const int j = i / kTile, t = i % kTile;                // position-fastest table: t fastest is coalesced
        cs[t * kRopePitch + j] = t < nt ? p.rope[(int64_t)j * p.rope_npos + p.pos_offset + t0 + t] : make_float2(0.f, 0.f);
      }
    }
    __syncthreads();
    for (int i = tid; i < NG * kTile * 4; i += kThreads) {
      const int t = i % kTile, q = (i / kTile) % 4, g = i / (4 * kTile);   // lanes: 32 tokens of one channel group
      constexpr int WQ = W / 4;                                // words of 32 channels: 4 / 3 / 2
      uint32_t w[WQ];
#pragma unroll
      for (int k = 0; k < WQ; ++k) w[k] = words[(g * kTile + t) * D::kWPitch + q * WQ + k];
      float* dst = tile + (g * kTile + t) * kTP + q * 32;
      if constexpr (IS_V) dq_quarter<BITS, true>(w, tab, 0, aff[2 * t], aff[2 * t + 1], dst);
      else dq_quarter<BITS, false>(w, tab + (g * kHeadDim + q * 32) * D::kLP, D::kLP, 0.f, 0.f, dst);
    }
    if (p.outliers != nullptr) {
      __syncthreads();
      if constexpr (PAGED) {
        for (int i = tid; i < nt * p.n_out; i += kThreads) {
          const int j = i / p.n_out;                          // token of the tile
          const int64_t e = page_row(pg, (int)(t0 + j)) * p.n_out + (i - j * p.n_out);
          const int idx = p.outlier_idx[e];
          const int g = (idx >> 7) - h0;
          if (g >= 0 && g < NG) dq_add_outlier(&tile[(g * kTile + j) * kTP + (idx & 127)], p.outliers[e]);
        }
      } else {
        const int64_t row0 = t0 * p.n_out;
        for (int i = tid; i < nt * p.n_out; i += kThreads) {
          const int idx = p.outlier_idx[row0 + i];
          const int g = (idx >> 7) - h0;
          if (g >= 0 && g < NG) {
            const float v = p.outliers[row0 + i];
            dq_add_outlier(&tile[(g * kTile + i / p.n_out) * kTP + (idx & 127)], v);
          }
        }
      }
    }
    __syncthreads();
    for (int i = tid; i < NG * kTile * (kHeadDim / 8); i += kThreads) {
      const int q = i % (kHeadDim / 8), gt = i / (kHeadDim / 8);
      const int t = gt % kTile, g = gt / kTile;
      if (t >= nt) continue;
      const int c0 = q * 8;
      // rotated K: k'[c] = cos*k[c] - sin*k[c+64] (c < 64), cos*k[c] + sin*k[c-64] (c >= 64); j = c mod 64
      const uint4 o = dq_finish8<!IS_V && ROPE>(tile + gt * kTP, c0, cs + t * kRopePitch + (c0 & 63));
      __half* dst = p.out + (int64_t)(h0 + g) * p.head_stride + (t0 - p.start + t) * kHeadDim + c0;
      *reinterpret_cast<uint4*>(dst) = o;
    }
  }
}

// contiguous cache of p.Lmax slots
template <int BITS, bool IS_V, bool ROPE>
__global__ void __launch_bounds__(kThreads, 3) dequant_kernel(const DqParams p) {
  dequant_body<BITS, IS_V, ROPE, false>(p, PageRef{});
}

// one paged sequence, pg.table its page-table row (a kernel of its own name: a PAGED template argument would rename
// the contiguous instantiations above)
template <int BITS, bool IS_V, bool ROPE>
__global__ void __launch_bounds__(kThreads, 3) dequant_paged_kernel(const DqParams p, const PageRef pg) {
  dequant_body<BITS, IS_V, ROPE, true>(p, pg);
}

// one KV head (H = 1, multi-query caches): CTAs of one head, contiguous (pg.table == nullptr) or paged.  Kernels of
// their own name: an NG template argument would rename the instantiations above.
template <int BITS, bool IS_V, bool ROPE>
__global__ void __launch_bounds__(kThreads, 3) dequant_one_kernel(const DqParams p, const PageRef pg) {
  if (pg.table == nullptr) dequant_body<BITS, IS_V, ROPE, false, 1>(p, pg);
  else dequant_body<BITS, IS_V, ROPE, true, 1>(p, pg);
}

template <int BITS, bool IS_V, bool ROPE>
int launch_dequant(const DqParams& p, int H, cudaStream_t st, const PageRef* pg) {
  const bool one = H == 1;
  const void* kern = one ? reinterpret_cast<const void*>(dequant_one_kernel<BITS, IS_V, ROPE>)
                     : pg != nullptr ? reinterpret_cast<const void*>(dequant_paged_kernel<BITS, IS_V, ROPE>)
                                     : reinterpret_cast<const void*>(dequant_kernel<BITS, IS_V, ROPE>);
  const size_t smem = one ? dq_smem_bytes<BITS, 1>(IS_V, ROPE) : dq_smem_bytes<BITS>(IS_V, ROPE);
  static PerDeviceOnce attr_once[3];   // (per form)
  bool& attr_done = attr_once[one ? 2 : pg != nullptr].cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  int dev = 0, sms = 0, per_sm = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem);
  if (e != cudaSuccess) return (int)e;
  // one wave of resident CTAs: the head groups side by side (they read the same tile's outlier rows and cos/sin at
  // about the same time), the token tiles split evenly over the rest
  const int groups = one ? 1 : H / kGroup;
  const int64_t n_tiles = (p.stop - p.start + kTile - 1) / kTile;
  const int64_t per_group = max(1, sms * max(per_sm, 1) / groups);
  const dim3 grid((unsigned)min(n_tiles, per_group), (unsigned)groups);
  if (one) dequant_one_kernel<BITS, IS_V, ROPE><<<grid, kThreads, smem, st>>>(p, pg != nullptr ? *pg : PageRef{});
  else if (pg != nullptr) dequant_paged_kernel<BITS, IS_V, ROPE><<<grid, kThreads, smem, st>>>(p, *pg);
  else dequant_kernel<BITS, IS_V, ROPE><<<grid, kThreads, smem, st>>>(p);
  KVQ_LAUNCH_CHECK();
  return 0;
}

template <int BITS>
int dequant_bits(const DqParams& pk, const DqParams& pv, int H, cudaStream_t st, const PageRef* pg) {
  int rc = 0;
  if (pk.out)
    rc = pk.rope ? launch_dequant<BITS, false, true>(pk, H, st, pg) : launch_dequant<BITS, false, false>(pk, H, st, pg);
  if (rc == 0 && pv.out) rc = launch_dequant<BITS, true, false>(pv, H, st, pg);
  return rc;
}

// the dequantisation of a contiguous cache (pg == nullptr; Lmax > 0) or of one paged sequence (Lmax = its mapped
// slots, possibly 0): every check, then the two launches
static int dequant_impl(int bits, int H, int64_t Lmax, int64_t start, int64_t stop, const int32_t* kcache,
                        const float* klut, const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                        const float* v_cent, const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx,
                        int n_out, const float* rope_cos_sin, int64_t rope_npos, int pos_offset, void* out_k,
                        void* out_v, int64_t head_stride, void* stream, const PageRef* pg) {
  if (bits < 2 || bits > 4) return KVQ_E_BITS;
  if (H <= 0 || ((H & 3) != 0 && H > 2) || H > 64 || Lmax < 0 || (Lmax == 0 && pg == nullptr) || start < 0 || start > stop ||
      stop > Lmax)
    return KVQ_E_SHAPE;
  if (n_out < 0 || (n_out & 1) != 0 || n_out > kMaxOutDq) return KVQ_E_SHAPE;
  if (head_stride < (stop - start) * kHeadDim) return KVQ_E_SHAPE;
  if (start == stop) return 0;   // nothing to write: outputs of zero elements may well be NULL
  if (!out_k && !out_v) return KVQ_E_NULL;
  if (out_k && (!kcache || !klut)) return KVQ_E_NULL;
  if (out_v && (!vcache || !v_cent || !v_aff)) return KVQ_E_NULL;
  if ((k_outliers == nullptr) != (k_outlier_idx == nullptr) || (v_outliers == nullptr) != (v_outlier_idx == nullptr))
    return KVQ_E_NULL;
  if (pg != nullptr && pg->table == nullptr) return KVQ_E_NULL;
  if ((k_outliers || v_outliers) && n_out == 0) return KVQ_E_SHAPE;
  if (out_k && rope_cos_sin && (pos_offset < 0 || rope_npos < (int64_t)pos_offset + stop)) return KVQ_E_SHAPE;
  if ((head_stride & 7) != 0 || (reinterpret_cast<uintptr_t>(out_k) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(out_v) & 15) != 0)
    return KVQ_E_ALIGN;

  DqParams pk{}, pv{};
  pk.Lmax = pv.Lmax = Lmax;
  pk.start = pv.start = start;
  pk.stop = pv.stop = stop;
  pk.head_stride = pv.head_stride = head_stride;
  pk.n_out = pv.n_out = n_out;
  pk.cache = kcache; pk.klut = klut; pk.outliers = k_outliers; pk.outlier_idx = k_outlier_idx;
  pk.rope = reinterpret_cast<const float2*>(rope_cos_sin); pk.rope_npos = rope_npos; pk.pos_offset = pos_offset;
  pk.out = static_cast<__half*>(out_k);
  pv.cache = vcache; pv.v_cent = v_cent; pv.v_aff = v_aff; pv.outliers = v_outliers; pv.outlier_idx = v_outlier_idx;
  pv.out = static_cast<__half*>(out_v);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (bits) {
    case 4: return dequant_bits<4>(pk, pv, H, st, pg);
    case 3: return dequant_bits<3>(pk, pv, H, st, pg);
    default: return dequant_bits<2>(pk, pv, H, st, pg);
  }
}

}  // namespace kvq

using namespace kvq;

extern "C" int kvq_dequant_kv(int bits, int H, int64_t Lmax, int64_t start, int64_t stop,
                              const int32_t* kcache, const float* klut, const float* k_outliers,
                              const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent,
                              const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx, int n_out,
                              const float* rope_cos_sin, int64_t rope_npos, int pos_offset, void* out_k, void* out_v,
                              int64_t head_stride, void* stream) {
  return dequant_impl(bits, H, Lmax, start, stop, kcache, klut, k_outliers, k_outlier_idx, vcache, v_cent, v_aff,
                      v_outliers, v_outlier_idx, n_out, rope_cos_sin, rope_npos, pos_offset, out_k, out_v, head_stride,
                      stream, nullptr);
}

extern "C" int kvq_dequant_kv_paged(int bits, int H, int n_pool, int64_t start, int64_t stop,
                                    const int32_t* kcache, const float* klut, const float* k_outliers,
                                    const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent,
                                    const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx,
                                    int n_out, const float* rope_cos_sin, int64_t rope_npos, int pos_offset,
                                    void* out_k, void* out_v, int64_t head_stride, void* stream,
                                    const int32_t* pages, int max_pages, int n_mapped, int P) {
  if (bits < 2 || bits > 4) return KVQ_E_BITS;
  if (H <= 0) return KVQ_E_SHAPE;
  const int rc = check_pages(n_pool, max_pages, P, (int64_t)H * kHeadDim * bits / 32);
  if (rc) return rc;
  if (n_mapped < 0 || n_mapped > max_pages) return KVQ_E_SHAPE;
  const PageRef pg{pages, nullptr, max_pages, P, n_pool};
  return dequant_impl(bits, H, (int64_t)n_mapped * P, start, stop, kcache, klut, k_outliers, k_outlier_idx, vcache,
                      v_cent, v_aff, v_outliers, v_outlier_idx, n_out, rope_cos_sin, rope_npos, pos_offset, out_k,
                      out_v, head_stride, stream, &pg);
}
