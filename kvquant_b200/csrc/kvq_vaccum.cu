// kvquant_b200 -- score.V decode matvec over the packed per-token-NUQ value cache, the fixed-width outlier
// stream fused in, optional fused softmax (exp(s - max) weights + denominators) for the attend path.
//
// Replaces (reference deployment/kvquant/quant_cuda_kernel.cu):
//   VecQuant{4,3,2}MatMulKernelNUQPerChannelTransposedMHABatchedFusedOpt   3211-3433, 4117-4491, 4998-5248
//   SPMV_ATOMIC_BALANCED                                                    436-470
//
//   O[h,c] = sum_t w[h,t] * (LUT[t, code(h,c,t)] (+) outlier(h,c,t))
//
// This file: the generic per-token-LUT kernel (legacy op surface kvq_v_matvec, and the fused attend over a cache given
// as materialised LUT rows only).  The native fused-path V kernel is kvq_vnative.cu, the attend itself kvq_attend.cu.
//
// Design (DESIGN.md section 4.2):
//   * one CTA streams a contiguous token range for ALL heads: the [H*W rows x 32 tokens] code slab of a tile is
//     fetched by TMA (cp.async.bulk.tensor.2d, 128B swizzle, boxes of 32 rows) into a 2-4 stage shared-memory ring
//     behind mbarriers, together with the tile's per-token LUT rows (cp.async.bulk); nothing is re-read;
//   * head split: where the whole slab does not fit shared memory next to the weights and the outlier accumulator
//     (4-bit H >= 48, 3-bit H >= 60), the grid gains a second dimension of G = 2 head groups and CTA (r, g) streams
//     only heads [g*H/2, (g+1)*H/2) of token range r, as the native kernel does (kvq_vnative.cu).  The two CTAs of a
//     range write disjoint heads of the same partial row (fused) or of `mul` (legacy);
//   * thread = packed word row (8 / 11 / 8 channels): channels stay in registers for the whole range, so there is
//     no cross-thread reduction per tile (the reference transposes through a 43.5 KB smem tile with 5 barriers
//     per 128 tokens and finishes with 128 global atomics per block);
//   * LUT rows are per token, all lanes of a warp work on the same token -> a lookup touches <= 16 distinct
//     consecutive words: conflict-free;
//   * outliers scatter into a shared-memory accumulator (42 shared atomics per token instead of 42 global
//     atomics onto 4096 hot addresses).
#include "kvq_attend.cuh"

namespace kvq {

constexpr int kVThreads = 512;
constexpr int kVT = 32;        // tokens per stage
constexpr int kVMaxStages = 4;
constexpr int kVMaxWPre = 4;   // prefetched weights per thread  (H*32/512 <= 4  -> H <= 64)
constexpr int kVMaxOPre = 4;   // prefetched outlier entries per thread (32*n_out/512 <= 4 -> n_out <= 64)
constexpr int kVBoxRows = 32;  // packed-word rows per TMA box
constexpr uint32_t kVBoxBytes = kVBoxRows * kVT * 4;   // 4 KiB: a box lands 1024-aligned, as the 128B swizzle needs

struct VParams {
  const float* score;        // [H, score_stride]: legacy = probabilities; fused = scaled scores
  const float* lut_tok;      // [Lmax, N]
  float* out;                // legacy: mul [H,128] (atomicAdd); fused: partial o [n_cta][H][128]
  float* out_l;              // fused: partial denominators [n_cta][H]; else null
  const float* gmax;         // fused: per-head max of the scaled scores; else null
  const float* outliers;     // [>=L, n_out] or null
  const int32_t* outlier_idx;
  int64_t Lmax, L, score_stride;
  int H, n_out, tiles_per_cta, n_stages, fused;
};

template <int BITS> struct VCfg {
  static constexpr int N = 1 << BITS;
  static constexpr int W = Layout<BITS>::kWords;
  static constexpr int CH = (BITS == 3) ? 11 : 8;  // channels per thread-unit
};

// smem carve-up (all offsets from a 1024-aligned base) for a CTA of Hg heads, rows = Hg*W packed-word rows.
// The stage holds whole 32-row boxes: the number of boxes issued and the bytes a stage's mbarrier expects both come
// from nbox (3-bit rows = 12*Hg is not a multiple of 32 when Hg % 8 == 4; the rows of the last box past the group
// are another group's or, past the tensor, zero-filled by TMA -- counted either way, never read).
struct VSmem {
  int nbox;              // 32-row TMA boxes per stage
  uint32_t stage_bytes;  // codes per stage (nbox * 4 KiB)
  uint32_t off_lut, off_w, off_oacc, off_bar, total;
};
__host__ __device__ inline VSmem v_smem_layout(int rows, int N, int Hg, int n_stages) {
  VSmem s;
  s.nbox = (rows + kVBoxRows - 1) / kVBoxRows;
  s.stage_bytes = (uint32_t)s.nbox * kVBoxBytes;
  s.off_lut = s.stage_bytes * n_stages;
  s.off_w = s.off_lut + (uint32_t)n_stages * kVT * N * 4;
  s.off_oacc = s.off_w + 2u * Hg * kVT * 4;
  s.off_bar = s.off_oacc + (uint32_t)Hg * kHeadDim * 4;
  s.total = s.off_bar + 8u * kVMaxStages;
  return s;
}

// one tile (32 tokens) of dense accumulation for one thread-unit.
// rowp: smem address of this unit's word row inside the stage (row_in_box*128 + box*4096), swz = row & 7.
template <int BITS, int SUB>
__device__ __forceinline__ void v_tile_unit(const unsigned char* stage, uint32_t row_off, uint32_t swz,
                                            uint32_t row_off2, uint32_t swz2, int part,
                                            const float* __restrict__ lut_tile, const float* __restrict__ wrow,
                                            float* __restrict__ acc) {
  constexpr int N = VCfg<BITS>::N;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const uint4 wa = *reinterpret_cast<const uint4*>(stage + row_off + ((q ^ swz) << 4));
    uint4 wb = make_uint4(0, 0, 0, 0);
    if constexpr (BITS == 3 && SUB < 2) wb = *reinterpret_cast<const uint4*>(stage + row_off2 + ((q ^ swz2) << 4));
    const float4 wt4 = *reinterpret_cast<const float4*>(wrow + 4 * q);
    const uint32_t wav[4] = {wa.x, wa.y, wa.z, wa.w};
    const uint32_t wbv[4] = {wb.x, wb.y, wb.z, wb.w};
    const float wtv[4] = {wt4.x, wt4.y, wt4.z, wt4.w};
#pragma unroll
    for (int tt = 0; tt < 4; ++tt) {
      const float* lr = lut_tile + (4 * q + tt) * N;
      const float wt = wtv[tt];
      if constexpr (BITS == 4) {
        const uint32_t w = wav[tt];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = fmaf(wt, lr[(w >> (4 * k)) & 0xFu], acc[k]);
      } else if constexpr (BITS == 2) {
        const uint32_t w = wav[tt] >> (16 * part);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = fmaf(wt, lr[(w >> (2 * k)) & 0x3u], acc[k]);
      } else {
        const uint32_t w = wav[tt];
#pragma unroll
        for (int k = 0; k < 10; ++k) acc[k] = fmaf(wt, lr[(w >> (SUB + 3 * k)) & 0x7u], acc[k]);
        if constexpr (SUB < 2) {
          const uint32_t c = ((w >> (30 + SUB)) | (wbv[tt] << (2 - SUB))) & 0x7u;
          acc[10] = fmaf(wt, lr[c], acc[10]);
        }
      }
    }
  }
}

// SPLIT: gridDim.y head groups (see the head split above); SPLIT = false is the whole-slab launch with h0 = 0
template <int BITS, bool SPLIT>
__global__ void __launch_bounds__(kVThreads, 1) v_accum_kernel(const __grid_constant__ CUtensorMap tmap, const VParams p) {
  using C = VCfg<BITS>;
  constexpr int N = C::N, W = C::W, CH = C::CH;
  extern __shared__ unsigned char smem_raw[];
  // 128B-swizzled TMA boxes need a 1024-byte aligned base
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int Hg = SPLIT ? p.H / (int)gridDim.y : p.H;     // heads of this CTA: [h0, h0 + Hg)
  const int h0 = SPLIT ? (int)blockIdx.y * Hg : 0;
  const int rows = Hg * W;
  const VSmem lay = v_smem_layout(rows, N, Hg, p.n_stages);
  float* s_lut = reinterpret_cast<float*>(smem + lay.off_lut);   // [n_stages][32][N]
  float* s_w = reinterpret_cast<float*>(smem + lay.off_w);       // [2][Hg][32]
  float* s_oacc = reinterpret_cast<float*>(smem + lay.off_oacc); // [Hg*128]
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(smem + lay.off_bar);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int S = p.n_stages;
  const int hidden = p.H * kHeadDim;

  // ---- thread -> unit mapping (up to 2 units per thread); u_head is relative to h0 ---------------------------
  // 4-bit: unit = word row (8 channels).  2-bit: unit = half a word row (8 channels).
  // 3-bit: warp-uniform SUB = warp % 3; unit = (32-channel group gi, SUB): row 3*gi+SUB (11/11/10 channels).
  int u_row[2], u_head[2], u_ch0[2], u_part[2];
  bool u_on[2];
  int sub = 0;
  if constexpr (BITS == 3) {
    sub = warp % 3;
    const int tri = warp / 3;            // 5 full warp-triples in 16 warps (warp 15 idles)
    const int ngroups = Hg * 4;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int gi = tri * 32 + lane + i * 160;
      u_on[i] = (warp < 15) && gi < ngroups;
      u_row[i] = 3 * gi + sub;
      u_head[i] = gi >> 2;
      u_ch0[i] = (gi & 3) * 32 + (sub == 0 ? 0 : (sub == 1 ? 11 : 22));
      u_part[i] = 0;
    }
  } else {
    const int nunits = Hg * 16;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int u = tid + i * kVThreads;
      u_on[i] = u < nunits;
      if constexpr (BITS == 4) { u_row[i] = u; u_part[i] = 0; u_head[i] = u >> 4; u_ch0[i] = (u & 15) * 8; }
      else { u_row[i] = u >> 1; u_part[i] = u & 1; u_head[i] = u >> 4; u_ch0[i] = ((u >> 1) & 7) * 16 + (u & 1) * 8; }
    }
  }
  uint32_t r_off[2], r_swz[2], r_off2[2], r_swz2[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = u_on[i] ? u_row[i] : 0;
    r_off[i] = (uint32_t)r * 128u;   // boxes of 32 rows back to back: row r sits at r*128 inside the stage
    r_swz[i] = (uint32_t)(r & 7);
    const int r2 = (r + 1 < rows) ? r + 1 : r;
    r_off2[i] = (uint32_t)r2 * 128u;
    r_swz2[i] = (uint32_t)(r2 & 7);
  }
  float acc[2][CH];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int k = 0; k < CH; ++k) acc[i][k] = 0.f;

  for (int i = tid; i < Hg * kHeadDim; i += kVThreads) s_oacc[i] = 0.f;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) mbar_init(&s_bar[s], 1);
    mbar_fence_init();
    prefetch_tensormap(&tmap);
  }

  const int64_t n_tiles_total = (p.L + kVT - 1) / kVT;
  const int64_t tile0 = (int64_t)blockIdx.x * p.tiles_per_cta;
  const int ntiles = (int)max((int64_t)0, min((int64_t)p.tiles_per_cta, n_tiles_total - tile0));

  auto issue_tile = [&](int it) {  // thread 0 only
    const int s = it % S;
    const int64_t t0 = (tile0 + it) * kVT;
    const uint32_t lut_bytes = (uint32_t)min((int64_t)kVT, p.Lmax - t0) * N * 4;  // never read past the LUT allocation
    mbar_expect_tx(&s_bar[s], lay.stage_bytes + lut_bytes);
    unsigned char* dst = smem + (size_t)s * lay.stage_bytes;
    for (int b = 0; b < lay.nbox; ++b)
      tma_load_2d(dst + b * kVBoxBytes, &tmap, &s_bar[s], (int)t0, h0 * W + b * kVBoxRows);
    bulk_load_1d(s_lut + s * kVT * N, p.lut_tok + t0 * N, lut_bytes, &s_bar[s]);
  };
  // weights of a tile: exp(s - max) in fused mode, the given probabilities otherwise; 0 beyond L
  const int n_w = Hg * kVT;  // values per tile
  float wpre[kVMaxWPre];
  auto load_weights = [&](int it) {
    const int64_t t0 = (tile0 + it) * kVT;
#pragma unroll
    for (int i = 0; i < kVMaxWPre; ++i) {
      const int e = tid + i * kVThreads;
      float w = 0.f;
      if (e < n_w) {
        const int h = e >> 5, tl = e & 31;
        if (t0 + tl < p.L) {
          w = p.score[(int64_t)(h0 + h) * p.score_stride + t0 + tl];
          if (p.fused) w = __expf(w - p.gmax[h0 + h]);
        }
      }
      wpre[i] = w;
    }
  };
  auto store_weights = [&](int buf) {
#pragma unroll
    for (int i = 0; i < kVMaxWPre; ++i) {
      const int e = tid + i * kVThreads;
      if (e < n_w) s_w[buf * n_w + e] = wpre[i];
    }
  };
  float opre_v[kVMaxOPre];
  int opre_i[kVMaxOPre];
  const bool has_out = p.outliers != nullptr;
  // a V outlier row spans all heads: a head-split CTA applies the entries of its own heads only
  auto own_head = [&](int idx) { return !SPLIT || (unsigned)((idx >> 7) - h0) < (unsigned)Hg; };
  auto load_outliers = [&](int it) {
    const int64_t t0 = (tile0 + it) * kVT;
    const int ntok = (int)min((int64_t)kVT, p.L - t0);
    const int total = ntok * p.n_out;
    const float* ov = p.outliers + t0 * p.n_out;
    const int32_t* oi = p.outlier_idx + t0 * p.n_out;
#pragma unroll
    for (int i = 0; i < kVMaxOPre; ++i) {
      const int e = tid + i * kVThreads;
      opre_v[i] = 0.f; opre_i[i] = 0;
      if (e < total) { opre_v[i] = ov[e]; opre_i[i] = oi[e]; }
    }
  };

  __syncthreads();  // barriers initialised, s_oacc zeroed
  if (ntiles > 0) {
    if (tid == 0)
      for (int it = 0; it < S - 1 && it < ntiles; ++it) issue_tile(it);
    load_weights(0);
    store_weights(0);
  }

  // per-head denominators (fused): every weight passes through exactly one thread's wpre[] -> accumulate there
  float lacc[kVMaxWPre];
#pragma unroll
  for (int i = 0; i < kVMaxWPre; ++i) lacc[i] = (ntiles > 0) ? wpre[i] : 0.f;

  for (int it = 0; it < ntiles; ++it) {
    __syncthreads();  // tile it-1 fully consumed (its stage and weight buffer are free); weights of `it` visible
    if (tid == 0 && it + S - 1 < ntiles) issue_tile(it + S - 1);
    const bool more = it + 1 < ntiles;
    if (more) load_weights(it + 1);
    if (has_out) load_outliers(it);
    const int s = it % S;
    mbar_wait(&s_bar[s], (uint32_t)((it / S) & 1));
    const unsigned char* stage = smem + (size_t)s * lay.stage_bytes;
    const float* lut_tile = s_lut + s * kVT * N;
    {
      // the allocation's last tile: LUT rows past Lmax were not loaded (issue_tile) and the stage may still hold
      // whatever an earlier kernel left in shared memory -- a NaN there would survive its zero weight.  Clear them
      // (CTA-uniform branch; this is the last tile any CTA streams, so no later copy lands on these rows)
      const int64_t t0 = (tile0 + it) * kVT;
      if (t0 + kVT > p.Lmax) {
        for (int i = (int)(p.Lmax - t0) * N + tid; i < kVT * N; i += kVThreads) s_lut[s * kVT * N + i] = 0.f;
        __syncthreads();
      }
    }
    const float* wbuf = s_w + (it & 1) * n_w;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (u_on[i]) {
        const float* wrow = wbuf + u_head[i] * kVT;
        if constexpr (BITS == 3) {
          if (sub == 0) v_tile_unit<3, 0>(stage, r_off[i], r_swz[i], r_off2[i], r_swz2[i], 0, lut_tile, wrow, acc[i]);
          else if (sub == 1) v_tile_unit<3, 1>(stage, r_off[i], r_swz[i], r_off2[i], r_swz2[i], 0, lut_tile, wrow, acc[i]);
          else v_tile_unit<3, 2>(stage, r_off[i], r_swz[i], r_off2[i], r_swz2[i], 0, lut_tile, wrow, acc[i]);
        } else {
          v_tile_unit<BITS, 0>(stage, r_off[i], r_swz[i], 0, 0, u_part[i], lut_tile, wrow, acc[i]);
        }
      }
    }
    if (has_out) {
      const int64_t t0 = (tile0 + it) * kVT;
      const int ntok = (int)min((int64_t)kVT, p.L - t0);
      const int total = ntok * p.n_out;
#pragma unroll
      for (int i = 0; i < kVMaxOPre; ++i) {
        const int e = tid + i * kVThreads;
        if (e < total && opre_v[i] != 0.f && own_head(opre_i[i])) {
          const int idx = opre_i[i] - h0 * kHeadDim;
          const int tl = e / p.n_out;
          atomicAdd(&s_oacc[idx], opre_v[i] * wbuf[(idx >> 7) * kVT + tl]);
        }
      }
      for (int e = tid + kVMaxOPre * kVThreads; e < total; e += kVThreads) {  // n_out > 64: unprefetched tail
        const float v = p.outliers[t0 * p.n_out + e];
        const int idx = p.outlier_idx[t0 * p.n_out + e] - h0 * kHeadDim;
        if (v != 0.f && own_head(idx + h0 * kHeadDim)) atomicAdd(&s_oacc[idx], v * wbuf[(idx >> 7) * kVT + e / p.n_out]);
      }
    }
    if (more) {
      store_weights((it + 1) & 1);
#pragma unroll
      for (int i = 0; i < kVMaxWPre; ++i) lacc[i] += wpre[i];
    }
  }
  __syncthreads();

  // ---- epilogue --------------------------------------------------------------------------------------------
  if (p.fused) {
    float* s_l = s_w;  // reuse: [Hg]
    for (int i = tid; i < Hg; i += kVThreads) s_l[i] = 0.f;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kVMaxWPre; ++i) {
      const int e = tid + i * kVThreads;
      if (e < n_w) {
        const float v = warp_sum(lacc[i]);   // a warp's 32 slots are the 32 tokens of one head
        if (lane == 0) atomicAdd(&s_l[e >> 5], v);
      }
    }
    __syncthreads();
    for (int i = tid; i < Hg; i += kVThreads) p.out_l[(int64_t)blockIdx.x * p.H + h0 + i] = s_l[i];
  }
  float* obase = p.fused ? (p.out + (int64_t)blockIdx.x * hidden) : p.out;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (u_on[i]) {
      const int nch = (BITS == 3 && sub == 2) ? 10 : CH;
#pragma unroll
      for (int k = 0; k < CH; ++k) {
        if (k < nch) {
          const int j = u_head[i] * kHeadDim + u_ch0[i] + k;
          const float v = acc[i][k] + s_oacc[j];
          if (p.fused) obase[h0 * kHeadDim + j] = v;
          else atomicAdd(&obase[h0 * kHeadDim + j], v);
        }
      }
    }
  }
}

// ---- host side -----------------------------------------------------------------------------------------------
constexpr uint32_t kSmemBudget = 227u * 1024u;

// ring stages that fit next to the LUT rows, weights and outlier accumulator for a slab of Hg heads (largest
// first); 0 when not even two do
template <int BITS>
static int v_stages(int Hg, VSmem* lay) {
  using C = VCfg<BITS>;
  for (int S = kVMaxStages; S >= 2; --S) {
    *lay = v_smem_layout(Hg * C::W, C::N, Hg, S);
    if (lay->total + 1024u <= kSmemBudget) return S;
  }
  return 0;
}

template <int BITS, bool SPLIT>
static int launch_v_kernel(const CUtensorMap& tmap, const VParams& p, dim3 grid, uint32_t smem, cudaStream_t st) {
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(v_accum_kernel<BITS, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  v_accum_kernel<BITS, SPLIT><<<grid, kVThreads, smem, st>>>(tmap, p);
  KVQ_LAUNCH_CHECK();
  return 0;
}

// returns 0 and the number of partial rows written (token ranges) in *n_cta_out, or an error
template <int BITS>
static int launch_v(VParams p, const int32_t* cache, int* n_cta_out, cudaStream_t st) {
  using C = VCfg<BITS>;
  // G head groups: 1 while the whole slab fits (4-bit H <= 44, 3-bit H <= 56, 2-bit H <= 64), else 2.  G = 2 always
  // fits for H <= 64: Hg = H/2 <= 32 heads is at most the 7B slab.
  VSmem lay{};
  int G = 1;
  int S = v_stages<BITS>(p.H, &lay);
  if (S < 2) { G = 2; S = v_stages<BITS>(p.H / G, &lay); }
  if (S < 2) return KVQ_E_UNSUPPORTED;
  p.n_stages = S;
  // one map over the whole cache; a head-split CTA offsets the row coordinate by its group's first row
  CUtensorMap tmap;
  int rc = make_cache_tensor_map(&tmap, cache, (uint64_t)p.H * C::W, (uint64_t)p.Lmax, kVT, kVBoxRows, 128);
  if (rc != 0) return rc;
  // token ranges x head groups ~ one CTA per SM; the partial index is the token range
  const int64_t n_tiles = (p.L + kVT - 1) / kVT;
  const int ranges = max(1, num_sms_cached() / G);
  p.tiles_per_cta = (int)((n_tiles + ranges - 1) / ranges);
  const int n_cta = (int)((n_tiles + p.tiles_per_cta - 1) / p.tiles_per_cta);
  const dim3 grid(n_cta, G);
  rc = G == 1 ? launch_v_kernel<BITS, false>(tmap, p, grid, lay.total + 1024u, st)
              : launch_v_kernel<BITS, true>(tmap, p, grid, lay.total + 1024u, st);
  if (rc != 0) return rc;
  *n_cta_out = n_cta;
  return 0;
}

static int v_accum_dispatch(int bits, const VParams& p, const int32_t* cache, int* n_cta, cudaStream_t st) {
  switch (bits) {
    case 4: return launch_v<4>(p, cache, n_cta, st);
    case 3: return launch_v<3>(p, cache, n_cta, st);
    case 2: return launch_v<2>(p, cache, n_cta, st);
    default: return KVQ_E_BITS;
  }
}

// the fused attend over a cache given as materialised LUT rows only (kvq_attend without v_cent / v_aff)
int v_accum_fused(const AttendCall& c, const AttendScratch& s, int* n_cta) {
  VParams p{};
  p.score = s.scores; p.lut_tok = c.vlut_tok; p.out = s.part_o; p.out_l = s.part_l; p.gmax = s.gmax;
  p.outliers = c.v_outliers; p.outlier_idx = c.v_outlier_idx;
  p.Lmax = c.Lmax; p.L = c.L; p.score_stride = s.stride; p.H = c.Hq; p.n_out = c.n_out; p.fused = 1;
  return v_accum_dispatch(c.bits, p, c.vcache, n_cta, c.stream);
}

}  // namespace kvq

using namespace kvq;

extern "C" int kvq_v_matvec(int bits, const float* score, const int32_t* cache, float* mul, const float* lut_tok, int B,
                            int H, int64_t Lmax, int64_t L, const float* outliers, const int32_t* outlier_idx, int n_out,
                            void* stream) {
  if (!score || !cache || !mul || !lut_tok) return KVQ_E_NULL;
  if (B <= 0) return KVQ_E_SHAPE;
  int rc = check_v_common(H, Lmax, L, cache);
  if (rc) return rc;
  if ((reinterpret_cast<uintptr_t>(lut_tok) & 15) != 0) return KVQ_E_ALIGN;
  if ((outliers == nullptr) != (outlier_idx == nullptr)) return KVQ_E_NULL;
  if (outliers && (B != 1 || n_out <= 0)) return KVQ_E_SHAPE;
  if (L == 0) return 0;
  for (int b = 0; b < B; ++b) {
    VParams p{};
    p.score = score + (int64_t)b * H * L;
    p.lut_tok = lut_tok;
    p.out = mul + (int64_t)b * H * kHeadDim;
    p.out_l = nullptr; p.gmax = nullptr;
    p.outliers = outliers; p.outlier_idx = outlier_idx;
    p.Lmax = Lmax; p.L = L; p.score_stride = L;
    p.H = H; p.n_out = n_out; p.fused = 0;
    int n_cta = 0;
    rc = v_accum_dispatch(bits, p, cache, &n_cta, static_cast<cudaStream_t>(stream));
    if (rc) return rc;
  }
  return 0;
}
