// kvquant_b200 -- score.V decode matvec over the packed per-token-NUQ value cache, the fixed-width outlier
// stream fused in, optional fused softmax (exp(s - max) weights + denominators) for the attend path.
//
// Replaces (reference deployment/kvquant/quant_cuda_kernel.cu):
//   VecQuant{4,3,2}MatMulKernelNUQPerChannelTransposedMHABatchedFusedOpt   3211-3433, 4117-4491, 4998-5248
//   SPMV_ATOMIC_BALANCED                                                    436-470
//
//   O[h,c] = sum_t w[h,t] * (LUT[t, code(h,c,t)] (+) outlier(h,c,t))
//
// This file: the generic per-token-LUT kernel (legacy op surface, and the fused path over a cache given as
// materialised LUT rows only), the attend_init / attend_combine / attend_merge kernels, the TMA descriptor helper
// and the kvq_attend entry points.  The native fused-path V kernel is kvq_vnative.cu.
//
// Design (DESIGN.md section 4.2):
//   * one CTA streams a contiguous token range for ALL heads: the [H*W rows x 32 tokens] code slab of a tile is
//     fetched by TMA (cp.async.bulk.tensor.2d, 128B swizzle) into a 2-4 stage shared-memory ring behind mbarriers,
//     together with the tile's per-token LUT rows (cp.async.bulk); nothing is re-read;
//   * thread = packed word row (8 / 11 / 8 channels): channels stay in registers for the whole range, so there is
//     no cross-thread reduction per tile (the reference transposes through a 43.5 KB smem tile with 5 barriers
//     per 128 tokens and finishes with 128 global atomics per block);
//   * LUT rows are per token, all lanes of a warp work on the same token -> a lookup touches <= 16 distinct
//     consecutive words: conflict-free;
//   * outliers scatter into a shared-memory accumulator (42 shared atomics per token instead of 42 global
//     atomics onto 4096 hot addresses).
#include "kvq_common.cuh"
#include <stdlib.h>
#include <cuda_fp16.h>
#include <dlfcn.h>

namespace kvq {

constexpr int kVThreads = 512;
constexpr int kVT = 32;        // tokens per stage
constexpr int kVMaxStages = 4;
constexpr int kVMaxWPre = 4;   // prefetched weights per thread  (H*32/512 <= 4  -> H <= 64)
constexpr int kVMaxOPre = 4;   // prefetched outlier entries per thread (32*n_out/512 <= 4 -> n_out <= 64)

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

// smem carve-up (all offsets from a 1024-aligned base)
struct VSmem {
  uint32_t stage_bytes;  // codes per stage (rows*128)
  uint32_t off_lut, off_w, off_oacc, off_bar, total;
};
__host__ __device__ inline VSmem v_smem_layout(int rows, int N, int H, int n_stages) {
  VSmem s;
  s.stage_bytes = (uint32_t)rows * 128u;
  s.off_lut = s.stage_bytes * n_stages;
  s.off_w = s.off_lut + (uint32_t)n_stages * kVT * N * 4;
  s.off_oacc = s.off_w + 2u * H * kVT * 4;
  s.off_bar = s.off_oacc + (uint32_t)H * kHeadDim * 4;
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

template <int BITS>
__global__ void __launch_bounds__(kVThreads, 1) v_accum_kernel(const __grid_constant__ CUtensorMap tmap, const VParams p) {
  using C = VCfg<BITS>;
  constexpr int N = C::N, W = C::W, CH = C::CH;
  extern __shared__ unsigned char smem_raw[];
  // 128B-swizzled TMA boxes need a 1024-byte aligned base
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int rows = p.H * W;
  const VSmem lay = v_smem_layout(rows, N, p.H, p.n_stages);
  float* s_lut = reinterpret_cast<float*>(smem + lay.off_lut);   // [n_stages][32][N]
  float* s_w = reinterpret_cast<float*>(smem + lay.off_w);       // [2][H][32]
  float* s_oacc = reinterpret_cast<float*>(smem + lay.off_oacc); // [H*128]
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(smem + lay.off_bar);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int S = p.n_stages;
  const int hidden = p.H * kHeadDim;

  // ---- thread -> unit mapping (up to 2 units per thread) ---------------------------------------------------
  // 4-bit: unit = word row (8 channels).  2-bit: unit = half a word row (8 channels).
  // 3-bit: warp-uniform SUB = warp % 3; unit = (32-channel group gi, SUB): row 3*gi+SUB (11/11/10 channels).
  int u_row[2], u_head[2], u_ch0[2], u_part[2];
  bool u_on[2];
  int sub = 0;
  if constexpr (BITS == 3) {
    sub = warp % 3;
    const int tri = warp / 3;            // 5 full warp-triples in 16 warps (warp 15 idles)
    const int ngroups = p.H * 4;
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
    const int nunits = p.H * 16;
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
    r_off[i] = (uint32_t)(r >> 5) * 4096u + (uint32_t)(r & 31) * 128u;
    r_swz[i] = (uint32_t)(r & 7);
    const int r2 = (r + 1 < rows) ? r + 1 : r;
    r_off2[i] = (uint32_t)(r2 >> 5) * 4096u + (uint32_t)(r2 & 31) * 128u;
    r_swz2[i] = (uint32_t)(r2 & 7);
  }
  float acc[2][CH];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int k = 0; k < CH; ++k) acc[i][k] = 0.f;

  for (int i = tid; i < hidden; i += kVThreads) s_oacc[i] = 0.f;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) mbar_init(&s_bar[s], 1);
    mbar_fence_init();
    prefetch_tensormap(&tmap);
  }

  const int64_t n_tiles_total = (p.L + kVT - 1) / kVT;
  const int64_t tile0 = (int64_t)blockIdx.x * p.tiles_per_cta;
  const int ntiles = (int)max((int64_t)0, min((int64_t)p.tiles_per_cta, n_tiles_total - tile0));
  const int nbox = rows >> 5;

  auto issue_tile = [&](int it) {  // thread 0 only
    const int s = it % S;
    const int64_t t0 = (tile0 + it) * kVT;
    const uint32_t lut_bytes = (uint32_t)min((int64_t)kVT, p.Lmax - t0) * N * 4;  // never read past the LUT allocation
    mbar_expect_tx(&s_bar[s], lay.stage_bytes + lut_bytes);
    unsigned char* dst = smem + (size_t)s * lay.stage_bytes;
    for (int b = 0; b < nbox; ++b) tma_load_2d(dst + b * 4096, &tmap, &s_bar[s], (int)t0, b * 32);
    bulk_load_1d(s_lut + s * kVT * N, p.lut_tok + t0 * N, lut_bytes, &s_bar[s]);
  };
  // weights of a tile: exp(s - max) in fused mode, the given probabilities otherwise; 0 beyond L
  const int n_w = p.H * kVT;  // values per tile
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
          w = p.score[(int64_t)h * p.score_stride + t0 + tl];
          if (p.fused) w = __expf(w - p.gmax[h]);
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
        if (e < total && opre_v[i] != 0.f) {
          const int idx = opre_i[i];
          const int tl = e / p.n_out;
          atomicAdd(&s_oacc[idx], opre_v[i] * wbuf[(idx >> 7) * kVT + tl]);
        }
      }
      for (int e = tid + kVMaxOPre * kVThreads; e < total; e += kVThreads) {  // n_out > 64: unprefetched tail
        const float v = p.outliers[t0 * p.n_out + e];
        const int idx = p.outlier_idx[t0 * p.n_out + e];
        if (v != 0.f) atomicAdd(&s_oacc[idx], v * wbuf[(idx >> 7) * kVT + e / p.n_out]);
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
    float* s_l = s_w;  // reuse: [H]
    for (int i = tid; i < p.H; i += kVThreads) s_l[i] = 0.f;
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
    for (int i = tid; i < p.H; i += kVThreads) p.out_l[(int64_t)blockIdx.x * p.H + i] = s_l[i];
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
          if (p.fused) obase[j] = v;
          else atomicAdd(&obase[j], v);
        }
      }
    }
  }
}

// ---- fused attend helpers ------------------------------------------------------------------------------------
// sink scores (fp16 post-RoPE keys, modeling_llama.py:1948-1949) and the initial per-head max
__global__ void attend_init_kernel(const float* __restrict__ q, const __half* __restrict__ sink_k, int n_sink,
                                   float* __restrict__ sink_scores, float* __restrict__ gmax, float scale) {
  // grid = H, block = 128 (thread = channel): s_i = scale * sum_c q[h,c] * sink_k[h,c,i], reduced per sink
  const int h = blockIdx.x, c = threadIdx.x;
  __shared__ float s_part[4];
  __shared__ float s_max;
  if (c == 0) s_max = -INFINITY;
  const float qc = q[h * kHeadDim + c];
  for (int i = 0; i < n_sink; ++i) {
    float v = qc * __half2float(sink_k[((int64_t)h * kHeadDim + c) * n_sink + i]);
    v = warp_sum(v);
    __syncthreads();
    if ((c & 31) == 0) s_part[c >> 5] = v;
    __syncthreads();
    if (c == 0) {
      const float s = (s_part[0] + s_part[1] + s_part[2] + s_part[3]) * scale;
      sink_scores[h * 64 + i] = s;
      s_max = fmaxf(s_max, s);
    }
  }
  __syncthreads();
  if (c == 0) gmax[h] = s_max;
}

// out[h,c] = (sum_s o[s,h,c] + sum_i p_i * sink_v[h,i,c]) / (sum_s l[s,h] + sum_i p_i),  p_i = exp(sink_s[h,i]-max)
// grid = H, block = 1024: 32 slices of the partials (one warp each, a lane owns 4 channels: 16-byte loads, all of a
// thread's <= 8 loads in flight at once), reduced through shared memory
__global__ void __launch_bounds__(1024) attend_combine_kernel(const float* __restrict__ po, const float* __restrict__ pl,
                                                              int n_part, int H, const float* __restrict__ gmax,
                                                              const float* __restrict__ sink_scores,
                                                              const __half* __restrict__ sink_v, int n_sink,
                                                              float* __restrict__ out, float* __restrict__ out_lse) {
  __shared__ float4 s_o[32][32];
  __shared__ float s_l[32];
  const int h = blockIdx.x, lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  float4 o4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float lsum = 0.f;
  constexpr int kU = 8;   // n_part <= 256 partials -> at most 8 per slice
  float4 v[kU];
  float lv[kU];
#pragma unroll
  for (int i = 0; i < kU; ++i) {
    const int s = g + 32 * i;
    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    lv[i] = 0.f;
    if (s < n_part) {
      v[i] = __ldcg(reinterpret_cast<const float4*>(po + ((int64_t)s * H + h) * kHeadDim) + lane);
      if (lane == 0) lv[i] = __ldcg(pl + (int64_t)s * H + h);
    }
  }
#pragma unroll
  for (int i = 0; i < kU; ++i) { o4.x += v[i].x; o4.y += v[i].y; o4.z += v[i].z; o4.w += v[i].w; lsum += lv[i]; }
  s_o[g][lane] = o4;
  if (lane == 0) s_l[g] = lsum;
  __syncthreads();
  if (threadIdx.x >= kHeadDim) return;
  const int c = threadIdx.x;
  float o = 0.f, l = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) { o += reinterpret_cast<const float*>(&s_o[i][0])[c]; l += s_l[i]; }
  const float m = gmax[h];
  for (int i = 0; i < n_sink; ++i) {
    const float pi = __expf(sink_scores[h * 64 + i] - m);
    o = fmaf(pi, __half2float(sink_v[((int64_t)h * n_sink + i) * kHeadDim + c]), o);
    l += pi;
  }
  out[h * kHeadDim + c] = o / l;
  if (out_lse != nullptr && c == 0) out_lse[h] = m + __logf(l);   // log-sum-exp of the scaled scores (for cross-GPU merges)
}

// merge N partial attention results (sequence-sharded decode): parts [N][H*128 + H] = (normalised out[H,128], lse[H])
__global__ void attend_merge_kernel(const float* __restrict__ parts, int n, int H, float* __restrict__ out) {
  const int h = blockIdx.x, c = threadIdx.x;   // block = 128
  const int stride = H * kHeadDim + H;
  float m = -INFINITY;
  for (int r = 0; r < n; ++r) m = fmaxf(m, parts[(int64_t)r * stride + H * kHeadDim + h]);
  float o = 0.f, l = 0.f;
  for (int r = 0; r < n; ++r) {
    const float* pr = parts + (int64_t)r * stride;
    const float w = __expf(pr[H * kHeadDim + h] - m);
    o = fmaf(w, pr[h * kHeadDim + c], o);
    l += w;
  }
  out[h * kHeadDim + c] = o / l;
}

// ---- host side -----------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_cache_tensor_map(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint32_t box_cols,
                          uint32_t box_rows, int swizzle_bytes) {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    // resolve the driver entry point directly (no link-time dependency on libcuda; the library must load on
    // GPU-less build hosts so that its exports can be checked there)
    void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return (int)cudaErrorInsufficientDriver;
    void* sym = dlsym(h, "cuTensorMapEncodeTiled");
    if (!sym) return (int)cudaErrorNotSupported;
    fn = reinterpret_cast<PFN_encodeTiled>(sym);
  }
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstride[1] = {cols * 4};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE),
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}

static int g_sms[64];   // per device (one process may drive several GPUs, see PerDeviceOnce)
int num_sms_cached();
static int num_sms() { return num_sms_cached(); }
int num_sms_cached() {
  int dev = 0;
  cudaGetDevice(&dev);
  int& n = g_sms[dev & 63];
  if (!n) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

constexpr uint32_t kSmemBudget = 227u * 1024u;

// returns number of CTAs launched (>0) or an error (<=0 mapped by caller)
template <int BITS>
static int launch_v(VParams p, const int32_t* cache, int* n_cta_out, cudaStream_t st) {
  using C = VCfg<BITS>;
  const int rows = p.H * C::W;
  int S = kVMaxStages;
  VSmem lay{};
  for (; S >= 2; --S) {
    lay = v_smem_layout(rows, C::N, p.H, S);
    if (lay.total + 1024u <= kSmemBudget) break;
  }
  if (S < 2) return KVQ_E_UNSUPPORTED;
  p.n_stages = S;
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(v_accum_kernel<BITS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBudget);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  CUtensorMap tmap;
  int rc = make_cache_tensor_map(&tmap, cache, (uint64_t)rows, (uint64_t)p.Lmax, kVT, 32, 128);
  if (rc != 0) return rc;
  const int64_t n_tiles = (p.L + kVT - 1) / kVT;
  const int sms = num_sms();
  p.tiles_per_cta = (int)((n_tiles + sms - 1) / sms);
  const int n_cta = (int)((n_tiles + p.tiles_per_cta - 1) / p.tiles_per_cta);
  v_accum_kernel<BITS><<<n_cta, kVThreads, lay.total + 1024u, st>>>(tmap, p);
  KVQ_LAUNCH_CHECK();
  *n_cta_out = n_cta;
  return 0;
}

int v_accum_dispatch(int bits, const VParams& p, const int32_t* cache, int* n_cta, cudaStream_t st) {
  switch (bits) {
    case 4: return launch_v<4>(p, cache, n_cta, st);
    case 3: return launch_v<3>(p, cache, n_cta, st);
    case 2: return launch_v<2>(p, cache, n_cta, st);
    default: return KVQ_E_BITS;
  }
}

struct KParams;  // kvq_kscore.cu
int k_scores_fused(int bits, const float* q, const int32_t* cache, float* scores, int64_t score_stride,
                   const float* lut, const float* outliers, const int32_t* outlier_idx, int n_out, int H,
                   int64_t Lmax, int64_t L, const float* rope, int64_t rope_npos, float theta, int pos_offset,
                   float* gmax, float scale, const int64_t* len_dev, int64_t len_add, float* opart, int opart_stride,
                   cudaStream_t st);

int v_native_dispatch(int bits, const float* score, int64_t score_stride, const float* gmax, const int32_t* cache,
                      const float* v_cent, const float* v_aff, const float* outliers, const int32_t* outlier_idx,
                      int n_out, int H, int64_t Lmax, int64_t L, float* out_o, float* out_l, int* n_cta,
                      const int64_t* len_dev, int64_t len_add, cudaStream_t st);

int k_scores_fused_fast(int bits, const float* q, const int32_t* cache, float* scores, int64_t score_stride,
                        const float* lut, const float* outliers, const int32_t* outlier_idx, int n_out, int H,
                        int64_t Lmax, int64_t L, const float* rope, const void* rope_half, int64_t rope_npos, float theta,
                        int pos_offset, float* gmax, float scale, const int64_t* len_dev, int64_t len_add, void* qtab,
                        cudaStream_t st);
// KVQ_K_IMPL set (generic / pair / kappa / lds64): round 1's 8-byte-entry kernels serve the exact mode of the fused attend
static int k_legacy_fused() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("KVQ_K_IMPL"); v = (e && e[0]) ? 1 : 0; }
  return v;
}

static int check_v_common(int H, int64_t Lmax, int64_t L, const void* cache) {
  if (H <= 0 || (H & 3) != 0 || H > 64 || L < 0 || L > Lmax) return KVQ_E_SHAPE;
  if ((Lmax & 3) != 0 || (reinterpret_cast<uintptr_t>(cache) & 15) != 0) return KVQ_E_ALIGN;
  return 0;
}

}  // namespace kvq

using namespace kvq;

extern "C" {

int kvq_v_matvec(int bits, const float* score, const int32_t* cache, float* mul, const float* lut_tok, int B, int H,
                 int64_t Lmax, int64_t L, const float* outliers, const int32_t* outlier_idx, int n_out, void* stream) {
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

static int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }
static const int kMaxPart = 256;

int64_t kvq_attend_scratch_bytes(int H, int64_t L) {
  // scores [H][L'] + gmax [H] + sink scores [H][64] + partial o / l of <= kMaxPart CTAs + token-major K-outlier
  // partials [L'][H'] (H' = H rounded up to 32) + the premultiplied K table [H][128][16] and ratios [H][128]
  return 4 * ((int64_t)H * round_up(L, 32) + H + (int64_t)H * 64 + (int64_t)kMaxPart * H * kHeadDim + (int64_t)kMaxPart * H +
              round_up(L, 32) * round_up(H, 32) + (int64_t)H * kHeadDim * 17) + 256;
}

}  // extern "C"

static int attend_impl(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
               const int32_t* k_outlier_idx, const int32_t* vcache, const float* vlut_tok, const float* v_cent,
               const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int H, int64_t Lmax, int64_t L, const float* rope_cos_sin,
               int64_t rope_npos, float theta, int pos_offset, const void* sink_k, const void* sink_v, int n_sink,
               float* out, float* out_lse, void* scratch, const int64_t* len_dev, int64_t len_add, const void* rope_half,
               void* stream) {
  if (!q || !kcache || !klut || !vcache || !rope_cos_sin || !out || !scratch) return KVQ_E_NULL;
  const bool native_v = (v_cent != nullptr && v_aff != nullptr);
  if (!native_v && !vlut_tok) return KVQ_E_NULL;
  int rc = check_v_common(H, Lmax, L, vcache);
  if (rc) return rc;
  if ((k_outliers == nullptr) != (k_outlier_idx == nullptr) || (v_outliers == nullptr) != (v_outlier_idx == nullptr)) return KVQ_E_NULL;
  if ((k_outliers || v_outliers) && n_out <= 0) return KVQ_E_SHAPE;
  if (n_sink < 0 || n_sink > 64 || (n_sink > 0 && (!sink_k || !sink_v))) return KVQ_E_SHAPE;
  if (L + n_sink == 0 || rope_npos < L + pos_offset || Lmax >= ((int64_t)1 << 30)) return KVQ_E_SHAPE;
  if (num_sms() > kMaxPart) return KVQ_E_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t stride = round_up(L, 32);
  float* scores = static_cast<float*>(scratch);
  float* gmax = scores + (int64_t)H * stride;
  float* sink_scores = gmax + H;
  float* part_o = sink_scores + (int64_t)H * 64;
  float* part_l = part_o + (int64_t)kMaxPart * H * kHeadDim;
  float* opart = part_l + (int64_t)kMaxPart * H;          // 16-byte aligned: every block above is a multiple of 4 floats
  const int opart_stride = (int)round_up(H, 32);
  float* qtab = opart + round_up(L, 32) * opart_stride;    // 16-byte aligned (rows of 32 floats)
  const bool fast = rope_half != nullptr;                  // fp16 tables (north_star's precision); NULL = exact fp32
  const float scale = 0.08838834764831845f;  // 1/sqrt(128)  (modeling_llama.py:1959,1973)
  attend_init_kernel<<<H, kHeadDim, 0, st>>>(q, static_cast<const __half*>(sink_k), n_sink, sink_scores, gmax, scale);
  KVQ_LAUNCH_CHECK();
  int n_cta = 0;
  if (L > 0) {
    // KVQ_K_IMPL (generic / pair / kappa) keeps round 1's LDS.64 kernels reachable for A/B runs; otherwise the
    // TMA-fed kernels: exact fp32 ratio form, or (rope_half given) the fp16-table form
    if (!fast && k_legacy_fused())
      rc = k_scores_fused(bits, q, kcache, scores, stride, klut, k_outliers, k_outlier_idx, n_out, H, Lmax, L,
                          rope_cos_sin, rope_npos, theta, pos_offset, gmax, scale, len_dev, len_add, opart, opart_stride, st);
    else
      rc = k_scores_fused_fast(bits, q, kcache, scores, stride, klut, k_outliers, k_outlier_idx, n_out, H, Lmax, L,
                               rope_cos_sin, rope_half, rope_npos, theta, pos_offset, gmax, scale, len_dev, len_add, qtab, st);
    if (rc) return rc;
    if (native_v) {
      rc = v_native_dispatch(bits, scores, stride, gmax, vcache, v_cent, v_aff, v_outliers, v_outlier_idx, n_out, H,
                             Lmax, L, part_o, part_l, &n_cta, len_dev, len_add, st);
    } else {   // materialised per-token LUT rows (kvq_attend without v_cent / v_aff)
      VParams p{};
      p.score = scores; p.lut_tok = vlut_tok; p.out = part_o; p.out_l = part_l; p.gmax = gmax;
      p.outliers = v_outliers; p.outlier_idx = v_outlier_idx;
      p.Lmax = Lmax; p.L = L; p.score_stride = stride; p.H = H; p.n_out = n_out; p.fused = 1;
      rc = v_accum_dispatch(bits, p, vcache, &n_cta, st);
    }
    if (rc) return rc;
  }
  attend_combine_kernel<<<H, 1024, 0, st>>>(part_o, part_l, n_cta, H, gmax, sink_scores,
                                                static_cast<const __half*>(sink_v), n_sink, out, out_lse);
  KVQ_LAUNCH_CHECK();
  return 0;
}

extern "C" {

int kvq_attend(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
               const int32_t* k_outlier_idx, const int32_t* vcache, const float* vlut_tok, const float* v_cent,
               const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int H, int64_t Lmax, int64_t L, const float* rope_cos_sin,
               int64_t rope_npos, float theta, int pos_offset, const void* sink_k, const void* sink_v, int n_sink,
               float* out, float* out_lse, void* scratch, const void* rope_half, void* stream) {
  return attend_impl(bits, q, kcache, klut, k_outliers, k_outlier_idx, vcache, vlut_tok, v_cent, v_aff, v_outliers,
                     v_outlier_idx, n_out, H, Lmax, L, rope_cos_sin, rope_npos, theta, pos_offset, sink_k, sink_v, n_sink,
                     out, out_lse, scratch, nullptr, 0, rope_half, stream);
}

int kvq_attend_dyn(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
                   const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent, const float* v_aff,
                   const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int H, int64_t Lmax, int64_t L_cap,
                   const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin, int64_t rope_npos, float theta,
                   int pos_offset, const void* sink_k, const void* sink_v, int n_sink, float* out, float* out_lse,
                   void* scratch, const void* rope_half, void* stream) {
  if (!len_dev || !v_cent || !v_aff) return KVQ_E_NULL;
  if (L_cap <= 0) return KVQ_E_SHAPE;
  return attend_impl(bits, q, kcache, klut, k_outliers, k_outlier_idx, vcache, nullptr, v_cent, v_aff, v_outliers,
                     v_outlier_idx, n_out, H, Lmax, L_cap, rope_cos_sin, rope_npos, theta, pos_offset, sink_k, sink_v,
                     n_sink, out, out_lse, scratch, len_dev, len_add, rope_half, stream);
}

int kvq_attend_merge(const float* parts, int n_parts, int H, float* out, void* stream) {
  if (!parts || !out) return KVQ_E_NULL;
  if (n_parts <= 0 || H <= 0) return KVQ_E_SHAPE;
  attend_merge_kernel<<<H, kHeadDim, 0, static_cast<cudaStream_t>(stream)>>>(parts, n_parts, H, out);
  KVQ_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
