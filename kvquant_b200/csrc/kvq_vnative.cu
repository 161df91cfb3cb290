// kvquant_b200 -- native score.V kernel of the fused attend path.
//
// The reference materialises a per-token LUT  LUT_t[i] = cent[i]*sf_t + off_t  (modeling_llama.py:1097-1114) and its
// V kernel looks values up in it (quant_cuda_kernel.cu:3238-3419).  Every value is therefore an affine image of ONE
// global 2^b-entry centroid table, so
//
//     O[h,c] = sum_t w[h,t] * (cent[code(h,c,t)]*sf_t + off_t)  =  sum_t (w*sf_t) * cent[code]  +  sum_t w*off_t
//
// The second term is one scalar per head.  The first needs only the global table, which lets TWO codes be looked up
// at once: a byte (4-bit), a 6-bit field (3-bit) or a nibble (2-bit) of the packed word indexes a lane-private
// table of float2 {cent[lo], cent[hi]} (lane-private = bank-conflict-free for any code pattern), and one packed
// lookup feeds both channels:   1 address op + 1 LDS.64 + 2 FFMA  per TWO elements.
// What bounds this kernel is the SM's load/store data path (one 8-byte lookup per 2 elements plus the outlier
// reductions), see DESIGN.md sections 4.2 and 7.
//
// Data movement: TMA (cp.async.bulk.tensor.2d, 128B swizzle, boxes of up to 256 rows) streams the
// [H*W rows x 32 tokens] code slab of a tile into a 2-3 stage ring behind mbarriers; thread = packed word row.
//
// Head split: where the whole slab does not fit shared memory next to the table (4-bit at H >= 36, 3-bit at H >= 60),
// the grid gains a second dimension of G = 2 head groups and CTA (r, g) streams only heads [g*H/2, (g+1)*H/2) of token
// range r.  The two CTAs of a range write disjoint heads of the same partial row, so the combine is unchanged.
//
// Grouped-query attention (GQA = true, p.grp query heads per KV head, p.H = query heads): the slab holds the H/grp KV
// heads' word rows, read from HBM once per token range; a thread unit is (query head, KV word row), so the g units of
// one KV row read the same staged words with their own head's weights.  Each V outlier entry (a KV channel) is applied
// with the weights of the grp query heads of its KV head.  A head-split CTA owns whole groups.
#include "kvq_attend.cuh"
#include <stdlib.h>

namespace kvq {

constexpr int kNThreads = 512;
constexpr int kNT = 32;          // tokens per stage (128-byte rows, 128B swizzle)
constexpr int kNMaxStages = 3;   // a 4th stage fits at 3 bits
constexpr int kNTokPerWarp = kNT / (kNThreads / 32);   // outlier rows handled by one warp per tile (2)
// row strides of the staged weights (floats).  Lanes of a warp sit in up to 8 different heads (3-bit) and read the SAME
// token columns: with 32-float rows every head's row starts in bank 0 -- an 8-way conflict on the LDS.128 of w*sf and a
// ~25-way one on the outlier weight gather.
constexpr int kNWStride = 33;    // w      : scalar gathers, head h token t -> bank (h + t) % 32
constexpr int kNWsStride = 36;   // w * sf : 16-byte reads, head h chunk q -> bank group (h + q) % 8
constexpr int kVNPad3 = 3 + 8;    // v_native_kernel's padded-box 3-bit form (below)

struct VNParams {
  const float* score;        // [H, score_stride] scaled scores
  const float* gmax;         // [H]
  const float* v_cent;       // [N] sorted centroids
  const float* v_aff;        // [Lmax][2] (sf, off) per token
  float* out_o;              // partial o [n_cta][H][128]
  float* out_l;              // partial denominators [n_cta][H]
  const float* outliers;     // [>=L, n_out] or null
  const int32_t* outlier_idx;
  int64_t Lmax, L, score_stride;
  const int64_t* len_dev;    // device-resident length (optional): L = min(*len_dev + len_add, L); L is then a cap
  int64_t len_add;
  int H, n_out, tiles_per_cta, n_stages, box_rows;   // H: query heads
  int grp;                   // query heads per KV head (GQA instantiation only)
};

template <int BITS> struct VNCfg {
  static constexpr int N = 1 << BITS;
  static constexpr int W = Layout<BITS>::kWords;
  static constexpr int IDXBITS = (BITS == 4) ? 8 : (BITS == 3 ? 6 : 4);  // two codes
  static constexpr int TABN = 1 << IDXBITS;                               // entries per lane
  static constexpr int NP = (BITS == 3) ? 6 : 4;                          // float2 accumulators per unit
};

struct VNSmem { uint32_t stage_bytes, off_tab, off_w, off_ws, off_oacc, off_bar, total; };
__host__ __device__ inline VNSmem vn_smem_layout(int rows, int tabn, int H, int n_stages) {
  VNSmem s;
  s.stage_bytes = (uint32_t)rows * (kNT * 4);
  s.off_tab = s.stage_bytes * n_stages;              // stages first (1024-aligned), then the table
  s.off_w = s.off_tab + (uint32_t)tabn * 256u;
  s.off_ws = (s.off_w + 2u * H * kNWStride * 4 + 15u) & ~15u;
  s.off_oacc = s.off_ws + 2u * H * kNWsStride * 4;
  s.off_bar = s.off_oacc;   // (the outlier accumulator lives in the partial-output row in global memory)
  s.total = s.off_bar + 8u * kNMaxStages;
  return s;
}

__device__ __forceinline__ float2 lds_f2_dyn(uint32_t addr) {
  float2 v;
  asm("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ void red_add_f32(float* addr, float v) {
  asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void ffma2v(float2& acc, const float2 a, const float2 b) {
  acc.x = __fmaf_rn(a.x, b.x, acc.x);
  acc.y = __fmaf_rn(a.y, b.y, acc.y);
}

// 32 tokens of one unit.  row_off/swz: this unit's word row in the 128B-swizzled stage; tab = shared address of the
// lane's table column (table base + lane*8); wsrow -> ws[head][0..31].
template <int BITS, int SUB>
__device__ __forceinline__ void vn_tile_unit(const unsigned char* stage, uint32_t row_off, uint32_t swz,
                                             uint32_t row_off2, uint32_t swz2, int part, uint32_t tab,
                                             const float* __restrict__ wsrow, float2* __restrict__ acc) {
#pragma unroll 2
  for (int q = 0; q < 8; ++q) {
    const uint4 wa = *reinterpret_cast<const uint4*>(stage + row_off + ((q ^ swz) << 4));
    uint4 wb = make_uint4(0, 0, 0, 0);
    if constexpr (BITS == 3 && SUB < 2) wb = *reinterpret_cast<const uint4*>(stage + row_off2 + ((q ^ swz2) << 4));
    const float4 ws4 = *reinterpret_cast<const float4*>(wsrow + 4 * q);
    const uint32_t wav[4] = {wa.x, wa.y, wa.z, wa.w};
    const uint32_t wbv[4] = {wb.x, wb.y, wb.z, wb.w};
    const float wsv[4] = {ws4.x, ws4.y, ws4.z, ws4.w};
#pragma unroll
    for (int tt = 0; tt < 4; ++tt) {
      const float2 ws2 = make_float2(wsv[tt], wsv[tt]);
      if constexpr (BITS == 4) {
        const uint32_t w = wav[tt];
#pragma unroll
        for (int b = 0; b < 4; ++b)  // byte b -> bits 8..15 of the table offset
          ffma2v(acc[b], ws2, lds_f2_dyn(__byte_perm(w, 0u, 0x4404 | (b << 4)) + tab));
      } else if constexpr (BITS == 2) {
        const uint32_t w = wav[tt] >> (16 * part);
#pragma unroll
        for (int b = 0; b < 4; ++b)  // nibble b of this thread's half word
          ffma2v(acc[b], ws2, lds_f2_dyn((b < 2 ? ((w << (8 - 4 * b)) & 0xF00u) : ((w >> (4 * b - 8)) & 0xF00u)) + tab));
      } else {
        const uint32_t w = wav[tt];
#pragma unroll
        for (int b = 0; b < 5; ++b) {  // 6-bit fields at bit SUB + 6b
          const int s = SUB + 6 * b;
          const uint32_t x = (s >= 8) ? (w >> (s - 8)) : (w << (8 - s));
          ffma2v(acc[b], ws2, lds_f2_dyn((x & 0x3F00u) + tab));
        }
        if constexpr (SUB < 2) {  // the straddling code (loc 10 / 21); high half of the index is 0 -> .y is unused
          const uint32_t c = ((w >> (30 + SUB)) | (wbv[tt] << (2 - SUB))) & 0x7u;
          ffma2v(acc[5], ws2, lds_f2_dyn((c << 8) + tab));
        }
      }
    }
  }
}

// SPLIT: gridDim.y head groups (see the head split above); SPLIT = false is the whole-slab launch with h0 = 0
// BATCH: sequence b = blockIdx.z of a batched attend (kvq_attend_batch): its scores, maximum and partials sit `bstride`
// floats after sequence b-1's, its (sf, off) and outlier rows are slice b of [B][Lmax][...], its length is
// p.len_dev[b], and its cache rows follow the b*Hkv*W rows of the sequences before it in the one tensor map.
// BATCH = false ignores `bstride`.
// PAGED (with BATCH; kvq_attend_paged): the tensor map covers the page pool (n_pool*Hkv*W rows x P columns) and the
// (sf, off) and outlier rows are pool rows.  A 32-token tile lies inside one page (P % 32 == 0), so each tile looks its
// page up for the TMA row base, and token t's (sf, off) and outlier rows sit at pool row page*P + t % P.
// The length is also capped at npages[b] * P.  Scores, maximum and partials are those of BATCH.  Others ignore `pg`.
// BITS = kVNPad3: the 3-bit kernel for a slab whose word rows are not a multiple of 8 -- one KV head, 12 rows.  One TMA
// box of p.box_rows (16) rows stages them with the next rows of the tensor, which no unit reads: the next sequence's or
// the next page's first rows of the same tokens, or TMA's zero fill past the tensor's last row.  Stages stay whole
// 1024-byte swizzle atoms.  (A pseudo bit width rather than a PAD template argument, which would rename every
// instantiation.)
template <int BITS, bool SPLIT, bool GQA, bool BATCH, bool PAGED = false>
__global__ void __launch_bounds__(kNThreads, 1) v_native_kernel(const __grid_constant__ CUtensorMap tmap, const VNParams p,
                                                                const int64_t bstride, const PageRef pg) {
  constexpr bool PAD = BITS == kVNPad3;
  constexpr int NB = PAD ? 3 : BITS;
  using C = VNCfg<NB>;
  constexpr int N = C::N, W = C::W, NP = C::NP, TABN = C::TABN;
  const int grp = GQA ? p.grp : 1;
  const int bz = BATCH ? (int)blockIdx.z : 0;
  const int64_t boff = BATCH ? bz * bstride : 0;                 // scores, gmax, partials
  const int64_t baff = BATCH ? bz * p.Lmax * 2 : 0;              // (sf, off) rows
  const int64_t bout = BATCH ? bz * p.Lmax * p.n_out : 0;        // outlier rows
  const int brow = BATCH ? bz * (p.H / grp) * W : 0;             // tensor-map rows
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int Hg = SPLIT ? p.H / (int)gridDim.y : p.H;     // heads of this CTA: [h0, h0 + Hg)
  const int h0 = SPLIT ? (int)blockIdx.y * Hg : 0;
  const int rows = Hg / grp * W;                          // word rows of the slab (KV heads)
  const VNSmem lay = vn_smem_layout(PAD ? p.box_rows : rows, TABN, Hg, p.n_stages);
  float2* s_tab = reinterpret_cast<float2*>(smem + lay.off_tab);   // [TABN][32 lanes]
  float* s_w = reinterpret_cast<float*>(smem + lay.off_w);         // [2][Hg][kNWStride]    w = exp(s - max)
  float* s_ws = reinterpret_cast<float*>(smem + lay.off_ws);       // [2][Hg][kNWsStride]   w * sf_t
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(smem + lay.off_bar);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int S = p.n_stages;
  const int hidden = p.H * kHeadDim;

  // ---- lane-private pair table: entry i -> {cent[i & (N-1)], cent[i >> BITS]} -------------------------------
  for (int i = tid; i < TABN * 32; i += kNThreads) {
    const int idx = i >> 5;
    s_tab[i] = make_float2(p.v_cent[idx & (N - 1)], p.v_cent[(idx >> NB) & (N - 1)]);
  }
  const uint32_t tab = smem_u32(s_tab) + lane * 8;

  // ---- thread -> unit mapping (same as kvq_vaccum.cu); u_head is relative to h0 -------------------------------------
  int u_row[2], u_head[2], u_ch0[2], u_part[2];
  bool u_on[2];
  int sub = 0;
  if constexpr (NB == 3) {
    sub = warp % 3;
    const int tri = warp / 3;
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
      const int u = tid + i * kNThreads;
      u_on[i] = u < nunits;
      if constexpr (NB == 4) { u_row[i] = u; u_part[i] = 0; u_head[i] = u >> 4; u_ch0[i] = (u & 15) * 8; }
      else { u_row[i] = u >> 1; u_part[i] = u & 1; u_head[i] = u >> 4; u_ch0[i] = ((u >> 1) & 7) * 16 + (u & 1) * 8; }
    }
  }
  // 128B swizzle: 16-byte chunk index ^= row & 7; TMA boxes are [32 tokens x box_rows rows] (box_rows % 8 == 0), laid
  // out back to back, so row r simply sits at r*128 inside the stage
  uint32_t r_off[2], r_swz[2], r_off2[2], r_swz2[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    // GQA: unit rows count query heads; the staged row is the same row of the head's KV head
    const int r = u_on[i] ? (GQA ? u_row[i] - (u_head[i] - u_head[i] / grp) * W : u_row[i]) : 0;
    r_off[i] = (uint32_t)r * 128u;
    r_swz[i] = (uint32_t)(r & 7);
    const int r2 = (r + 1 < rows) ? r + 1 : r;
    r_off2[i] = (uint32_t)r2 * 128u;
    r_swz2[i] = (uint32_t)(r2 & 7);
  }
  float2 acc[2][NP];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int k = 0; k < NP; ++k) acc[i][k] = make_float2(0.f, 0.f);

  // this CTA's row of the partial-output buffer doubles as the outlier accumulator: cleared here, reduced into by
  // the outlier rows, read back (after a fence) and completed in the epilogue.  Only this CTA's heads are touched.
  float* obase = p.out_o + boff + (int64_t)blockIdx.x * hidden;
  if (p.outliers != nullptr) {
    for (int i = h0 * kHeadDim + tid; i < (h0 + Hg) * kHeadDim; i += kNThreads) obase[i] = 0.f;
    __threadfence();   // the clears reach L2 before any reduction (ordered by the __syncthreads below)
  }
  if (tid == 0) {
    for (int s = 0; s < S; ++s) mbar_init(&s_bar[s], 1);
    mbar_fence_init();
    prefetch_tensormap(&tmap);
  }

  // device-resident length: the grid was sized for the cap p.L; CTAs past the current length write zero partials
  int64_t L_eff = p.L;
  if constexpr (PAGED) {   // (p.len_dev is set: the paged attend reads device lengths)
    const int64_t l = p.len_dev[bz] + p.len_add, cap = min(p.L, page_cap(pg, bz));
    L_eff = l < 0 ? 0 : (l < cap ? l : cap);
  } else {
    if (p.len_dev != nullptr) { const int64_t l = p.len_dev[bz] + p.len_add; L_eff = l < 0 ? 0 : (l < p.L ? l : p.L); }
  }
  const int64_t n_tiles_total = (L_eff + kNT - 1) / kNT;
  const int64_t tiles_per_cta = p.len_dev != nullptr ? (n_tiles_total + gridDim.x - 1) / gridDim.x : p.tiles_per_cta;
  const int64_t tile0 = (int64_t)blockIdx.x * tiles_per_cta;
  const int ntiles = (int)max((int64_t)0, min(tiles_per_cta, n_tiles_total - tile0));
  const int nbox = PAD ? 1 : rows / p.box_rows;

  auto issue_tile = [&](int it) {  // thread 0 only
    const int s = it % S;
    const int64_t t0 = (tile0 + it) * kNT;
    mbar_expect_tx(&s_bar[s], lay.stage_bytes);
    unsigned char* dst = smem + (size_t)s * lay.stage_bytes;
    if constexpr (PAGED) {
      const int row0 = page_of(pg, bz, (int)t0) * (p.H / grp) * W + h0 / grp * W;
      for (int b = 0; b < nbox; ++b) tma_load_2d(dst + (size_t)b * p.box_rows * 128, &tmap, &s_bar[s], (int)t0 % pg.P, row0 + b * p.box_rows);
    } else {
      for (int b = 0; b < nbox; ++b) tma_load_2d(dst + (size_t)b * p.box_rows * 128, &tmap, &s_bar[s], (int)t0, h0 / grp * W + b * p.box_rows + brow);
    }
  };
  // PAGED: pool row of token t (below the length, so its page is mapped; n_pool * P < 2^31)
  auto pool_row = [&](int64_t t) -> int { const int ti = (int)t; return page_of(pg, bz, ti) * pg.P + ti % pg.P; };
  // weights: Hg*32 (head, token) values per tile -> 2 per thread at Hg = 32 (up to 4 at Hg = 64)
  const int n_w = Hg * kNT;
  constexpr int NW = 4;
  float wpre[NW], wspre[NW], offpre[NW];
  float lacc[NW], oacc_off[NW];
#pragma unroll
  for (int i = 0; i < NW; ++i) { lacc[i] = 0.f; oacc_off[i] = 0.f; wpre[i] = wspre[i] = offpre[i] = 0.f; }
  // raw loads only (consumed in finish_weights after the tile's compute, so their latency is hidden)
  float w_s[NW], w_m[NW];
  float2 w_a[NW];
  auto load_weights = [&](int it) {
    const int64_t t0 = (tile0 + it) * kNT;
    const int r0 = PAGED ? pool_row(t0) : 0;   // (one page per tile)
#pragma unroll
    for (int i = 0; i < NW; ++i) {
      const int e = tid + i * kNThreads;
      w_s[i] = -INFINITY; w_m[i] = 0.f; w_a[i] = make_float2(0.f, 0.f);
      if (e < n_w) {
        const int h = e >> 5, tl = e & 31;
        if (t0 + tl < L_eff) {
          if constexpr (PAGED) {
            w_s[i] = p.score[boff + (int64_t)(h0 + h) * p.score_stride + t0 + tl];
            w_m[i] = p.gmax[boff + h0 + h];
            w_a[i] = *reinterpret_cast<const float2*>(p.v_aff + 2 * (int64_t)(r0 + tl));
          } else if constexpr (BATCH) {
            w_s[i] = p.score[boff + (int64_t)(h0 + h) * p.score_stride + t0 + tl];
            w_m[i] = p.gmax[boff + h0 + h];
            w_a[i] = *reinterpret_cast<const float2*>(p.v_aff + baff + 2 * (t0 + tl));
          } else {   // (kept apart: the single-sequence kernels compile exactly as before)
            w_s[i] = p.score[(int64_t)(h0 + h) * p.score_stride + t0 + tl];
            w_m[i] = p.gmax[h0 + h];
            w_a[i] = *reinterpret_cast<const float2*>(p.v_aff + 2 * (t0 + tl));
          }
        }
      }
    }
  };
  auto finish_weights = [&]() {
#pragma unroll
    for (int i = 0; i < NW; ++i) {
      const float w = (w_s[i] == -INFINITY) ? 0.f : __expf(w_s[i] - w_m[i]);
      wpre[i] = w;
      wspre[i] = w * w_a[i].x;
      lacc[i] += w;
      oacc_off[i] = fmaf(w, w_a[i].y, oacc_off[i]);
    }
  };
  auto store_weights = [&](int buf) {
#pragma unroll
    for (int i = 0; i < NW; ++i) {
      const int e = tid + i * kNThreads;
      if (e < n_w) {
        const int h = e >> 5, tl = e & 31;
        s_w[(buf * Hg + h) * kNWStride + tl] = wpre[i];
        s_ws[(buf * Hg + h) * kNWsStride + tl] = wspre[i];
      }
    }
  };
  // outliers: O[j] += w[h(j), t] * val(t, j).  Warp w owns tokens {w, w+16} of the tile; lanes walk the row (no
  // divisions), prefetched into registers.  The sums go straight to this CTA's row of the partial-output buffer with
  // fire-and-forget global reductions (RED.ADD.F32): shared memory has no native fp32 atomic add -- atomicAdd on
  // shared compiles to a compare-and-swap loop that ncu charged with 55 % of this kernel's shared-memory
  // wavefronts, more than the table lookups -- whereas a RED costs one L1 pass per lane and no return trip.
  constexpr int NO = 2 * kNTokPerWarp;   // (value, index) pairs per lane per tile for n_out <= 64
  float opre_v[NO];
  int opre_i[NO];
  const bool has_out = p.outliers != nullptr;
  // a V outlier row spans all heads: a head-split CTA applies the entries of its own heads only
  auto own_head = [&](int idx) { return !SPLIT || (unsigned)((idx >> 7) - h0 / grp) < (unsigned)(Hg / grp); };
  // O[j] += w * val for entry (val, idx) of slot tl; GQA: idx is a KV channel, applied to each query head of its group
  auto apply_outlier = [&](const float* wbuf, int tl, float v, int idx) {
    if constexpr (GQA) {
      const int hk = idx >> 7, c = idx & (kHeadDim - 1);
      for (int j = 0; j < grp; ++j) {
        const int hq = hk * grp + j;
        red_add_f32(obase + hq * kHeadDim + c, v * wbuf[(hq - h0) * kNWStride + tl]);
      }
    } else {
      red_add_f32(obase + idx, v * wbuf[((idx >> 7) - h0) * kNWStride + tl]);
    }
  };
  auto load_outliers = [&](int it) {
    const int64_t t0 = (tile0 + it) * kNT;
    const int r0 = PAGED ? pool_row(t0) : 0;   // (one page per tile)
#pragma unroll
    for (int j = 0; j < kNTokPerWarp; ++j) {
      const int64_t t = t0 + warp + j * (kNThreads / 32);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int k = lane + 32 * r;
        const bool in = (t < L_eff) && (k < p.n_out);
        if constexpr (PAGED) {
          const int64_t row = r0 + (int)(t - t0);
          opre_v[2 * j + r] = in ? p.outliers[row * p.n_out + k] : 0.f;
          opre_i[2 * j + r] = in ? p.outlier_idx[row * p.n_out + k] : 0;
        } else {
          opre_v[2 * j + r] = in ? p.outliers[bout + t * p.n_out + k] : 0.f;
          opre_i[2 * j + r] = in ? p.outlier_idx[bout + t * p.n_out + k] : 0;
        }
      }
    }
  };

  __syncthreads();
  if (ntiles > 0) {
    if (tid == 0)
      for (int it = 0; it < S - 1 && it < ntiles; ++it) issue_tile(it);
    load_weights(0);
    finish_weights();
    store_weights(0);
  }

  for (int it = 0; it < ntiles; ++it) {
    __syncthreads();
    if (tid == 0 && it + S - 1 < ntiles) issue_tile(it + S - 1);
    const bool more = it + 1 < ntiles;
    if (more) load_weights(it + 1);
    if (has_out) load_outliers(it);
    const int s = it % S;
    mbar_wait(&s_bar[s], (uint32_t)((it / S) & 1));
    const unsigned char* stage = smem + (size_t)s * lay.stage_bytes;
    const float* wsbuf = s_ws + (it & 1) * Hg * kNWsStride;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (u_on[i]) {
        const float* wsrow = wsbuf + u_head[i] * kNWsStride;
        if constexpr (NB == 3) {
          if (sub == 0) vn_tile_unit<3, 0>(stage, r_off[i], r_swz[i], r_off2[i], r_swz2[i], 0, tab, wsrow, acc[i]);
          else if (sub == 1) vn_tile_unit<3, 1>(stage, r_off[i], r_swz[i], r_off2[i], r_swz2[i], 0, tab, wsrow, acc[i]);
          else vn_tile_unit<3, 2>(stage, r_off[i], r_swz[i], r_off2[i], r_swz2[i], 0, tab, wsrow, acc[i]);
        } else {
          vn_tile_unit<NB, 0>(stage, r_off[i], r_swz[i], 0, 0, u_part[i], tab, wsrow, acc[i]);
        }
      }
    }
    if (has_out) {
      const float* wbuf = s_w + (it & 1) * Hg * kNWStride;
#pragma unroll
      for (int j = 0; j < kNTokPerWarp; ++j) {
        const int tl = warp + j * (kNThreads / 32);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float v = opre_v[2 * j + r];
          const int idx = opre_i[2 * j + r];
          if (v != 0.f && own_head(idx)) apply_outlier(wbuf, tl, v, idx);
        }
        for (int k = lane + 64; k < p.n_out; k += 32) {   // n_out > 64: unprefetched tail
          const int64_t t = (tile0 + it) * kNT + tl;
          if (t < L_eff) {
            const int64_t e = PAGED ? (int64_t)pool_row(t) * p.n_out + k : bout + t * p.n_out + k;
            const float v = p.outliers[e];
            const int idx = p.outlier_idx[e];
            if (v != 0.f && own_head(idx)) apply_outlier(wbuf, tl, v, idx);
          }
        }
      }
    }
    if (more) { finish_weights(); store_weights((it + 1) & 1); }
  }
  __threadfence();   // this thread's reductions are performed at L2 before anyone reads the row back
  __syncthreads();

  // ---- epilogue: per-head scalars (denominator, offset term), then the partial output -----------------------------
  float* s_l = s_w;            // [Hg]
  float* s_off = s_w + Hg;     // [Hg]
  for (int i = tid; i < 2 * Hg; i += kNThreads) s_w[i] = 0.f;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < NW; ++i) {
    const int e = tid + i * kNThreads;
    // a warp's 32 slots are the 32 tokens of one head
    const float a = warp_sum(lacc[i]), b = warp_sum(oacc_off[i]);
    if (e < n_w && lane == 0) { atomicAdd(&s_l[e >> 5], a); atomicAdd(&s_off[e >> 5], b); }
  }
  __syncthreads();
  for (int i = tid; i < Hg; i += kNThreads) p.out_l[boff + (int64_t)blockIdx.x * p.H + h0 + i] = s_l[i];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (u_on[i]) {
      const float hoff = s_off[u_head[i]];
      const int nch = (NB == 3) ? (sub == 2 ? 10 : 11) : 8;
#pragma unroll
      for (int k = 0; k < 2 * NP; ++k) {
        if (k < nch) {
          const int j = (h0 + u_head[i]) * kHeadDim + u_ch0[i] + k;
          const float v = (k & 1) ? acc[i][k >> 1].y : acc[i][k >> 1].x;
          obase[j] = v + hoff + (has_out ? __ldcg(obase + j) : 0.f);
        }
      }
    }
  }
}

constexpr uint32_t kVNSmemBudget = 227u * 1024u;

// ring stages that fit next to the table for a slab of Hg query heads, grp per KV head (largest first); 0 when not
// even two do
template <int BITS>
static int vn_stages(int Hg, int grp, VNSmem* lay) {
  using C = VNCfg<BITS>;
  for (int S = kNMaxStages; S >= 2; --S) {
    *lay = vn_smem_layout((Hg / grp * C::W + 7) / 8 * 8, C::TABN, Hg, S);   // staged rows: whole 8-row atoms
    if (lay->total + 1024u <= kVNSmemBudget) return S;
  }
  return 0;
}

template <int BITS, bool SPLIT, bool GQA, bool BATCH, bool PAGED>
static int launch_vn_kernel(const CUtensorMap& tmap, const VNParams& p, dim3 grid, uint32_t smem, cudaStream_t st,
                            int64_t bstride, const PageRef& pg) {
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(v_native_kernel<BITS, SPLIT, GQA, BATCH, PAGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kVNSmemBudget);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  v_native_kernel<BITS, SPLIT, GQA, BATCH, PAGED><<<grid, kNThreads, smem, st>>>(tmap, p, bstride, pg);
  KVQ_LAUNCH_CHECK();
  return 0;
}

// c.B == 0: one sequence; c.B >= 1: a batch (grid dimension z = sequence, each with its own scratch block of s.bstride
// floats); c.pg != nullptr: a paged batch
template <int BITS>
static int launch_vn(VNParams p, const AttendCall& c, const AttendScratch& s, int* n_cta_out) {
  using C = VNCfg<BITS>;
  const int B = c.B;
  const bool batch = B > 0, paged = c.pg != nullptr;
  // G head groups: 1 while the whole slab fits (every shape up to 4-bit H = 32, 3-bit H = 56, 2-bit H = 64), else 2.
  // G = 2 always fits for H <= 64: Hg = H/2 <= 32 heads is at most the 7B slab, and H % 4 == 0 keeps Hg even, so
  // the 3-bit group rows (Hg*12) stay a multiple of 8 for the TMA box below.
  // GQA: the slab holds H/grp KV heads, and each of the G = 2 groups whole KV-head groups (H/grp % 4 == 0).  One or two
  // KV heads are a slab of at most 32 rows, which always fits whole (G = 1).
  VNSmem lay{};
  int G = 1;
  int S = vn_stages<BITS>(p.H, p.grp, &lay);
  if (S < 2) { G = 2; S = vn_stages<BITS>(p.H / G, p.grp, &lay); }
  if (S < 2 || (G == 2 && (p.H / p.grp) % 4 != 0)) return KVQ_E_UNSUPPORTED;
  p.n_stages = S;
  const int rows = p.H / G / p.grp * C::W;   // word rows of one head group
  CUtensorMap tmap;
  // largest TMA box height <= 256 that divides the group's row count (a multiple of 8); one map over the whole
  // cache, the kernel offsets the row coordinate by its group's first row.  One 3-bit KV head (12 rows): one box of 16
  // rows, the kVNPad3 kernel.
  const bool pad = rows % 8 != 0;
  if (pad) {
    p.box_rows = (rows + 7) / 8 * 8;
  } else {
    int nb = (rows + 255) / 256;
    while (rows % nb != 0 || (rows / nb) % 8 != 0) ++nb;
    p.box_rows = rows / nb;
  }
  // a batch: one map over the B sequences' caches (sequence b's rows follow b*Hkv*W others); a paged batch: one map
  // over the pool (n_pool*Hkv*W rows of P tokens)
  int rc = paged
      ? make_cache_tensor_map(&tmap, c.vcache, (uint64_t)c.pg->n_pool * (p.H / p.grp) * C::W, (uint64_t)c.pg->P, kNT,
                              (uint32_t)p.box_rows, /*swizzle bytes*/ 128)
      : make_cache_tensor_map(&tmap, c.vcache, (uint64_t)(batch ? B : 1) * (p.H / p.grp) * C::W, (uint64_t)p.Lmax, kNT,
                              (uint32_t)p.box_rows, /*swizzle bytes*/ 128);
  if (rc != 0) return rc;
  // token ranges x head groups (x sequences) ~ one CTA per SM; the partial index is the token range
  const int64_t n_tiles = (p.L + kNT - 1) / kNT;
  const int ranges = max(1, num_sms_cached() / (G * (batch ? B : 1)));
  p.tiles_per_cta = (int)((n_tiles + ranges - 1) / ranges);
  const int n_cta = (int)((n_tiles + p.tiles_per_cta - 1) / p.tiles_per_cta);
  const dim3 grid = batch ? dim3(n_cta, G, B) : dim3(n_cta, G);
  const uint32_t smem = lay.total + 1024u;
  const PageRef pg = paged ? *c.pg : PageRef{};
  rc = with_flavour(p.grp > 1, batch, paged, [&](auto GQA, auto BATCH, auto PAGED) {
    if constexpr (BITS == 3 && GQA())   // (pad implies one 3-bit KV head under GQA, G = 1)
      if (pad) return launch_vn_kernel<kVNPad3, false, true, BATCH(), PAGED()>(tmap, p, grid, smem, c.stream, s.bstride, pg);
    return G == 1 ? launch_vn_kernel<BITS, false, GQA(), BATCH(), PAGED()>(tmap, p, grid, smem, c.stream, s.bstride, pg)
                  : launch_vn_kernel<BITS, true, GQA(), BATCH(), PAGED()>(tmap, p, grid, smem, c.stream, s.bstride, pg);
  });
  if (rc != 0) return rc;
  *n_cta_out = n_cta;
  return 0;
}

int v_native_dispatch(const AttendCall& c, const AttendScratch& s, int* n_cta) {
  VNParams p{};
  p.grp = c.grp();
  p.len_dev = c.len_dev; p.len_add = c.len_add;
  p.score = s.scores; p.gmax = s.gmax; p.v_cent = c.v_cent; p.v_aff = c.v_aff; p.out_o = s.part_o; p.out_l = s.part_l;
  p.outliers = c.v_outliers; p.outlier_idx = c.v_outlier_idx; p.Lmax = c.Lmax; p.L = c.L; p.score_stride = s.stride;
  p.H = c.Hq; p.n_out = c.n_out;
  switch (c.bits) {
    case 4: return launch_vn<4>(p, c, s, n_cta);
    case 3: return launch_vn<3>(p, c, s, n_cta);
    case 2: return launch_vn<2>(p, c, s, n_cta);
    default: return KVQ_E_BITS;
  }
}

}  // namespace kvq
