// kvquant_b200 -- the fused append's device code shared by kvq_append.cu and kvq_append_ragged.cu: the exact top-k
// selection, the per-token K and V work, the word packing, the outlier-row writer and the chunk append's body.  Each
// translation unit instantiates what it launches.
#pragma once
#include "kvq_common.cuh"

namespace kvq {

constexpr int kFusedThreads = 1024;
constexpr int kMaxHidden = 8192;
constexpr int kMaxOut = 128;  // 2*n_each upper bound

__device__ __forceinline__ uint32_t f2key(float f) {  // monotone float -> uint (larger float => larger key)
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

struct SelectSmem {
  uint32_t hist[2][256];
  uint32_t prefix[2];
  uint32_t krem[2];
  uint32_t kth[2];
  uint32_t need_eq[2];
  uint32_t n_sel;
};

// Exact top-k on both ends at once.  keys[] (monotone uint keys, n of them) live in shared memory.
// side 0 = k largest, side 1 = k smallest (run on inverted keys).  After return:
//   sel.kth[s]     = key of the k-th element on that side (in that side's key space)
//   sel.need_eq[s] = how many elements equal to kth must be taken (lowest index first)
// 4 passes of 8-bit digits; histogram updates are warp-aggregated with match_any.
static __device__ void radix_select_both(const uint32_t* keys, int n, int k, SelectSmem& sel) {
  const int tid = threadIdx.x;
  if (tid < 2) { sel.prefix[tid] = 0; sel.krem[tid] = k; }
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = tid; i < 512; i += blockDim.x) (&sel.hist[0][0])[i] = 0;
    __syncthreads();
    const uint32_t himask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + 8));
    const uint32_t p0 = sel.prefix[0], p1 = sel.prefix[1];
    for (int base = 0; base < n; base += blockDim.x) {
      const int i = base + tid;
      const bool valid = i < n;
      const uint32_t ka = valid ? keys[i] : 0u;
      const uint32_t kb = ~ka;
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const uint32_t key = s == 0 ? ka : kb;
        const bool in = valid && ((key & himask) == (s == 0 ? p0 : p1));
        const uint32_t act = __ballot_sync(0xffffffffu, in);
        if (in) {
          const uint32_t d = (key >> shift) & 0xFFu;
          const uint32_t peers = __match_any_sync(act, d);
          if ((int)(__ffs(peers) - 1) == (tid & 31)) atomicAdd(&sel.hist[s][d], __popc(peers));
        }
      }
    }
    __syncthreads();
    // warps 0 and 1 resolve side 0 and 1: find digit d with count(>d) < krem <= count(>=d)
    if (tid < 64) {
      const int s = tid >> 5, lane = tid & 31;
      uint32_t c[8];
      uint32_t tot = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) { c[q] = sel.hist[s][lane * 8 + q]; tot += c[q]; }
      // suffix sum over lanes: above = sum of totals of lanes > lane
      uint32_t incl = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_down_sync(0xffffffffu, incl, o);
        if (lane + o < 32) incl += v;
      }
      uint32_t above = incl - tot;  // elements in higher lanes' bins
      const uint32_t kr = sel.krem[s];
      __syncwarp();   // every lane has read krem before the one winning lane below rewrites it (racecheck: WAR hazard)
      // the k-th element lies in this lane's 8 bins iff above < kr <= above + tot
      if (above < kr && kr <= above + tot) {
#pragma unroll
        for (int q = 7; q >= 0; --q) {
          if (above < kr && kr <= above + c[q]) {
            sel.prefix[s] = sel.prefix[s] | ((uint32_t)(lane * 8 + q) << shift);
            sel.krem[s] = kr - above;
            above = 0xFFFFFFFFu;  // done
          } else if (above != 0xFFFFFFFFu) {
            above += c[q];
          }
        }
      }
    }
    __syncthreads();
  }
  if (tid < 2) { sel.kth[tid] = sel.prefix[tid]; sel.need_eq[tid] = sel.krem[tid]; }
  __syncthreads();
}

// Collect selected elements: side 0 -> slots [0, k), side 1 -> [k, 2k) of out_idx (unordered within a side).
// Elements with key beyond kth are taken; `need_eq` elements equal to kth are taken lowest-index-first.
static __device__ void collect_selected(const uint32_t* keys, int n, int k, SelectSmem& sel, int* out_idx, uint32_t* counters) {
  __shared__ uint32_t eq_cnt[2];
  __shared__ int eq_list[2][8];
  const int tid = threadIdx.x;
  if (tid < 2) { counters[tid] = 0; eq_cnt[tid] = 0; }
  __syncthreads();
  const uint32_t kth0 = sel.kth[0], kth1 = sel.kth[1];
  for (int i = tid; i < n; i += blockDim.x) {
    const uint32_t ka = keys[i], kb = ~ka;
    if (ka > kth0) out_idx[atomicAdd(&counters[0], 1u)] = i;
    if (kb > kth1) out_idx[k + atomicAdd(&counters[1], 1u)] = i;
    if (ka == kth0) { const uint32_t p = atomicAdd(&eq_cnt[0], 1u); if (p < 8) eq_list[0][p] = i; }
    if (kb == kth1) { const uint32_t p = atomicAdd(&eq_cnt[1], 1u); if (p < 8) eq_list[1][p] = i; }
  }
  __syncthreads();
  if (tid < 2) {
    const int s = tid;
    uint32_t need = sel.need_eq[s];
    uint32_t pos = counters[s];
    if (eq_cnt[s] == need && need <= 8) {
      // common case: every element equal to the k-th key is selected (their mutual order is irrelevant,
      // the row is sorted by channel index afterwards)
      for (uint32_t q = 0; q < need; ++q) out_idx[s * k + pos++] = eq_list[s][q];
    } else {
      // exact ties straddling the boundary: deterministic serial scan, lowest index first
      const uint32_t kth = sel.kth[s];
      for (int i = 0; i < n && need > 0; ++i) {
        const uint32_t key = s == 0 ? keys[i] : ~keys[i];
        if (key == kth) { out_idx[s * k + pos++] = i; --need; }
      }
    }
  }
  __syncthreads();
}

// ---- the per-token work of the fused append, shared by the single-token and the chunk kernel --------------------
// Each function is run by the whole CTA (blockDim.x a multiple of 32 and >= kMaxOut) on one token of one side, with
// that token's scratch in shared memory: s_x / s_key [hidden], s_code [hidden], s_sel_idx / s_sel_val [kMaxOut + 2].

// K: codes + normalised value, then the n_each largest / smallest normalised values and their outlier values
// (k - LUT end entry, zeroed when |r| <= 1).  Leaves s_code, and s_sel_idx / s_sel_val [0, 2*n_each) unordered.
template <int BITS>
__device__ __forceinline__ void k_token(int hidden, int n_each, const float* __restrict__ k_new,
                                        const float* __restrict__ klut, const float* __restrict__ klut_sub,
                                        const float* __restrict__ k_thr_lo, const float* __restrict__ k_thr_hi,
                                        float* s_x, uint32_t* s_key, uint8_t* s_code, SelectSmem& sel, int* s_sel_idx,
                                        float* s_sel_val, uint32_t* s_cnt) {
  constexpr int N = Layout<BITS>::kLevels;
  const int tid = threadIdx.x;
  const int n_out = 2 * n_each;
  for (int j = tid; j < hidden; j += blockDim.x) {
    const float x = k_new[j];
    float l[N];
#pragma unroll
    for (int i = 0; i < N; i += 4) {
      const float4 t = *reinterpret_cast<const float4*>(klut + (int64_t)j * N + i);
      l[i] = t.x; l[i + 1] = t.y; l[i + 2] = t.z; l[i + 3] = t.w;
    }
    s_code[j] = (uint8_t)nearest_code<BITS>(l, x);
    const float lo = k_thr_lo[j], hi = k_thr_hi[j];
    const float r = (x - (hi + lo) / 2) / ((hi - lo) / 2);
    s_x[j] = x;
    s_key[j] = f2key(r);
  }
  __syncthreads();
  if (n_each > 0) {
    radix_select_both(s_key, hidden, n_each, sel);
    collect_selected(s_key, hidden, n_each, sel, s_sel_idx, s_cnt);
  }
  // values: k - LUT end entry, zeroed when |r| <= 1 (modeling_llama.py:730-747)
  if (tid < n_out) {
    const int j = s_sel_idx[tid];
    const bool upper = tid < n_each;
    const float x = s_x[j];
    const float lo = k_thr_lo[j], hi = k_thr_hi[j];
    const float r = (x - (hi + lo) / 2) / ((hi - lo) / 2);
    float val = x - klut_sub[(int64_t)j * N + (upper ? N - 1 : 0)];
    if (upper ? (r <= 1.f) : (r >= -1.f)) val = 0.f;
    s_sel_val[tid] = val;
  }
  __syncthreads();
}

// V: thresholds = the (n_each+1)-th order statistics, the token's LUT row (written to row `row` of vlut [., N]) and
// (sf, off) (row `row` of aff [., 2] unless aff is NULL), codes, and the strict outlier row (pads for a short side).
template <int BITS>
__device__ __forceinline__ void v_token(int hidden, int n_each, const float* __restrict__ v_new,
                                        const float* __restrict__ v_cent, const float* __restrict__ v_cent_deq,
                                        float* vlut, float* aff, int64_t row, float* s_x, uint32_t* s_key, uint8_t* s_code,
                                        SelectSmem& sel, int* s_sel_idx, float* s_sel_val, uint32_t* s_cnt,
                                        float* s_vlut, float* s_thr, float& s_vzp) {
  constexpr int N = Layout<BITS>::kLevels;
  const int tid = threadIdx.x;
  const int n_out = 2 * n_each;
  for (int j = tid; j < hidden; j += blockDim.x) {
    const float x = v_new[j];
    s_x[j] = x;
    s_key[j] = f2key(x);
  }
  __syncthreads();
  radix_select_both(s_key, hidden, n_each + 1, sel);
  if (tid == 0) {
    // invert the key transform to recover the threshold values
    auto key2f = [](uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); };
    const float hi = key2f(sel.kth[0]);
    const float lo = key2f(~sel.kth[1]);
    s_thr[0] = lo; s_thr[1] = hi;
  }
  __syncthreads();
  const float lo = s_thr[0], hi = s_thr[1];
  if (tid < N) {
    const float off = (hi + lo) / 2;   // modeling_llama.py:1097-1098
    const float sf = (hi - lo) / 2;
    const float e = __fadd_rn(__fmul_rn(v_cent[tid], sf), off);  // two roundings, as torch mul then add
    s_vlut[tid] = e;
    vlut[row * N + tid] = e;
    if (tid == Layout<BITS>::kZeroPoint)   // modeling_llama.py:1126,1149-1152
      s_vzp = (v_cent_deq != nullptr) ? __fadd_rn(__fmul_rn(v_cent_deq[tid], sf), off) : e;
    if (tid == 0 && aff != nullptr) { aff[2 * row] = sf; aff[2 * row + 1] = off; }
  }
  // outliers are the elements strictly beyond the thresholds (the n_each larger / smaller ones)
  if (tid < 2) s_cnt[tid] = 0;
  __syncthreads();
  float lv[N];
#pragma unroll
  for (int i = 0; i < N; ++i) lv[i] = s_vlut[i];
  for (int j = tid; j < hidden; j += blockDim.x) {
    const float x = s_x[j];
    uint32_t code;
    if (x < lo || x > hi) {
      code = Layout<BITS>::kZeroPoint;
      const int side = x > hi ? 0 : 1;
      const uint32_t p = atomicAdd(&s_cnt[side], 1u);
      if (p < (uint32_t)n_each) s_sel_idx[side * n_each + p] = j;
    } else {
      code = nearest_code<BITS>(lv, x);
    }
    s_code[j] = (uint8_t)code;
  }
  __syncthreads();
  if (tid < n_out) {
    const bool upper = tid < n_each;
    const uint32_t have = s_cnt[upper ? 0 : 1];
    const int local = upper ? tid : tid - n_each;
    if ((uint32_t)local < have) {
      const int j = s_sel_idx[tid];
      s_sel_val[tid] = s_x[j] - s_vzp;  // modeling_llama.py:1169
    } else {  // exact ties at the threshold: fewer than n_each strict outliers -> pad (value 0, index 0)
      s_sel_idx[tid] = 0;
      s_sel_val[tid] = 0.f;
    }
  }
  __syncthreads();
}

// Packed word R (R < hidden*BITS/32) of the token's codes.
template <int BITS>
__device__ __forceinline__ uint32_t pack_word(const uint8_t* s_code, int R) {
  uint32_t w = 0;
  if constexpr (BITS == 4) {
#pragma unroll
    for (int q = 0; q < 8; ++q) w |= (uint32_t)s_code[R * 8 + q] << (4 * q);
  } else if constexpr (BITS == 2) {
#pragma unroll
    for (int q = 0; q < 16; ++q) w |= (uint32_t)s_code[R * 16 + q] << (2 * q);
  } else {
    const int g = R / 3, sub = R - g * 3;
    for (int l = 0; l < 32; ++l) {
      int row, shift, row2, rs2;
      pack_slot<3>(g * 32 + l, row, shift, row2, rs2);
      const uint32_t c = s_code[g * 32 + l];
      if (row == g * 3 + sub) w |= c << shift;
      if (row2 == g * 3 + sub) w |= c >> rs2;
    }
  }
  return w;
}

// The outlier row, sorted by channel index (rank by counting; indices are distinct except pads), to orow / irow.
__device__ __forceinline__ void write_outlier_row(int n_out, const int* s_sel_idx, const float* s_sel_val, float* orow,
                                                  int32_t* irow) {
  const int tid = threadIdx.x;
  if (tid < n_out) {
    const int my = s_sel_idx[tid];
    int rank = 0;
    for (int q = 0; q < n_out; ++q) {
      const int o = s_sel_idx[q];
      rank += (o < my) || (o == my && q < tid);
    }
    orow[rank] = s_sel_val[tid];
    irow[rank] = my;
  }
}
// ------------------------------------------------------------------------------------------------------------
// chunk append: T consecutive tokens at slots slot0 .. slot0+T-1 in one launch (a prompt).  grid = (tiles, 2):
// CTA (x, 0) runs the K side, (x, 1) the V side of tokens [x*kChunkTile, (x+1)*kChunkTile).  The CTA runs the
// per-token functions above on one token after the other, keeps the tile's packed words, outlier rows, LUT rows and
// (sf, off) in shared memory, and stores them at the end: each packed-word row as kChunkTile consecutive words (one
// 32-byte sector) instead of one scattered 4-byte store per token, the row tensors as one contiguous block each.
// Dynamic shared memory: chunk_smem_bytes (DESIGN.md section 4.4).
// ------------------------------------------------------------------------------------------------------------
constexpr int kChunkThreads = 256;
constexpr int kChunkTile = 8;
constexpr int kChunkPitch = kChunkTile + 1;   // words per packed-word row in shared memory (odd: no bank conflicts)

template <int BITS>
__host__ __device__ constexpr size_t chunk_smem_bytes(int hidden, int n_out) {
  return (size_t)hidden * (4 + 4)                                      // s_x, s_key
         + (size_t)hidden * BITS / 32 * kChunkPitch * 4                 // packed words of the tile
         + (size_t)kChunkTile * n_out * 8                               // outlier rows (values, indices)
         + (size_t)kChunkTile * (Layout<BITS>::kLevels + 2) * 4         // LUT rows, (sf, off)
         + (size_t)hidden;                                              // s_code
}

// The chunk kernel's body.  PAGED (append_kv_chunk_paged_kernel, DESIGN.md section 4.12): the cache pointers are page
// pools and pg.table is ONE sequence's page-table row; logical slot s goes to page pg.table[s / P], column s % P, a
// block laid out as a cache with Lmax = P.  Only the store phase differs, and it looks the page up per token: a tile
// straddles a page boundary whenever slot0 % 8 != 0.  The host has checked that every slot written is mapped.
template <int BITS, bool PAGED>
__device__ __forceinline__ void append_kv_chunk_body(
    int hidden, int64_t Lmax, int64_t slot0, int64_t T, int n_each,
    const float* __restrict__ k_new, uint32_t* __restrict__ kcache, const float* __restrict__ klut,
    const float* __restrict__ klut_sub, const float* __restrict__ k_thr_lo, const float* __restrict__ k_thr_hi,
    float* __restrict__ k_out, int32_t* __restrict__ k_idx,
    const float* __restrict__ v_new, uint32_t* __restrict__ vcache, const float* __restrict__ v_cent,
    const float* __restrict__ v_cent_deq, float* __restrict__ vlut_tok, float* __restrict__ v_aff, float* __restrict__ v_out,
    int32_t* __restrict__ v_idx, const PageRef& pg) {
  constexpr int N = Layout<BITS>::kLevels;
  const int nwords = hidden * BITS / 32;
  const int row_cap = 2 * n_each;   // outlier-row length the shared-memory layout was sized for
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* s_x = reinterpret_cast<float*>(smem_raw);                        // [hidden]
  uint32_t* s_key = reinterpret_cast<uint32_t*>(s_x + hidden);            // [hidden]
  uint32_t* s_words = s_key + hidden;                                     // [nwords][kChunkPitch]
  float* s_orow = reinterpret_cast<float*>(s_words + nwords * kChunkPitch);  // [kChunkTile][row_cap]
  int32_t* s_irow = reinterpret_cast<int32_t*>(s_orow + kChunkTile * row_cap);
  float* s_trow = reinterpret_cast<float*>(s_irow + kChunkTile * row_cap);  // [kChunkTile][N] LUT rows
  float* s_taff = s_trow + kChunkTile * N;                                // [kChunkTile][2]
  uint8_t* s_code = reinterpret_cast<uint8_t*>(s_taff + kChunkTile * 2);  // [hidden]
  __shared__ SelectSmem sel;
  __shared__ int s_sel_idx[kMaxOut + 2];
  __shared__ float s_sel_val[kMaxOut + 2];
  __shared__ uint32_t s_cnt[2];
  __shared__ float s_vlut[16];
  __shared__ float s_thr[2];
  __shared__ float s_vzp;
  const int tid = threadIdx.x;
  const bool isV = blockIdx.y == 1;
  if ((isV ? v_out : k_out) == nullptr) n_each = 0;   // dense-only side (as in append_kv_fused_kernel)
  const int n_out = 2 * n_each;
  const int64_t t0 = (int64_t)blockIdx.x * kChunkTile;
  const int ntok = (int)min((int64_t)kChunkTile, T - t0);

  for (int i = 0; i < ntok; ++i) {
    const int64_t t = t0 + i;
    if (!isV)
      k_token<BITS>(hidden, n_each, k_new + t * hidden, klut, klut_sub, k_thr_lo, k_thr_hi, s_x, s_key, s_code, sel,
                    s_sel_idx, s_sel_val, s_cnt);
    else
      v_token<BITS>(hidden, n_each, v_new + t * hidden, v_cent, v_cent_deq, s_trow, s_taff, i, s_x, s_key, s_code, sel,
                    s_sel_idx, s_sel_val, s_cnt, s_vlut, s_thr, s_vzp);
    for (int R = tid; R < nwords; R += blockDim.x) s_words[R * kChunkPitch + i] = pack_word<BITS>(s_code, R);
    if (n_out > 0) write_outlier_row(n_out, s_sel_idx, s_sel_val, s_orow + i * n_out, s_irow + i * n_out);
    __syncthreads();   // the next token overwrites s_code and the selection
  }

  // ---- stores: the tile's segment of every packed-word row, then the row tensors -------------------------------
  const int64_t slot = slot0 + t0;
  uint32_t* cache = isV ? vcache : kcache;
  if constexpr (PAGED) {   // the same stores, each token's through its own page
    for (int e = tid; e < nwords * kChunkTile; e += blockDim.x) {
      const int R = e / kChunkTile, i = e - R * kChunkTile;
      if (i < ntok) {
        const PageCol pc = page_col(pg, (int)(slot + i));
        cache[((int64_t)pc.page * nwords + R) * pg.P + pc.col] = s_words[R * kChunkPitch + i];
      }
    }
    if (n_out > 0) {
      float* orow = isV ? v_out : k_out;
      int32_t* irow = isV ? v_idx : k_idx;
      for (int e = tid; e < ntok * n_out; e += blockDim.x) {
        const int i = e / n_out;
        const int64_t r = page_row(pg, (int)(slot + i)) * n_out + (e - i * n_out);
        orow[r] = s_orow[e];
        irow[r] = s_irow[e];
      }
    }
    if (isV) {
      for (int e = tid; e < ntok * N; e += blockDim.x)
        vlut_tok[page_row(pg, (int)(slot + e / N)) * N + e % N] = s_trow[e];
      if (v_aff != nullptr)
        for (int e = tid; e < ntok * 2; e += blockDim.x) v_aff[2 * page_row(pg, (int)(slot + e / 2)) + e % 2] = s_taff[e];
    }
  } else {
    for (int e = tid; e < nwords * kChunkTile; e += blockDim.x) {
      const int R = e / kChunkTile, i = e - R * kChunkTile;
      if (i < ntok) cache[(int64_t)R * Lmax + slot + i] = s_words[R * kChunkPitch + i];
    }
    if (n_out > 0) {
      float* orow = (isV ? v_out : k_out) + slot * n_out;
      int32_t* irow = (isV ? v_idx : k_idx) + slot * n_out;
      for (int e = tid; e < ntok * n_out; e += blockDim.x) { orow[e] = s_orow[e]; irow[e] = s_irow[e]; }
    }
    if (isV) {
      for (int e = tid; e < ntok * N; e += blockDim.x) vlut_tok[slot * N + e] = s_trow[e];
      if (v_aff != nullptr)
        for (int e = tid; e < ntok * 2; e += blockDim.x) v_aff[2 * slot + e] = s_taff[e];
    }
  }
}
}  // namespace kvq
