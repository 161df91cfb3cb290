// kvquant_b200 -- append path: NUQ nearest-entry quantise + 4/3/2-bit pack (legacy single-token ops,
// prefill packers) and the fused device-side append (top-K outlier split + V thresholds + pack + row build) of one
// token or of a chunk of consecutive tokens.
//
// Reference semantics: deployment/kvquant/quant_cuda_kernel.cu:1167-2102 (appends), and the host-side glue
// in deployment/transformers/.../modeling_llama.py:664-751 (K), 1803-1820 + 1091-1176 (V).
#include "kvq_common.cuh"

namespace kvq {

// ------------------------------------------------------------------------------------------------------------
// legacy single-token appends.  One thread per channel; a warp covers 32 consecutive channels, i.e. 4 / 3 / 2
// packed words, assembled with REDUX (warp OR) and ADDED to the cache word by one lane (the reference adds with
// atomicAdd; each word has exactly one writer here).
// MODE 0: K dense, 1: K sparse (writes rescaled), 2: V dense (per-token LUT), 3: V sparse (zero-point for outliers)
// ------------------------------------------------------------------------------------------------------------
template <int BITS, int MODE>
__global__ void __launch_bounds__(128) append_one_kernel(
    uint32_t* __restrict__ cache, const float* __restrict__ lut, const float* __restrict__ newvec,
    float* __restrict__ rescaled, const float* __restrict__ thr_lo, const float* __restrict__ thr_hi,
    float v_lo, float v_hi, int hidden, int64_t Lmax, int64_t slot) {
  constexpr int N = Layout<BITS>::kLevels;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  uint32_t code = 0;
  if (j < hidden) {
    const float x = newvec[j];
    const float* row = (MODE >= 2) ? (lut + (int64_t)slot * N) : (lut + (int64_t)j * N);
    float l[N];
#pragma unroll
    for (int i = 0; i < N; i += 4) {
      const float4 t = *reinterpret_cast<const float4*>(row + i);
      l[i] = t.x; l[i + 1] = t.y; l[i + 2] = t.z; l[i + 3] = t.w;
    }
    code = nearest_code<BITS>(l, x);
    if (MODE == 1) {
      const float lo = thr_lo[j], hi = thr_hi[j];
      const float rg = (hi - lo) / 2;  // quant_cuda_kernel.cu:1759-1764
      const float zp = (hi + lo) / 2;
      rescaled[j] = (x - zp) / rg;
    }
    if (MODE == 3) {
      if (x < v_lo || x > v_hi) code = Layout<BITS>::kZeroPoint;  // quant_cuda_kernel.cu:2083-2084
    }
  }
  // assemble the warp's words (hidden is a multiple of 128, so whole warps are active together)
  const int jw = j & ~31;  // first channel of this warp
  if constexpr (BITS == 4) {
    const uint32_t v = code << ((lane & 7) * 4);
    const uint32_t m = 0xFFu << (lane & 24);
    const uint32_t w = __reduce_or_sync(m, v);
    if ((lane & 7) == 0 && j < hidden) {
      uint32_t* p = cache + (int64_t)(j >> 3) * Lmax + slot;
      *p = *p + w;
    }
  } else if constexpr (BITS == 2) {
    const uint32_t v = code << ((lane & 15) * 2);
    const uint32_t m = 0xFFFFu << (lane & 16);
    const uint32_t w = __reduce_or_sync(m, v);
    if ((lane & 15) == 0 && j < hidden) {
      uint32_t* p = cache + (int64_t)(j >> 4) * Lmax + slot;
      *p = *p + w;
    }
  } else {
    uint32_t c0 = 0, c1 = 0, c2 = 0;
    const int l = lane;
    if (l < 10) c0 = code << (3 * l);
    else if (l == 10) { c0 = code << 30; c1 = code >> 2; }
    else if (l < 21) c1 = code << ((3 * l) & 31);
    else if (l == 21) { c1 = code << 31; c2 = code >> 1; }
    else c2 = code << ((3 * l) & 31);
    c0 = __reduce_or_sync(0xffffffffu, c0);
    c1 = __reduce_or_sync(0xffffffffu, c1);
    c2 = __reduce_or_sync(0xffffffffu, c2);
    if (lane < 3 && jw < hidden) {
      const uint32_t w = lane == 0 ? c0 : (lane == 1 ? c1 : c2);
      uint32_t* p = cache + (int64_t)((jw >> 5) * 3 + lane) * Lmax + slot;
      *p = *p + w;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// prefill packers: newvec f32 [H,128,T] (token fastest).  thread = token (coalesced along T), loops the head's
// 128 channels; the per-channel LUT of the head is staged once per CTA in shared memory (broadcast reads).
// Words are ADDED to the cache (reference: non-atomic `mat[dst] += code<<shift`, quant_cuda_kernel.cu:1893).
// ISV = false: K (per-channel LUT + thresholds, writes rescaled); true: V (per-token LUT, per-token thresholds).
// ------------------------------------------------------------------------------------------------------------
template <int BITS, bool ISV>
__global__ void __launch_bounds__(128) append_parallel_kernel(
    uint32_t* __restrict__ cache, const float* __restrict__ lut, const float* __restrict__ newvec,
    float* __restrict__ rescaled, const float* __restrict__ thr_lo, const float* __restrict__ thr_hi,
    int64_t Lmax, int64_t T) {
  constexpr int N = Layout<BITS>::kLevels;
  constexpr int W = Layout<BITS>::kWords;
  __shared__ float s_lut[ISV ? 1 : kHeadDim * N];
  __shared__ float s_rg[ISV ? 1 : kHeadDim];
  __shared__ float s_zp[ISV ? 1 : kHeadDim];
  const int h = blockIdx.y;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if constexpr (!ISV) {
    for (int i = threadIdx.x; i < kHeadDim * N; i += blockDim.x) s_lut[i] = lut[(int64_t)h * kHeadDim * N + i];
    for (int i = threadIdx.x; i < kHeadDim; i += blockDim.x) {
      const float lo = thr_lo[h * kHeadDim + i], hi = thr_hi[h * kHeadDim + i];
      s_rg[i] = (hi - lo) / 2;
      s_zp[i] = (hi + lo) / 2;
    }
    __syncthreads();
  }
  if (t >= T) return;
  float lt[N];
  float vlo = 0.f, vhi = 0.f;
  if constexpr (ISV) {
#pragma unroll
    for (int i = 0; i < N; ++i) lt[i] = lut[t * N + i];
    vlo = thr_lo[t];
    vhi = thr_hi[t];
  }
  uint32_t w[W];
#pragma unroll
  for (int i = 0; i < W; ++i) w[i] = 0;
  const float* src = newvec + (int64_t)h * kHeadDim * T + t;
#pragma unroll 8
  for (int c = 0; c < kHeadDim; ++c) {
    const float x = src[(int64_t)c * T];
    uint32_t code;
    if constexpr (ISV) {
      code = nearest_code<BITS>(lt, x);
      if (x < vlo || x > vhi) code = Layout<BITS>::kZeroPoint;
    } else {
      code = nearest_code<BITS>(&s_lut[c * N], x);
      rescaled[(int64_t)h * kHeadDim * T + (int64_t)c * T + t] = (x - s_zp[c]) / s_rg[c];
    }
    int row, shift, row2, rs2;
    pack_slot<BITS>(c, row, shift, row2, rs2);
    // static indexing after unrolling keeps w[] in registers
#pragma unroll
    for (int i = 0; i < W; ++i) {
      if (i == row) w[i] |= code << shift;
      if (i == row2) w[i] |= code >> rs2;
    }
  }
#pragma unroll
  for (int i = 0; i < W; ++i) {
    uint32_t* p = cache + ((int64_t)h * W + i) * Lmax + t;
    *p = *p + w[i];
  }
}

// ------------------------------------------------------------------------------------------------------------
// fused device-side append.  grid = 2 CTAs (0: K, 1: V), 1024 threads each.
// ------------------------------------------------------------------------------------------------------------
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
__device__ void radix_select_both(const uint32_t* keys, int n, int k, SelectSmem& sel) {
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
__device__ void collect_selected(const uint32_t* keys, int n, int k, SelectSmem& sel, int* out_idx, uint32_t* counters) {
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

// BATCH: sequence b = blockIdx.y of a batch-strided cache (kvq_append_kv_fused_batch): every pointer but the shared
// tables is rebased on sequence b's slice, slot_dev points at the [B] lengths, and `active` (int32 [B] or null) skips
// inactive sequences.  BATCH = false is the single-sequence kernel (`active` unused).
// PAGED (with BATCH; kvq_append_kv_fused_paged): the cache pointers are page pools; slot s = len_dev[b] + slot_add of
// sequence b goes to column s % P of page page_of(b, s), a block laid out as a cache with Lmax = P, so the pointers are
// rebased on that page and the rest of the kernel runs with (Lmax, slot) = (P, s % P).  A slot at or past
// npages[b] * P is dropped, as a full cache drops it.  Other instantiations ignore `pg`.
template <int BITS, bool BATCH, bool PAGED = false>
__global__ void __launch_bounds__(kFusedThreads, 1) append_kv_fused_kernel(
    int hidden, int64_t Lmax, int64_t slot, const int64_t* __restrict__ slot_dev, int n_each,
    const float* __restrict__ k_new, uint32_t* __restrict__ kcache, const float* __restrict__ klut,
    const float* __restrict__ klut_sub, const float* __restrict__ k_thr_lo, const float* __restrict__ k_thr_hi,
    float* __restrict__ k_out, int32_t* __restrict__ k_idx,
    const float* __restrict__ v_new, uint32_t* __restrict__ vcache, const float* __restrict__ v_cent,
    const float* __restrict__ v_cent_deq, float* __restrict__ vlut_tok, float* __restrict__ v_aff, float* __restrict__ v_out, int32_t* __restrict__ v_idx,
    const int32_t* __restrict__ active, const PageRef pg) {
  constexpr int N = Layout<BITS>::kLevels;
  if constexpr (PAGED) {
    const int b = blockIdx.y;
    if (active != nullptr && active[b] == 0) return;
    slot += slot_dev[b];
    if (slot < 0 || slot >= page_cap(pg, b)) return;   // unmapped: dropped like a full cache's token
    const int64_t page = page_of(pg, b, slot);
    Lmax = pg.P;
    slot -= slot / Lmax * Lmax;
    const int64_t words = (int64_t)hidden * BITS / 32 * Lmax, rows = Lmax * 2 * n_each;
    k_new += (int64_t)b * hidden; v_new += (int64_t)b * hidden;
    kcache += page * words; vcache += page * words;
    if (k_out != nullptr) { k_out += page * rows; k_idx += page * rows; }
    if (v_out != nullptr) { v_out += page * rows; v_idx += page * rows; }
    vlut_tok += page * Lmax * (1 << BITS);
    if (v_aff != nullptr) v_aff += page * Lmax * 2;
    slot_dev = nullptr;
  } else if constexpr (BATCH) {
    const int b = blockIdx.y;
    if (active != nullptr && active[b] == 0) return;
    const int64_t words = (int64_t)hidden * BITS / 32 * Lmax, rows = Lmax * 2 * n_each;
    k_new += (int64_t)b * hidden; v_new += (int64_t)b * hidden;
    kcache += b * words; vcache += b * words;
    if (k_out != nullptr) { k_out += b * rows; k_idx += b * rows; }
    if (v_out != nullptr) { v_out += b * rows; v_idx += b * rows; }
    vlut_tok += b * Lmax * (1 << BITS);
    if (v_aff != nullptr) v_aff += b * Lmax * 2;
    slot_dev += b;
  }
  if constexpr (!PAGED) {
    if (slot_dev != nullptr) {   // device-resident length (CUDA-graph replays with a growing cache): slot = *slot_dev + slot
      slot += *slot_dev;
      if (slot < 0 || slot >= Lmax) return;   // a full cache drops the token instead of writing out of bounds
    }
  }
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* s_x = reinterpret_cast<float*>(smem_raw);                 // [hidden] raw values
  uint32_t* s_key = reinterpret_cast<uint32_t*>(s_x + hidden);     // [hidden] select keys
  uint8_t* s_code = reinterpret_cast<uint8_t*>(s_key + hidden);    // [hidden]
  __shared__ SelectSmem sel;
  __shared__ int s_sel_idx[kMaxOut + 2];
  __shared__ float s_sel_val[kMaxOut + 2];
  __shared__ uint32_t s_cnt[2];
  __shared__ float s_vlut[16];
  __shared__ float s_thr[2];
  __shared__ float s_vzp;   // value the zero-point code dequantises to (Q-Norm: from the shifted centroids)
  const int tid = threadIdx.x;
  const bool isV = blockIdx.x == 1;
  // a cache without an outlier row pointer is dense-only (the reference's include_sparse=False branch,
  // modeling_llama.py:753-779, 1178-1201): K keeps every value as its nearest code, V's range is the min / max of
  // the vector (compute_lut, modeling_llama.py:318-349) -- which is the order-statistics rule below with n_each = 0
  if ((isV ? v_out : k_out) == nullptr) n_each = 0;
  const int n_out = 2 * n_each;

  if (!isV)
    k_token<BITS>(hidden, n_each, k_new, klut, klut_sub, k_thr_lo, k_thr_hi, s_x, s_key, s_code, sel, s_sel_idx,
                  s_sel_val, s_cnt);
  else
    v_token<BITS>(hidden, n_each, v_new, v_cent, v_cent_deq, vlut_tok, v_aff, slot, s_x, s_key, s_code, sel,
                  s_sel_idx, s_sel_val, s_cnt, s_vlut, s_thr, s_vzp);

  // ---- pack codes (thread per word, assembled from s_code) and write (overwrite) ---------------------------
  uint32_t* cache = isV ? vcache : kcache;
  const int nwords = hidden * BITS / 32;
  for (int R = tid; R < nwords; R += blockDim.x) cache[(int64_t)R * Lmax + slot] = pack_word<BITS>(s_code, R);
  if (n_out == 0) return;
  write_outlier_row(n_out, s_sel_idx, s_sel_val, (isV ? v_out : k_out) + slot * n_out,
                    (isV ? v_idx : k_idx) + slot * n_out);
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

// contiguous cache of Lmax slots
template <int BITS>
__global__ void __launch_bounds__(kChunkThreads, 4) append_kv_chunk_kernel(
    int hidden, int64_t Lmax, int64_t slot0, int64_t T, int n_each,
    const float* __restrict__ k_new, uint32_t* __restrict__ kcache, const float* __restrict__ klut,
    const float* __restrict__ klut_sub, const float* __restrict__ k_thr_lo, const float* __restrict__ k_thr_hi,
    float* __restrict__ k_out, int32_t* __restrict__ k_idx,
    const float* __restrict__ v_new, uint32_t* __restrict__ vcache, const float* __restrict__ v_cent,
    const float* __restrict__ v_cent_deq, float* __restrict__ vlut_tok, float* __restrict__ v_aff, float* __restrict__ v_out, int32_t* __restrict__ v_idx) {
  append_kv_chunk_body<BITS, false>(hidden, Lmax, slot0, T, n_each, k_new, kcache, klut, klut_sub, k_thr_lo, k_thr_hi,
                                    k_out, k_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok, v_aff, v_out, v_idx,
                                    PageRef{});
}

// one paged sequence, pg.table its page-table row (a kernel of its own name: a PAGED template argument would rename
// the contiguous instantiations above)
template <int BITS>
__global__ void __launch_bounds__(kChunkThreads, 4) append_kv_chunk_paged_kernel(
    int hidden, int64_t slot0, int64_t T, int n_each,
    const float* __restrict__ k_new, uint32_t* __restrict__ kcache, const float* __restrict__ klut,
    const float* __restrict__ klut_sub, const float* __restrict__ k_thr_lo, const float* __restrict__ k_thr_hi,
    float* __restrict__ k_out, int32_t* __restrict__ k_idx,
    const float* __restrict__ v_new, uint32_t* __restrict__ vcache, const float* __restrict__ v_cent,
    const float* __restrict__ v_cent_deq, float* __restrict__ vlut_tok, float* __restrict__ v_aff, float* __restrict__ v_out, int32_t* __restrict__ v_idx,
    const PageRef pg) {
  append_kv_chunk_body<BITS, true>(hidden, pg.P, slot0, T, n_each, k_new, kcache, klut, klut_sub, k_thr_lo, k_thr_hi,
                                   k_out, k_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok, v_aff, v_out, v_idx, pg);
}

template <int BITS>
static int launch_append_one(int mode, uint32_t* cache, const float* lut, const float* newvec, float* rescaled,
                             const float* tlo, const float* thi, float vlo, float vhi, int H, int64_t Lmax,
                             int64_t slot, cudaStream_t st) {
  const int hidden = H * kHeadDim;
  const dim3 grid((hidden + 127) / 128), block(128);
  switch (mode) {
    case 0: append_one_kernel<BITS, 0><<<grid, block, 0, st>>>(cache, lut, newvec, rescaled, tlo, thi, vlo, vhi, hidden, Lmax, slot); break;
    case 1: append_one_kernel<BITS, 1><<<grid, block, 0, st>>>(cache, lut, newvec, rescaled, tlo, thi, vlo, vhi, hidden, Lmax, slot); break;
    case 2: append_one_kernel<BITS, 2><<<grid, block, 0, st>>>(cache, lut, newvec, rescaled, tlo, thi, vlo, vhi, hidden, Lmax, slot); break;
    default: append_one_kernel<BITS, 3><<<grid, block, 0, st>>>(cache, lut, newvec, rescaled, tlo, thi, vlo, vhi, hidden, Lmax, slot); break;
  }
  KVQ_LAUNCH_CHECK();
  return 0;
}

static int append_one(int bits, int mode, int32_t* cache, const float* lut, const float* newvec, float* rescaled,
                      const float* tlo, const float* thi, float vlo, float vhi, int H, int64_t Lmax, int64_t slot,
                      void* stream) {
  if (!cache || !lut || !newvec) return KVQ_E_NULL;
  if (mode == 1 && (!rescaled || !tlo || !thi)) return KVQ_E_NULL;
  if (H <= 0 || Lmax <= 0 || slot < 0 || slot >= Lmax) return KVQ_E_SHAPE;
  if ((reinterpret_cast<uintptr_t>(lut) & 15) != 0) return KVQ_E_ALIGN;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint32_t* c = reinterpret_cast<uint32_t*>(cache);
  switch (bits) {
    case 4: return launch_append_one<4>(mode, c, lut, newvec, rescaled, tlo, thi, vlo, vhi, H, Lmax, slot, st);
    case 3: return launch_append_one<3>(mode, c, lut, newvec, rescaled, tlo, thi, vlo, vhi, H, Lmax, slot, st);
    case 2: return launch_append_one<2>(mode, c, lut, newvec, rescaled, tlo, thi, vlo, vhi, H, Lmax, slot, st);
    default: return KVQ_E_BITS;
  }
}

template <int BITS>
static int launch_parallel(bool isv, uint32_t* cache, const float* lut, const float* newvec, float* rescaled,
                           const float* tlo, const float* thi, int H, int64_t Lmax, int64_t T, cudaStream_t st) {
  const dim3 grid((unsigned)((T + 127) / 128), H), block(128);
  if (isv) append_parallel_kernel<BITS, true><<<grid, block, 0, st>>>(cache, lut, newvec, rescaled, tlo, thi, Lmax, T);
  else append_parallel_kernel<BITS, false><<<grid, block, 0, st>>>(cache, lut, newvec, rescaled, tlo, thi, Lmax, T);
  KVQ_LAUNCH_CHECK();
  return 0;
}

static int append_parallel(int bits, bool isv, int32_t* cache, const float* lut, const float* newvec,
                           float* rescaled, const float* tlo, const float* thi, int H, int64_t Lmax, int64_t T,
                           void* stream) {
  if (!cache || !lut || !newvec || !tlo || !thi) return KVQ_E_NULL;
  if (!isv && !rescaled) return KVQ_E_NULL;
  if (H <= 0 || Lmax <= 0 || T < 0 || T > Lmax) return KVQ_E_SHAPE;
  if (T == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint32_t* c = reinterpret_cast<uint32_t*>(cache);
  switch (bits) {
    case 4: return launch_parallel<4>(isv, c, lut, newvec, rescaled, tlo, thi, H, Lmax, T, st);
    case 3: return launch_parallel<3>(isv, c, lut, newvec, rescaled, tlo, thi, H, Lmax, T, st);
    case 2: return launch_parallel<2>(isv, c, lut, newvec, rescaled, tlo, thi, H, Lmax, T, st);
    default: return KVQ_E_BITS;
  }
}

// B == 0: the single-sequence kernel; B >= 1: the batched one, grid (2, B); pg != nullptr: the paged one, grid (2, B)
template <int BITS>
static int launch_fused(int hidden, int64_t Lmax, int64_t slot, const int64_t* slot_dev, int n_each, const float* k_new, uint32_t* kcache,
                        const float* klut, const float* klut_sub, const float* ktl, const float* kth, float* kout,
                        int32_t* kidx, const float* v_new, uint32_t* vcache, const float* vcent, const float* vcent_deq,
                        float* vlut, float* vaff, float* vout, int32_t* vidx, cudaStream_t st, int B = 0,
                        const int32_t* active = nullptr, const PageRef* pg = nullptr) {
  const size_t smem = (size_t)hidden * (4 + 4 + 1);
  static PerDeviceOnce attr_once[3];   // (one instance per BITS instantiation and form)
  const int form = pg != nullptr ? 2 : (B > 0 ? 1 : 0);
  bool& attr_done = attr_once[form].cur();
  if (!attr_done) {
    const int a = cudaFuncAttributeMaxDynamicSharedMemorySize;
    cudaError_t e = form == 2 ? cudaFuncSetAttribute(append_kv_fused_kernel<BITS, true, true>, (cudaFuncAttribute)a, 96 * 1024)
                  : form == 1 ? cudaFuncSetAttribute(append_kv_fused_kernel<BITS, true>, (cudaFuncAttribute)a, 96 * 1024)
                              : cudaFuncSetAttribute(append_kv_fused_kernel<BITS, false>, (cudaFuncAttribute)a, 96 * 1024);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  if (pg != nullptr)
    append_kv_fused_kernel<BITS, true, true><<<dim3(2, B), kFusedThreads, smem, st>>>(
        hidden, Lmax, slot, slot_dev, n_each, k_new, kcache, klut, klut_sub, ktl, kth, kout, kidx, v_new, vcache, vcent,
        vcent_deq, vlut, vaff, vout, vidx, active, *pg);
  else if (B > 0)
    append_kv_fused_kernel<BITS, true><<<dim3(2, B), kFusedThreads, smem, st>>>(
        hidden, Lmax, slot, slot_dev, n_each, k_new, kcache, klut, klut_sub, ktl, kth, kout, kidx, v_new, vcache, vcent,
        vcent_deq, vlut, vaff, vout, vidx, active, PageRef{});
  else
    append_kv_fused_kernel<BITS, false><<<2, kFusedThreads, smem, st>>>(hidden, Lmax, slot, slot_dev, n_each, k_new, kcache, klut,
                                                                       klut_sub, ktl, kth, kout, kidx, v_new, vcache, vcent,
                                                                       vcent_deq, vlut, vaff, vout, vidx, nullptr, PageRef{});
  KVQ_LAUNCH_CHECK();
  return 0;
}

template <int BITS>
static int launch_fused_chunk(int hidden, int64_t Lmax, int64_t slot, int64_t T, int n_each, const float* k_new,
                              uint32_t* kcache, const float* klut, const float* klut_sub, const float* ktl,
                              const float* kth, float* kout, int32_t* kidx, const float* v_new, uint32_t* vcache,
                              const float* vcent, const float* vcent_deq, float* vlut, float* vaff, float* vout,
                              int32_t* vidx, cudaStream_t st, const PageRef* pg) {
  const size_t smem = chunk_smem_bytes<BITS>(hidden, 2 * n_each);
  static PerDeviceOnce attr_once[2];   // (one instance per BITS instantiation and form)
  bool& attr_done = attr_once[pg != nullptr].cur();
  if (!attr_done) {
    const int most = (int)chunk_smem_bytes<BITS>(kMaxHidden, kMaxOut);
    const cudaFuncAttribute a = cudaFuncAttributeMaxDynamicSharedMemorySize;
    cudaError_t e = pg != nullptr ? cudaFuncSetAttribute(append_kv_chunk_paged_kernel<BITS>, a, most)
                                  : cudaFuncSetAttribute(append_kv_chunk_kernel<BITS>, a, most);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  const dim3 grid((unsigned)((T + kChunkTile - 1) / kChunkTile), 2);
  if (pg != nullptr)
    append_kv_chunk_paged_kernel<BITS><<<grid, kChunkThreads, smem, st>>>(
        hidden, slot, T, n_each, k_new, kcache, klut, klut_sub, ktl, kth, kout, kidx, v_new, vcache, vcent, vcent_deq,
        vlut, vaff, vout, vidx, *pg);
  else
    append_kv_chunk_kernel<BITS><<<grid, kChunkThreads, smem, st>>>(hidden, Lmax, slot, T, n_each, k_new, kcache, klut,
                                                                    klut_sub, ktl, kth, kout, kidx, v_new, vcache, vcent,
                                                                    vcent_deq, vlut, vaff, vout, vidx);
  KVQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace kvq

using namespace kvq;

extern "C" {

int kvq_append_k(int bits, int32_t* cache, const float* lut, const float* newvec, int H, int64_t Lmax,
                 int64_t slot, void* stream) {
  return append_one(bits, 0, cache, lut, newvec, nullptr, nullptr, nullptr, 0.f, 0.f, H, Lmax, slot, stream);
}
int kvq_append_v(int bits, int32_t* cache, const float* lut_tok, const float* newvec, int H, int64_t Lmax,
                 int64_t slot, void* stream) {
  return append_one(bits, 2, cache, lut_tok, newvec, nullptr, nullptr, nullptr, 0.f, 0.f, H, Lmax, slot, stream);
}
int kvq_append_k_sparse(int bits, int32_t* cache, const float* lut, const float* newvec, float* outliers_rescaled,
                        const float* thr_lower, const float* thr_upper, int H, int64_t Lmax, int64_t slot,
                        void* stream) {
  return append_one(bits, 1, cache, lut, newvec, outliers_rescaled, thr_lower, thr_upper, 0.f, 0.f, H, Lmax, slot, stream);
}
int kvq_append_v_sparse(int bits, int32_t* cache, const float* lut_tok, const float* newvec, float zeropoint,
                        float thr_lower, float thr_upper, int H, int64_t Lmax, int64_t slot, void* stream) {
  (void)zeropoint;  // accepted and unused, as in the reference kernel (quant_cuda_kernel.cu:2049-2057)
  return append_one(bits, 3, cache, lut_tok, newvec, nullptr, nullptr, nullptr, thr_lower, thr_upper, H, Lmax, slot, stream);
}
int kvq_append_k_sparse_parallel(int bits, int32_t* cache, const float* lut, const float* newvec,
                                 float* outliers_rescaled, const float* thr_lower, const float* thr_upper, int H,
                                 int64_t Lmax, int64_t T, void* stream) {
  return append_parallel(bits, false, cache, lut, newvec, outliers_rescaled, thr_lower, thr_upper, H, Lmax, T, stream);
}
int kvq_append_v_sparse_parallel(int bits, int32_t* cache, const float* lut_tok, const float* newvec,
                                 const float* thr_lower, const float* thr_upper, int H, int64_t Lmax, int64_t T,
                                 void* stream) {
  return append_parallel(bits, true, cache, lut_tok, newvec, nullptr, thr_lower, thr_upper, H, Lmax, T, stream);
}

static int append_kv_fused_impl(int bits, int H, int64_t Lmax, int64_t slot, const int64_t* slot_dev, int n_each,
                                const float* k_new, int32_t* kcache, const float* klut, const float* klut_sub,
                                const float* k_thr_lower, const float* k_thr_upper, float* k_outliers,
                                int32_t* k_outlier_idx, const float* v_new, int32_t* vcache, const float* v_cent,
                                const float* v_cent_deq, float* vlut_tok, float* v_aff, float* v_outliers,
                                int32_t* v_outlier_idx, void* stream, int B = 0, const int32_t* active = nullptr,
                                const PageRef* pg = nullptr) {
  if (!k_new || !kcache || !klut || !klut_sub || !k_thr_lower || !k_thr_upper || !v_new || !vcache || !v_cent || !vlut_tok)
    return KVQ_E_NULL;
  // outlier rows are optional per cache: NULL = that cache is dense-only (value and index pointers go together)
  if ((k_outliers == nullptr) != (k_outlier_idx == nullptr) || (v_outliers == nullptr) != (v_outlier_idx == nullptr))
    return KVQ_E_NULL;
  const int hidden = H * kHeadDim;
  if (H <= 0 || hidden > kMaxHidden || Lmax <= 0) return KVQ_E_SHAPE;
  // the batch strides keep every slice 16-byte aligned (Lmax % 4 == 0); H as the attends accept it: H % 4 == 0 or H <= 2
  if (B > 0 && ((H % 4 != 0 && H > 2) || Lmax % 4 != 0)) return KVQ_E_SHAPE;
  if (slot_dev == nullptr && (slot < 0 || slot >= Lmax)) return KVQ_E_SHAPE;
  const bool any_sparse = k_outliers != nullptr || v_outliers != nullptr;
  if (any_sparse && (n_each <= 0 || 2 * n_each > kMaxOut || 2 * (n_each + 1) > hidden)) return KVQ_E_SHAPE;
  if (!any_sparse) n_each = 0;
  if ((reinterpret_cast<uintptr_t>(klut) & 15) != 0) return KVQ_E_ALIGN;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint32_t* kc = reinterpret_cast<uint32_t*>(kcache);
  uint32_t* vc = reinterpret_cast<uint32_t*>(vcache);
  switch (bits) {
    case 4: return launch_fused<4>(hidden, Lmax, slot, slot_dev, n_each, k_new, kc, klut, klut_sub, k_thr_lower, k_thr_upper, k_outliers, k_outlier_idx, v_new, vc, v_cent, v_cent_deq, vlut_tok, v_aff, v_outliers, v_outlier_idx, st, B, active, pg);
    case 3: return launch_fused<3>(hidden, Lmax, slot, slot_dev, n_each, k_new, kc, klut, klut_sub, k_thr_lower, k_thr_upper, k_outliers, k_outlier_idx, v_new, vc, v_cent, v_cent_deq, vlut_tok, v_aff, v_outliers, v_outlier_idx, st, B, active, pg);
    case 2: return launch_fused<2>(hidden, Lmax, slot, slot_dev, n_each, k_new, kc, klut, klut_sub, k_thr_lower, k_thr_upper, k_outliers, k_outlier_idx, v_new, vc, v_cent, v_cent_deq, vlut_tok, v_aff, v_outliers, v_outlier_idx, st, B, active, pg);
    default: return KVQ_E_BITS;
  }
}

int kvq_append_kv_fused(int bits, int H, int64_t Lmax, int64_t slot, int n_each, const float* k_new,
                        int32_t* kcache, const float* klut, const float* klut_sub, const float* k_thr_lower,
                        const float* k_thr_upper, float* k_outliers, int32_t* k_outlier_idx, const float* v_new,
                        int32_t* vcache, const float* v_cent, const float* v_cent_deq, float* vlut_tok, float* v_aff,
                        float* v_outliers, int32_t* v_outlier_idx, void* stream) {
  return append_kv_fused_impl(bits, H, Lmax, slot, nullptr, n_each, k_new, kcache, klut, klut_sub, k_thr_lower,
                              k_thr_upper, k_outliers, k_outlier_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok,
                              v_aff, v_outliers, v_outlier_idx, stream);
}

int kvq_append_kv_fused_dyn(int bits, int H, int64_t Lmax, const int64_t* len_dev, int64_t slot_add, int n_each,
                            const float* k_new, int32_t* kcache, const float* klut, const float* klut_sub,
                            const float* k_thr_lower, const float* k_thr_upper, float* k_outliers,
                            int32_t* k_outlier_idx, const float* v_new, int32_t* vcache, const float* v_cent,
                            const float* v_cent_deq, float* vlut_tok, float* v_aff, float* v_outliers,
                            int32_t* v_outlier_idx, void* stream) {
  if (!len_dev) return KVQ_E_NULL;
  return append_kv_fused_impl(bits, H, Lmax, slot_add, len_dev, n_each, k_new, kcache, klut, klut_sub, k_thr_lower,
                              k_thr_upper, k_outliers, k_outlier_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok,
                              v_aff, v_outliers, v_outlier_idx, stream);
}

int kvq_append_kv_fused_batch(int bits, int B, int H, int64_t Lmax, const int64_t* len_dev, int64_t slot_add,
                              const int32_t* active, int n_each, const float* k_new, int32_t* kcache, const float* klut,
                              const float* klut_sub, const float* k_thr_lower, const float* k_thr_upper, float* k_outliers,
                              int32_t* k_outlier_idx, const float* v_new, int32_t* vcache, const float* v_cent,
                              const float* v_cent_deq, float* vlut_tok, float* v_aff, float* v_outliers,
                              int32_t* v_outlier_idx, void* stream) {
  if (!len_dev) return KVQ_E_NULL;
  if (B < 1 || B > 256) return KVQ_E_SHAPE;
  return append_kv_fused_impl(bits, H, Lmax, slot_add, len_dev, n_each, k_new, kcache, klut, klut_sub, k_thr_lower,
                              k_thr_upper, k_outliers, k_outlier_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok,
                              v_aff, v_outliers, v_outlier_idx, stream, B, active);
}

int kvq_append_kv_fused_paged(int bits, int B, int H, int n_pool, const int64_t* len_dev, int64_t slot_add,
                              const int32_t* active, int n_each, const float* k_new, int32_t* kcache, const float* klut,
                              const float* klut_sub, const float* k_thr_lower, const float* k_thr_upper, float* k_outliers,
                              int32_t* k_outlier_idx, const float* v_new, int32_t* vcache, const float* v_cent,
                              const float* v_cent_deq, float* vlut_tok, float* v_aff, float* v_outliers,
                              int32_t* v_outlier_idx, void* stream, const int32_t* page_table, int max_pages,
                              const int32_t* npages, int P) {
  if (!len_dev || !page_table || !npages) return KVQ_E_NULL;
  if (B < 1 || B > 256) return KVQ_E_SHAPE;
  const int rc = check_pages(n_pool, max_pages, P, (int64_t)H * kHeadDim * bits / 32);
  if (rc) return rc;
  const PageRef pg{page_table, npages, max_pages, P, n_pool};
  return append_kv_fused_impl(bits, H, P, slot_add, len_dev, n_each, k_new, kcache, klut, klut_sub, k_thr_lower,
                              k_thr_upper, k_outliers, k_outlier_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok,
                              v_aff, v_outliers, v_outlier_idx, stream, B, active, &pg);
}

// the chunk append into a contiguous cache (pg == nullptr; Lmax > 0) or one paged sequence (Lmax = its mapped slots,
// possibly 0): every check, then the launch
static int append_chunk_impl(int bits, int H, int64_t Lmax, int64_t slot, int64_t T, int n_each, const float* k_new,
                             int32_t* kcache, const float* klut, const float* klut_sub, const float* k_thr_lower,
                             const float* k_thr_upper, float* k_outliers, int32_t* k_outlier_idx, const float* v_new,
                             int32_t* vcache, const float* v_cent, const float* v_cent_deq, float* vlut_tok,
                             float* v_aff, float* v_outliers, int32_t* v_outlier_idx, void* stream, const PageRef* pg) {
  // sizes first: an empty chunk returns 0 once they are valid, whatever the pointers (as kvq_dequant_kv)
  const int hidden = H * kHeadDim;
  if (H <= 0 || hidden > kMaxHidden || Lmax < 0 || (Lmax == 0 && pg == nullptr)) return KVQ_E_SHAPE;
  if (slot < 0 || T < 0 || slot > Lmax || T > Lmax - slot) return KVQ_E_SHAPE;
  const bool any_sparse = k_outliers != nullptr || v_outliers != nullptr;
  if (any_sparse && (n_each <= 0 || 2 * n_each > kMaxOut || 2 * (n_each + 1) > hidden)) return KVQ_E_SHAPE;
  if (!any_sparse) n_each = 0;
  if (bits < 2 || bits > 4) return KVQ_E_BITS;
  if (T == 0) return 0;
  if (!k_new || !kcache || !klut || !klut_sub || !k_thr_lower || !k_thr_upper || !v_new || !vcache || !v_cent || !vlut_tok)
    return KVQ_E_NULL;
  if ((k_outliers == nullptr) != (k_outlier_idx == nullptr) || (v_outliers == nullptr) != (v_outlier_idx == nullptr))
    return KVQ_E_NULL;
  if (pg != nullptr && pg->table == nullptr) return KVQ_E_NULL;
  if ((reinterpret_cast<uintptr_t>(klut) & 15) != 0) return KVQ_E_ALIGN;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint32_t* kc = reinterpret_cast<uint32_t*>(kcache);
  uint32_t* vc = reinterpret_cast<uint32_t*>(vcache);
  switch (bits) {
    case 4: return launch_fused_chunk<4>(hidden, Lmax, slot, T, n_each, k_new, kc, klut, klut_sub, k_thr_lower, k_thr_upper, k_outliers, k_outlier_idx, v_new, vc, v_cent, v_cent_deq, vlut_tok, v_aff, v_outliers, v_outlier_idx, st, pg);
    case 3: return launch_fused_chunk<3>(hidden, Lmax, slot, T, n_each, k_new, kc, klut, klut_sub, k_thr_lower, k_thr_upper, k_outliers, k_outlier_idx, v_new, vc, v_cent, v_cent_deq, vlut_tok, v_aff, v_outliers, v_outlier_idx, st, pg);
    default: return launch_fused_chunk<2>(hidden, Lmax, slot, T, n_each, k_new, kc, klut, klut_sub, k_thr_lower, k_thr_upper, k_outliers, k_outlier_idx, v_new, vc, v_cent, v_cent_deq, vlut_tok, v_aff, v_outliers, v_outlier_idx, st, pg);
  }
}

int kvq_append_kv_fused_chunk(int bits, int H, int64_t Lmax, int64_t slot, int64_t T, int n_each, const float* k_new,
                              int32_t* kcache, const float* klut, const float* klut_sub, const float* k_thr_lower,
                              const float* k_thr_upper, float* k_outliers, int32_t* k_outlier_idx, const float* v_new,
                              int32_t* vcache, const float* v_cent, const float* v_cent_deq, float* vlut_tok,
                              float* v_aff, float* v_outliers, int32_t* v_outlier_idx, void* stream) {
  return append_chunk_impl(bits, H, Lmax, slot, T, n_each, k_new, kcache, klut, klut_sub, k_thr_lower, k_thr_upper,
                           k_outliers, k_outlier_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok, v_aff, v_outliers,
                           v_outlier_idx, stream, nullptr);
}

int kvq_append_kv_fused_chunk_paged(int bits, int H, int n_pool, int64_t slot, int64_t T, int n_each,
                                    const float* k_new, int32_t* kcache, const float* klut, const float* klut_sub,
                                    const float* k_thr_lower, const float* k_thr_upper, float* k_outliers,
                                    int32_t* k_outlier_idx, const float* v_new, int32_t* vcache, const float* v_cent,
                                    const float* v_cent_deq, float* vlut_tok, float* v_aff, float* v_outliers,
                                    int32_t* v_outlier_idx, void* stream, const int32_t* pages, int max_pages,
                                    int n_mapped, int P) {
  if (H <= 0) return KVQ_E_SHAPE;
  const int rc = check_pages(n_pool, max_pages, P, (int64_t)H * kHeadDim * bits / 32);
  if (rc) return rc;
  if (n_mapped < 0 || n_mapped > max_pages) return KVQ_E_SHAPE;
  const PageRef pg{pages, nullptr, max_pages, P, n_pool};
  return append_chunk_impl(bits, H, (int64_t)n_mapped * P, slot, T, n_each, k_new, kcache, klut, klut_sub, k_thr_lower,
                           k_thr_upper, k_outliers, k_outlier_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok, v_aff,
                           v_outliers, v_outlier_idx, stream, &pg);
}

}  // extern "C"
