// kvquant_b200 -- append path: NUQ nearest-entry quantise + 4/3/2-bit pack (legacy single-token ops,
// prefill packers) and the fused device-side append (top-K outlier split + V thresholds + pack + row build) of one
// token or of a chunk of consecutive tokens.
//
// Reference semantics: deployment/kvquant/quant_cuda_kernel.cu:1167-2102 (appends), and the host-side glue
// in deployment/transformers/.../modeling_llama.py:664-751 (K), 1803-1820 + 1091-1176 (V).
#include "kvq_append.cuh"

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
// fused device-side append.  grid = 2 CTAs (0: K, 1: V), 1024 threads each.  The selection, the per-token work and
// the chunk append's body are in kvq_append.cuh, shared with the ragged chunk append (kvq_append_ragged.cu).
// ------------------------------------------------------------------------------------------------------------

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
