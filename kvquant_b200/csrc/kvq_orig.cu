// kvquant_b200 -- the uncapped "orig" dense-and-sparse path (4-bit only in the reference):
//   * append: pack one token, threshold-crossing elements get the zero-point code 7 and are emitted compacted in
//     channel order as (index, value - zeropoint)     (reference quant_cuda_kernel.cu:846-931 and 1078-1163);
//     the reference needs two launches + a blocking D2H read of the count in between (745-747); here one launch
//     emits indices, values and the count, and the host glue (kvquant_b200/quant_cuda.py) grows the CSR arrays.
//   * SpMV: nnz-balanced CSR (K, rows = tokens, RoPE per nonzero; 523-614) and CSC (V, cols = tokens; 616-689),
//     10 nonzeros per thread, `start` gives each thread its first row/col.
#include "kvq_common.cuh"

namespace kvq {

constexpr int kOrigThreads = 1024;

// ISV=false: per-channel thresholds/zeropoint arrays, per-channel LUT [hidden,16]
// ISV=true : scalar thresholds/zeropoint, per-token LUT row lut[slot*16 ...]
template <bool ISV>
__global__ void __launch_bounds__(kOrigThreads, 1) orig_append_kernel(
    uint32_t* __restrict__ cache, const float* __restrict__ lut, const float* __restrict__ newvec,
    const float* __restrict__ zp_arr, const float* __restrict__ lo_arr, const float* __restrict__ hi_arr,
    float zp_s, float lo_s, float hi_s, int32_t* __restrict__ out_idx, float* __restrict__ out_val,
    int32_t* __restrict__ out_count, int hidden, int64_t Lmax, int64_t slot) {
  extern __shared__ unsigned char s_code[];  // [hidden]
  __shared__ int s_warp[32];
  __shared__ int s_total;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = (hidden + kOrigThreads - 1) / kOrigThreads;  // consecutive channels per thread
  const int j0 = tid * per;
  int cnt = 0;
  for (int e = 0; e < per; ++e) {
    const int j = j0 + e;
    if (j >= hidden) break;
    const float x = newvec[j];
    const float lo = ISV ? lo_s : lo_arr[j];
    const float hi = ISV ? hi_s : hi_arr[j];
    uint32_t code;
    if (x < lo || x > hi) { code = 7; ++cnt; }   // zero-point (quant_cuda_kernel.cu:905-909)
    else code = nearest_code<4>(lut + (ISV ? slot * 16 : (int64_t)j * 16), x);
    s_code[j] = (unsigned char)code;
  }
  // exclusive prefix sum of cnt over the block (channel order == thread order)
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = s_warp[lane];
    int wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += v;
    }
    s_warp[lane] = wi - w;  // exclusive
    if (lane == 31) s_total = wi;
  }
  __syncthreads();
  int pos = s_warp[warp] + incl - cnt;
  for (int e = 0; e < per; ++e) {
    const int j = j0 + e;
    if (j >= hidden) break;
    const float x = newvec[j];
    const float lo = ISV ? lo_s : lo_arr[j];
    const float hi = ISV ? hi_s : hi_arr[j];
    if (x < lo || x > hi) {
      out_idx[pos] = j;
      out_val[pos] = x - (ISV ? zp_s : zp_arr[j]);
      ++pos;
    }
  }
  if (tid == 0) *out_count = s_total;
  // pack (4-bit), words ADDED to the cache like the reference's atomicAdd
  for (int R = tid; R < hidden / 8; R += kOrigThreads) {
    uint32_t w = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) w |= (uint32_t)s_code[R * 8 + q] << (4 * q);
    uint32_t* p = cache + (int64_t)R * Lmax + slot;
    *p = *p + w;
  }
}

// ---- SpMV halves of the uncapped path ----------------------------------------------------------------------------------
// Same results as SPMV_ATOMIC_CSR_ROPE_BALANCED / SPMV_ATOMIC_CSC_BALANCED (quant_cuda_kernel.cu:523-614, 616-689), built
// the way the capped kernels of this library are (kvq_kscore.cu): the reference gives every thread ten consecutive
// non-zeros, walks the row pointers to find out which token each belongs to, re-evaluates powf / cosf / sinf per
// non-zero and issues one global atomic per non-zero (its start_rows / num_threads arguments only describe that work
// split and do not influence the result -- they are accepted and ignored here).
//
// K (CSR, row = token): one WARP per token.  The lanes stride over the token's non-zeros (coalesced), cos/sin come from
// the rope table (the reference's own expressions, evaluated once per (pair, position)), and because a row is sorted by
// channel the non-zeros of one head are adjacent: a warp-level segmented sum leaves one atomic per (token, head).
constexpr int kSpmvThreads = 256;

__global__ void __launch_bounds__(kSpmvThreads) csr_k_spmv_kernel(
    const int* __restrict__ row_ptr, const int* __restrict__ cols, const float* __restrict__ vals,
    const float* __restrict__ q, float* __restrict__ mul, int num_rows, int64_t seqlen,
    const float2* __restrict__ rope, int64_t rope_npos, int pos_offset) {
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * kSpmvThreads) >> 5;
  for (int row = (blockIdx.x * kSpmvThreads + threadIdx.x) >> 5; row < num_rows; row += warps) {
    const int beg = row_ptr[row], end = row_ptr[row + 1];
    for (int base = beg; base < end; base += 32) {      // warp-uniform trip count
      const int i = base + lane;
      float contrib = 0.f;
      int head = -1 - lane;                              // idle lanes never merge
      if (i < end) {
        const int col = cols[i];
        const float v = vals[i];
        head = col >> 7;
        const int ch = col & (kHeadDim - 1);
        const float2 cs = rope[(int64_t)(ch & (kHalf - 1)) * rope_npos + row + pos_offset];
        float dot = v * cs.x * __ldg(q + col);                                  // operation order of DK.cu:599-601
        dot += ((ch < kHalf) ? 1.f : -1.f) * v * cs.y * __ldg(q + (col ^ kHalf));
        contrib = dot;
      }
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {                 // segmented sum over runs of equal heads
        const float v2 = __shfl_down_sync(0xffffffffu, contrib, o);
        const int h2 = __shfl_down_sync(0xffffffffu, head, o);
        if (lane + o < 32 && h2 == head) contrib += v2;
      }
      const int hprev = __shfl_up_sync(0xffffffffu, head, 1);
      if (i < end && (lane == 0 || hprev != head)) atomicAdd(&mul[(int64_t)head * seqlen + row], contrib);
    }
  }
}

// V (CSC, column = token): one warp per token again; the products value * score[head, token] are summed per CHANNEL in a
// shared-memory image of the output that the CTA flushes once at the end -- `hidden` global atomics per CTA instead
// of one per non-zero onto the same 4096 addresses.
__global__ void __launch_bounds__(kSpmvThreads) csc_v_spmv_kernel(
    const int* __restrict__ rows, const int* __restrict__ col_ptr, const float* __restrict__ vals,
    const float* __restrict__ score, float* __restrict__ mul, int num_cols, int64_t seqlen, int hidden) {
  extern __shared__ float s_acc[];                       // [hidden]
  for (int j = threadIdx.x; j < hidden; j += kSpmvThreads) s_acc[j] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * kSpmvThreads) >> 5;
  for (int col = (blockIdx.x * kSpmvThreads + threadIdx.x) >> 5; col < num_cols; col += warps) {
    const int beg = col_ptr[col], end = col_ptr[col + 1];
    for (int i = beg + lane; i < end; i += 32) {
      const int ch = rows[i];
      atomicAdd(&s_acc[ch], vals[i] * __ldg(score + (int64_t)(ch >> 7) * seqlen + col));
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < hidden; j += kSpmvThreads) {
    const float v = s_acc[j];
    if (v != 0.f) atomicAdd(&mul[j], v);
  }
}

}  // namespace kvq

using namespace kvq;

extern "C" {

int kvq_k_spmv_csr(const int32_t* rows, const int32_t* cols, const int32_t* start_rows, const float* vals,
                   const float* q, float* mul, int H, int64_t L, int num_rows, int num_threads, int nnz,
                   const float* rope_cos_sin, int64_t rope_npos, int pos_offset, void* stream) {
  (void)start_rows; (void)num_threads;                  // the reference's work split, not part of the result
  if (!rows || !cols || !vals || !q || !mul || !rope_cos_sin) return KVQ_E_NULL;
  if (H <= 0 || L < 0 || nnz < 0 || num_rows < 0 || num_rows > L || rope_npos < num_rows + pos_offset) return KVQ_E_SHAPE;
  if (nnz == 0 || num_rows == 0) return 0;
  int grid = (num_rows * 32 + kSpmvThreads - 1) / kSpmvThreads;
  const int cap = num_sms_cached() * 8;
  if (grid > cap) grid = cap;
  csr_k_spmv_kernel<<<grid, kSpmvThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      rows, cols, vals, q, mul, num_rows, L, reinterpret_cast<const float2*>(rope_cos_sin), rope_npos, pos_offset);
  KVQ_LAUNCH_CHECK();
  return 0;
}

int kvq_v_spmv_csc(const int32_t* rows, const int32_t* cols, const int32_t* start_cols, const float* vals,
                   const float* score, float* mul, int H, int64_t L, int num_cols, int num_threads, int nnz,
                   void* stream) {
  (void)start_cols; (void)num_threads;
  if (!rows || !cols || !vals || !score || !mul) return KVQ_E_NULL;
  if (H <= 0 || H * kHeadDim > 12288 || L < 0 || nnz < 0 || num_cols < 0 || num_cols > L) return KVQ_E_SHAPE;
  if (nnz == 0 || num_cols == 0) return 0;
  const int hidden = H * kHeadDim;
  int grid = (num_cols * 32 + kSpmvThreads - 1) / kSpmvThreads;
  const int cap = num_sms_cached() * 2;
  if (grid > cap) grid = cap;
  csc_v_spmv_kernel<<<grid, kSpmvThreads, hidden * sizeof(float), static_cast<cudaStream_t>(stream)>>>(
      rows, cols, vals, score, mul, num_cols, L, hidden);
  KVQ_LAUNCH_CHECK();
  return 0;
}

int kvq_append_k_orig(int32_t* cache, const float* lut, const float* newvec, const float* zeropoint,
                      const float* thr_lower, const float* thr_upper, int32_t* out_cols, float* out_vals,
                      int32_t* out_count, int H, int64_t Lmax, int64_t slot, void* stream) {
  if (!cache || !lut || !newvec || !zeropoint || !thr_lower || !thr_upper || !out_cols || !out_vals || !out_count) return KVQ_E_NULL;
  if (H <= 0 || Lmax <= 0 || slot < 0 || slot >= Lmax) return KVQ_E_SHAPE;
  const int hidden = H * kHeadDim;
  orig_append_kernel<false><<<1, kOrigThreads, hidden, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<uint32_t*>(cache), lut, newvec, zeropoint, thr_lower, thr_upper, 0.f, 0.f, 0.f, out_cols,
      out_vals, out_count, hidden, Lmax, slot);
  KVQ_LAUNCH_CHECK();
  return 0;
}

int kvq_append_v_orig(int32_t* cache, const float* lut_tok, const float* newvec, float zeropoint, float thr_lower,
                      float thr_upper, int32_t* out_rows, float* out_vals, int32_t* out_count, int H, int64_t Lmax,
                      int64_t slot, void* stream) {
  if (!cache || !lut_tok || !newvec || !out_rows || !out_vals || !out_count) return KVQ_E_NULL;
  if (H <= 0 || Lmax <= 0 || slot < 0 || slot >= Lmax) return KVQ_E_SHAPE;
  const int hidden = H * kHeadDim;
  orig_append_kernel<true><<<1, kOrigThreads, hidden, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<uint32_t*>(cache), lut_tok, newvec, nullptr, nullptr, nullptr, zeropoint, thr_lower,
      thr_upper, out_rows, out_vals, out_count, hidden, Lmax, slot);
  KVQ_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
