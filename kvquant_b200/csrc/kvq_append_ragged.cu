// kvquant_b200 -- ragged chunk append: the chunks of several slots of a batch in one launch (DESIGN.md section 4.15).
// A translation unit of its own, so that kvq_append.cu's kernels compile exactly as before.
#include "kvq_append.cuh"

namespace kvq {

// ------------------------------------------------------------------------------------------------------------
// ragged chunk append (kvq_append_kv_fused_chunk_ragged[_paged], DESIGN.md section 4.15): the chunks of several slots
// in one launch, grid (sum of the segments' tiles, 2).  Segment i owns tiles [tile0[i], tile0[i + 1]).  A CTA finds its
// segment, rebases the pointers on it and runs append_kv_chunk_body unchanged: the body numbers tiles from blockIdx.x,
// so the segment is presented as starting tile0[i] tiles early (rows row0 - 8 * tile0[i], slots s0 - 8 * tile0[i]),
// and the CTA's tile is then exactly the tile the lone call for that segment would give it.
// ------------------------------------------------------------------------------------------------------------
struct RagSeg {
  int64_t s0;     // first slot written
  int b, T, row0; // slot, tokens, first row of k_new / v_new
};
struct RaggedAppend {
  int n_seg;
  int tile0[kMaxSeg + 1];   // first tile of each segment; tile0[n_seg] = the grid's x extent
  RagSeg seg[kMaxSeg];
};

// PAGED: the cache pointers are page pools and pg.table the batch page table [B][max_pages]; the body gets the
// segment's row of it.  Contiguous: the pointers are rebased on the segment's slot of a [B, ...] batch (the layout of
// kvq_append_kv_fused_batch).
template <int BITS, bool PAGED>
__global__ void __launch_bounds__(kChunkThreads, 4) append_kv_chunk_ragged_kernel(
    int hidden, int64_t Lmax, int n_each,
    const float* __restrict__ k_new, uint32_t* __restrict__ kcache, const float* __restrict__ klut,
    const float* __restrict__ klut_sub, const float* __restrict__ k_thr_lo, const float* __restrict__ k_thr_hi,
    float* __restrict__ k_out, int32_t* __restrict__ k_idx,
    const float* __restrict__ v_new, uint32_t* __restrict__ vcache, const float* __restrict__ v_cent,
    const float* __restrict__ v_cent_deq, float* __restrict__ vlut_tok, float* __restrict__ v_aff, float* __restrict__ v_out,
    int32_t* __restrict__ v_idx, const PageRef pg, const __grid_constant__ RaggedAppend rg) {
  const int i = find_segment(rg.tile0, rg.n_seg, (int)blockIdx.x);
  const RagSeg sg = rg.seg[i];
  const int64_t back = (int64_t)rg.tile0[i] * kChunkTile;
  const int64_t r0 = sg.row0 - back;
  k_new += r0 * hidden;
  v_new += r0 * hidden;
  if constexpr (PAGED) {
    PageRef row = pg;
    row.table += (int64_t)sg.b * pg.max_pages;
    append_kv_chunk_body<BITS, true>(hidden, pg.P, sg.s0 - back, sg.T + back, n_each, k_new, kcache, klut, klut_sub,
                                     k_thr_lo, k_thr_hi, k_out, k_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok, v_aff,
                                     v_out, v_idx, row);
  } else {
    const int64_t b = sg.b;
    const int64_t words = (int64_t)hidden * BITS / 32 * Lmax, rows = Lmax * 2 * n_each;
    kcache += b * words; vcache += b * words;
    if (k_out != nullptr) { k_out += b * rows; k_idx += b * rows; }
    if (v_out != nullptr) { v_out += b * rows; v_idx += b * rows; }
    vlut_tok += b * Lmax * (1 << BITS);
    if (v_aff != nullptr) v_aff += b * Lmax * 2;
    append_kv_chunk_body<BITS, false>(hidden, Lmax, sg.s0 - back, sg.T + back, n_each, k_new, kcache, klut, klut_sub,
                                      k_thr_lo, k_thr_hi, k_out, k_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok,
                                      v_aff, v_out, v_idx, PageRef{});
  }
}

// segments checked; empty ones get no tiles
template <int BITS>
static int launch_fused_chunk_ragged(int hidden, int64_t Lmax, int n_seg, const int64_t* segs, int n_each,
                                     const float* k_new, uint32_t* kcache, const float* klut, const float* klut_sub,
                                     const float* ktl, const float* kth, float* kout, int32_t* kidx, const float* v_new,
                                     uint32_t* vcache, const float* vcent, const float* vcent_deq, float* vlut,
                                     float* vaff, float* vout, int32_t* vidx, cudaStream_t st, const PageRef* pg) {
  RaggedAppend rg{};
  rg.n_seg = n_seg;
  int64_t tiles = 0;
  for (int i = 0; i < n_seg; ++i) {
    rg.tile0[i] = (int)tiles;
    rg.seg[i] = RagSeg{segs[4 * i + 1], (int)segs[4 * i], (int)segs[4 * i + 2], (int)segs[4 * i + 3]};
    tiles += (segs[4 * i + 2] + kChunkTile - 1) / kChunkTile;
  }
  rg.tile0[n_seg] = (int)tiles;
  const size_t smem = chunk_smem_bytes<BITS>(hidden, 2 * n_each);
  static PerDeviceOnce attr_once[2];   // (one instance per BITS instantiation and form)
  bool& attr_done = attr_once[pg != nullptr].cur();
  if (!attr_done) {
    const int most = (int)chunk_smem_bytes<BITS>(kMaxHidden, kMaxOut);
    const cudaFuncAttribute a = cudaFuncAttributeMaxDynamicSharedMemorySize;
    cudaError_t e = pg != nullptr ? cudaFuncSetAttribute(append_kv_chunk_ragged_kernel<BITS, true>, a, most)
                                  : cudaFuncSetAttribute(append_kv_chunk_ragged_kernel<BITS, false>, a, most);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  const dim3 grid((unsigned)tiles, 2);
  if (pg != nullptr)
    append_kv_chunk_ragged_kernel<BITS, true><<<grid, kChunkThreads, smem, st>>>(
        hidden, pg->P, n_each, k_new, kcache, klut, klut_sub, ktl, kth, kout, kidx, v_new, vcache, vcent, vcent_deq,
        vlut, vaff, vout, vidx, *pg, rg);
  else
    append_kv_chunk_ragged_kernel<BITS, false><<<grid, kChunkThreads, smem, st>>>(
        hidden, Lmax, n_each, k_new, kcache, klut, klut_sub, ktl, kth, kout, kidx, v_new, vcache, vcent, vcent_deq,
        vlut, vaff, vout, vidx, PageRef{}, rg);
  KVQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace kvq

using namespace kvq;

extern "C" {

// the ragged chunk append into a contiguous batch (pg == nullptr) or a page pool (n_mapped: host, one per segment):
// every check, in the order of append_chunk_impl with the segment table's in front of its pointer checks, then one launch
static int append_chunk_ragged_impl(int bits, int B, int H, int64_t Lmax, int n_seg, const int64_t* segs, int64_t N,
                                    int n_each, const float* k_new, int32_t* kcache, const float* klut,
                                    const float* klut_sub, const float* k_thr_lower, const float* k_thr_upper,
                                    float* k_outliers, int32_t* k_outlier_idx, const float* v_new, int32_t* vcache,
                                    const float* v_cent, const float* v_cent_deq, float* vlut_tok, float* v_aff,
                                    float* v_outliers, int32_t* v_outlier_idx, void* stream, const PageRef* pg,
                                    const int32_t* n_mapped) {
  const int hidden = H * kHeadDim;
  if (H <= 0 || hidden > kMaxHidden || Lmax <= 0) return KVQ_E_SHAPE;
  if (B < 1 || B > kMaxSeg || n_seg < 0 || n_seg > B || N < 0) return KVQ_E_SHAPE;
  // the batch strides keep every slice 16-byte aligned, as kvq_append_kv_fused_batch
  if (pg == nullptr && ((H % 4 != 0 && H > 2) || Lmax % 4 != 0)) return KVQ_E_SHAPE;
  if (n_seg > 0 && (segs == nullptr || (pg != nullptr && n_mapped == nullptr))) return KVQ_E_NULL;
  int rc = check_segments(B, n_seg, segs, N, Lmax, pg != nullptr ? n_mapped : nullptr, pg != nullptr ? pg->max_pages : 0,
                          pg != nullptr ? pg->P : 0, true, nullptr);
  if (rc) return rc;
  const bool any_sparse = k_outliers != nullptr || v_outliers != nullptr;
  if (any_sparse && (n_each <= 0 || 2 * n_each > kMaxOut || 2 * (n_each + 1) > hidden)) return KVQ_E_SHAPE;
  if (!any_sparse) n_each = 0;
  if (bits < 2 || bits > 4) return KVQ_E_BITS;
  if (N == 0) return 0;
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
    case 4: return launch_fused_chunk_ragged<4>(hidden, Lmax, n_seg, segs, n_each, k_new, kc, klut, klut_sub, k_thr_lower, k_thr_upper, k_outliers, k_outlier_idx, v_new, vc, v_cent, v_cent_deq, vlut_tok, v_aff, v_outliers, v_outlier_idx, st, pg);
    case 3: return launch_fused_chunk_ragged<3>(hidden, Lmax, n_seg, segs, n_each, k_new, kc, klut, klut_sub, k_thr_lower, k_thr_upper, k_outliers, k_outlier_idx, v_new, vc, v_cent, v_cent_deq, vlut_tok, v_aff, v_outliers, v_outlier_idx, st, pg);
    default: return launch_fused_chunk_ragged<2>(hidden, Lmax, n_seg, segs, n_each, k_new, kc, klut, klut_sub, k_thr_lower, k_thr_upper, k_outliers, k_outlier_idx, v_new, vc, v_cent, v_cent_deq, vlut_tok, v_aff, v_outliers, v_outlier_idx, st, pg);
  }
}

int kvq_append_kv_fused_chunk_ragged(int bits, int B, int H, int64_t Lmax, int n_seg, const int64_t* segs, int64_t N,
                                     int n_each, const float* k_new, int32_t* kcache, const float* klut,
                                     const float* klut_sub, const float* k_thr_lower, const float* k_thr_upper,
                                     float* k_outliers, int32_t* k_outlier_idx, const float* v_new, int32_t* vcache,
                                     const float* v_cent, const float* v_cent_deq, float* vlut_tok, float* v_aff,
                                     float* v_outliers, int32_t* v_outlier_idx, void* stream) {
  return append_chunk_ragged_impl(bits, B, H, Lmax, n_seg, segs, N, n_each, k_new, kcache, klut, klut_sub, k_thr_lower,
                                  k_thr_upper, k_outliers, k_outlier_idx, v_new, vcache, v_cent, v_cent_deq, vlut_tok,
                                  v_aff, v_outliers, v_outlier_idx, stream, nullptr, nullptr);
}

int kvq_append_kv_fused_chunk_ragged_paged(int bits, int B, int H, int n_pool, int n_seg, const int64_t* segs,
                                           int64_t N, int n_each, const float* k_new, int32_t* kcache,
                                           const float* klut, const float* klut_sub, const float* k_thr_lower,
                                           const float* k_thr_upper, float* k_outliers, int32_t* k_outlier_idx,
                                           const float* v_new, int32_t* vcache, const float* v_cent,
                                           const float* v_cent_deq, float* vlut_tok, float* v_aff, float* v_outliers,
                                           int32_t* v_outlier_idx, void* stream, const int32_t* page_table,
                                           int max_pages, const int32_t* n_mapped, int P) {
  if (H <= 0) return KVQ_E_SHAPE;
  const int rc = check_pages(n_pool, max_pages, P, (int64_t)H * kHeadDim * bits / 32);
  if (rc) return rc;
  const PageRef pg{page_table, nullptr, max_pages, P, n_pool};
  return append_chunk_ragged_impl(bits, B, H, (int64_t)max_pages * P, n_seg, segs, N, n_each, k_new, kcache, klut,
                                  klut_sub, k_thr_lower, k_thr_upper, k_outliers, k_outlier_idx, v_new, vcache, v_cent,
                                  v_cent_deq, vlut_tok, v_aff, v_outliers, v_outlier_idx, stream, &pg, n_mapped);
}

}  // extern "C"
