// kvquant_b200 -- paged batch helpers (DESIGN.md section 4.11): the page-geometry checks of the paged entry points and
// kvq_page_copy, which moves a slot range of one sequence between a contiguous single-sequence cache and a paged
// sequence (or between two paged sequences), bit for bit.
//
// A paged sequence's token t lives in page pages[t / P], column t % P; a page is laid out as a single-sequence cache
// with Lmax = P.  So word row R of token t sits at (page * rows + R) * P + t % P of the pool's packed words (rows =
// Hkv * W), and its per-token rows (outliers, vlut, (sf, off)) at pool row page * P + t % P.
#include "kvq_common.cuh"
#include <algorithm>

namespace kvq {

int check_pages(int n_pool, int max_pages, int P, int64_t rows) {
  if (P <= 0 || P % kPageQuantum != 0) return KVQ_E_SHAPE;
  if (max_pages < 1 || (int64_t)max_pages * P >= ((int64_t)1 << 30)) return KVQ_E_SHAPE;
  if (n_pool < 1 || rows <= 0 || (int64_t)n_pool * rows >= ((int64_t)1 << 31) || (int64_t)n_pool * P >= ((int64_t)1 << 31))
    return KVQ_E_SHAPE;
  return 0;
}

int check_segments(int B, int n_seg, const int64_t* segs, int64_t N, int64_t Lmax, const int32_t* n_mapped,
                   int max_pages, int P, bool writes, int64_t* max_s0) {
  bool seen[kMaxSeg] = {};
  int64_t row = 0, top = 0;
  for (int i = 0; i < n_seg; ++i) {
    const int64_t b = segs[4 * i], s0 = segs[4 * i + 1], T = segs[4 * i + 2], row0 = segs[4 * i + 3];
    if (b < 0 || b >= B || seen[b]) return KVQ_E_SHAPE;
    seen[b] = true;
    if (s0 < 0 || T < 0 || row0 != row) return KVQ_E_SHAPE;
    if (s0 > Lmax || T > Lmax - s0) return KVQ_E_SHAPE;
    if (n_mapped != nullptr) {   // the slots read (s0) or written (s0 + T) must be mapped
      if (n_mapped[i] < 0 || n_mapped[i] > max_pages) return KVQ_E_SHAPE;
      if ((writes ? s0 + T : s0) > (int64_t)n_mapped[i] * P) return KVQ_E_SHAPE;
    }
    row += T;
    top = std::max(top, s0);
  }
  if (row != N || N >= ((int64_t)1 << 31)) return KVQ_E_SHAPE;
  if (max_s0 != nullptr) *max_s0 = top;
  return 0;
}

// one side of a copy: the eight tensors as 32-bit words (kcache, vcache, k values, k indices, v values, v indices,
// vlut, (sf, off)); pages == nullptr: a contiguous cache of Lmax slots
struct CopySide {
  uint32_t* t[8];
  int64_t Lmax;
  const int32_t* pages;
};

__device__ __forceinline__ int64_t copy_word_at(const CopySide& s, int rows, int P, int64_t R, int64_t t) {
  if (s.pages == nullptr) return R * s.Lmax + t;
  return ((int64_t)s.pages[t / P] * rows + R) * P + t % P;
}
__device__ __forceinline__ int64_t copy_row_at(const CopySide& s, int P, int64_t t) {
  return s.pages == nullptr ? t : (int64_t)s.pages[t / P] * P + t % P;
}

// grid (x, 8): blockIdx.y = tensor; grid-stride over its elements of tokens [s0, s0 + n), token-fastest for the
// packed words (a word row's tokens are consecutive in both layouts) and element-fastest for the per-token rows
constexpr int kCopyThreads = 256;
__global__ void __launch_bounds__(kCopyThreads) page_copy_kernel(const CopySide src, const CopySide dst, int64_t s0,
                                                                 int64_t n, int rows, int n_out, int nlev, int P) {
  const int which = blockIdx.y;
  const uint32_t* __restrict__ a = src.t[which];
  uint32_t* __restrict__ d = dst.t[which];
  if (a == nullptr) return;
  const int w = which < 2 ? 1 : (which < 6 ? n_out : (which == 6 ? nlev : 2));
  const int64_t total = which < 2 ? (int64_t)rows * n : n * w;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (which < 2) {
      const int64_t R = i / n, t = s0 + (i - R * n);
      d[copy_word_at(dst, rows, P, R, t)] = a[copy_word_at(src, rows, P, R, t)];
    } else {
      const int64_t j = i / w, c = i - j * w, t = s0 + j;
      d[copy_row_at(dst, P, t) * w + c] = a[copy_row_at(src, P, t) * w + c];
    }
  }
}

static int copy_side(const kvq_seq_ref* r, CopySide* s, int P, int64_t s1) {
  if (!r || !r->kcache || !r->vcache || !r->vlut_tok || !r->v_aff) return KVQ_E_NULL;
  if ((r->k_outliers == nullptr) != (r->k_outlier_idx == nullptr) || (r->v_outliers == nullptr) != (r->v_outlier_idx == nullptr))
    return KVQ_E_NULL;
  if (r->pages == nullptr && (r->Lmax <= 0 || s1 > r->Lmax)) return KVQ_E_SHAPE;
  if (r->pages != nullptr && (P <= 0 || P % kPageQuantum != 0)) return KVQ_E_SHAPE;
  s->t[0] = reinterpret_cast<uint32_t*>(r->kcache);
  s->t[1] = reinterpret_cast<uint32_t*>(r->vcache);
  s->t[2] = reinterpret_cast<uint32_t*>(r->k_outliers);
  s->t[3] = reinterpret_cast<uint32_t*>(r->k_outlier_idx);
  s->t[4] = reinterpret_cast<uint32_t*>(r->v_outliers);
  s->t[5] = reinterpret_cast<uint32_t*>(r->v_outlier_idx);
  s->t[6] = reinterpret_cast<uint32_t*>(r->vlut_tok);
  s->t[7] = reinterpret_cast<uint32_t*>(r->v_aff);
  s->Lmax = r->Lmax;
  s->pages = r->pages;
  return 0;
}

}  // namespace kvq

using namespace kvq;

extern "C" {

int kvq_page_copy(int bits, int H, int n_out, int P, int64_t s0, int64_t s1, const kvq_seq_ref* src,
                  const kvq_seq_ref* dst, void* stream) {
  if (bits < 2 || bits > 4) return KVQ_E_BITS;
  if (H <= 0 || s0 < 0 || s1 < s0 || s1 >= ((int64_t)1 << 30)) return KVQ_E_SHAPE;
  CopySide a{}, d{};
  int rc = copy_side(src, &a, P, s1);
  if (rc) return rc;
  if ((rc = copy_side(dst, &d, P, s1)) != 0) return rc;
  if (a.pages == nullptr && d.pages == nullptr) return KVQ_E_SHAPE;   // one side at least is paged
  // the two sides hold the same tensors: a dense-only side on one end must be dense-only on the other
  if ((a.t[2] == nullptr) != (d.t[2] == nullptr) || (a.t[4] == nullptr) != (d.t[4] == nullptr)) return KVQ_E_NULL;
  if ((a.t[2] != nullptr || a.t[4] != nullptr) && n_out <= 0) return KVQ_E_SHAPE;
  if (s1 == s0) return 0;
  const int rows = H * kHeadDim * bits / 32;
  const int64_t n = s1 - s0;
  const int64_t most = std::max<int64_t>((int64_t)rows * n, n * std::max(n_out, 1 << bits));
  const unsigned gx = (unsigned)std::min<int64_t>((most + kCopyThreads - 1) / kCopyThreads, 4 * num_sms_cached());
  page_copy_kernel<<<dim3(gx, 8), kCopyThreads, 0, static_cast<cudaStream_t>(stream)>>>(a, d, s0, n, rows, n_out,
                                                                                        1 << bits, P);
  KVQ_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
