// kvquant_b200 -- host-side description of one fused decode attend call (kvq_attend.cu) and of its scratch, and the
// K-side / V-side drivers that take them.
#pragma once
#include "kvq_common.cuh"

namespace kvq {

constexpr int kMaxPart = 256;                            // partial (o, l) rows: one per V-pass token range, <= one per SM
constexpr float kAttendScale = 0.08838834764831845f;     // 1/sqrt(128)  (modeling_llama.py:1959,1973)

// shape and alignment rules every reader of the V cache shares (the attend and kvq_v_matvec)
inline int check_v_common(int H, int64_t Lmax, int64_t L, const void* cache) {
  if (H <= 0 || (H & 3) != 0 || H > 64 || L < 0 || L > Lmax) return KVQ_E_SHAPE;
  if ((Lmax & 3) != 0 || (reinterpret_cast<uintptr_t>(cache) & 15) != 0) return KVQ_E_ALIGN;
  return 0;
}

// One attend call: a field per argument of the widest entry point (kvq_attend_paged).  Hq query heads, Hq / Hkv of them
// per KV head; the caches, tables, outlier rows and sinks hold Hkv heads.
struct AttendCall {
  int bits;
  const float* q;                    // [Hq][128], a batch [B][Hq][128]
  const int32_t* kcache;
  const float* klut;
  const float* k_outliers;           // outlier rows: values and channel indices, both or neither
  const int32_t* k_outlier_idx;
  const int32_t* vcache;
  const float* vlut_tok;             // materialised per-token LUT rows (the V form used when v_cent / v_aff are null)
  const float* v_cent;
  const float* v_aff;
  const float* v_outliers;
  const int32_t* v_outlier_idx;
  int n_out, Hq, Hkv;
  int64_t Lmax;                      // slots per sequence (a paged batch: max_pages * P)
  int64_t L;                         // tokens attended; with len_dev the cap the grids and the scratch are sized for
  const int64_t* len_dev;            // device-resident length(s), L = min(len_dev[b] + len_add, L); null: L as given
  int64_t len_add;
  const float* rope;                 // float2 [64][rope_npos] (cos, sin)
  const void* rope_half;             // half2 copy of it: selects the fp16-table K form; null = exact fp32
  int64_t rope_npos;
  float theta;
  bool freq;                         // the *_freq entry points: the table was built from rope_freq and attn_factor
  const float* rope_freq;            // f32 [64] (device): the outlier pass's rotary frequencies, theta unused
  float attn_factor;
  bool rope_per_seq;                 // batched *_seq entry points: sequence b's table and rope_freq sit b * 64 * rope_npos
                                     // entries and b * 64 floats after sequence 0's (length-dependent frequencies)
  int pos_offset;
  const void* sink_k;
  const void* sink_v;
  int n_sink;
  float* out;
  float* lse;                        // optional
  void* scratch;
  int B;                             // 0: one sequence; >= 1: a batch, sequence b's scratch block b * bstride floats on
  const PageRef* pg;                 // null: contiguous caches; else a paged batch (B >= 1)
  cudaStream_t stream;

  int grp() const { return Hq / Hkv; }
};

// The scratch of one sequence as the kernels see it; a batch repeats the block every `bstride` floats.
struct AttendScratch {
  float* scores;        // [Hq][stride]
  float* gmax;          // [Hq]
  float* sink_scores;   // [Hq][64]
  float* part_o;        // [kMaxPart][Hq][128]
  float* part_l;        // [kMaxPart][Hq]
  float* qtab;          // premultiplied K table [Hq][128][2^bits] ...
  float* qrat;          // ... and ratios [Hq][128] of the exact K form
  int64_t stride;       // L rounded up to 32
  int64_t bstride;      // floats per sequence block (a multiple of 4)
};
// the layout for Hq heads and L tokens over `scratch` (null: sizes only); every block starts 16-byte aligned
AttendScratch attend_scratch(void* scratch, int H, int64_t L, int bits);

// K side.  k_scores_fused: outlier scatter + the TMA-fed dense kernel (exact ratio form, or the fp16-table form when
// c.rope_half is set); k_scores_batch: the same for a (paged) batch, exact form only.  Both in kvq_kscore.cu.
int k_scores_fused(const AttendCall& c, const AttendScratch& s);
int k_scores_batch(const AttendCall& c, const AttendScratch& s);
// dense K kernels over tokens [0, c.L): kvq_kratio.cu, kvq_kfast.cu.
// accumulate != 0: s.scores holds the unscaled outlier partial sums on entry.
int k_ratio_dispatch(const AttendCall& c, const AttendScratch& s, int accumulate);
int k_fast_dispatch(const AttendCall& c, const AttendScratch& s, int accumulate);
// V side: softmax weights from s.scores / s.gmax, partial rows into s.part_o / s.part_l, their count in *n_cta.
// Native form (kvq_vnative.cu) and the form over materialised LUT rows (kvq_vaccum.cu).
int v_native_dispatch(const AttendCall& c, const AttendScratch& s, int* n_cta);
int v_accum_fused(const AttendCall& c, const AttendScratch& s, int* n_cta);

}  // namespace kvq
