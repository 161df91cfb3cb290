// kvquant_b200 -- the fused decode attend: softmax(q.K^T / sqrt(128)).V over the sinks and the quantised slots of one
// sequence, a batch of sequences or a paged batch (DESIGN.md section 4.3).
//
// One call is an AttendCall (kvq_attend.cuh): every kvq_attend* entry point fills one, attend_validate() rejects what
// cannot run before anything is launched, and attend_run() enqueues the chain
//   attend_init -> K outliers + dense K scores (kvq_kscore.cu) -> softmax . V partials (kvq_vnative.cu) -> attend_combine
// over a scratch laid out by attend_scratch().  This file holds the init / combine / merge kernels and that host side.
#include "kvq_attend.cuh"
#include <cuda_fp16.h>

namespace kvq {

// sink scores (fp16 post-RoPE keys, modeling_llama.py:1948-1949) and the initial per-head max.  GQA: the sinks belong
// to the cache, query head h reads those of KV head h / grp.
// BATCH: sequence b = blockIdx.y of a batched attend: q [B][H][128], sink_k [B][H/grp][128][n_sink], sink scores and
// maximum `bstride` floats after sequence b-1's.  BATCH = false ignores `bstride`.
template <bool GQA, bool BATCH>
__global__ void attend_init_kernel(const float* __restrict__ q, const __half* __restrict__ sink_k, int n_sink,
                                   float* __restrict__ sink_scores, float* __restrict__ gmax, float scale, int grp,
                                   const int64_t bstride) {
  // grid = H, block = 128 (thread = channel): s_i = scale * sum_c q[h,c] * sink_k[h,c,i], reduced per sink
  const int h = blockIdx.x, c = threadIdx.x;
  const int hk = GQA ? h / grp : h;
  if constexpr (BATCH) {
    const int b = blockIdx.y;
    q += (int64_t)b * gridDim.x * kHeadDim;
    if (sink_k != nullptr) sink_k += (int64_t)b * (gridDim.x / grp) * kHeadDim * n_sink;
    sink_scores += b * bstride;
    gmax += b * bstride;
  }
  __shared__ float s_part[4];
  __shared__ float s_max;
  if (c == 0) s_max = -INFINITY;
  const float qc = q[h * kHeadDim + c];
  for (int i = 0; i < n_sink; ++i) {
    float v = qc * __half2float(sink_k[((int64_t)hk * kHeadDim + c) * n_sink + i]);
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
// GQA: sink_v of KV head h / grp
// BATCH: sequence b = blockIdx.y of a batched attend: partials, maximum and sink scores `bstride` floats after sequence
// b-1's, sink_v [B][H/grp][n_sink][128], out [B][H][128], out_lse [B][H].  A sequence with no slot and no sink (an idle
// serving slot: l == 0) writes out = 0 and lse = -inf.  BATCH = false ignores `bstride`.
template <bool GQA, bool BATCH>
__global__ void __launch_bounds__(1024) attend_combine_kernel(const float* __restrict__ po, const float* __restrict__ pl,
                                                              int n_part, int H, const float* __restrict__ gmax,
                                                              const float* __restrict__ sink_scores,
                                                              const __half* __restrict__ sink_v, int n_sink,
                                                              float* __restrict__ out, float* __restrict__ out_lse,
                                                              int grp, const int64_t bstride) {
  __shared__ float4 s_o[32][32];
  __shared__ float s_l[32];
  const int h = blockIdx.x, lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  if constexpr (BATCH) {
    const int b = blockIdx.y;
    po += b * bstride; pl += b * bstride; gmax += b * bstride; sink_scores += b * bstride;
    if (sink_v != nullptr) sink_v += (int64_t)b * (H / grp) * n_sink * kHeadDim;
    out += (int64_t)b * H * kHeadDim;
    if (out_lse != nullptr) out_lse += (int64_t)b * H;
  }
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
  float m = gmax[h];
  for (int i = 0; i < n_sink; ++i) {
    const float pi = __expf(sink_scores[h * 64 + i] - m);
    o = fmaf(pi, __half2float(sink_v[((int64_t)(GQA ? h / grp : h) * n_sink + i) * kHeadDim + c]), o);
    l += pi;
  }
  if (BATCH && l == 0.f) o = 0.f, l = 1.f, m = -INFINITY;   // idle slot: nothing attended
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
static int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

AttendScratch attend_scratch(void* scratch, int H, int64_t L, int bits) {
  AttendScratch s{};
  float* const base = static_cast<float*>(scratch);
  int64_t off = 0;   // floats; every block below is a multiple of 4 floats (H % 4 == 0), so each starts 16-byte aligned
  auto take = [&](int64_t n) { float* p = base ? base + off : nullptr; off += n; return p; };
  s.stride = round_up(L, 32);
  s.scores = take(H * s.stride);
  s.gmax = take(H);
  s.sink_scores = take((int64_t)H * 64);
  s.part_o = take((int64_t)kMaxPart * H * kHeadDim);
  s.part_l = take((int64_t)kMaxPart * H);
  s.qtab = take((int64_t)H * kHeadDim * 17);   // sized for 4 bits: 16 table entries and one ratio per channel
  s.qrat = base ? s.qtab + (int64_t)H * kHeadDim * (1 << bits) : nullptr;
  s.bstride = off + 64;
  return s;
}

// Grouped-query attention: Hq query heads over an Hkv-head cache, query head h attending over KV head h / (Hq / Hkv).
// Hq == Hkv is multi-head attention, every K and V form; otherwise the exact-table, native-V path only.
// Hq % 4 == 0, Hq <= 64, and Hkv % 4 == 0 or Hkv <= 2 (two-KV-head and multi-query models, DESIGN.md section 4.9).
static int check_gqa(int Hq, int Hkv) {
  if (Hkv <= 0 || Hq <= 0 || Hq > 64 || (Hq & 3) != 0 || ((Hkv & 3) != 0 && Hkv > 2) || Hq % Hkv != 0) return KVQ_E_SHAPE;
  return 0;
}
static int gqa_unsupported(const AttendCall& c) {
  return (c.v_cent == nullptr || c.v_aff == nullptr || c.rope_half != nullptr) ? KVQ_E_UNSUPPORTED : 0;
}
// the preconditions of kvq_attend_gqa[_dyn] and kvq_attend_dyn, checked ahead of attend_validate
static int check_gqa_call(const AttendCall& c) {
  const int rc = check_gqa(c.Hq, c.Hkv);
  return rc ? rc : (c.Hq != c.Hkv ? gqa_unsupported(c) : 0);
}
static int check_dyn_call(const AttendCall& c) {
  if (!c.len_dev || !c.v_cent || !c.v_aff) return KVQ_E_NULL;
  return c.L <= 0 ? KVQ_E_SHAPE : 0;
}

// Everything that can be rejected from the arguments alone, before anything is launched.  The order is part of the
// ABI: an input with several faults gets the first code below.  That is why the bits and the kcache / scratch alignment
// checks appear twice: a batch reports them ahead of its pointer and shape checks, a single sequence after them.
static int attend_validate(const AttendCall& c) {
  const bool batch = c.B > 0;
  const bool bad_bits = c.bits < 2 || c.bits > 4;
  const bool misaligned = ((reinterpret_cast<uintptr_t>(c.kcache) | reinterpret_cast<uintptr_t>(c.scratch)) & 15) != 0;
  int rc;
  if (batch) {
    if ((rc = check_gqa(c.Hq, c.Hkv)) != 0) return rc;
    if (c.B > 256 || c.L <= 0) return KVQ_E_SHAPE;
    if (bad_bits) return KVQ_E_BITS;
    if ((rc = gqa_unsupported(c)) != 0) return rc;
    if (!c.len_dev) return KVQ_E_NULL;
  }
  if (!c.q || !c.kcache || !c.klut || !c.vcache || !c.rope || !c.out || !c.scratch) return KVQ_E_NULL;
  if ((!c.v_cent || !c.v_aff) && !c.vlut_tok) return KVQ_E_NULL;
  if (c.pg != nullptr) {
    if (!c.pg->table || !c.pg->npages) return KVQ_E_NULL;
    if ((rc = check_pages(c.pg->n_pool, c.pg->max_pages, c.pg->P, (int64_t)c.Hkv * kHeadDim * c.bits / 32)) != 0) return rc;
  }
  if ((rc = check_v_common(c.Hq, c.Lmax, c.L, c.vcache)) != 0) return rc;
  if (batch && misaligned) return KVQ_E_ALIGN;
  if ((c.k_outliers == nullptr) != (c.k_outlier_idx == nullptr) || (c.v_outliers == nullptr) != (c.v_outlier_idx == nullptr)) return KVQ_E_NULL;
  if ((c.k_outliers || c.v_outliers) && c.n_out <= 0) return KVQ_E_SHAPE;
  if (c.n_sink < 0 || c.n_sink > 64 || (c.n_sink > 0 && (!c.sink_k || !c.sink_v))) return KVQ_E_SHAPE;
  if (c.L + c.n_sink == 0 || c.rope_npos < c.L + c.pos_offset || c.pos_offset < 0 || c.Lmax >= ((int64_t)1 << 30)) return KVQ_E_SHAPE;
  if (num_sms_cached() > kMaxPart) return KVQ_E_UNSUPPORTED;
  if (misaligned) return KVQ_E_ALIGN;
  if (bad_bits) return KVQ_E_BITS;
  if (c.freq && !c.rope_freq) return KVQ_E_NULL;
  if (c.freq && !(c.attn_factor > 0.f && c.attn_factor < INFINITY)) return KVQ_E_SHAPE;
  if (c.rope_per_seq && (c.B < 1 || c.rope_npos > ((int64_t)1 << 30))) return KVQ_E_SHAPE;
  return 0;
}

// One sequence: init -> score clear (cudaMemset2DAsync) -> K outliers -> dense K -> V -> combine, the K and V kernels
// skipped when L == 0 (sinks only).  A batch (c.B >= 1): the same chain with the sequence a grid dimension, the clear
// done by a kernel that reads each sequence's length, and nothing skipped.  A paged batch (c.pg) differs only inside
// the kernels that read the cache (K outliers, dense K, V): init, clear and combine work on logical token indices in
// the scratch, and the grids are sized by (B, Hq, L) alone, so it runs the contiguous batch's grids.
static int attend_run(const AttendCall& c) {
  const int H = c.Hq, grp = c.grp();
  const bool batch = c.B > 0;
  AttendScratch s = attend_scratch(c.scratch, H, c.L, c.bits);
  if (!batch) s.bstride = 0;   // one sequence: no block offset is handed to the kernels
  const dim3 heads = batch ? dim3(H, c.B) : dim3(H);
  const __half* sink_k = static_cast<const __half*>(c.sink_k);
  const __half* sink_v = static_cast<const __half*>(c.sink_v);
  with_flavour(grp > 1, batch, false, [&](auto GQA, auto BATCH, auto) {
    attend_init_kernel<GQA(), BATCH()><<<heads, kHeadDim, 0, c.stream>>>(
        c.q, sink_k, c.n_sink, s.sink_scores, s.gmax, kAttendScale, grp, s.bstride);
  });
  KVQ_LAUNCH_CHECK();
  int n_cta = 0;
  if (batch || c.L > 0) {
    int rc = batch ? k_scores_batch(c, s) : k_scores_fused(c, s);
    if (rc) return rc;
    rc = (c.v_cent != nullptr && c.v_aff != nullptr) ? v_native_dispatch(c, s, &n_cta) : v_accum_fused(c, s, &n_cta);
    if (rc) return rc;
  }
  with_flavour(grp > 1, batch, false, [&](auto GQA, auto BATCH, auto) {
    attend_combine_kernel<GQA(), BATCH()><<<heads, 1024, 0, c.stream>>>(
        s.part_o, s.part_l, n_cta, H, s.gmax, s.sink_scores, sink_v, c.n_sink, c.out, c.lse, grp, s.bstride);
  });
  KVQ_LAUNCH_CHECK();
  return 0;
}

static int attend(const AttendCall& c) {
  const int rc = attend_validate(c);
  return rc ? rc : attend_run(c);
}

}  // namespace kvq

using namespace kvq;

extern "C" {

int64_t kvq_attend_scratch_bytes(int H, int64_t L) { return 4 * attend_scratch(nullptr, H, L, 4).bstride; }

// Sequence b's scratch block is bytes [b*S, (b+1)*S) of scratch, S = kvq_attend_scratch_bytes(Hq, L_cap) (a multiple of
// 16 bytes), laid out as the single-sequence call lays it out.
int64_t kvq_attend_batch_scratch_bytes(int B, int Hq, int64_t L_cap) {
  if (B < 1 || B > 256 || Hq <= 0 || L_cap <= 0) return 0;
  return (int64_t)B * kvq_attend_scratch_bytes(Hq, L_cap);
}

int kvq_attend(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
               const int32_t* k_outlier_idx, const int32_t* vcache, const float* vlut_tok, const float* v_cent,
               const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int H, int64_t Lmax, int64_t L, const float* rope_cos_sin,
               int64_t rope_npos, float theta, int pos_offset, const void* sink_k, const void* sink_v, int n_sink,
               float* out, float* out_lse, void* scratch, const void* rope_half, void* stream) {
  AttendCall c{};
  c.bits = bits; c.q = q; c.kcache = kcache; c.klut = klut; c.k_outliers = k_outliers; c.k_outlier_idx = k_outlier_idx;
  c.vcache = vcache; c.vlut_tok = vlut_tok; c.v_cent = v_cent; c.v_aff = v_aff; c.v_outliers = v_outliers; c.v_outlier_idx = v_outlier_idx;
  c.n_out = n_out; c.Hq = H; c.Hkv = H; c.Lmax = Lmax; c.L = L;
  c.rope = rope_cos_sin; c.rope_half = rope_half; c.rope_npos = rope_npos; c.theta = theta; c.pos_offset = pos_offset;
  c.sink_k = sink_k; c.sink_v = sink_v; c.n_sink = n_sink; c.out = out; c.lse = out_lse; c.scratch = scratch;
  c.stream = static_cast<cudaStream_t>(stream);
  return attend(c);
}

int kvq_attend_dyn(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
                   const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent, const float* v_aff,
                   const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int H, int64_t Lmax, int64_t L_cap,
                   const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin, int64_t rope_npos, float theta,
                   int pos_offset, const void* sink_k, const void* sink_v, int n_sink, float* out, float* out_lse,
                   void* scratch, const void* rope_half, void* stream) {
  AttendCall c{};
  c.bits = bits; c.q = q; c.kcache = kcache; c.klut = klut; c.k_outliers = k_outliers; c.k_outlier_idx = k_outlier_idx;
  c.vcache = vcache; c.v_cent = v_cent; c.v_aff = v_aff; c.v_outliers = v_outliers; c.v_outlier_idx = v_outlier_idx;
  c.n_out = n_out; c.Hq = H; c.Hkv = H; c.Lmax = Lmax; c.L = L_cap; c.len_dev = len_dev; c.len_add = len_add;
  c.rope = rope_cos_sin; c.rope_half = rope_half; c.rope_npos = rope_npos; c.theta = theta; c.pos_offset = pos_offset;
  c.sink_k = sink_k; c.sink_v = sink_v; c.n_sink = n_sink; c.out = out; c.lse = out_lse; c.scratch = scratch;
  c.stream = static_cast<cudaStream_t>(stream);
  const int rc = check_dyn_call(c);
  return rc ? rc : attend(c);
}

}  // extern "C"

// The rotary side of a call: theta (the kvq_attend* entry points) or a frequency vector and attention factor (their
// *_freq siblings), stored into the AttendCall by the shared bodies below.
// The *_freq_seq entry points: one table and frequency vector per sequence of a batch (length-dependent rotary).
struct RopeArg {
  float theta;
  const float* freq;
  float attn;
  bool scaled;
  bool per_seq;
  void set(AttendCall& c) const {
    c.theta = theta; c.freq = scaled; c.rope_freq = freq; c.attn_factor = attn; c.rope_per_seq = per_seq;
  }
};
static RopeArg theta_arg(float theta) { return RopeArg{theta, nullptr, 1.f, false, false}; }
static RopeArg freq_arg(const float* freq, float attn) { return RopeArg{0.f, freq, attn, true, false}; }
static RopeArg freq_seq_arg(const float* freq, float attn) { return RopeArg{0.f, freq, attn, true, true}; }

static int attend_gqa(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
                      const int32_t* k_outlier_idx, const int32_t* vcache, const float* vlut_tok, const float* v_cent,
                      const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int Hq,
                      int Hkv, int64_t Lmax, int64_t L, const float* rope_cos_sin, int64_t rope_npos, RopeArg ra,
                      int pos_offset, const void* sink_k, const void* sink_v, int n_sink, float* out, float* out_lse,
                      void* scratch, const void* rope_half, void* stream) {
  AttendCall c{};
  c.bits = bits; c.q = q; c.kcache = kcache; c.klut = klut; c.k_outliers = k_outliers; c.k_outlier_idx = k_outlier_idx;
  c.vcache = vcache; c.vlut_tok = vlut_tok; c.v_cent = v_cent; c.v_aff = v_aff; c.v_outliers = v_outliers; c.v_outlier_idx = v_outlier_idx;
  c.n_out = n_out; c.Hq = Hq; c.Hkv = Hkv; c.Lmax = Lmax; c.L = L;
  c.rope = rope_cos_sin; c.rope_half = rope_half; c.rope_npos = rope_npos; ra.set(c); c.pos_offset = pos_offset;
  c.sink_k = sink_k; c.sink_v = sink_v; c.n_sink = n_sink; c.out = out; c.lse = out_lse; c.scratch = scratch;
  c.stream = static_cast<cudaStream_t>(stream);
  const int rc = check_gqa_call(c);
  return rc ? rc : attend(c);
}

static int attend_gqa_dyn(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
                          const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent, const float* v_aff,
                          const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv,
                          int64_t Lmax, int64_t L_cap, const int64_t* len_dev, int64_t len_add,
                          const float* rope_cos_sin, int64_t rope_npos, RopeArg ra, int pos_offset, const void* sink_k,
                          const void* sink_v, int n_sink, float* out, float* out_lse, void* scratch,
                          const void* rope_half, void* stream) {
  AttendCall c{};
  c.bits = bits; c.q = q; c.kcache = kcache; c.klut = klut; c.k_outliers = k_outliers; c.k_outlier_idx = k_outlier_idx;
  c.vcache = vcache; c.v_cent = v_cent; c.v_aff = v_aff; c.v_outliers = v_outliers; c.v_outlier_idx = v_outlier_idx;
  c.n_out = n_out; c.Hq = Hq; c.Hkv = Hkv; c.Lmax = Lmax; c.L = L_cap; c.len_dev = len_dev; c.len_add = len_add;
  c.rope = rope_cos_sin; c.rope_half = rope_half; c.rope_npos = rope_npos; ra.set(c); c.pos_offset = pos_offset;
  c.sink_k = sink_k; c.sink_v = sink_v; c.n_sink = n_sink; c.out = out; c.lse = out_lse; c.scratch = scratch;
  c.stream = static_cast<cudaStream_t>(stream);
  int rc = check_gqa_call(c);
  if (rc == 0) rc = check_dyn_call(c);
  return rc ? rc : attend(c);
}

// Batched decode attend: B sequences of one layer in one launch set, over a batch-strided cache of Lmax slots per
// sequence
static int attend_batch(int bits, int B, const float* q, const int32_t* kcache, const float* klut,
                        const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                        const float* v_cent, const float* v_aff, const float* v_outliers,
                        const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv, int64_t Lmax, int64_t L_cap,
                        const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin, int64_t rope_npos,
                        RopeArg ra, int pos_offset, const void* sink_k, const void* sink_v, int n_sink, float* out,
                        float* out_lse, void* scratch, const void* rope_half, void* stream) {
  if (B < 1) return KVQ_E_SHAPE;
  AttendCall c{};
  c.bits = bits; c.q = q; c.kcache = kcache; c.klut = klut; c.k_outliers = k_outliers; c.k_outlier_idx = k_outlier_idx;
  c.vcache = vcache; c.v_cent = v_cent; c.v_aff = v_aff; c.v_outliers = v_outliers; c.v_outlier_idx = v_outlier_idx;
  c.n_out = n_out; c.Hq = Hq; c.Hkv = Hkv; c.Lmax = Lmax; c.L = L_cap; c.len_dev = len_dev; c.len_add = len_add;
  c.rope = rope_cos_sin; c.rope_half = rope_half; c.rope_npos = rope_npos; ra.set(c); c.pos_offset = pos_offset;
  c.sink_k = sink_k; c.sink_v = sink_v; c.n_sink = n_sink; c.out = out; c.lse = out_lse; c.scratch = scratch;
  c.stream = static_cast<cudaStream_t>(stream);
  c.B = B;
  return attend(c);
}

// Paged batch: the argument list of kvq_attend_batch with the pool size n_pool in place of Lmax, plus the page table;
// the caches and row tensors are page pools and the per-sequence cap is max_pages * P
static int attend_paged(int bits, int B, const float* q, const int32_t* kcache, const float* klut,
                        const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                        const float* v_cent, const float* v_aff, const float* v_outliers,
                        const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv, int n_pool, int64_t L_cap,
                        const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin, int64_t rope_npos,
                        RopeArg ra, int pos_offset, const void* sink_k, const void* sink_v, int n_sink, float* out,
                        float* out_lse, void* scratch, const void* rope_half, void* stream,
                        const int32_t* page_table, int max_pages, const int32_t* npages, int P) {
  if (B < 1) return KVQ_E_SHAPE;
  const PageRef pg{page_table, npages, max_pages, P, n_pool};
  AttendCall c{};
  c.bits = bits; c.q = q; c.kcache = kcache; c.klut = klut; c.k_outliers = k_outliers; c.k_outlier_idx = k_outlier_idx;
  c.vcache = vcache; c.v_cent = v_cent; c.v_aff = v_aff; c.v_outliers = v_outliers; c.v_outlier_idx = v_outlier_idx;
  c.n_out = n_out; c.Hq = Hq; c.Hkv = Hkv; c.Lmax = (int64_t)max_pages * P; c.L = L_cap; c.len_dev = len_dev; c.len_add = len_add;
  c.rope = rope_cos_sin; c.rope_half = rope_half; c.rope_npos = rope_npos; ra.set(c); c.pos_offset = pos_offset;
  c.sink_k = sink_k; c.sink_v = sink_v; c.n_sink = n_sink; c.out = out; c.lse = out_lse; c.scratch = scratch;
  c.stream = static_cast<cudaStream_t>(stream);
  c.B = B; c.pg = &pg;
  return attend(c);
}

extern "C" {

#define KVQ_GQA_ARGS(ROPE)                                                                                               \
  bits, q, kcache, klut, k_outliers, k_outlier_idx, vcache, vlut_tok, v_cent, v_aff, v_outliers, v_outlier_idx, n_out,   \
      Hq, Hkv, Lmax, L, rope_cos_sin, rope_npos, ROPE, pos_offset, sink_k, sink_v, n_sink, out, out_lse, scratch,       \
      rope_half, stream
#define KVQ_DYN_ARGS(ROPE)                                                                                               \
  bits, q, kcache, klut, k_outliers, k_outlier_idx, vcache, v_cent, v_aff, v_outliers, v_outlier_idx, n_out, Hq, Hkv,    \
      Lmax, L_cap, len_dev, len_add, rope_cos_sin, rope_npos, ROPE, pos_offset, sink_k, sink_v, n_sink, out, out_lse,   \
      scratch, rope_half, stream
#define KVQ_BATCH_ARGS(EXTENT, ROPE)                                                                                     \
  bits, B, q, kcache, klut, k_outliers, k_outlier_idx, vcache, v_cent, v_aff, v_outliers, v_outlier_idx, n_out, Hq, Hkv, \
      EXTENT, L_cap, len_dev, len_add, rope_cos_sin, rope_npos, ROPE, pos_offset, sink_k, sink_v, n_sink, out, out_lse, \
      scratch, rope_half, stream

int kvq_attend_gqa(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
                   const int32_t* k_outlier_idx, const int32_t* vcache, const float* vlut_tok, const float* v_cent,
                   const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv,
                   int64_t Lmax, int64_t L, const float* rope_cos_sin, int64_t rope_npos, float theta, int pos_offset,
                   const void* sink_k, const void* sink_v, int n_sink, float* out, float* out_lse, void* scratch,
                   const void* rope_half, void* stream) {
  return attend_gqa(KVQ_GQA_ARGS(theta_arg(theta)));
}

int kvq_attend_gqa_freq(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
                        const int32_t* k_outlier_idx, const int32_t* vcache, const float* vlut_tok, const float* v_cent,
                        const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int Hq,
                        int Hkv, int64_t Lmax, int64_t L, const float* rope_cos_sin, int64_t rope_npos,
                        const float* rope_freq, float attn_factor, int pos_offset, const void* sink_k,
                        const void* sink_v, int n_sink, float* out, float* out_lse, void* scratch,
                        const void* rope_half, void* stream) {
  return attend_gqa(KVQ_GQA_ARGS(freq_arg(rope_freq, attn_factor)));
}

int kvq_attend_gqa_dyn(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
                       const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent, const float* v_aff,
                       const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv, int64_t Lmax,
                       int64_t L_cap, const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin,
                       int64_t rope_npos, float theta, int pos_offset, const void* sink_k, const void* sink_v, int n_sink,
                       float* out, float* out_lse, void* scratch, const void* rope_half, void* stream) {
  return attend_gqa_dyn(KVQ_DYN_ARGS(theta_arg(theta)));
}

int kvq_attend_gqa_dyn_freq(int bits, const float* q, const int32_t* kcache, const float* klut,
                            const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                            const float* v_cent, const float* v_aff, const float* v_outliers,
                            const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv, int64_t Lmax, int64_t L_cap,
                            const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin, int64_t rope_npos,
                            const float* rope_freq, float attn_factor, int pos_offset, const void* sink_k,
                            const void* sink_v, int n_sink, float* out, float* out_lse, void* scratch,
                            const void* rope_half, void* stream) {
  return attend_gqa_dyn(KVQ_DYN_ARGS(freq_arg(rope_freq, attn_factor)));
}

int kvq_attend_batch(int bits, int B, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
                     const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent, const float* v_aff,
                     const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv, int64_t Lmax,
                     int64_t L_cap, const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin,
                     int64_t rope_npos, float theta, int pos_offset, const void* sink_k, const void* sink_v, int n_sink,
                     float* out, float* out_lse, void* scratch, const void* rope_half, void* stream) {
  return attend_batch(KVQ_BATCH_ARGS(Lmax, theta_arg(theta)));
}

int kvq_attend_batch_freq(int bits, int B, const float* q, const int32_t* kcache, const float* klut,
                          const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                          const float* v_cent, const float* v_aff, const float* v_outliers,
                          const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv, int64_t Lmax, int64_t L_cap,
                          const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin, int64_t rope_npos,
                          const float* rope_freq, float attn_factor, int pos_offset, const void* sink_k,
                          const void* sink_v, int n_sink, float* out, float* out_lse, void* scratch,
                          const void* rope_half, void* stream) {
  return attend_batch(KVQ_BATCH_ARGS(Lmax, freq_arg(rope_freq, attn_factor)));
}

int kvq_attend_paged(int bits, int B, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
                     const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent, const float* v_aff,
                     const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv, int n_pool,
                     int64_t L_cap, const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin,
                     int64_t rope_npos, float theta, int pos_offset, const void* sink_k, const void* sink_v, int n_sink,
                     float* out, float* out_lse, void* scratch, const void* rope_half, void* stream,
                     const int32_t* page_table, int max_pages, const int32_t* npages, int P) {
  return attend_paged(KVQ_BATCH_ARGS(n_pool, theta_arg(theta)), page_table, max_pages, npages, P);
}

int kvq_attend_paged_freq(int bits, int B, const float* q, const int32_t* kcache, const float* klut,
                          const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                          const float* v_cent, const float* v_aff, const float* v_outliers,
                          const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv, int n_pool, int64_t L_cap,
                          const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin, int64_t rope_npos,
                          const float* rope_freq, float attn_factor, int pos_offset, const void* sink_k,
                          const void* sink_v, int n_sink, float* out, float* out_lse, void* scratch,
                          const void* rope_half, void* stream, const int32_t* page_table, int max_pages,
                          const int32_t* npages, int P) {
  return attend_paged(KVQ_BATCH_ARGS(n_pool, freq_arg(rope_freq, attn_factor)), page_table, max_pages, npages, P);
}

int kvq_attend_batch_freq_seq(int bits, int B, const float* q, const int32_t* kcache, const float* klut,
                              const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                              const float* v_cent, const float* v_aff, const float* v_outliers,
                              const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv, int64_t Lmax, int64_t L_cap,
                              const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin, int64_t rope_npos,
                              const float* rope_freq, float attn_factor, int pos_offset, const void* sink_k,
                              const void* sink_v, int n_sink, float* out, float* out_lse, void* scratch,
                              const void* rope_half, void* stream) {
  return attend_batch(KVQ_BATCH_ARGS(Lmax, freq_seq_arg(rope_freq, attn_factor)));
}

int kvq_attend_paged_freq_seq(int bits, int B, const float* q, const int32_t* kcache, const float* klut,
                              const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                              const float* v_cent, const float* v_aff, const float* v_outliers,
                              const int32_t* v_outlier_idx, int n_out, int Hq, int Hkv, int n_pool, int64_t L_cap,
                              const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin, int64_t rope_npos,
                              const float* rope_freq, float attn_factor, int pos_offset, const void* sink_k,
                              const void* sink_v, int n_sink, float* out, float* out_lse, void* scratch,
                              const void* rope_half, void* stream, const int32_t* page_table, int max_pages,
                              const int32_t* npages, int P) {
  return attend_paged(KVQ_BATCH_ARGS(n_pool, freq_seq_arg(rope_freq, attn_factor)), page_table, max_pages, npages, P);
}

int kvq_attend_merge(const float* parts, int n_parts, int H, float* out, void* stream) {
  if (!parts || !out) return KVQ_E_NULL;
  if (n_parts <= 0 || H <= 0) return KVQ_E_SHAPE;
  attend_merge_kernel<<<H, kHeadDim, 0, static_cast<cudaStream_t>(stream)>>>(parts, n_parts, H, out);
  KVQ_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
