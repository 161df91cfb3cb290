// kvquant_b200 -- Q.K^T decode matvec over the packed pre-RoPE key cache with RoPE applied at read time: the dense
// kernel of kvq_k_matvec at 4 and 2 bits (3-bit has its own in kvq_k3.cu), the outlier scatter that runs in front of
// it and of the fused attend's dense kernels, the rope table builder, and the K side of the fused attend.
//
// Replaces (reference deployment/kvquant/quant_cuda_kernel.cu):
//   VecQuant{4,3,2}MatMulKernelNUQPerChannelTransposedRopeMHABatchedFusedOpt   3040-3209, 3692-4115, 4747-4996
//   SPMV_ATOMIC_ROPE_BALANCED                                                   472-521
//
//   S[h,t] = sum_c (LUT[h,c,code(h,c,t)] (+) outlier(h,c,t)) * (cos(th_j p) q[h,c] + s_c sin(th_j p) q[h,(c+64)%128])
//   j = c % 64, p = t + pos_offset.
//
// Design (DESIGN.md section 4.1):
//   * The reference evaluates powf+cosf+sinf per (head, channel, token): 4096 sincos per token per layer make it
//     ALU-bound.  cos/sin depend on (j, p) only, so they come from a table rope[j][p] built ONCE with the
//     reference's own expressions (bit-identical values); a thread loads the 16 pairs it needs for its token and
//     reuses them across all heads of its CTA (G heads) -> 64 table reads per token per CTA.
//   * thread = token (coalesced 128-byte warp loads straight from the sequence-fastest cache rows), per-channel
//     premultiplied tables T[h][c][code] = (LUT*q[h,c], s_c*LUT*q[h,c^64]) in shared memory: 16 (4) entries per
//     channel are 16 distinct consecutive 8-byte slots -> conflict-free multicast for any code pattern.
//   * per element: 1 address op (PRMT), 1 LDS.64, 2 FFMA; words and rope values are prefetched into rotating
//     register buffers; token ranges are cut at warp granularity so that every SM gets an equal share.
#include "kvq_kscore.cuh"
#include "kvq_attend.cuh"
#include <cuda_fp16.h>
#include <math_constants.h>
#include <stdlib.h>
#include <algorithm>

namespace kvq {

template <int BITS> struct KCfg {
  static_assert(BITS == 4 || BITS == 2, "3-bit caches have their own kernel (kvq_k3.cu)");
  static constexpr int N = 1 << BITS;
  static constexpr int W = Layout<BITS>::kWords;
  static constexpr int G = (BITS == 2) ? 16 : 128 / N;  // heads per CTA: 8 / 16 -> table = 128 / 64 KiB
  static constexpr int kThreads = 512;
  static constexpr int TT = kThreads;          // tokens per tile (thread = token)
  static constexpr int NRW = 2;                // packed words a thread needs per (head, 8-pair chunk)
};

// packed-word rows (relative to the head) needed for 8-pair chunk a (pairs 8a..8a+7): channels 8a..8a+7 and +64
template <int BITS> __device__ __forceinline__ int chunk_word_row(int a, int i) {
  if constexpr (BITS == 4) { return i == 0 ? a : a + 8; }
  else { return i == 0 ? (a >> 1) : 4 + (a >> 1); }
}

// One work item = (head hl, 8-pair chunk a): 16 table lookups + 16 packed FMAs into the head's accumulator.
//   base = shared address of T[hl][8a][0] (256-byte aligned: the low address byte carries code*8);
//   codes pre-masked into byte lanes, ONE PRMT per element builds the address.
template <int BITS>
__device__ __forceinline__ void k_item(const uint32_t* __restrict__ w, const int a, const uint32_t base,
                                       const float2* __restrict__ cs, float2& acc) {
  constexpr int N = 1 << BITS;
  constexpr int HI = kHalf * N * 8;  // byte offset of the +64 partner channel's table
  if constexpr (BITS == 4) {
    const uint32_t e0 = (w[0] << 3) & 0x78787878u, o0 = (w[0] >> 1) & 0x78787878u;
    const uint32_t e1 = (w[1] << 3) & 0x78787878u, o1 = (w[1] >> 1) & 0x78787878u;
    static_for<0, 8>([&](auto ik) {
      constexpr int k = decltype(ik)::v;
      ffma2(acc, cs[k], lds_f2<k * N * 8>(__byte_perm((k & 1) ? o0 : e0, base, 0x7650 | (k >> 1))));
      ffma2(acc, cs[k], lds_f2<k * N * 8 + HI>(__byte_perm((k & 1) ? o1 : e1, base, 0x7650 | (k >> 1))));
    });
  } else {
    const int sh = 16 * (a & 1);
    const uint32_t x0 = w[0] >> sh, x1 = w[1] >> sh;
    const uint32_t m00 = (x0 << 3) & 0x1818u, m01 = (x0 << 1) & 0x1818u, m02 = (x0 >> 1) & 0x1818u, m03 = (x0 >> 3) & 0x1818u;
    const uint32_t m10 = (x1 << 3) & 0x1818u, m11 = (x1 << 1) & 0x1818u, m12 = (x1 >> 1) & 0x1818u, m13 = (x1 >> 3) & 0x1818u;
    static_for<0, 8>([&](auto ik) {
      constexpr int k = decltype(ik)::v;
      const uint32_t s0 = (k & 3) == 0 ? m00 : ((k & 3) == 1 ? m01 : ((k & 3) == 2 ? m02 : m03));
      const uint32_t s1 = (k & 3) == 0 ? m10 : ((k & 3) == 1 ? m11 : ((k & 3) == 2 ? m12 : m13));
      ffma2(acc, cs[k], lds_f2<k * N * 8>(__byte_perm(s0, base, 0x7650 | (k >> 2))));
      ffma2(acc, cs[k], lds_f2<k * N * 8 + HI>(__byte_perm(s1, base, 0x7650 | (k >> 2))));
    });
  }
}

// FULL = the CTA owns a complete group of G heads (the common case: H % G == 0) -> no per-item head checks.
template <int BITS, bool FULL>
__global__ void __launch_bounds__(KCfg<BITS>::kThreads, 1) k_scores_kernel(const KParams p) {
  using C = KCfg<BITS>;
  constexpr int N = C::N, W = C::W, G = C::G, TT = C::TT, NRW = C::NRW;
  constexpr int PD = (BITS == 4) ? 8 : 4;   // register prefetch distance in work items (G % PD == 0)
  extern __shared__ unsigned char smem_raw[];
  // table base must be 256-byte aligned (the low address byte carries code*8)
  unsigned char* smem = smem_raw + ((256u - (smem_u32(smem_raw) & 255u)) & 255u);
  float2* s_tab = reinterpret_cast<float2*>(smem);                  // [G][128][N]
  float* s_q = reinterpret_cast<float*>(s_tab + G * kHeadDim * N);   // [G][128]

  const int tid = threadIdx.x;
  const uint64_t pol_stream = policy_evict_first(), pol_keep = policy_evict_last();
  const int h0 = blockIdx.y * G;
  const int nh = FULL ? G : min(G, p.H - h0);

  // ---- premultiplied tables T[hl][c][code] = (LUT*q[c], s_c*LUT*q[c^64]) -----------------------------------------
  for (int i = tid; i < nh * kHeadDim; i += C::kThreads) s_q[i] = p.q[(int64_t)h0 * kHeadDim + i];
  __syncthreads();
  for (int i = tid; i < G * kHeadDim * N; i += C::kThreads) {
    float2 e = make_float2(0.f, 0.f);   // heads past nh: zero tables (their items still run, results are dropped)
    if (i < nh * kHeadDim * N) {
      const int hc = i / N;             // hl*128 + c
      const int c = hc & (kHeadDim - 1);
      const float l = p.lut[((int64_t)h0 * kHeadDim) * N + i];
      const float qa = s_q[hc];
      const float qb = s_q[hc ^ kHalf];  // (c+64)%128 within the same head
      e = make_float2(l * qa, (c < kHalf) ? (l * qb) : -(l * qb));
    }
    s_tab[i] = e;
  }
  __syncthreads();
  const uint32_t tab0 = smem_u32(s_tab);

  // The CTA walks its token range [t_begin, t_limit) (a multiple of 32 tokens, cut so that every SM gets an equal
  // share) in tiles of TT tokens; a thread's work items are linearised as (tile, chunk a = 0..7, head hl = 0..G-1);
  // the packed words of item i+PD are loaded into a rotating register buffer while item i computes, the rope
  // values of the next chunk likewise.  A warp whose 32 tokens lie past the range skips the (last) tile, so a
  // partial tile costs only its live warps.
  const int64_t t_begin = (int64_t)blockIdx.x * p.range;
  const int64_t t_limit = min(p.L, t_begin + p.range);   // tokens this CTA may touch
  if (t_begin >= t_limit) return;
  const uint32_t pitch = (uint32_t)p.Lmax * 4u;      // row pitch in bytes (host checks Lmax < 2^30)
  const unsigned char* cb0 = reinterpret_cast<const unsigned char*>(p.cache + (int64_t)h0 * W * p.Lmax);

  // pointers of the current / next tile's column for this thread, and whether those columns exist
  const unsigned char* src_cur = cb0 + (t_begin + tid) * 4;
  bool ok_cur = (t_begin + tid) < t_limit;

  uint32_t wq[PD][NRW];   // rotating prefetch buffer (compile-time indices only)
#pragma unroll
  for (int d = 0; d < PD; ++d)
#pragma unroll
    for (int i = 0; i < NRW; ++i) wq[d][i] = 0;
  auto fetch = [&](uint32_t* dst, const unsigned char* base, bool ok, int a, int hl) {
    if (ok && (FULL || hl < nh)) {   // heads past nh do not exist in the cache: never touch them
#pragma unroll
      for (int i = 0; i < NRW; ++i)
        dst[i] = ld_stream_u32(reinterpret_cast<const uint32_t*>(
                                   base + (uint64_t)(uint32_t)(hl * W + chunk_word_row<BITS>(a, i)) * pitch), pol_stream);
    }
  };
  auto load_cs = [&](float2* dst, const int64_t t, int a) {
    if (t < t_limit) {
      const float2* rp = p.rope + (t + p.pos_offset) + (int64_t)(8 * a) * p.rope_npos;
#pragma unroll
      for (int k = 0; k < 8; ++k) dst[k] = ld_keep_f2(rp + (int64_t)k * p.rope_npos, pol_keep);
    }
  };

  // prologue: first PD items (chunk 0, heads 0..PD-1), rope values of chunk 0
  static_for<0, PD>([&](auto id) { constexpr int d = decltype(id)::v; fetch(wq[d], src_cur, ok_cur, 0, d); });
  float2 cs[8], csn[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { cs[k] = make_float2(0.f, 0.f); csn[k] = make_float2(0.f, 0.f); }
  load_cs(cs, t_begin + tid, 0);

  for (int64_t tb = t_begin; tb < t_limit; tb += TT) {
    const int64_t t = tb + tid;
    const bool live = t < t_limit;
    const unsigned char* src_nxt = src_cur + TT * 4;
    const bool ok_nxt = (t + TT) < t_limit;
    if (tb + (tid & ~31) < t_limit) {   // warp-uniform
    float2 acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = make_float2(0.f, 0.f);

    for (int a = 0; a < 8; ++a) {
      // rope values of the next chunk (next tile's chunk 0 after the last one) travel while this chunk computes
      load_cs(csn, a == 7 ? t + TT : t, (a + 1) & 7);
      // prefetch targets of this chunk's items: same chunk (hl+PD < G) or the next chunk / next tile's chunk 0
      const unsigned char* src_w = (a == 7) ? src_nxt : src_cur;
      const bool ok_w = (a == 7) ? ok_nxt : ok_cur;
      const int a_w = (a + 1) & 7;
      static_for<0, G>([&](auto ig) {
        constexpr int hl = decltype(ig)::v;
        uint32_t w[NRW];
#pragma unroll
        for (int i = 0; i < NRW; ++i) w[i] = wq[hl % PD][i];
        if constexpr (hl + PD < G) fetch(wq[hl % PD], src_cur, ok_cur, a, hl + PD);
        else fetch(wq[hl % PD], src_w, ok_w, a_w, hl + PD - G);
        // no per-thread guard: lanes past the range (and heads past nh) compute on zero / stale inputs and are dropped at the store
        k_item<BITS>(w, a, tab0 + (uint32_t)hl * (kHeadDim * N * 8) + (uint32_t)a * (8 * N * 8), cs, acc[hl]);
      });
#pragma unroll
      for (int k = 0; k < 8; ++k) cs[k] = csn[k];
    }

    // ---- write back: this thread owns column t of the score matrix for the CTA's heads ---------------------------
#pragma unroll
    for (int hl = 0; hl < G; ++hl) {
      if (live && hl < nh) {
        float* o = p.out + (int64_t)(h0 + hl) * p.out_stride + t;
        *o = (acc[hl].x + acc[hl].y) + *o;
      }
    }
    }
    src_cur = src_nxt;
    ok_cur = ok_nxt;
  }
}

// ------------------------------------------------------------------------------------------------------------
// Outlier scatter (replaces SPMV_ATOMIC_ROPE_BALANCED, quant_cuda_kernel.cu:472-521).  Runs before the dense
// kernel, which then adds its own sum into `out`.
// ------------------------------------------------------------------------------------------------------------
constexpr int kOutThreads = 256;

// theta_j of rotary row j, and (cos, sin)(theta_j * pos): the reference's expressions (quant_cuda_kernel.cu:3081 and
// 3123-3126).  The rope table is built from them and the outlier pass evaluates them, so both hold the same bits.
// rope_row_theta runs once per row, not per entry: out of line, its powf leaves the outlier pass's register allocation
// alone (inlined, ptxas puts cosf / sinf's slow-path reduction buffer of the one-sequence MHA pass in local memory).
__device__ __noinline__ float rope_row_theta(float rope_theta, int j) {
  const int headdim = kHeadDim;
  const int headdim2 = headdim / 2;
  return powf(rope_theta, (-2 * __int2float_rd(j % headdim2) / __int2float_rd(headdim)));
}
__device__ __forceinline__ float2 rope_cos_sin(float theta, int pos) {
  const float c = cosf(theta * pos);
  const float s = sinf(theta * pos);
  return make_float2(c, s);
}
// The frequency of rotary row j: f[j] for a frequency vector (scaled or length-dependent rotary), else theta_j of base
// theta.  Every table entry and every factor the outlier pass computes is (cos, sin)(f_j * pos) * a of this value (a =
// 1 for theta, where the product is exact), so the two hold the same bits.
__device__ __forceinline__ float rotary_row_freq(float theta, const float* __restrict__ f, int j) {
  return f != nullptr ? f[j] : rope_row_theta(theta, j);
}

// thread = one (token, outlier slot) entry.  cos/sin come from the RoPE table (bit-identical to the reference's
// cosf/sinf(theta*pos)); entries of one (token, head) are adjacent (rows are sorted by channel), so a warp-level
// segmented sum leaves ~1 atomic per (token, head) instead of the reference's one per entry.
__global__ void __launch_bounds__(kOutThreads) k_outlier_kernel(
    const float* __restrict__ q, const float* __restrict__ outliers, const int32_t* __restrict__ outlier_idx,
    float* __restrict__ out, int64_t out_stride, int64_t L, int H, int n_out, const float2* __restrict__ rope,
    int64_t rope_npos, int pos_offset, float scale) {
  const int64_t e = (int64_t)blockIdx.x * kOutThreads + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int64_t total = L * n_out;
  float contrib = 0.f;
  int64_t key = -1 - lane;   // unique negative keys for idle lanes (never merge)
  int64_t t = 0;
  int h = 0;
  if (e < total) {
    t = e / n_out;
    const float v = outliers[e];
    const int col = outlier_idx[e];
    h = col >> 7;
    const int c = col & (kHeadDim - 1);
    key = t * 64 + h;
    if (v != 0.f) {   // pads / non-outliers contribute exactly 0 in the reference too
      const float2 cs = rope[(int64_t)(c & (kHalf - 1)) * rope_npos + t + pos_offset];
      const float sign = (c < kHalf) ? 1.f : -1.f;
      float dot = v * cs.x * __ldg(q + col);            // same operation order as DK.cu:513-515
      dot += sign * v * cs.y * __ldg(q + (col ^ kHalf));
      contrib = dot * scale;
    }
  }
  // segmented sum over runs of equal keys (runs are contiguous in lane order)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v2 = __shfl_down_sync(0xffffffffu, contrib, o);
    const int64_t k2 = __shfl_down_sync(0xffffffffu, key, o);
    if (lane + o < 32 && k2 == key) contrib += v2;
  }
  const int64_t kprev = __shfl_up_sync(0xffffffffu, key, 1);
  const bool leader = (lane == 0) || (kprev != key);
  if (leader && e < total && contrib != 0.f) atomicAdd(out + (int64_t)h * out_stride + t, contrib);
}

// Persistent form (default).  ncu on the kernel above: load/store data path 75 % busy -- per ENTRY one scattered
// 8-byte rope read plus TWO scattered reads of q.  Here CTAs are persistent and keep (q[c], q[c^64]) for all channels
// in shared memory (one 8-byte shared read per entry instead of two scattered global ones); the rotary factors are
// computed (direct, k_out_direct) or gathered from the table.
// Alternatives considered (DESIGN.md section 4.1): a second, token-major copy of the rope table read with coalesced
// row loads + shuffles instead of the gather (it loads rows for the zero-valued pads too and adds 8 shuffles per
// entry); gathering every entry's rotary factors from the rope table (slower than computing them, even at 32K);
// accumulating into a per-CTA [H][256-token] shared tile with coalesced write-out
// instead of global atomics (shared-memory fp32 atomics are compare-and-swap loops).
//
// GQA (grp query heads per KV head, H = query heads): an entry's channel is a KV channel; it is read once and adds its
// contribution to each of the grp query heads of its KV head, one segmented sum per group member (keys token * 64 +
// query head: the entries of one (token, KV head) are adjacent, so each member's runs stay contiguous).
//
// BATCH: sequence b = blockIdx.y of a batched attend: q [B][H][128], outlier rows `b_rows` entries after sequence b-1's,
// score rows `b_out` floats after sequence b-1's, length len_dev[b].  BATCH = false ignores b_out / b_rows.
// PAGED (with BATCH, b_rows = 0): the outlier rows are a page pool; logical entry e = t * n_out + k of sequence b is
// read from row page_of(b, t) * P + t % P, and the length is also capped at npages[b] * P.  Others ignore `pg`.
constexpr int kOutPersThreads = 512;
constexpr size_t kOutThetaBytes = kHalf * sizeof(float);   // dynamic shared memory past the q table: s_th
//
// Rotary factors: rotary row j turns at f_j = rotary_row_freq(rope_theta, rope_freq, j) -- theta_j of rope_theta when
// rope_freq is null, else rope_freq[j] (scaled or length-dependent frequencies, DESIGN.md sections 4.13, 4.14) -- and
// the factors are (cos, sin)(f_j * pos) * attn (attn = 1 for theta), as rope_table_kernel builds the table.  direct:
// the pass computes them (past CUDART_TRIG_PLOSS_F it gathers them); otherwise every factor comes from the table.
// With BATCH, sequence b's table and frequency vector sit b * rope_bstride entries and b * freq_bstride floats after
// sequence 0's: 64 * rope_npos and 64 for a rotation per sequence, 0 for one shared by the batch.
template <bool GQA, bool BATCH, bool PAGED>
__global__ void __launch_bounds__(kOutPersThreads) k_outlier_pers_kernel(
    const float* __restrict__ q, const float* __restrict__ outliers, const int32_t* __restrict__ outlier_idx,
    float* __restrict__ out, int64_t stride_h, int64_t stride_t, int64_t L, int H, int n_out,
    const float2* __restrict__ rope, int64_t rope_npos, int pos_offset, float scale,
    const int64_t* __restrict__ len_dev, int64_t len_add, const uint32_t* __restrict__ rope_h, float rope_theta,
    const float* __restrict__ rope_freq, float attn, bool direct, int grp, const int64_t b_out, const int64_t b_rows,
    const PageRef pg, const int64_t rope_bstride, const int freq_bstride) {
  extern __shared__ float2 s_qq[];                       // [H*128] = (q[c], q[c^64]), query heads
  float* const s_th = reinterpret_cast<float*>(s_qq + H * kHeadDim);   // [64]: f_j of rotary row j (direct)
  if constexpr (BATCH) {
    const int b = blockIdx.y;
    q += (int64_t)b * H * kHeadDim;
    outliers += b * b_rows; outlier_idx += b * b_rows;
    out += b * b_out;
    len_dev += b;
    rope += b * rope_bstride;
    if (rope_freq != nullptr) rope_freq += b * freq_bstride;
  }
  if (len_dev != nullptr) {                              // device-resident length: L is the cap the grid was sized for
    const int64_t l = *len_dev + len_add;
    L = l < 0 ? 0 : (l < L ? l : L);
  }
  if constexpr (PAGED) {
    const int64_t cap = page_cap(pg, blockIdx.y);
    L = L < cap ? L : cap;
  }
  const uint32_t total = (uint32_t)(L * n_out);          // host checks L * n_out < 2^31
  const int tid = threadIdx.x, lane = tid & 31;
  for (int i = tid; i < H * kHeadDim; i += kOutPersThreads) s_qq[i] = make_float2(q[i], q[i ^ kHalf]);
  if (direct && tid < kHalf) s_th[tid] = rotary_row_freq(rope_theta, rope_freq, tid);
  __syncthreads();
  const uint32_t stride = gridDim.x * kOutPersThreads;
  // outlier rows are read once: evict them first, so that the score rows the atomics add into (just cleared) stay in L2
  const uint64_t pol_keep = policy_evict_last(), pol_stream = policy_evict_first();
  for (uint32_t base = blockIdx.x * kOutPersThreads + (tid & ~31); base < total; base += stride) {
    const uint32_t e = base + lane;
    float contrib = 0.f;
    int key = -1 - lane;   // unique negative keys for idle lanes (never merge)
    uint32_t t = 0;
    int h = 0;
    float gv = 0.f, gsign = 0.f;                       // GQA: the entry's value and rotation, applied per group member
    float2 gcs = make_float2(0.f, 0.f);
    int gc = 0;
    if (e < total) {
      t = e / (uint32_t)n_out;
      float v;
      int col;
      if constexpr (PAGED) {
        const int64_t pe = ((int64_t)page_of(pg, blockIdx.y, (int)t) * pg.P + t % (uint32_t)pg.P) * n_out + (e - t * (uint32_t)n_out);
        v = __uint_as_float(ld_stream_u32(reinterpret_cast<const uint32_t*>(outliers + pe), pol_stream));
        col = (int)ld_stream_u32(reinterpret_cast<const uint32_t*>(outlier_idx + pe), pol_stream);
      } else {
        v = __uint_as_float(ld_stream_u32(reinterpret_cast<const uint32_t*>(outliers + e), pol_stream));
        col = (int)ld_stream_u32(reinterpret_cast<const uint32_t*>(outlier_idx + e), pol_stream);
      }
      h = col >> 7;
      const int c = col & (kHeadDim - 1);
      key = (int)(t * 64u) + h;                          // t < 2^25
      if (v != 0.f) {   // pads / non-outliers contribute exactly 0 in the reference too
        float2 cs;
        if (direct) {
          // the table builder's own expressions (same device functions, same arguments: bit-identical values) cost
          // less than a scattered 8-byte gather, which past L2-sized tables is a 32-byte DRAM sector.  Past
          // CUDART_TRIG_PLOSS_F, cosf / sinf leave their fast argument reduction for a local-memory one that stalls
          // the whole warp; those arguments (rows j < 2 at 128K, j < 16 at 1M) come from the table, whose few rows
          // stay in L2.
          const int j = c & (kHalf - 1), pos = (int)t + pos_offset;
          const float th = s_th[j];
          const bool fast = th * pos <= CUDART_TRIG_PLOSS_F;
          if (fast) cs = rope_cos_sin(th, pos);
          else cs = ld_keep_f2(rope + (int64_t)j * rope_npos + pos, pol_keep);
          const float m = fast ? attn : 1.f;   // the table's entries already carry attn (a product with 1 is exact)
          cs = make_float2(cs.x * m, cs.y * m);
        } else if (rope_h != nullptr) {   // fp16 mode: the half2 table the dense kernel streams (half the bytes per gather)
          uint32_t u;
          asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(u)
                       : "l"(rope_h + (int64_t)(c & (kHalf - 1)) * rope_npos + t + pos_offset), "l"(pol_keep));
          cs = __half22float2(*reinterpret_cast<const __half2*>(&u));
        } else {
          cs = ld_keep_f2(rope + (int64_t)(c & (kHalf - 1)) * rope_npos + t + pos_offset, pol_keep);
        }
        const float sign = (c < kHalf) ? 1.f : -1.f;
        if constexpr (GQA) {
          gv = v; gsign = sign; gcs = cs;
        } else {
          const float2 qq = s_qq[col];
          float dot = v * cs.x * qq.x;            // same operation order as DK.cu:513-515
          dot += sign * v * cs.y * qq.y;
          contrib = dot * scale;
        }
      }
      gc = c;
    }
    // segmented sum over runs of equal keys, one atomic per run, into score row hq
    auto reduce_add = [&](float v, const int k, const int hq) {
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float v2 = __shfl_down_sync(0xffffffffu, v, o);
        const int k2 = __shfl_down_sync(0xffffffffu, k, o);
        if (lane + o < 32 && k2 == k) v += v2;
      }
      const int kprev = __shfl_up_sync(0xffffffffu, k, 1);
      const bool leader = (lane == 0) || (kprev != k);
      if (leader && e < total && v != 0.f) atomicAdd(out + (int64_t)hq * stride_h + (int64_t)t * stride_t, v);
    };
    if constexpr (GQA) {
      for (int j = 0; j < grp; ++j) {
        const int hq = h * grp + j;
        float cj = 0.f;
        if (gv != 0.f) {
          const float2 qq = s_qq[hq * kHeadDim + gc];
          float dot = gv * gcs.x * qq.x;
          dot += gsign * gv * gcs.y * qq.y;
          cj = dot * scale;
        }
        reduce_add(cj, e < total ? (int)(t * 64u) + hq : key, hq);
      }
    } else {
      reduce_add(contrib, key, h);
    }
  }
}

static int k_out_impl_table() {   // KVQ_KOUT_IMPL=table selects the non-persistent gather form for A/B runs
  static int v = -1;
  if (v < 0) { const char* e = getenv("KVQ_KOUT_IMPL"); v = (e && e[0] == 't') ? 1 : 0; }
  return v;
}

// Whether the outlier scatter computes its rotary factors (rope_row_theta / rope_cos_sin, bit-identical to the table)
// instead of gathering them from the rope table.  Exact mode: at every length (one layer of 7B at 3 bits on an H100:
// 15.4 against 20.0 us at 32K, DESIGN.md section 5).  fp16 mode (half_table): its half2 gather up to 64K positions
// (64 pairs x 8 bytes x 64K = 32 MB of fp32 table, about what stays in the 50 MB L2 next to the streams), the exact
// factors beyond.  KVQ_KOUT_DIRECT_NPOS=N overrides both: compute beyond N positions, gather up to N.
static bool k_out_direct(int64_t n_positions, bool half_table) {
  static int64_t thr = -2;
  if (thr == -2) { const char* e = getenv("KVQ_KOUT_DIRECT_NPOS"); thr = e ? atoll(e) : -1; }
  return n_positions > (thr >= 0 ? thr : (half_table ? 64 * 1024 : 0));
}

static int set_k_outlier_smem(size_t smem, bool gqa, bool batch, bool paged) {
  static size_t smem_set_dev[6][64];   // per kernel and device: largest dynamic shared memory opted in so far (0 = 48 KiB)
  int dev_idx = 0;
  cudaGetDevice(&dev_idx);
  size_t& smem_set = smem_set_dev[gqa + 2 * (batch + paged)][dev_idx & 63];
  if (smem_set == 0) smem_set = 48 * 1024;
  if (smem > smem_set) {
    const cudaError_t e = with_flavour(gqa, batch, paged, [&](auto GQA, auto BATCH, auto PAGED) {
      return cudaFuncSetAttribute(k_outlier_pers_kernel<GQA(), BATCH(), PAGED()>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    });
    if (e != cudaSuccess) return (int)e;
    smem_set = smem;
  }
  return 0;
}

// persistent outlier CTAs along x for `total` entries per sequence: a few per SM (fewer when the q table is large),
// that allowance shared among the nseq sequences of a batch
static unsigned k_outlier_grid(int64_t total, size_t smem, int nseq) {
  const int64_t want = (total + kOutPersThreads - 1) / kOutPersThreads;
  const int per_sm = smem > 56 * 1024 ? 2 : 4;
  const int64_t cap = std::max<int64_t>(1, (int64_t)num_sms_cached() * per_sm / nseq);
  return (unsigned)std::max<int64_t>(1, std::min(want, cap));
}

// adds the outlier entries' contributions into the head-major score rows p.out
// p.H counts query heads, p.grp of them per KV head (the entries' channels are KV channels)
static int launch_k_outliers(const KParams& p, cudaStream_t st) {
  const bool gqa = p.grp > 1;
  const int64_t total = p.L * p.n_out;
  const size_t smem = (size_t)p.H * kHeadDim * sizeof(float2);
  if (k_out_impl_table() || smem > 100 * 1024 || total >= ((int64_t)1 << 31) || p.L >= ((int64_t)1 << 25)) {
    if (p.len_dev != nullptr || gqa) return KVQ_E_UNSUPPORTED;   // host length, MHA only
    const unsigned grid = (unsigned)((total + kOutThreads - 1) / kOutThreads);
    k_outlier_kernel<<<grid, kOutThreads, 0, st>>>(p.q, p.outliers, p.outlier_idx, p.out, p.out_stride, p.L, p.H,
                                                   p.n_out, p.rope, p.rope_npos, p.pos_offset, 1.f);
    KVQ_LAUNCH_CHECK();
    return 0;
  }
  const int rc = set_k_outlier_smem(smem + kOutThetaBytes, gqa, false, false);
  if (rc != 0) return rc;
  const unsigned grid = k_outlier_grid(total, smem, 1);
  const bool direct = k_out_direct(p.L + p.pos_offset, p.rope_h != nullptr);
  with_flavour(gqa, false, false, [&](auto GQA, auto BATCH, auto PAGED) {
    k_outlier_pers_kernel<GQA(), BATCH(), PAGED()><<<grid, kOutPersThreads, smem + kOutThetaBytes, st>>>(
        p.q, p.outliers, p.outlier_idx, p.out, p.out_stride, 1, p.L, p.H, p.n_out, p.rope, p.rope_npos, p.pos_offset, 1.f,
        p.len_dev, p.len_add, p.rope_h, p.theta, p.freq ? p.rope_freq : nullptr, p.freq ? p.attn : 1.f, direct,
        gqa ? p.grp : 1, 0, 0, PageRef{}, 0, 0);
  });
  KVQ_LAUNCH_CHECK();
  return 0;
}

// rope table [B][64][n_pos]: entry (j, p) = (cosf(f_j p) * attn, sinf(f_j p) * attn), f_j = rotary_row_freq(theta, f, j)
// -- the factors k_outlier_pers_kernel computes.  HALF: the same values rounded once to fp16 (half2 entries).
// Sequence b = blockIdx.z: its table and f follow b * 64 * n_pos entries and b * 64 floats after sequence 0's.
// st (the length-dependent rebuild, kvq_rope_len_update): sequence b writes positions [0, st[b][1]) of its table;
// null: every position.  grid = (x, 64, B).
template <bool HALF>
__global__ void rope_table_kernel(void* __restrict__ out, float theta, const float* __restrict__ f, float attn,
                                  int64_t n_pos, const int64_t* __restrict__ st) {
  const int j = blockIdx.y, b = blockIdx.z;
  const int64_t n = st != nullptr ? st[2 * b + 1] : n_pos;
  const float fj = rotary_row_freq(theta, f != nullptr ? f + (int64_t)b * kHalf : nullptr, j);
  const int64_t row = ((int64_t)b * kHalf + j) * n_pos;
  for (int64_t pos64 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pos64 < n; pos64 += (int64_t)gridDim.x * blockDim.x) {
    const float2 cs = rope_cos_sin(fj, (int)pos64);
    const float2 e = make_float2(cs.x * attn, cs.y * attn);
    if constexpr (HALF) {
      const __half2 h = __floats2half2_rn(e.x, e.y);
      static_cast<uint32_t*>(out)[row + pos64] = *reinterpret_cast<const uint32_t*>(&h);
    } else {
      static_cast<float2*>(out)[row + pos64] = e;
    }
  }
}

// the static tables of kvq_rope_table_build*: one shared table, every argument checked before anything is launched
static int rope_table_build(void* out, float theta, const float* freq, float attn, int64_t n_pos, void* stream,
                            bool half) {
  const dim3 grid((unsigned)((n_pos + 255) / 256 > 4096 ? 4096 : (n_pos + 255) / 256), kHalf);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (half) rope_table_kernel<true><<<grid, 256, 0, st>>>(out, theta, freq, attn, n_pos, nullptr);
  else rope_table_kernel<false><<<grid, 256, 0, st>>>(out, theta, freq, attn, n_pos, nullptr);
  KVQ_LAUNCH_CHECK();
  return 0;
}

// Length-dependent rotary frequencies (kvq_rope_len_update, DESIGN.md section 4.14).  Per sequence b: f_cur [b][64],
// st [b][2] = (key of the frequencies the table holds, positions the rebuild writes) and a table [b][64][npos] in the
// rope table layout.  s = one plus the last query position: s_host, or pos_offset + min(max(len_dev[b] + len_add, 0),
// L_cap).  Dynamic NTK (mode 0): s <= m_pos reads f_lo (the default vector, one key for the whole range); s > m_pos is
// HF's formula in double precision, rounded once to fp32, and a key per length.  LongRoPE (mode 1): f_lo (short) up
// to m_pos (original_max_position_embeddings), f_hi (long) above, one key each.  A rebuild writes the positions its key
// covers: [0, s) for a per-length key, [0, m_pos) or [0, npos) for a range key.  grid = B, block = 64.
constexpr int kRopeLenDynamic = 0;
__global__ void rope_len_prepare_kernel(int mode, double theta, double factor, int64_t m_pos, const float* __restrict__ f_lo,
                                        const float* __restrict__ f_hi, int64_t s_host, const int64_t* __restrict__ len_dev,
                                        int64_t len_add, int64_t L_cap, int pos_offset, float* __restrict__ f_cur,
                                        int64_t* __restrict__ st, int64_t npos) {
  const int b = blockIdx.x, j = threadIdx.x;
  int64_t s = s_host;
  if (len_dev != nullptr) {
    const int64_t l = len_dev[b] + len_add;
    s = pos_offset + (l < 0 ? 0 : (l < L_cap ? l : L_cap));
  }
  const bool above = s > m_pos;
  const bool per_len = mode == kRopeLenDynamic && above;
  float f;
  if (per_len) {   // base * ((factor * s / M) - (factor - 1)) ** (128 / 126), then 1 / base' ** (2j / 128)
    const double base = theta * pow(factor * (double)s / (double)m_pos - (factor - 1.0), 128.0 / 126.0);
    f = (float)(1.0 / pow(base, (double)(2 * j) / 128.0));
  } else {
    f = (above ? f_hi : f_lo)[j];
  }
  f_cur[(int64_t)b * kHalf + j] = f;
  if (j == 0) {
    const int64_t key = per_len ? s : (above ? 1 : 0);   // a per-length key is s > m_pos >= 1: never 0 or 1
    const int64_t end = per_len ? s : (above ? npos : m_pos);
    int64_t* sb = st + 2 * b;
    const bool rebuild = sb[0] != key;
    sb[0] = key;
    sb[1] = rebuild ? (end < npos ? end : npos) : 0;
  }
}

template <int BITS>
static int launch_k_scores(const KParams& p, cudaStream_t st) {
  using C = KCfg<BITS>;
  const size_t smem = 256 + (size_t)C::G * kHeadDim * C::N * sizeof(float2) + (size_t)C::G * kHeadDim * 4;
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(k_scores_kernel<BITS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(k_scores_kernel<BITS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  const int n_groups = (p.H + C::G - 1) / C::G;
  const int sms = num_sms_cached();
  const int64_t max_splits = sms / n_groups > 0 ? sms / n_groups : 1;
  KParams q = p;
  q.range = k_token_range(p.L, max_splits);
  const int64_t splits = (p.L + q.range - 1) / q.range;
  const dim3 grid((unsigned)splits, (unsigned)n_groups);
  if (p.H % C::G == 0) k_scores_kernel<BITS, true><<<grid, C::kThreads, smem, st>>>(q);
  else k_scores_kernel<BITS, false><<<grid, C::kThreads, smem, st>>>(q);
  KVQ_LAUNCH_CHECK();
  return 0;
}

// dense K scores of kvq_k_matvec: out += S
int k_scores_dispatch(int bits, const KParams& p, cudaStream_t st) {
  switch (bits) {
    case 4: return launch_k_scores<4>(p, st);
    case 3: return k_scores3_dispatch(p, st);
    case 2: return launch_k_scores<2>(p, st);
    default: return KVQ_E_BITS;
  }
}

// K side of the fused attend: outlier scatter straight into the head-major score buffer (cleared first), then the
// TMA-fed dense kernel folds it in: out = (partial + S) * scale.  rope_half == null: exact fp32 ratio form
// (kvq_kratio.cu); otherwise the fp16-table form (kvq_kfast.cu).
// GQA: Hq query heads, grp per KV head (exact ratio form only: rope_half must be null when grp > 1)
int k_scores_fused(const AttendCall& c, const AttendScratch& s) {
  int accumulate = 0;
  if (c.k_outliers != nullptr) {
    KParams p{};
    p.len_dev = c.len_dev; p.len_add = c.len_add;
    p.q = c.q; p.out = s.scores; p.rope = reinterpret_cast<const float2*>(c.rope);
    p.Lmax = c.Lmax; p.L = c.L; p.out_stride = s.stride; p.rope_npos = c.rope_npos;
    p.H = c.Hq; p.n_out = c.n_out; p.pos_offset = c.pos_offset; p.theta = c.theta;
    p.outliers = c.k_outliers; p.outlier_idx = c.k_outlier_idx;
    p.rope_h = static_cast<const uint32_t*>(c.rope_half); p.grp = c.grp();
    p.freq = c.freq; p.rope_freq = c.rope_freq; p.attn = c.attn_factor;
    cudaError_t e = cudaMemset2DAsync(s.scores, sizeof(float) * (size_t)s.stride, 0, sizeof(float) * (size_t)c.L, (size_t)c.Hq, c.stream);
    if (e != cudaSuccess) return (int)e;
    const int rc = launch_k_outliers(p, c.stream);
    if (rc != 0) return rc;
    accumulate = 1;
  }
  return (c.rope_half == nullptr) ? k_ratio_dispatch(c, s, accumulate) : k_fast_dispatch(c, s, accumulate);
}

// Score rows [h][0, L_eff) of every sequence of a batch cleared before the outlier pass adds into them (L_eff =
// min(len_dev[b] + len_add, L_cap): nothing past a sequence's length is read).  grid = (x, H, B).
__global__ void k_batch_zero_kernel(float* __restrict__ scores, int64_t stride, int64_t bstride, const int64_t* __restrict__ len_dev,
                                    int64_t len_add, int64_t L_cap) {
  const int h = blockIdx.y, b = blockIdx.z;
  const int64_t l = len_dev[b] + len_add;
  const int64_t L = l < 0 ? 0 : (l < L_cap ? l : L_cap);
  float* row = scores + b * bstride + (int64_t)h * stride;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < L; t += (int64_t)gridDim.x * blockDim.x) row[t] = 0.f;
}

// K side of the batched attend (kvq_attend_batch): exact fp32 ratio form, one launch per kernel for all B sequences.
// q [B][H][128]; cache [B][Hkv*W][Lmax]; outlier rows [B][Lmax][n_out]; scores, gmax and qtab of sequence b at
// b * bstride floats (sequence b's scratch block); the grids are sized for the cap c.L, each CTA reads its own length.
// c.pg != nullptr: the paged batch (kvq_attend_paged), cache and outlier rows page pools; the score clear works on
// logical token indices in the scratch and is the same.
int k_scores_batch(const AttendCall& c, const AttendScratch& s) {
  const int H = c.Hq, B = c.B, grp = c.grp();
  int accumulate = 0;
  if (c.k_outliers != nullptr) {
    const size_t smem = (size_t)H * kHeadDim * sizeof(float2);
    if (c.L * c.n_out >= ((int64_t)1 << 31) || c.L >= ((int64_t)1 << 25)) return KVQ_E_UNSUPPORTED;
    k_batch_zero_kernel<<<dim3((unsigned)std::min<int64_t>((c.L + 2047) / 2048, 64), H, B), 256, 0, c.stream>>>(
        s.scores, s.stride, s.bstride, c.len_dev, c.len_add, c.L);
    KVQ_LAUNCH_CHECK();
    const int rc = set_k_outlier_smem(smem + kOutThetaBytes, grp > 1, true, c.pg != nullptr);
    if (rc != 0) return rc;
    const dim3 grid(k_outlier_grid(c.L * c.n_out, smem, B), (unsigned)B);
    const bool direct = k_out_direct(c.L + c.pos_offset, false);
    const int64_t b_rows = c.pg != nullptr ? 0 : c.Lmax * c.n_out;   // a pool has no per-sequence row block
    const float2* rope = reinterpret_cast<const float2*>(c.rope);
    const PageRef pg = c.pg != nullptr ? *c.pg : PageRef{};
    with_flavour(grp > 1, true, c.pg != nullptr, [&](auto GQA, auto BATCH, auto PAGED) {
      k_outlier_pers_kernel<GQA(), BATCH(), PAGED()><<<grid, kOutPersThreads, smem + kOutThetaBytes, c.stream>>>(
          c.q, c.k_outliers, c.k_outlier_idx, s.scores, s.stride, 1, c.L, H, c.n_out, rope, c.rope_npos, c.pos_offset,
          1.f, c.len_dev, c.len_add, nullptr, c.theta, c.freq ? c.rope_freq : nullptr, c.freq ? c.attn_factor : 1.f,
          direct, grp, s.bstride, b_rows, pg, c.rope_per_seq ? kHalf * c.rope_npos : 0, c.rope_per_seq ? kHalf : 0);
    });
    KVQ_LAUNCH_CHECK();
    accumulate = 1;
  }
  return k_ratio_dispatch(c, s, accumulate);
}

}  // namespace kvq

using namespace kvq;

extern "C" {

int kvq_rope_table_build(float* rope_cos_sin, float theta, int64_t n_pos, void* stream) {
  if (!rope_cos_sin) return KVQ_E_NULL;
  if (n_pos <= 0 || n_pos > (int64_t)1 << 30) return KVQ_E_SHAPE;
  return rope_table_build(rope_cos_sin, theta, nullptr, 1.f, n_pos, stream, false);
}

int kvq_rope_table_build_half(void* rope_half, float theta, int64_t n_pos, void* stream) {
  if (!rope_half) return KVQ_E_NULL;
  if (n_pos <= 0 || n_pos > (int64_t)1 << 30) return KVQ_E_SHAPE;
  return rope_table_build(rope_half, theta, nullptr, 1.f, n_pos, stream, true);
}

// scaled tables: the frequency vector is read on the device
static int rope_table_freq_build(void* out, const float* freq, float attn_factor, int64_t n_pos, void* stream, bool half) {
  if (!out || !freq) return KVQ_E_NULL;
  if (n_pos <= 0 || n_pos > (int64_t)1 << 30 || !(attn_factor > 0.f && attn_factor < INFINITY)) return KVQ_E_SHAPE;
  return rope_table_build(out, 0.f, freq, attn_factor, n_pos, stream, half);
}

int kvq_rope_table_build_freq(float* rope_cos_sin, const float* freq, float attn_factor, int64_t n_pos, void* stream) {
  return rope_table_freq_build(rope_cos_sin, freq, attn_factor, n_pos, stream, false);
}

int kvq_rope_table_build_freq_half(void* rope_half, const float* freq, float attn_factor, int64_t n_pos, void* stream) {
  return rope_table_freq_build(rope_half, freq, attn_factor, n_pos, stream, true);
}

int kvq_rope_len_update(int mode, const double* params, int64_t m_pos, const float* f_lo, const float* f_hi,
                        float attn_factor, int64_t s, const int64_t* len_dev, int64_t len_add, int64_t L_cap,
                        int pos_offset, int B, float* f_cur, int64_t* state, float* table, int64_t npos, void* stream) {
  if (!params || !f_lo || !f_cur || !state || !table || (mode == 1 && !f_hi)) return KVQ_E_NULL;
  if ((mode != 0 && mode != 1) || m_pos <= 0 || npos <= 0 || npos > (int64_t)1 << 30 || B < 1 || B > 256) return KVQ_E_SHAPE;
  const double theta = params[0], factor = params[1];
  if (!(theta > 1.0 && theta < INFINITY) || (mode == 0 && !(factor > 0.0 && factor < INFINITY))) return KVQ_E_SHAPE;
  if (!(attn_factor > 0.f && attn_factor < INFINITY)) return KVQ_E_SHAPE;
  if (len_dev == nullptr ? (B != 1 || s < 0 || s > npos) : (L_cap < 0 || pos_offset < 0 || pos_offset + L_cap > npos))
    return KVQ_E_SHAPE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rope_len_prepare_kernel<<<B, kHalf, 0, st>>>(mode, theta, factor, m_pos, f_lo, f_hi, s, len_dev, len_add, L_cap,
                                                pos_offset, f_cur, state, npos);
  KVQ_LAUNCH_CHECK();
  // a second launch: no rebuild CTA reads a sequence's decision while the prepare CTA writes it
  const dim3 grid((unsigned)((npos + 255) / 256 > 16 ? 16 : (npos + 255) / 256), kHalf, (unsigned)B);
  rope_table_kernel<false><<<grid, 256, 0, st>>>(table, 0.f, f_cur, attn_factor, npos, state);
  KVQ_LAUNCH_CHECK();
  return 0;
}

int kvq_k_matvec(int bits, const float* q, const int32_t* cache, float* mul, const float* lut, int B, int H,
                 int64_t Lmax, int64_t L, const float* outliers, const int32_t* outlier_idx, int n_out,
                 const float* rope_cos_sin, int64_t rope_npos, float theta, int pos_offset, void* stream) {
  if (!q || !cache || !mul || !lut || !rope_cos_sin) return KVQ_E_NULL;
  if (B <= 0 || H <= 0 || L < 0 || L > Lmax || pos_offset < 0 || Lmax >= ((int64_t)1 << 30)) return KVQ_E_SHAPE;
  if ((outliers == nullptr) != (outlier_idx == nullptr)) return KVQ_E_NULL;
  if (outliers && (B != 1 || n_out <= 0)) return KVQ_E_SHAPE;  // reference: sparse part is batch-1 only (DK.cu:3605)
  if (outliers && H > 64) return KVQ_E_SHAPE;                  // the outlier scatter keys its segments on token * 64 + head
  if (rope_npos < L + pos_offset) return KVQ_E_SHAPE;
  if (L == 0) return 0;
  for (int b = 0; b < B; ++b) {
    KParams p{};
    p.q = q + (int64_t)b * H * kHeadDim;
    p.cache = reinterpret_cast<const uint32_t*>(cache);
    p.out = mul + (int64_t)b * H * L;
    p.lut = lut;
    p.outliers = outliers;
    p.outlier_idx = outlier_idx;
    p.rope = reinterpret_cast<const float2*>(rope_cos_sin);
    p.Lmax = Lmax; p.L = L; p.out_stride = L; p.rope_npos = rope_npos;
    p.H = H; p.n_out = n_out; p.pos_offset = pos_offset; p.theta = theta;
    if (outliers != nullptr) {
      const int rc0 = launch_k_outliers(p, static_cast<cudaStream_t>(stream));
      if (rc0 != 0) return rc0;
    }
    const int rc = k_scores_dispatch(bits, p, static_cast<cudaStream_t>(stream));
    if (rc != 0) return rc;
  }
  return 0;
}

}  // extern "C"
