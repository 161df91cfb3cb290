// kvquant_b200 -- Q.K^T decode matvec of the fused attend, exact fp32 "ratio" form (the default of kvq_attend).
//
// Replaces (reference deployment/kvquant/quant_cuda_kernel.cu):
//   VecQuant{4,3,2}MatMulKernelNUQPerChannelTransposedRopeMHABatchedFusedOpt   3040-3209, 3692-4115, 4747-4996
//
//   S[h,t] = sum_c LUT[h,c,code(h,c,t)] * (cos(th_j p) q[h,c] + s_c sin(th_j p) q[h,(c+64)%128]),  j = c % 64, p = t + off
//
// Round 1's kernels looked an 8-byte entry (LUT q_c, s_c LUT q_{c^64}) up per element: two shared-memory wavefronts
// per warp lookup, and that data path was 78-86 % busy.  An fp16 entry halves the wavefronts (kvq_kfast.cu) but costs
// precision: 1.4e-3 .. 1.7e-3 at 128K tokens, above north_star's 1e-3.  This form gets the single wavefront without
// giving up fp32:
//
//     LUT (q_c cos + s_c q_{c^64} sin)  =  (LUT q_c) * (cos + r_c sin),     r_c = s_c q_{c^64} / q_c
//
//   * the table holds ONE fp32 per (channel, code), T[h][c][code] = LUT * q_c: a 4-byte lookup, one wavefront;
//   * r_c depends on (head, channel) only: 128 floats per head next to the table, fetched four at a time by a
//     broadcast LDS.128 (q_c = 0 is replaced by +-1e-30: the product LUT q_c r_c = LUT s_c q_{c^64} is unchanged and
//     stays finite);
//   * per element: PRMT (3-bit: SHF + LOP3), LDS.32, FFMA g = r sin + cos (independent of the lookup, hides its
//     latency), FFMA acc += T g  -- the instruction count of the fp16 form, every operand fp32.
// Everything else is the structure measured on kvq_kfast.cu: table and ratios built once per call by a prep kernel and
// bulk-copied into shared memory; packed codes through a TMA ring of [W rows x 64 tokens] boxes behind full / empty
// mbarriers; a warp covers 16 tokens x 2 channel halves (even channels / odd channels: disjoint table banks, same
// packed word -> broadcast) so that a lane keeps cos/sin of 32 pairs (64 registers); lookups of the next word pair
// are issued before the FMAs of the current one.  512 threads = 15 consumer warps + 1 producer warp: a 17th warp would
// cut the register budget from 128 to 96 (a lane holds 64 registers of cos/sin), and a TMA issue rotating over the
// consumer warps measured 40 % slower (the issuing warp waits for the slowest warp before it may start its own slab).
#include "kvq_kscore.cuh"
#include "kvq_attend.cuh"

namespace kvq {

constexpr int kKRWarps = 15;                       // consumer warps; the 16th warp feeds the TMA ring
constexpr int kKRThreads = (kKRWarps + 1) * 32;    // 512 threads -> 128 registers each
constexpr int kKRColTok = 16;                      // tokens per warp column
constexpr int kKRBoxWarps = 5;                     // one TMA box: W rows x 80 tokens (5 warp columns of 16)
constexpr int kKRRow = kKRBoxWarps * kKRColTok * 4;   // bytes between packed-word rows inside a TMA box
constexpr uint32_t kKRSmemBudget = 227u * 1024u;

struct KRParams {
  const float* qtab;         // f32 [H][128][N]   LUT * q_c (k_ratio_prep_kernel)
  const float* qrat;         // f32 [H][128]      r_c, permuted: [group 0..7][half][x|y][k 0..3]
  const float2* rope;        // float2 [64][rope_npos] (cos, sin)
  float* out;                // [H][out_stride]
  float* gmax;               // [H] or null
  int64_t Lmax, L, out_stride, rope_npos, range;
  const int64_t* len_dev;
  int64_t len_add;
  int H, G, pos_offset, accumulate, n_stages;   // H, G: query heads (of the call, of one CTA)
  float scale;
};

template <int BITS> struct KRCfg {
  static constexpr int N = 1 << BITS;
  static constexpr int W = Layout<BITS>::kWords;
  static constexpr int GMAX = (BITS == 4) ? 16 : 32;       // heads per CTA: table = G * 128 * N * 4 bytes <= 128 KiB
  static constexpr uint32_t kHeadTab = kHeadDim * N * 4;   // bytes of one head's table
  static constexpr uint32_t kHeadRat = kHeadDim * 4;       // bytes of one head's ratios
  static constexpr int kBoxWarps = kKRBoxWarps;
  static constexpr uint32_t kBox = W * kKRRow;
  static constexpr uint32_t kStage = (kKRWarps / kBoxWarps) * kBox;   // one slab = one head x 240 tokens
};

// tokens per CTA when L tokens are cut into at most `splits` ranges of whole 16-token warp columns: the finest rounding
// the kernel allows, so that long caches give every SM a range (the last round's columns are spread over the warps)
__host__ __device__ __forceinline__ int64_t kr_range(int64_t L, int64_t splits) {
  const int64_t r = (L + splits - 1) / splits;
  return (r + kKRColTok - 1) / kKRColTok * kKRColTok;
}

template <int IMM> __device__ __forceinline__ uint32_t kr_lds_word(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(IMM));
  return v;
}
template <int IMM> __device__ __forceinline__ float kr_lds_tab(uint32_t addr) {   // keeps its place in the stream
  float v;
  asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(addr), "n"(IMM));
  return v;
}
template <int IMM> __device__ __forceinline__ float4 kr_lds_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4+%5];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr), "n"(IMM));
  return v;
}

struct KRHalf {
  uint32_t half;     // 0: even channels, 1: odd channels
  uint32_t rot;      // 4-bit: left-rotation that brings this half's nibbles to bits 2..5 of each byte (2 / 30)
  uint32_t bias;     // byte-replicated offset of the odd channel's table (one channel = 64 / 32 / 16 bytes)
};

// One head, this lane's half of one token.  st = shared address of the lane's token column in the slab, base = the
// head's table (256-byte aligned), rat = the head's ratios + half * 32 bytes, cs[i] = (cos, sin) of the lane's pair i.
// Group gi (0..7) = channels 8 gi .. 8 gi + 7 (and their rotary partners +64); the lane owns 8 gi + 2k + half, k < 4.
template <int BITS>
__device__ __forceinline__ float k_ratio_head(const uint32_t st, const uint32_t base, const uint32_t rat, const KRHalf hs,
                                             const float2 (&cs)[32]) {
  float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
  constexpr int kRow = kKRRow;
  float xs[2][4], ys[2][4];
  // packed words of a group: loaded once per word (a 2-bit word spans two groups, a 3-bit group three words)
  uint32_t wa4 = 0, wb4 = 0, w3a[2][3], w3b[2][3];
  if constexpr (BITS == 3) {
    static_for<0, 2>([&](auto ig) {
      constexpr int g = decltype(ig)::v;
      w3a[g][0] = kr_lds_word<(3 * g) * kRow>(st); w3a[g][1] = kr_lds_word<(3 * g + 1) * kRow>(st); w3a[g][2] = kr_lds_word<(3 * g + 2) * kRow>(st);
      w3b[g][0] = kr_lds_word<(3 * g + 6) * kRow>(st); w3b[g][1] = kr_lds_word<(3 * g + 7) * kRow>(st); w3b[g][2] = kr_lds_word<(3 * g + 8) * kRow>(st);
    });
  }
  auto window3 = [&](const uint32_t (&w)[3], auto ia) -> uint32_t {
    constexpr int a = decltype(ia)::v;
    return (a == 0 ? w[0] : (a == 1 ? __funnelshift_r(w[0], w[1], 24) : (a == 2 ? __funnelshift_r(w[1], w[2], 16) : (w[2] >> 8))))
           >> (3 * hs.half);
  };
  auto issue = [&](auto igi, float (&x)[4], float (&y)[4]) {
    constexpr int gi = decltype(igi)::v;
    if constexpr (BITS == 4) {
      const uint32_t wa = kr_lds_word<gi * kRow>(st), wb = kr_lds_word<(gi + 8) * kRow>(st);
      // byte b <- (code 2b + half) * 4 + half * 64   (the rotation wraps only into masked-out bits)
      const uint32_t ma = (__funnelshift_l(wa, wa, hs.rot) & 0x3C3C3C3Cu) | hs.bias;
      const uint32_t mb = (__funnelshift_l(wb, wb, hs.rot) & 0x3C3C3C3Cu) | hs.bias;
      static_for<0, 4>([&](auto ik) {
        constexpr int k = decltype(ik)::v;
        x[k] = kr_lds_tab<(8 * gi + 2 * k) * 64>(__byte_perm(ma, base, 0x7650 | k));
        y[k] = kr_lds_tab<(8 * gi + 2 * k + kHalf) * 64>(__byte_perm(mb, base, 0x7650 | k));
      });
    } else if constexpr (BITS == 2) {
      if constexpr ((gi & 1) == 0) {              // word gi/2: channels 16 (gi/2) .. +15, partners in word gi/2 + 4
        wa4 = kr_lds_word<(gi / 2) * kRow>(st) >> (2 * hs.half);
        wb4 = kr_lds_word<(gi / 2 + 4) * kRow>(st) >> (2 * hs.half);
      }
      // code 2k' + half of the word (k' = 4 (gi & 1) + k) sits at bits 4k': byte k' >> 1, bits 0..1 / 4..5
      const uint32_t ma[2] = {((wa4 << 2) & 0x0C0C0C0Cu) | hs.bias, ((wa4 >> 2) & 0x0C0C0C0Cu) | hs.bias};
      const uint32_t mb[2] = {((wb4 << 2) & 0x0C0C0C0Cu) | hs.bias, ((wb4 >> 2) & 0x0C0C0C0Cu) | hs.bias};
      static_for<0, 4>([&](auto ik) {
        constexpr int k = decltype(ik)::v, kk = 4 * (gi & 1) + k;
        x[k] = kr_lds_tab<(8 * gi + 2 * k) * 16>(__byte_perm(ma[kk & 1], base, 0x7650 | (kk >> 1)));
        y[k] = kr_lds_tab<(8 * gi + 2 * k + kHalf) * 16>(__byte_perm(mb[kk & 1], base, 0x7650 | (kk >> 1)));
      });
    } else {
      constexpr int g = gi >> 2, a = gi & 3;      // 24-bit window a of group g: channels 32g + 8a .. +7
      const uint32_t hb = base | hs.bias;         // bias = half * 32: bit 5, clear of the code bits 2..4
      const uint32_t x0 = window3(w3a[g], IC<a>{}), x1 = window3(w3b[g], IC<a>{});   // this half's codes at bits 6k
      static_for<0, 4>([&](auto ik) {
        constexpr int k = decltype(ik)::v;
        const uint32_t ax = ((k == 0 ? (x0 << 2) : (x0 >> (6 * k - 2))) & 0x1Cu) | hb;
        const uint32_t ay = ((k == 0 ? (x1 << 2) : (x1 >> (6 * k - 2))) & 0x1Cu) | hb;
        x[k] = kr_lds_tab<(8 * gi + 2 * k) * 32>(ax);
        y[k] = kr_lds_tab<(8 * gi + 2 * k + kHalf) * 32>(ay);
      });
    }
  };
  auto consume = [&](auto igi, const float (&x)[4], const float (&y)[4]) {
    constexpr int gi = decltype(igi)::v;
    const float4 rx = kr_lds_f4<gi * 64>(rat), ry = kr_lds_f4<gi * 64 + 16>(rat);   // broadcast within the half
    const float rxv[4] = {rx.x, rx.y, rx.z, rx.w}, ryv[4] = {ry.x, ry.y, ry.z, ry.w};
    static_for<0, 4>([&](auto ik) {
      constexpr int k = decltype(ik)::v;
      constexpr int i = 4 * gi + k;               // this lane's pair index: channel 8 gi + 2k + half
      const float gx = fmaf(rxv[k], cs[i].y, cs[i].x);
      const float gy = fmaf(ryv[k], cs[i].y, cs[i].x);
      if constexpr (k & 1) { a1 = fmaf(x[k], gx, a1); b1 = fmaf(y[k], gy, b1); }
      else { a0 = fmaf(x[k], gx, a0); b0 = fmaf(y[k], gy, b0); }
    });
  };
  issue(IC<0>{}, xs[0], ys[0]);
  static_for<0, 8>([&](auto igi) {
    constexpr int gi = decltype(igi)::v;
    if constexpr (gi + 1 < 8) issue(IC<gi + 1>{}, xs[(gi + 1) & 1], ys[(gi + 1) & 1]);
    consume(igi, xs[gi & 1], ys[gi & 1]);
  });
  return (a0 + b0) + (a1 + b1);
}

// GQA: p.H and p.G count query heads, `group` of them per KV head.  A CTA owns whole groups (p.G is a multiple of
// `group`); the slab of a KV head is consumed by the tables of its query heads before its stage is released, so the
// packed words are read from HBM once per token range.  GQA = false is the one-KV-head-per-query-head kernel (`group`
// unused; it is a kernel argument rather than a KRParams field so that this instantiation compiles as before).
// BATCH: sequence b = blockIdx.z of a batched attend (kvq_attend_batch): its tables, ratios, score rows and maximum sit
// `bstride` floats after sequence b-1's, its length is p.len_dev[b], and its cache rows follow the b*Hkv*W rows of the
// sequences before it in the one tensor map.  BATCH = false ignores `bstride`.
// PAGED (with BATCH; kvq_attend_paged): the tensor map covers the page pool, n_pool*Hkv*W rows x P columns, and each
// box is looked up in sequence b's page table: token x -> column x % P of rows page_of(b, x)*Hkv*W + ...  Ranges are
// rounded to 160 tokens (not 32) so that every 80-token box starts on a multiple of 80 and, P being a multiple of
// 160, lies inside one page; the box's first token is below the sequence's length, so its page is mapped.  The
// length is also capped at npages[b] * P.  A token's score is the same instruction sequence whatever the range, so
// the scores equal the contiguous batch's bit for bit.  Other instantiations ignore `pg`.
// With BATCH, sequence b's rope table sits b * rope_bstride entries after sequence 0's: 64 * rope_npos for a rotation
// per sequence (length-dependent frequencies, DESIGN.md section 4.14), 0 for one table shared by the batch.  It is the
// last kernel argument, not a KRParams field, so that every other argument keeps its parameter-bank offset.
// SUB (with GQA; k_ratio_sub_kernel): a KV head has more query heads than one CTA's table holds (grp > GMAX, one or
// two KV heads), so a CTA owns a sub-range of one KV head's query heads.  The grp heads of each KV head are cut into
// nsub = ceil(grp / p.G) ranges of at most p.G heads, CTA row y being range y % nsub of KV head y / nsub; its producer
// loads that KV head's slab once per round, and its first and last heads wait for and release the stage.  The nsub
// CTAs of a KV head each read its slab (DESIGN.md section 4.9).
template <int BITS, bool GQA, bool BATCH, bool PAGED, bool SUB>
__device__ __forceinline__ void k_ratio_body(const CUtensorMap& tmap, const KRParams& p, const int group,
                                             const int64_t bstride, const PageRef& pg, const int64_t rope_bstride) {
  using C = KRCfg<BITS>;
  constexpr int W = C::W;
  const int grp = GQA ? group : 1;
  const int bz = BATCH ? (int)blockIdx.z : 0;
  const int64_t boff = BATCH ? bz * bstride : 0;
  const int brow = BATCH ? bz * (p.H / grp) * W : 0;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int S = p.n_stages;
  const int nsub = SUB ? (grp + p.G - 1) / p.G : 1;
  const int h0 = SUB ? (int)blockIdx.y / nsub * grp + (int)blockIdx.y % nsub * p.G : blockIdx.y * p.G;
  const int nh = min(p.G, SUB ? ((int)blockIdx.y / nsub + 1) * grp - h0 : p.H - h0);
  const uint32_t tab_span = (uint32_t)p.G * C::kHeadTab;
  const uint32_t rat_span = (uint32_t)p.G * C::kHeadRat;
  unsigned char* s_tab = smem;                                         // [G][128][N] f32
  unsigned char* s_rat = smem + tab_span;                              // [G][128] f32 (permuted)
  unsigned char* s_stage = s_rat + rat_span;                           // [S][4 boxes][W][64] u32
  uint64_t* s_full = reinterpret_cast<uint64_t*>(s_stage + (size_t)S * C::kStage);
  uint64_t* s_empty = s_full + S;
  uint64_t* s_tabbar = s_empty + S;
  int* s_max = reinterpret_cast<int*>(s_tabbar + 1);                    // [G] running max (ordered-int encoding)

  int64_t L_eff = p.L;
  int64_t range = p.range;
  if (p.len_dev != nullptr) {
    const int64_t l = p.len_dev[bz] + p.len_add;
    L_eff = l < 0 ? 0 : (l < p.L ? l : p.L);
    if constexpr (PAGED) {
      const int64_t cap = page_cap(pg, bz);
      L_eff = L_eff < cap ? L_eff : cap;
      const int64_t r = (L_eff + gridDim.x - 1) / gridDim.x;
      range = (r + kPageQuantum - 1) / kPageQuantum * kPageQuantum;
    } else {
      range = kr_range(L_eff, gridDim.x);
    }
  }
  const int64_t t_begin = (int64_t)blockIdx.x * range;
  const int64_t t_limit = min(L_eff, ((int64_t)blockIdx.x + 1) * range);
  if (t_begin >= t_limit) return;
  const int ncols = (int)((t_limit - t_begin + kKRColTok - 1) / kKRColTok);
  const int nrounds = (ncols + kKRWarps - 1) / kKRWarps;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(&s_full[s], 1); mbar_init(&s_empty[s], kKRWarps); }
    mbar_init(s_tabbar, 1);
    mbar_fence_init();
    prefetch_tensormap(&tmap);
  }
  if (tid < p.G) s_max[tid] = (int)(0xFF800000u ^ 0x7FFFFFFFu);   // -inf in the ordered-int encoding
  __syncthreads();

  if (warp == kKRWarps) {
    // ---------------- producer warp: table + ratios, then the slab ring ----------------------------------------------
    if (lane == 0) {
      mbar_expect_tx(s_tabbar, (uint32_t)nh * (C::kHeadTab + C::kHeadRat));
      const unsigned char* src = reinterpret_cast<const unsigned char*>(p.qtab + boff) + (size_t)h0 * C::kHeadTab;
      const uint32_t tab_bytes = (uint32_t)nh * C::kHeadTab;
      for (uint32_t o = 0; o < tab_bytes; o += 16384u) bulk_load_1d(s_tab + o, src + o, min(16384u, tab_bytes - o), s_tabbar);
      bulk_load_1d(s_rat, reinterpret_cast<const unsigned char*>(p.qrat + boff) + (size_t)h0 * C::kHeadRat, (uint32_t)nh * C::kHeadRat, s_tabbar);
      int s = 0;
      uint32_t ph = 1;   // parity of the previous use of stage s (first pass: nothing to wait for)
      bool wrapped = false;
      for (int r = 0; r < nrounds; ++r) {
        const int nlive = min(kKRWarps, ncols - r * kKRWarps);
        const int nbox = (nlive + C::kBoxWarps - 1) / C::kBoxWarps;    // the last box may reach past the range: read-only
        const int x0 = (int)(t_begin + (int64_t)r * kKRWarps * kKRColTok);
        for (int hl = 0; hl < (SUB ? 1 : (GQA ? nh / grp : nh)); ++hl) {   // one slab per KV head
          if (wrapped) mbar_wait(&s_empty[s], ph);
          mbar_expect_tx(&s_full[s], (uint32_t)nbox * C::kBox);
          unsigned char* dst = s_stage + (size_t)s * C::kStage;
          for (int b = 0; b < nbox; ++b) {
            const int x = x0 + kKRColTok * C::kBoxWarps * b;
            if constexpr (PAGED) {
              const int page = page_of(pg, bz, x);
              tma_load_2d(dst + (size_t)b * C::kBox, &tmap, &s_full[s], x % pg.P,
                          (page * (p.H / grp) + (GQA ? h0 / grp + hl : h0 + hl)) * W);
            } else {
              tma_load_2d(dst + (size_t)b * C::kBox, &tmap, &s_full[s], x, (GQA ? h0 / grp + hl : h0 + hl) * W + brow);
            }
          }
          if (++s == S) { s = 0; ph ^= 1u; wrapped = true; }
        }
      }
    }
    if (p.gmax != nullptr) __syncthreads();
    return;
  }

  const uint64_t pol_keep = policy_evict_last();
  uint32_t tab0 = smem_u32(s_tab);
  const int tl = lane & 15;
  KRHalf hs;
  hs.half = (uint32_t)lane >> 4;
  hs.rot = hs.half ? 30u : 2u;
  hs.bias = hs.half * (BITS == 4 ? 0x40404040u : (BITS == 2 ? 0x10101010u : 0x20u));
  uint32_t rat0 = smem_u32(s_rat) + hs.half * 32u;
  asm volatile("" : "+r"(tab0), "+r"(rat0));   // kept in registers, not rebuilt from the shared window every head
  mbar_wait(s_tabbar, 0);
  int s = 0;
  uint32_t ph = 0;
  for (int r = 0; r < nrounds; ++r) {
    // A round's slabs hold nlive columns (15; fewer in a CTA's last round).  Every column gets the warps w with
    // w % nlive == c; the m of them split its heads round-robin (warp w takes heads w / nlive, + m, ...), so a short last
    // round keeps all 15 warps busy on the slabs the ring holds at once, and a warp keeps one column (one cos/sin
    // load) per round.  A full round is one column per warp for every head.
    const int nlive = min(kKRWarps, ncols - r * kKRWarps);
    const int c = warp % nlive;
    const int64_t t = t_begin + (int64_t)(r * kKRWarps + c) * kKRColTok + tl;
    const bool mine = t < t_limit;
    float2 cs[32];
    if (warp / nlive < nh) {
      // a lane past the range loads the range's last token's factors (its score is dropped at the store and the max)
      const float2* rope = p.rope;
      if constexpr (BATCH) rope += bz * rope_bstride;
      const float2* rp = rope + ((mine ? t : t_limit - 1) + p.pos_offset) + (int64_t)hs.half * p.rope_npos;
      // pair k sits 2k rows below pair 0 (channel 8 (k/4) + 2 (k%4) + half = 2k + half).  The row step is passed
      // through an empty asm so that the 32 row offsets are walked per round: hoisted out of the round loop they are
      // 64 live registers, which ptxas spills to the stack and reloads every round.
      int64_t step = 2 * p.rope_npos;
      asm volatile("" : "+l"(step));
#pragma unroll
      for (int k = 0; k < 32; ++k, rp += step) cs[k] = ld_keep_f2(rp, pol_keep);
    }
    const int m = (kKRWarps - 1 - c) / nlive + 1;
    int next_h = warp / nlive;                           // this warp's next head (warp-uniform)
    const uint32_t stage0 = smem_u32(s_stage) + (uint32_t)(c / C::kBoxWarps) * C::kBox +
                            (uint32_t)((c % C::kBoxWarps) * kKRColTok + tl) * 4u;
    // GQA: the grp query heads of a KV head are consecutive; the first waits for the slab, the last releases it.
    // Every warp waits for and releases every slab, its heads or not, so the ring's arrive counts stay kKRWarps.
    for (int hl = 0; hl < nh; ++hl) {
      const bool live = hl == next_h;                    // warp-uniform
      if (live) next_h += m;
      float* optr = p.out + boff + (int64_t)(h0 + hl) * p.out_stride + t;
      float old = 0.f;
      if (p.accumulate && live && mine && hs.half == 0) old = __ldcg(optr);
      if (SUB ? hl == 0 : (!GQA || hl % grp == 0)) mbar_wait(&s_full[s], ph);
      if (live) {
        float acc = k_ratio_head<BITS>(stage0 + (uint32_t)s * C::kStage, tab0 + (uint32_t)hl * C::kHeadTab,
                                       rat0 + (uint32_t)hl * C::kHeadRat, hs, cs);
        acc += __shfl_xor_sync(0xffffffffu, acc, 16);    // even + odd channels
        const float sc = (acc + old) * p.scale;
        if (mine && hs.half == 0) *optr = sc;
        if (p.gmax != nullptr) {
          // warp max in ONE instruction: floats compare like their bit patterns once the negative range is mirrored
          const int bits = __float_as_int((mine && hs.half == 0) ? sc : -INFINITY);
          const int key = __reduce_max_sync(0xffffffffu, bits >= 0 ? bits : (bits ^ 0x7FFFFFFF));
          if (lane == 0) atomicMax(&s_max[hl], key);
        }
      }
      if (SUB ? hl == nh - 1 : (!GQA || hl % grp == grp - 1)) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&s_empty[s]);
        if (++s == S) { s = 0; ph ^= 1u; }
      }
    }
  }
  if (p.gmax != nullptr) {
    __syncthreads();
    if (tid < nh) {
      const int key = s_max[tid];
      const float m = __int_as_float(key >= 0 ? key : (key ^ 0x7FFFFFFF));
      if (m > -INFINITY) atomic_max_float(p.gmax + boff + h0 + tid, m);
    }
  }
}

template <int BITS, bool GQA, bool BATCH, bool PAGED = false>
__global__ void __launch_bounds__(kKRThreads, 1) k_ratio_kernel(const __grid_constant__ CUtensorMap tmap, const KRParams p,
                                                                const int group, const int64_t bstride, const PageRef pg,
                                                                const int64_t rope_bstride) {
  k_ratio_body<BITS, GQA, BATCH, PAGED, false>(tmap, p, group, bstride, pg, rope_bstride);
}

// a kernel of its own name: a SUB template argument would rename the instantiations above
template <int BITS, bool BATCH, bool PAGED>
__global__ void __launch_bounds__(kKRThreads, 1) k_ratio_sub_kernel(const __grid_constant__ CUtensorMap tmap, const KRParams p,
                                                                    const int group, const int64_t bstride, const PageRef pg,
                                                                    const int64_t rope_bstride) {
  k_ratio_body<BITS, true, BATCH, PAGED, true>(tmap, p, group, bstride, pg, rope_bstride);
}

// table T[h][c][code] = LUT * qe_c and ratios r_c = s_c q_{c^64} / qe_c (qe = q, or +-1e-30 where q is exactly 0);
// grid = H query heads, block = 128 (thread = channel).  GQA: query head h reads the LUT of KV head h / grp.
// BATCH: sequence b = blockIdx.y, q [B][H][128], its tables and ratios `bstride` floats after sequence b-1's.
template <int BITS, bool GQA, bool BATCH>
__global__ void k_ratio_prep_kernel(const float* __restrict__ q, const float* __restrict__ lut, float* __restrict__ qtab,
                                    float* __restrict__ qrat, int grp, const int64_t bstride) {
  constexpr int N = 1 << BITS;
  const int h = blockIdx.x, c = threadIdx.x;
  if constexpr (BATCH) {
    const int b = blockIdx.y;
    q += (int64_t)b * gridDim.x * kHeadDim;
    qtab += b * bstride;
    qrat += b * bstride;
  }
  const int hk = GQA ? h / grp : h;
  float qa = q[h * kHeadDim + c];
  const float qb = q[h * kHeadDim + (c ^ kHalf)];
  if (qa == 0.f) qa = 1e-30f;
  const float sg = (c < kHalf) ? 1.f : -1.f;
  const float* l = lut + ((int64_t)hk * kHeadDim + c) * N;
  float* o = qtab + ((int64_t)h * kHeadDim + c) * N;
#pragma unroll
  for (int i = 0; i < N; ++i) o[i] = l[i] * qa;
  const int cc = c & (kHalf - 1), xy = c >> 6;           // channel 8 gi + 2k + half (+64 for y)
  const int gi = cc >> 3, k = (cc & 7) >> 1, half = cc & 1;
  qrat[(int64_t)h * kHeadDim + gi * 16 + half * 8 + xy * 4 + k] = sg * qb / qa;
}

template <int BITS, bool GQA, bool BATCH, bool PAGED, bool SUB>
static int set_k_ratio_smem() {
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    const void* kern = SUB ? reinterpret_cast<const void*>(k_ratio_sub_kernel<BITS, BATCH, PAGED>)
                           : reinterpret_cast<const void*>(k_ratio_kernel<BITS, GQA, BATCH, PAGED>);
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kKRSmemBudget);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  return 0;
}

// c.B == 0: one sequence; c.B >= 1: a batch of B sequences, each with its own scratch block of s.bstride floats;
// c.pg != nullptr: a paged batch (the grid is the contiguous batch's)
template <int BITS>
static int launch_k_ratio(KRParams p, const AttendCall& c, const AttendScratch& s) {
  using C = KRCfg<BITS>;
  const int B = c.B, grp = c.grp();
  const bool gqa = grp > 1, batch = B > 0, paged = c.pg != nullptr;
  cudaStream_t st = c.stream;
  with_flavour(gqa, batch, false, [&](auto GQA, auto BATCH, auto) {
    k_ratio_prep_kernel<BITS, GQA(), BATCH()><<<batch ? dim3(p.H, B) : dim3(p.H), kHeadDim, 0, st>>>(
        c.q, c.klut, s.qtab, s.qrat, grp, s.bstride);
  });
  KVQ_LAUNCH_CHECK();
  // CTA head groups of at most GMAX query heads: whole KV-head groups while grp <= GMAX (every shape with Hkv % 4 == 0),
  // else (one or two KV heads) nsub CTAs per KV head, each a sub-range of its query heads (k_ratio_sub_kernel)
  const int Hkv = p.H / grp;
  const bool sub = grp > C::GMAX;
  int groups;
  if (sub) {
    const int nsub = (grp + C::GMAX - 1) / C::GMAX;
    p.G = (grp + nsub - 1) / nsub;
    groups = Hkv * nsub;
  } else {
    const int kv_max = C::GMAX / grp;
    groups = (Hkv + kv_max - 1) / kv_max;
    p.G = (Hkv + groups - 1) / groups * grp;
  }
  const uint32_t tab_span = (uint32_t)p.G * (C::kHeadTab + C::kHeadRat);
  const uint32_t fixed = tab_span + 1024u /*align*/ + 8u * 20u + 4u * 64u + 64u;
  int S = (int)((kKRSmemBudget - fixed) / C::kStage);
  if (S > 8) S = 8;
  if (S < 2) return KVQ_E_UNSUPPORTED;
  p.n_stages = S;
  const size_t smem = (size_t)tab_span + (size_t)S * C::kStage + 8u * (2 * S + 1) + 4u * p.G + 1024u;
  int rc = with_flavour(gqa, batch, paged, [&](auto GQA, auto BATCH, auto PAGED) {
    return sub ? set_k_ratio_smem<BITS, GQA(), BATCH(), PAGED(), true>() : set_k_ratio_smem<BITS, GQA(), BATCH(), PAGED(), false>();
  });
  if (rc != 0) return rc;
  CUtensorMap tmap;
  // a batch: one map over the B sequences' caches, B*Hkv*W rows (sequence b's rows follow b*Hkv*W others);
  // a paged batch: one map over the pool, n_pool*Hkv*W rows of P tokens
  if (paged)
    rc = make_cache_tensor_map(&tmap, c.kcache, (uint64_t)c.pg->n_pool * Hkv * C::W, (uint64_t)c.pg->P,
                               kKRColTok * C::kBoxWarps, C::W, /*swizzle*/ 0);
  else
    rc = make_cache_tensor_map(&tmap, c.kcache, (uint64_t)(batch ? B : 1) * Hkv * C::W, (uint64_t)p.Lmax,
                               kKRColTok * C::kBoxWarps, C::W, /*swizzle*/ 0);
  if (rc != 0) return rc;
  const int sms = num_sms_cached();
  const int per = batch ? groups * B : groups;   // a batch shares the SMs among its B x groups CTA columns
  const int64_t max_splits = sms / per > 0 ? sms / per : 1;
  p.range = kr_range(p.L, max_splits);
  const int64_t splits = (p.L + p.range - 1) / p.range;
  const dim3 grid = batch ? dim3((unsigned)splits, (unsigned)groups, (unsigned)B) : dim3((unsigned)splits, (unsigned)groups);
  const int64_t rope_bstride = c.rope_per_seq ? kHalf * p.rope_npos : 0;
  const PageRef pg = paged ? *c.pg : PageRef{};
  with_flavour(gqa, batch, paged, [&](auto GQA, auto BATCH, auto PAGED) {
    if (sub)
      k_ratio_sub_kernel<BITS, BATCH(), PAGED()><<<grid, kKRThreads, smem, st>>>(tmap, p, grp, s.bstride, pg, rope_bstride);
    else
      k_ratio_kernel<BITS, GQA(), BATCH(), PAGED()><<<grid, kKRThreads, smem, st>>>(tmap, p, grp, s.bstride, pg, rope_bstride);
  });
  KVQ_LAUNCH_CHECK();
  return 0;
}

// dense K scores of the fused attend, fp32 ratio form.  s.scores holds the (unscaled) outlier partial sums on entry
// when accumulate != 0.  s.qtab / s.qrat: Hq * 128 * (2^bits + 1) floats of scratch.
int k_ratio_dispatch(const AttendCall& c, const AttendScratch& s, int accumulate) {
  KRParams p{};
  p.qtab = s.qtab; p.qrat = s.qrat;
  p.rope = reinterpret_cast<const float2*>(c.rope);
  p.out = s.scores; p.gmax = s.gmax;
  p.Lmax = c.Lmax; p.L = c.L; p.out_stride = s.stride; p.rope_npos = c.rope_npos;
  p.len_dev = c.len_dev; p.len_add = c.len_add;
  p.H = c.Hq; p.pos_offset = c.pos_offset; p.accumulate = accumulate; p.scale = kAttendScale;
  switch (c.bits) {
    case 4: return launch_k_ratio<4>(p, c, s);
    case 3: return launch_k_ratio<3>(p, c, s);
    case 2: return launch_k_ratio<2>(p, c, s);
    default: return KVQ_E_BITS;
  }
}

}  // namespace kvq
