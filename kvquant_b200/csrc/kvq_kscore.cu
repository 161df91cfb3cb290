// kvquant_b200 -- Q.K^T decode matvec over the packed pre-RoPE key cache with RoPE applied at read time: the dense
// kernel (all widths; 3-bit has its own in kvq_k3.cu), the outlier scatter that runs in front of it, the rope table
// builder, and the A/B variants kept behind KVQ_K_IMPL.
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
//     premultiplied tables T[h][c][code] = (LUT*q[h,c], s_c*LUT*q[h,c^64]) in shared memory: 16 (8, 4) entries per
//     channel are 16 distinct consecutive 8-byte slots -> conflict-free multicast for any code pattern.
//   * per element: 1 address op (PRMT), 1 LDS.64, 2 FFMA; words and rope values are prefetched into rotating
//     register buffers; token ranges are cut at warp granularity so that every SM gets an equal share.
#include "kvq_kscore.cuh"
#include <cuda_fp16.h>
#include <stdlib.h>

namespace kvq {

template <int BITS> struct KCfg {
  static constexpr int N = 1 << BITS;
  static constexpr int W = Layout<BITS>::kWords;
  static constexpr int G = (BITS == 2) ? 16 : 128 / N;  // heads per CTA: 8 / 16 / 16 -> table = 128 / 128 / 64 KiB
  static constexpr int kThreads = 512;
  static constexpr int TT = kThreads;          // tokens per tile (thread = token)
  static constexpr int NRW = (BITS == 3) ? 4 : 2;  // packed words a thread needs per (head, 8-pair chunk)
  static constexpr int D = (BITS == 4) ? 8 : 4;    // cp.async prefetch distance in (head, chunk) work items
};

// 4-byte asynchronous global->shared copy (LDGSTS) with an L2 eviction policy; per-thread software pipeline
__device__ __forceinline__ void cp_async4(uint32_t smem_dst, const void* gsrc, uint64_t pol, int pred) {
  asm volatile("{ .reg .pred p; setp.ne.s32 p, %3, 0;"
               " @p cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 4, %2; }"
               ::"r"(smem_dst), "l"(gsrc), "l"(pol), "r"(pred) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

// packed-word rows (relative to the head) needed for 8-pair chunk a (pairs 8a..8a+7): channels 8a..8a+7 and +64
template <int BITS> __device__ __forceinline__ int chunk_word_row(int a, int i) {
  if constexpr (BITS == 4) { return i == 0 ? a : a + 8; }
  else if constexpr (BITS == 2) { return i == 0 ? (a >> 1) : 4 + (a >> 1); }
  else {
    // 24-bit window at bit 24*(a&3) of the 96-bit group a>>2 (words 3g..3g+2); i=0/1 low pair of words, i=2/3 high (+2 groups)
    const int first = (24 * (a & 3)) >> 5;            // 0,0,1,2
    const int w = (i & 1) ? min(first + 1, 2) : first;
    return 3 * ((a >> 2) + ((i >> 1) ? 2 : 0)) + w;
  }
}

// One work item = (head hl, 8-pair chunk a): 16 table lookups + 16 packed FMAs into the head's accumulator.
//   base = shared address of T[hl][8a][0] (256-byte aligned: the low address byte carries code*8);
//   4-bit / 2-bit: codes pre-masked into byte lanes, ONE PRMT per element builds the address;
//   3-bit: one shift + one LOP3 (and-or) per element on the funnel-shifted 24-bit window.
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
  } else if constexpr (BITS == 2) {
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
  } else {
    const int sh = (24 * (a & 3)) & 31;  // 0, 24, 16, 8
    const uint32_t x0 = __funnelshift_r(w[0], w[1], sh), x1 = __funnelshift_r(w[2], w[3], sh);
    static_for<0, 8>([&](auto ik) {
      constexpr int k = decltype(ik)::v;
      const uint32_t a0 = ((k == 0 ? (x0 << 3) : (x0 >> (3 * k - 3))) & 0x38u) | base;
      const uint32_t a1 = ((k == 0 ? (x1 << 3) : (x1 >> (3 * k - 3))) & 0x38u) | base;
      ffma2(acc, cs[k], lds_f2<k * N * 8>(a0));
      ffma2(acc, cs[k], lds_f2<k * N * 8 + HI>(a1));
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
  const int64_t L_eff = k_eff_len(p);
  const int64_t range = k_eff_range(p, L_eff);
  const int64_t t_begin = (int64_t)blockIdx.x * range;
  const int64_t t_limit = min(L_eff, t_begin + range);   // tokens this CTA may touch
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
    float old[G];
#pragma unroll
    for (int hl = 0; hl < G; ++hl) {
      old[hl] = 0.f;
      if (p.accumulate && live && hl < nh) old[hl] = p.out[(int64_t)(h0 + hl) * p.out_stride + t];
    }
    if (p.opart != nullptr && live) {   // outlier partials of this token's G heads: G/4 16-byte loads (rows are padded)
      const float4* src = reinterpret_cast<const float4*>(p.opart + t * p.opart_stride + h0);
#pragma unroll
      for (int i = 0; i < G / 4; ++i) {
        const float4 v = __ldcg(src + i);
        old[4 * i] += v.x; old[4 * i + 1] += v.y; old[4 * i + 2] += v.z; old[4 * i + 3] += v.w;
      }
    }
#pragma unroll
    for (int hl = 0; hl < G; ++hl) {
      if (hl < nh) {
        const float s = ((acc[hl].x + acc[hl].y) + old[hl]) * p.scale;
        if (live) p.out[(int64_t)(h0 + hl) * p.out_stride + t] = s;
        if (p.gmax != nullptr) {
          const float m = warp_max(live ? s : -INFINITY);
          if ((tid & 31) == 0 && m > -INFINITY) atomic_max_float(p.gmax + h0 + hl, m);
        }
      }
    }
    }
    src_cur = src_nxt;
    ok_cur = ok_nxt;
  }
}

// ------------------------------------------------------------------------------------------------------------
// kappa form of the dense kernel (alternative, KVQ_K_IMPL=kappa).  The LDS.64 form above pays two shared-memory wavefronts per 32
// elements, and the shared-memory pipe is what limits it.
// Here the shared table holds the RAW per-channel LUT (4 bytes per entry -> one wavefront per 32 elements) and the
// query-dependent factor is applied arithmetically per (head, pair, token):
//
//     kappa = cos*(q_c, q_c64) + sin*(q_c64, -q_c)            4 scalar ops, q pairs are uniform operands from the
//     acc  += (LUT_c[code_c], LUT_c64[code_c64]) * kappa      constant bank (LDC.128 -> FMUL / FFMA UR operands)
//
// per pair: 2 PRMT + 2 LDS.32 + LDC.128 + 2 FMUL + 4 FFMA  = 8 issue slots and 1 shared wavefront per element.
// The rotated-query constants live in __constant__ memory, refreshed per call by a tiny prep kernel + a D2D
// cudaMemcpyToSymbolAsync (stream-ordered, graph-capturable).  K launches of one device must be stream-ordered.
// ------------------------------------------------------------------------------------------------------------
constexpr int kMaxConstHeads = 48;
__constant__ float4 c_qrot[kMaxConstHeads * kHalf];   // [h][j] = (q_c, q_c64, q_c64, -q_c), c = j < 64

template <int BITS> struct KKCfg {
  static constexpr int N = 1 << BITS;
  static constexpr int W = Layout<BITS>::kWords;
  static constexpr int CS = (N * 4 < 32) ? 32 : N * 4;   // bytes per channel in the table (8 channels = multiple of 256 B)
  static constexpr int G = (BITS == 4) ? 16 : 32;        // heads per CTA: table = G*128*CS = 128 KiB
  static constexpr int kThreads = 512;
  static constexpr int TT = kThreads;
  static constexpr int NRW = (BITS == 3) ? 4 : 2;
  static constexpr int D = 4;                            // cp.async prefetch distance in work items
};

template <int IMM>
__device__ __forceinline__ float lds_f1(uint32_t addr) {
  float v;
  asm("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(addr), "n"(IMM));
  return v;
}
__device__ __forceinline__ float2 fmul2(const float2 a, const float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}

// one work item (head h (global), chunk a): 8 pairs
template <int BITS>
__device__ __forceinline__ void kk_item(const uint32_t* __restrict__ w, const int a, const uint32_t base, const int hq,
                                        const float2* __restrict__ cs, float2& acc) {
  using C = KKCfg<BITS>;
  constexpr int CS = C::CS;
  constexpr int HI = kHalf * CS;
  uint32_t alo[8], ahi[8];
  if constexpr (BITS == 4) {
    const uint32_t e0 = (w[0] << 2) & 0x3C3C3C3Cu, o0 = (w[0] >> 2) & 0x3C3C3C3Cu;
    const uint32_t e1 = (w[1] << 2) & 0x3C3C3C3Cu, o1 = (w[1] >> 2) & 0x3C3C3C3Cu;
    static_for<0, 8>([&](auto ik) {
      constexpr int k = decltype(ik)::v;
      alo[k] = __byte_perm((k & 1) ? o0 : e0, base, 0x7650 | (k >> 1));
      ahi[k] = __byte_perm((k & 1) ? o1 : e1, base, 0x7650 | (k >> 1));
    });
  } else if constexpr (BITS == 2) {
    const int sh = 16 * (a & 1);
    const uint32_t x0 = w[0] >> sh, x1 = w[1] >> sh;
    const uint32_t m00 = (x0 << 2) & 0x0C0Cu, m01 = x0 & 0x0C0Cu, m02 = (x0 >> 2) & 0x0C0Cu, m03 = (x0 >> 4) & 0x0C0Cu;
    const uint32_t m10 = (x1 << 2) & 0x0C0Cu, m11 = x1 & 0x0C0Cu, m12 = (x1 >> 2) & 0x0C0Cu, m13 = (x1 >> 4) & 0x0C0Cu;
    static_for<0, 8>([&](auto ik) {
      constexpr int k = decltype(ik)::v;
      const uint32_t s0 = (k & 3) == 0 ? m00 : ((k & 3) == 1 ? m01 : ((k & 3) == 2 ? m02 : m03));
      const uint32_t s1 = (k & 3) == 0 ? m10 : ((k & 3) == 1 ? m11 : ((k & 3) == 2 ? m12 : m13));
      alo[k] = __byte_perm(s0, base, 0x7650 | (k >> 2));
      ahi[k] = __byte_perm(s1, base, 0x7650 | (k >> 2));
    });
  } else {
    const int sh = (24 * (a & 3)) & 31;
    const uint32_t x0 = __funnelshift_r(w[0], w[1], sh), x1 = __funnelshift_r(w[2], w[3], sh);
    static_for<0, 8>([&](auto ik) {
      constexpr int k = decltype(ik)::v;
      alo[k] = ((3 * k >= 2 ? (x0 >> (3 * k - 2)) : (x0 << (2 - 3 * k))) & 0x1Cu) | base;
      ahi[k] = ((3 * k >= 2 ? (x1 >> (3 * k - 2)) : (x1 << (2 - 3 * k))) & 0x1Cu) | base;
    });
  }
  static_for<0, 8>([&](auto ik) {
    constexpr int k = decltype(ik)::v;
    const float2 x = make_float2(lds_f1<k * CS>(alo[k]), lds_f1<k * CS + HI>(ahi[k]));
    const float4 qr = c_qrot[hq * kHalf + 8 * a + k];   // uniform: one LDCU.128
    const float2 kap = [&] {
      const float2 t = fmul2(make_float2(cs[k].y, cs[k].y), make_float2(qr.z, qr.w));
      float2 r = t;
      ffma2(r, make_float2(cs[k].x, cs[k].x), make_float2(qr.x, qr.y));
      return r;
    }();
    ffma2(acc, x, kap);
  });
}

template <int BITS>
__global__ void __launch_bounds__(KKCfg<BITS>::kThreads, 1) k_scores_kappa_kernel(const KParams p) {
  using C = KKCfg<BITS>;
  constexpr int N = C::N, W = C::W, G = C::G, TT = C::TT, NRW = C::NRW, D = C::D, CS = C::CS;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((256u - (smem_u32(smem_raw) & 255u)) & 255u);
  unsigned char* s_tab = smem;                                                   // [G][128][CS bytes]
  uint32_t* s_ring = reinterpret_cast<uint32_t*>(smem + (size_t)G * kHeadDim * CS);  // [D][NRW][TT]

  const int tid = threadIdx.x;
  const uint64_t pol_stream = policy_evict_first(), pol_keep = policy_evict_last();
  const int h0 = blockIdx.y * G;
  const int nh = min(G, p.H - h0);

  // raw per-channel LUT, CS bytes per channel
  for (int i = tid; i < nh * kHeadDim * N; i += C::kThreads) {
    const int hc = i / N, code = i - hc * N;
    *reinterpret_cast<float*>(s_tab + (size_t)hc * CS + code * 4) = p.lut[((int64_t)h0 * kHeadDim) * N + i];
  }
  __syncthreads();
  const uint32_t tab0 = smem_u32(s_tab);
  const uint32_t ring0 = smem_u32(s_ring) + tid * 4;

  const int64_t tile_first = (int64_t)blockIdx.x * p.tiles_per_cta;
  const int64_t tile_end = min(tile_first + p.tiles_per_cta, (p.L + TT - 1) / TT);
  const int64_t t_limit = min(p.L, tile_end * TT);
  const uint32_t* cbase = p.cache + (int64_t)h0 * W * p.Lmax;
  const uint32_t pitch = (uint32_t)p.Lmax * 4u;
  const unsigned char* cb0 = reinterpret_cast<const unsigned char*>(cbase);
  int64_t t_cur = tile_first * TT + tid;
  auto prefetch = [&](int nxt, int a, int hl, int slot) {
    const int64_t t = t_cur + (nxt ? TT : 0);
    const int ok = (t < t_limit) && (hl < nh);
    const unsigned char* src = cb0 + t * 4;
#pragma unroll
    for (int i = 0; i < NRW; ++i)
      cp_async4(ring0 + (uint32_t)(slot * NRW + i) * (TT * 4),
                src + (uint64_t)(uint32_t)(hl * W + chunk_word_row<BITS>(a, i)) * pitch, pol_stream, ok);
    cp_async_commit();
  };
  auto load_cs = [&](float2* dst, int64_t tile, int a) {
    const int64_t t = tile * TT + tid;
    if (t < t_limit) {
      const float2* rp = p.rope + (t + p.pos_offset) + (int64_t)(8 * a) * p.rope_npos;
#pragma unroll
      for (int k = 0; k < 8; ++k) dst[k] = ld_keep_f2(rp + (int64_t)k * p.rope_npos, pol_keep);
    }
  };

  static_for<0, D>([&](auto id) {
    constexpr int d = decltype(id)::v;
    prefetch((d / G) / 8, (d / G) % 8, d % G, d % D);
  });
  float2 cs[8], csn[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { cs[k] = make_float2(0.f, 0.f); csn[k] = make_float2(0.f, 0.f); }
  load_cs(cs, tile_first, 0);

  for (int64_t tile = tile_first; tile < tile_end; ++tile) {
    const int64_t t = tile * TT + tid;
    t_cur = t;
    const bool live = t < p.L;
    float2 acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = make_float2(0.f, 0.f);

    for (int a = 0; a < 8; ++a) {
      load_cs(csn, a == 7 ? tile + 1 : tile, (a + 1) & 7);
      static_for<0, G>([&](auto ig) {
        constexpr int hl = decltype(ig)::v;
        cp_async_wait<D - 1>();
        uint32_t w[NRW];
        constexpr int slot = hl % D;
#pragma unroll
        for (int i = 0; i < NRW; ++i) w[i] = lds_u32(ring0 + (uint32_t)(slot * NRW + i) * (TT * 4));
        {
          constexpr int hn = (hl + D) % G;
          constexpr int wrap = (hl + D) / G;
          const int an = a + wrap;
          prefetch(an >> 3, an & 7, hn, slot);
        }
        // no per-thread guard here: lanes past L compute on stale ring words (always in-bounds table reads) and are
        // masked at the store; keeping the region convergent lets the q constants use the uniform datapath (LDCU)
        if (hl < nh)
          kk_item<BITS>(w, a, tab0 + (uint32_t)hl * (kHeadDim * CS) + (uint32_t)a * (8 * CS), h0 + hl, cs, acc[hl]);
      });
#pragma unroll
      for (int k = 0; k < 8; ++k) cs[k] = csn[k];
    }

#pragma unroll
    for (int hl = 0; hl < G; ++hl) {
      if (hl < nh) {
        float s = acc[hl].x + acc[hl].y;
        if (live) {
          float* o = p.out + (int64_t)(h0 + hl) * p.out_stride + t;
          if (p.accumulate) s += *o;
          s *= p.scale;
          *o = s;
        }
        if (p.gmax != nullptr) {
          const float m = warp_max(live ? s : -INFINITY);
          if ((tid & 31) == 0 && m > -INFINITY) atomic_max_float(p.gmax + h0 + hl, m);
        }
      }
    }
  }
  cp_async_wait<0>();
}

// rotated-query constants: scratch[h*64+j] = (q_c, q_c64, q_c64, -q_c)
__global__ void k_qrot_prep_kernel(const float* __restrict__ q, float4* __restrict__ scratch, int H) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * kHalf) return;
  const int h = i / kHalf, j = i - h * kHalf;
  const float a = q[h * kHeadDim + j], b = q[h * kHeadDim + j + kHalf];
  scratch[i] = make_float4(a, b, b, -a);
}

static float4* g_qrot_scratch[32] = {nullptr};

static int upload_qrot(const float* q, int H, cudaStream_t st) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 32) return KVQ_E_UNSUPPORTED;
  if (!g_qrot_scratch[dev]) {
    cudaError_t e = cudaMalloc(&g_qrot_scratch[dev], sizeof(float4) * kMaxConstHeads * kHalf);
    if (e != cudaSuccess) return (int)e;
  }
  k_qrot_prep_kernel<<<(H * kHalf + 255) / 256, 256, 0, st>>>(q, g_qrot_scratch[dev], H);
  KVQ_LAUNCH_CHECK();
  cudaError_t e = cudaMemcpyToSymbolAsync(c_qrot, g_qrot_scratch[dev], sizeof(float4) * H * kHalf, 0,
                                          cudaMemcpyDeviceToDevice, st);
  return e == cudaSuccess ? 0 : (int)e;
}

template <int BITS>
static int launch_k_kappa(const KParams& p, cudaStream_t st) {
  using C = KKCfg<BITS>;
  const size_t smem = 256 + (size_t)C::G * kHeadDim * C::CS + (size_t)C::D * C::NRW * C::TT * 4;
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(k_scores_kappa_kernel<BITS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  int rc = upload_qrot(p.q, p.H, st);
  if (rc != 0) return rc;
  const int n_groups = (p.H + C::G - 1) / C::G;
  const int64_t n_tiles = (p.L + C::TT - 1) / C::TT;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t max_splits = sms / n_groups > 0 ? sms / n_groups : 1;
  KParams q = p;
  q.tiles_per_cta = (int)((n_tiles + max_splits - 1) / max_splits);
  const int64_t splits = (n_tiles + q.tiles_per_cta - 1) / q.tiles_per_cta;
  k_scores_kappa_kernel<BITS><<<dim3((unsigned)splits, (unsigned)n_groups), C::kThreads, smem, st>>>(q);
  KVQ_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// Outlier scatter (replaces SPMV_ATOMIC_ROPE_BALANCED, quant_cuda_kernel.cu:472-521).  Runs before the dense
// kernel, which then folds `out` into its own sum: out = (out + S) * scale.
// ------------------------------------------------------------------------------------------------------------
constexpr int kOutThreads = 256;

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
// in shared memory (one 8-byte shared read per entry instead of two scattered global ones); the rope values still
// come from the table.  In the fused path the sums go to a TOKEN-major partial buffer (a token's heads share one
// 128-byte line, so a warp's ~25 reductions coalesce into one or two L1 requests).
// Alternatives considered (DESIGN.md section 4.1): a second, token-major copy of the rope table read with coalesced
// row loads + shuffles instead of the gather (it loads rows for the zero-valued pads too and adds 8 shuffles per
// entry); evaluating cosf/sinf(theta_j * pos) per entry instead of the gather (more instructions; used beyond
// L2-sized rope tables, k_out_direct); accumulating into a per-CTA [H][256-token] shared tile with coalesced write-out
// instead of global atomics (shared-memory fp32 atomics are compare-and-swap loops).
constexpr int kOutPersThreads = 512;
__global__ void __launch_bounds__(kOutPersThreads) k_outlier_pers_kernel(
    const float* __restrict__ q, const float* __restrict__ outliers, const int32_t* __restrict__ outlier_idx,
    float* __restrict__ out, int64_t stride_h, int64_t stride_t, int64_t L, int H, int n_out,
    const float2* __restrict__ rope, int64_t rope_npos, int pos_offset, float scale,
    const int64_t* __restrict__ len_dev, int64_t len_add, const uint32_t* __restrict__ rope_h, float rope_theta) {
  extern __shared__ float2 s_qq[];                       // [H*128] = (q[c], q[c^64])
  if (len_dev != nullptr) {                              // device-resident length: L is the cap the grid was sized for
    const int64_t l = *len_dev + len_add;
    L = l < 0 ? 0 : (l < L ? l : L);
  }
  const int tid = threadIdx.x, lane = tid & 31;
  for (int i = tid; i < H * kHeadDim; i += kOutPersThreads) s_qq[i] = make_float2(q[i], q[i ^ kHalf]);
  __syncthreads();
  const uint32_t total = (uint32_t)(L * n_out);          // host checks L * n_out < 2^31
  const uint32_t stride = gridDim.x * kOutPersThreads;
  const uint64_t pol_keep = policy_evict_last();
  for (uint32_t base = blockIdx.x * kOutPersThreads + (tid & ~31); base < total; base += stride) {
    const uint32_t e = base + lane;
    float contrib = 0.f;
    int key = -1 - lane;   // unique negative keys for idle lanes (never merge)
    uint32_t t = 0;
    int h = 0;
    if (e < total) {
      t = e / (uint32_t)n_out;
      const float v = outliers[e];
      const int col = outlier_idx[e];
      h = col >> 7;
      const int c = col & (kHeadDim - 1);
      key = (int)(t * 64u) + h;                          // t < 2^25
      if (v != 0.f) {   // pads / non-outliers contribute exactly 0 in the reference too
        float2 cs;
        if (rope_theta > 0.f) {
          // long contexts: the rope table no longer fits L2 and a scattered 8-byte gather costs a 32-byte DRAM sector
          // (1M tokens: 17x the 128K cost for 8x the tokens) -- evaluate the table builder's own expressions instead
          // (same device functions, same arguments: bit-identical values)
          const int headdim = kHeadDim, headdim2 = headdim / 2;
          const float th = powf(rope_theta, (-2 * __int2float_rd((c & (kHalf - 1)) % headdim2) / __int2float_rd(headdim)));
          const int pos = (int)t + pos_offset;
          cs = make_float2(cosf(th * pos), sinf(th * pos));
        } else if (rope_h != nullptr) {   // fp16 mode: the half2 table the dense kernel streams (half the bytes per gather)
          uint32_t u;
          asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(u)
                       : "l"(rope_h + (int64_t)(c & (kHalf - 1)) * rope_npos + t + pos_offset), "l"(pol_keep));
          cs = __half22float2(*reinterpret_cast<const __half2*>(&u));
        } else {
          cs = ld_keep_f2(rope + (int64_t)(c & (kHalf - 1)) * rope_npos + t + pos_offset, pol_keep);
        }
        const float2 qq = s_qq[col];
        const float sign = (c < kHalf) ? 1.f : -1.f;
        float dot = v * cs.x * qq.x;            // same operation order as DK.cu:513-515
        dot += sign * v * cs.y * qq.y;
        contrib = dot * scale;
      }
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float v2 = __shfl_down_sync(0xffffffffu, contrib, o);
      const int k2 = __shfl_down_sync(0xffffffffu, key, o);
      if (lane + o < 32 && k2 == key) contrib += v2;
    }
    const int kprev = __shfl_up_sync(0xffffffffu, key, 1);
    const bool leader = (lane == 0) || (kprev != key);
    if (leader && e < total && contrib != 0.f) atomicAdd(out + (int64_t)h * stride_h + (int64_t)t * stride_t, contrib);
  }
}

static int k_out_impl_table() {   // KVQ_KOUT_IMPL=table selects the non-persistent gather form for A/B runs
  static int v = -1;
  if (v < 0) { const char* e = getenv("KVQ_KOUT_IMPL"); v = (e && e[0] == 't') ? 1 : 0; }
  return v;
}

// rope tables beyond this many positions are not gathered from by the outlier scatter (KVQ_KOUT_DIRECT_NPOS overrides):
// 64 pairs x 8 bytes x 64K positions = 32 MB, about what stays resident in the 50 MB L2 next to the streams
static bool k_out_direct(int64_t n_positions) {
  static int64_t thr = -1;
  if (thr < 0) { const char* e = getenv("KVQ_KOUT_DIRECT_NPOS"); thr = e ? atoll(e) : 64 * 1024; }
  return n_positions > thr;
}

// zero_first = 1: `out` is a fresh score buffer (fused path) and is cleared before the scatter
static int launch_k_outliers(const KParams& p, int zero_first, float scale, cudaStream_t st) {
  if (zero_first) {
    cudaError_t e = p.opart != nullptr
        ? cudaMemsetAsync(const_cast<float*>(p.opart), 0, sizeof(float) * (size_t)p.L * (size_t)p.opart_stride, st)
        : cudaMemsetAsync(p.out, 0, sizeof(float) * (size_t)p.H * (size_t)p.out_stride, st);
    if (e != cudaSuccess) return (int)e;
  }
  const int64_t total = p.L * p.n_out;
  const size_t smem = (size_t)p.H * kHeadDim * sizeof(float2);
  if (k_out_impl_table() || smem > 100 * 1024 || total >= ((int64_t)1 << 31) || p.L >= ((int64_t)1 << 25)) {
    if (p.len_dev != nullptr || p.opart != nullptr) return KVQ_E_UNSUPPORTED;   // host length, head-major target only
    const unsigned grid = (unsigned)((total + kOutThreads - 1) / kOutThreads);
    k_outlier_kernel<<<grid, kOutThreads, 0, st>>>(p.q, p.outliers, p.outlier_idx, p.out, p.out_stride, p.L, p.H,
                                                   p.n_out, p.rope, p.rope_npos, p.pos_offset, scale);
    KVQ_LAUNCH_CHECK();
    return 0;
  }
  static size_t smem_set_dev[64];   // per device: largest dynamic shared memory opted in so far (0 = default 48 KiB)
  int dev_idx = 0;
  cudaGetDevice(&dev_idx);
  size_t& smem_set = smem_set_dev[dev_idx & 63];
  if (smem_set == 0) smem_set = 48 * 1024;
  if (smem > smem_set) {
    cudaError_t e = cudaFuncSetAttribute(k_outlier_pers_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    smem_set = smem;
  }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t want = (total + kOutPersThreads - 1) / kOutPersThreads;
  const int per_sm = smem > 56 * 1024 ? 2 : 4;
  const unsigned grid = (unsigned)(want < (int64_t)sms * per_sm ? want : (int64_t)sms * per_sm);
  // token-major target (fused path): a token's heads share one 128-byte line, so a warp's ~25 reductions (one or
  // two tokens) coalesce into one or two L1 requests instead of one per head row
  float* dst = p.opart != nullptr ? const_cast<float*>(p.opart) : p.out;
  const int64_t sh = p.opart != nullptr ? 1 : p.out_stride, stt = p.opart != nullptr ? p.opart_stride : 1;
  k_outlier_pers_kernel<<<grid, kOutPersThreads, smem, st>>>(p.q, p.outliers, p.outlier_idx, dst, sh, stt, p.L,
                                                             p.H, p.n_out, p.rope, p.rope_npos, p.pos_offset, scale,
                                                             p.len_dev, p.len_add, p.rope_h,
                                                             k_out_direct(p.L + p.pos_offset) ? p.theta : 0.f);
  KVQ_LAUNCH_CHECK();
  return 0;
}

// rope table: reference expressions quant_cuda_kernel.cu:3081 (theta) and 3123-3126 (cos/sin), once per (j, p)
__global__ void rope_table_kernel(float2* __restrict__ out, float rope_theta, int64_t n_pos) {
  const int j = blockIdx.y;
  const int headdim = kHeadDim;
  const int headdim2 = headdim / 2;
  const float theta = powf(rope_theta, (-2 * __int2float_rd(j % headdim2) / __int2float_rd(headdim)));
  for (int64_t pos64 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pos64 < n_pos; pos64 += (int64_t)gridDim.x * blockDim.x) {
    const int pos = (int)pos64;
    const float c = cosf(theta * pos);
    const float s = sinf(theta * pos);
    out[(int64_t)j * n_pos + pos64] = make_float2(c, s);
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
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
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

// KVQ_K_IMPL selects the dense kernel for A/B runs.  Default: 4-bit / 2-bit -> k_scores_kernel (this file),
// 3-bit -> k_scores3_kernel (kvq_k3.cu).  "generic": k_scores_kernel for every width; "pair": pair-table form
// (kvq_kpair.cu, 4/3-bit); "kappa": 4-byte entries + constant-bank q.  Measurements: DESIGN.md section 4.1.
static int k_impl() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("KVQ_K_IMPL");
    v = !e ? 0 : (e[0] == 'g' ? 1 : (e[0] == 'p' ? 2 : (e[0] == 'k' ? 3 : 0)));
  }
  return v;
}

int k_scores_dispatch(int bits, const KParams& p, cudaStream_t st) {
  const int impl = p.len_dev != nullptr ? 0 : k_impl();   // the A/B variants take their length from the host
  if (impl == 0 && bits == 3) return k_scores3_dispatch(p, st);
  if (impl == 2 && (bits == 4 || bits == 3)) return k_pair_dispatch(bits, p, st);
  if (impl == 3 && p.H <= kMaxConstHeads) {
    switch (bits) {
      case 4: return launch_k_kappa<4>(p, st);
      case 3: return launch_k_kappa<3>(p, st);
      case 2: return launch_k_kappa<2>(p, st);
      default: return KVQ_E_BITS;
    }
  }
  switch (bits) {
    case 4: return launch_k_scores<4>(p, st);
    case 3: return launch_k_scores<3>(p, st);
    case 2: return launch_k_scores<2>(p, st);
    default: return KVQ_E_BITS;
  }
}

int k_scores_fused(int bits, const float* q, const int32_t* cache, float* scores, int64_t score_stride,
                   const float* lut, const float* outliers, const int32_t* outlier_idx, int n_out, int H,
                   int64_t Lmax, int64_t L, const float* rope, int64_t rope_npos, float theta, int pos_offset,
                   float* gmax, float scale, const int64_t* len_dev, int64_t len_add, float* opart, int opart_stride,
                   cudaStream_t st) {
  KParams p{};
  p.len_dev = len_dev; p.len_add = len_add;
  p.q = q; p.cache = reinterpret_cast<const uint32_t*>(cache); p.out = scores; p.lut = lut;
  p.outliers = outliers; p.outlier_idx = outlier_idx; p.rope = reinterpret_cast<const float2*>(rope);
  p.gmax = gmax; p.Lmax = Lmax; p.L = L; p.out_stride = score_stride; p.rope_npos = rope_npos;
  p.H = H; p.n_out = n_out; p.pos_offset = pos_offset; p.scale = scale; p.accumulate = 0; p.theta = theta;
  if (outliers != nullptr) {
    // outlier contributions are deposited UNSCALED (the dense kernel applies `scale` to partial + S), token-major
    // when the caller provides the partial buffer (and the variant in use supports it)
    const bool tm = opart != nullptr && !k_out_impl_table() && k_impl() == 0;
    if (tm) { p.opart = opart; p.opart_stride = opart_stride; }
    const int rc = launch_k_outliers(p, /*zero_first=*/1, 1.f, st);
    if (rc != 0) return rc;
    if (!tm) p.accumulate = 1;
  }
  return k_scores_dispatch(bits, p, st);
}

// K side of the fused attend: outlier scatter straight into the head-major score buffer (cleared first), then the
// TMA-fed dense kernel folds it in: out = (partial + S) * scale.  rope_half == null: exact fp32 ratio form
// (kvq_kratio.cu); otherwise the fp16-table form (kvq_kfast.cu).
int k_scores_fused_fast(int bits, const float* q, const int32_t* cache, float* scores, int64_t score_stride,
                        const float* lut, const float* outliers, const int32_t* outlier_idx, int n_out, int H,
                        int64_t Lmax, int64_t L, const float* rope, const void* rope_half, int64_t rope_npos, float theta,
                        int pos_offset, float* gmax, float scale, const int64_t* len_dev, int64_t len_add, void* qtab,
                        cudaStream_t st) {
  // KVQ_K_BLOCK=<tokens>: walk the cache in blocks whose score rows (H x block floats) stay L2-resident between the
  // outlier scatter (atomic adds) and the dense kernel.  The default is ONE pass; the switch stays for A/B runs and is
  // covered by tests/test_gpu_variants.py.
  static int64_t kBlock = 0;
  if (kBlock == 0) {
    const char* e = getenv("KVQ_K_BLOCK");
    kBlock = e ? (atoll(e) + 31) / 32 * 32 : ((int64_t)1 << 40);
    if (kBlock < 32) kBlock = (int64_t)1 << 40;
  }
  int run_prep = 1;
  for (int64_t t0 = 0; t0 < L; t0 += kBlock) {
    const int64_t Lb = (L - t0 > kBlock + kBlock / 2) ? kBlock : (L - t0);   // the last block may be up to 1.5 blocks
    int accumulate = 0;
    if (outliers != nullptr) {
      KParams p{};
      p.len_dev = len_dev; p.len_add = len_add - t0;
      p.q = q; p.out = scores + t0; p.outliers = outliers + t0 * n_out; p.outlier_idx = outlier_idx + t0 * n_out;
      p.rope = reinterpret_cast<const float2*>(rope); p.rope_h = static_cast<const uint32_t*>(rope_half);
      p.Lmax = Lmax; p.L = Lb; p.out_stride = score_stride; p.rope_npos = rope_npos;
      p.H = H; p.n_out = n_out; p.pos_offset = pos_offset + (int)t0; p.theta = theta;
      cudaError_t e = cudaMemset2DAsync(scores + t0, sizeof(float) * (size_t)score_stride, 0, sizeof(float) * (size_t)Lb, (size_t)H, st);
      if (e != cudaSuccess) return (int)e;
      const int rc = launch_k_outliers(p, /*zero_first=*/0, 1.f, st);
      if (rc != 0) return rc;
      accumulate = 1;
    }
    const int rc = (rope_half == nullptr)     // exact mode: fp32 ratio form (kvq_kratio.cu); else the fp16-table form
        ? k_ratio_dispatch(bits, q, cache, scores, score_stride, lut, H, Lmax, Lb, rope, rope_npos, pos_offset, gmax, scale,
                           accumulate, len_dev, len_add, qtab, t0, run_prep, st)
        : k_fast_dispatch(bits, q, cache, scores, score_stride, lut, H, Lmax, Lb, rope_half, rope_npos, pos_offset, gmax,
                          scale, accumulate, len_dev, len_add, qtab, t0, run_prep, st);
    if (rc != 0) return rc;
    run_prep = 0;
    if (Lb != kBlock) break;
  }
  return 0;
}

}  // namespace kvq

using namespace kvq;

extern "C" {

int kvq_rope_table_build(float* rope_cos_sin, float theta, int64_t n_pos, void* stream) {
  if (!rope_cos_sin) return KVQ_E_NULL;
  if (n_pos <= 0 || n_pos > (int64_t)1 << 30) return KVQ_E_SHAPE;
  const dim3 grid((unsigned)((n_pos + 255) / 256 > 4096 ? 4096 : (n_pos + 255) / 256), kHalf);
  rope_table_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<float2*>(rope_cos_sin), theta, n_pos);
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
    p.gmax = nullptr;
    p.Lmax = Lmax; p.L = L; p.out_stride = L; p.rope_npos = rope_npos;
    p.H = H; p.n_out = n_out; p.pos_offset = pos_offset;
    p.scale = 1.f; p.accumulate = 1; p.theta = theta;
    if (outliers != nullptr) {
      const int rc0 = launch_k_outliers(p, /*zero_first=*/0, 1.f, static_cast<cudaStream_t>(stream));
      if (rc0 != 0) return rc0;
    }
    const int rc = k_scores_dispatch(bits, p, static_cast<cudaStream_t>(stream));
    if (rc != 0) return rc;
  }
  return 0;
}

}  // extern "C"
