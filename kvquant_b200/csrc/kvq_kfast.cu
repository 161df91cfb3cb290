// kvquant_b200 -- Q.K^T decode matvec of the fused attend, fp16-table form (opt-in: kvq_attend with rope_half != NULL;
// the default is the exact ratio form, kvq_kratio.cu).
//
// Replaces (reference deployment/kvquant/quant_cuda_kernel.cu):
//   VecQuant{4,3,2}MatMulKernelNUQPerChannelTransposedRopeMHABatchedFusedOpt   3040-3209, 3692-4115, 4747-4996
//
//   S[h,t] = sum_c LUT[h,c,code(h,c,t)] * (cos(th_j p) q[h,c] + s_c sin(th_j p) q[h,(c+64)%128]),  j = c % 64, p = t + off
//
// What bounded the fp32 kernels (kvq_kscore.cu / kvq_k3.cu) was the SM's shared-memory data path: an 8-byte table
// entry per element costs two 128-byte wavefronts per warp lookup (ncu: 78-86 % busy).  north_star asks for an fp16
// LUT and a 1e-3 tolerance (measured: within 1e-3 at a few thousand tokens, 1.4e-3 .. 2.2e-3 at 128K -- which is why
// this form is opt-in), so here
//   * the premultiplied table T[h][c][code] = half2(LUT*q_c, s_c*LUT*q_{c^64}) is built ONCE per call by a prep
//     kernel (k_fast_prep_kernel) and bulk-copied into shared memory (cp.async.bulk): one LDS.32 = one wavefront per
//     warp lookup, and G = 16 (4-bit) / 32 (3-, 2-bit) heads share one CTA, so a token's cos/sin are loaded once per
//     16-32 heads instead of once per 8;
//   * cos/sin come from a half2 copy of the rope table (same reference expressions, rounded once), held in
//     registers for all 64 pairs of the thread's token; products are exact in fp32 and accumulate in fp32 (each
//     half is widened to fp32, then one FFMA);
//   * the packed codes reach shared memory by TMA (cp.async.bulk.tensor.2d boxes of [W rows x 64 tokens], four per
//     head slab) through a 5-8 stage full/empty mbarrier ring filled by a producer warp: 64+ KiB in flight per SM
//     without spending registers or issue slots on global loads; a warp = 16 tokens x 2 channel halves, warps drift
//     apart by up to a ring.
// Per element: 1 PRMT (3-bit: SHF+LOP3) + 1 LDS.32 + 2 half->float conversions + 2 FFMA.
#include "kvq_kscore.cuh"
#include "kvq_attend.cuh"
#include <cuda_fp16.h>

namespace kvq {

constexpr int kKFWarps = 16;                       // consumer warps (16 tokens x 2 channel halves per warp column)
constexpr int kKFColTok = 16;                      // tokens per warp column
constexpr int kKFThreads = kKFWarps * 32 + 32;     // + one producer warp
constexpr uint32_t kKFSmemBudget = 227u * 1024u;

struct KFParams {
  const uint32_t* qtab;      // half2 [H][128][N] premultiplied table (k_fast_prep_kernel)
  const uint32_t* rope_h;    // half2 [64][rope_npos] (cos, sin)
  float* out;                // [H][out_stride]
  float* gmax;               // [H] or null
  int64_t Lmax, L, out_stride, rope_npos, range;
  int64_t t0;                // always 0.  The kernel adds it to its token range because ptxas then schedules it
                             // faster: without it the 4-bit fp16-table attend at 128K (7B shapes) takes 0.448 instead
                             // of 0.430 ms on an H100 80GB HBM3 (SXM, 700 W)
  const int64_t* len_dev;
  int64_t len_add;
  int H, G, pos_offset, accumulate, n_stages;
  float scale;
};

template <int BITS> struct KFCfg {
  static constexpr int N = 1 << BITS;
  static constexpr int W = Layout<BITS>::kWords;
  static constexpr int GMAX = (BITS == 4) ? 16 : 32;       // heads per CTA: table = G * 128 * N * 4 bytes <= 128 KiB
  static constexpr uint32_t kHeadTab = kHeadDim * N * 4;   // bytes of one head's table
  static constexpr int kBoxWarps = 4;                      // one TMA box: W rows x 64 tokens (4 warp columns of 16)
  static constexpr uint32_t kBox = W * kKFColTok * 4 * kBoxWarps;
  static constexpr uint32_t kStage = (kKFWarps / kBoxWarps) * kBox;   // one slab = one head x 16 warp columns = 256 tokens
};

// acc += a.h{0,1} * b.h{0,1}: fp16 -> fp32 is exact and so is the product of two fp16 in fp32, so widening first and
// one fp32 FMA round exactly as a mixed-precision fp16 x fp16 + fp32 FMA would (sm_90 has no such instruction)
__device__ __forceinline__ void fhfma_lo(float& acc, uint32_t a, uint32_t b) {
  acc = __fmaf_rn(__low2float(*reinterpret_cast<const __half2*>(&a)), __low2float(*reinterpret_cast<const __half2*>(&b)), acc);
}
__device__ __forceinline__ void fhfma_hi(float& acc, uint32_t a, uint32_t b) {
  acc = __fmaf_rn(__high2float(*reinterpret_cast<const __half2*>(&a)), __high2float(*reinterpret_cast<const __half2*>(&b)), acc);
}
template <int IMM> __device__ __forceinline__ uint32_t lds_u32i(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(IMM));
  return v;
}
// table read that keeps its place in the instruction stream (the hand-pipelined loops rely on the source order)
template <int IMM> __device__ __forceinline__ uint32_t lds_tabv(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(IMM));
  return v;
}
template <int IMM> __device__ __forceinline__ uint32_t lds_tab(uint32_t addr) {   // table reads: not volatile
  uint32_t v;
  asm("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(IMM));
  return v;
}
__device__ __forceinline__ uint32_t ld_keep_u32(const uint32_t* p, uint64_t pol) {
  uint32_t v;
  asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}

// One head, this lane's half of one token.  A warp covers 16 tokens x 2 halves: lane = half * 16 + token, half 0 owns
// the even channels of the head, half 1 the odd ones (even- and odd-channel tables sit in disjoint banks, and both
// halves read the same packed word -> a broadcast), so a thread keeps cos/sin of only 32 pairs in registers and the
// compiler has room to keep many lookups in flight (the 64-pair form stalls on shared-memory latency).  The two halves meet in one shuffle per head.
//   st   = shared address of this lane's token column in the slab (row r at st + r * kRow)
//   base = shared address of the head's table (256-byte aligned)
//   hs   = per-lane constants of its half (see KFHalf)
//   cs[i] = half2 (cos, sin) of this lane's i-th pair
struct KFHalf {
  uint32_t half;     // 0 / 1
  uint32_t rot;      // 4-bit: left-rotation that brings this half's nibbles to bits 2..5 of each byte (2 / 30)
  uint32_t bias;     // byte-replicated offset of the odd channel's table (one channel = 64 / 32 / 16 bytes)
};
constexpr int kKFRow = 256;   // bytes between packed-word rows inside a TMA box (64 tokens)

template <int BITS>
__device__ __forceinline__ float k_fast_head(const uint32_t st, const uint32_t base, const KFHalf hs, const uint32_t (&cs)[32]) {
  float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
  constexpr int kRow = kKFRow;
  if constexpr (BITS == 4) {
    // software-pipelined by hand: the 8 lookups of word pair w+1 are issued before the 16 FMAs of word pair w, so
    // that a warp always has 8-16 shared-memory loads in flight (ptxas left to itself keeps 2-4: ncu showed the warps
    // waiting on the short scoreboard most of the time)
    uint32_t xs[2][4], ys[2][4];
    auto issue = [&](auto iw, uint32_t (&x)[4], uint32_t (&y)[4]) {
      constexpr int w = decltype(iw)::v;          // word w: channels 8w..8w+7, word w+8: their rotary partners
      const uint32_t wa = lds_u32i<w * kRow>(st), wb = lds_u32i<(w + 8) * kRow>(st);
      // byte b <- (code 2b + half) * 4 + half * 64   (the rotation wraps only into masked-out bits)
      const uint32_t ma = (__funnelshift_l(wa, wa, hs.rot) & 0x3C3C3C3Cu) | hs.bias;
      const uint32_t mb = (__funnelshift_l(wb, wb, hs.rot) & 0x3C3C3C3Cu) | hs.bias;
      static_for<0, 4>([&](auto ik) {
        constexpr int k = decltype(ik)::v;         // channel 8w + 2k + half
        x[k] = lds_tabv<(8 * w + 2 * k) * 64>(__byte_perm(ma, base, 0x7650 | k));
        y[k] = lds_tabv<(8 * w + 2 * k + kHalf) * 64>(__byte_perm(mb, base, 0x7650 | k));
      });
    };
    auto consume = [&](auto iw, const uint32_t (&x)[4], const uint32_t (&y)[4]) {
      constexpr int w = decltype(iw)::v;
      static_for<0, 4>([&](auto ik) {
        constexpr int k = decltype(ik)::v;
        constexpr int i = 4 * w + k;
        fhfma_lo(a0, x[k], cs[i]); fhfma_hi(a1, x[k], cs[i]);
        fhfma_lo(b0, y[k], cs[i]); fhfma_hi(b1, y[k], cs[i]);
      });
    };
    issue(IC<0>{}, xs[0], ys[0]);
    static_for<0, 8>([&](auto iw) {
      constexpr int w = decltype(iw)::v;
      if constexpr (w + 1 < 8) issue(IC<w + 1>{}, xs[(w + 1) & 1], ys[(w + 1) & 1]);
      consume(iw, xs[w & 1], ys[w & 1]);
    });
  } else if constexpr (BITS == 2) {
    static_for<0, 4>([&](auto iw) {
      constexpr int w = decltype(iw)::v;          // word w: channels 16w..16w+15, word w+4: partners
      const uint32_t wa = lds_u32i<w * kRow>(st) >> (2 * hs.half), wb = lds_u32i<(w + 4) * kRow>(st) >> (2 * hs.half);
      // code 2k + half now sits at bits 4k of the shifted word: byte k>>1, bits 0..1 (k even) / 4..5 (k odd)
      const uint32_t ma[2] = {((wa << 2) & 0x0C0C0C0Cu) | hs.bias, ((wa >> 2) & 0x0C0C0C0Cu) | hs.bias};
      const uint32_t mb[2] = {((wb << 2) & 0x0C0C0C0Cu) | hs.bias, ((wb >> 2) & 0x0C0C0C0Cu) | hs.bias};
      static_for<0, 8>([&](auto ik) {
        constexpr int k = decltype(ik)::v;         // channel 16w + 2k + half
        constexpr int i = 8 * w + k;
        const uint32_t x = lds_tab<(16 * w + 2 * k) * 16>(__byte_perm(ma[k & 1], base, 0x7650 | (k >> 1)));
        const uint32_t y = lds_tab<(16 * w + 2 * k + kHalf) * 16>(__byte_perm(mb[k & 1], base, 0x7650 | (k >> 1)));
        fhfma_lo(a0, x, cs[i]); fhfma_hi(a1, x, cs[i]);
        fhfma_lo(b0, y, cs[i]); fhfma_hi(b1, y, cs[i]);
      });
    });
  } else {
    const uint32_t hb = base | hs.bias;            // bias = half * 32: bit 5, clear of the code bits 2..4
    // the six words of groups g (channels 32g..) and g+2 (their rotary partners), then the same hand pipelining over
    // the eight 24-bit windows
    uint32_t wa[2][3], wb[2][3];
    static_for<0, 2>([&](auto ig) {
      constexpr int g = decltype(ig)::v;
      wa[g][0] = lds_u32i<(3 * g) * kRow>(st); wa[g][1] = lds_u32i<(3 * g + 1) * kRow>(st); wa[g][2] = lds_u32i<(3 * g + 2) * kRow>(st);
      wb[g][0] = lds_u32i<(3 * g + 6) * kRow>(st); wb[g][1] = lds_u32i<(3 * g + 7) * kRow>(st); wb[g][2] = lds_u32i<(3 * g + 8) * kRow>(st);
    });
    uint32_t xs[2][4], ys[2][4];
    auto window = [&](const uint32_t (&w)[3], auto ia) -> uint32_t {
      constexpr int a = decltype(ia)::v;           // 24-bit window a of a 96-bit group
      return (a == 0 ? w[0] : (a == 1 ? __funnelshift_r(w[0], w[1], 24) : (a == 2 ? __funnelshift_r(w[1], w[2], 16) : (w[2] >> 8))))
             >> (3 * hs.half);                     // this half's codes now sit at bits 6k
    };
    auto issue = [&](auto iv, uint32_t (&x)[4], uint32_t (&y)[4]) {
      constexpr int v = decltype(iv)::v, g = v >> 2, a = v & 3;   // channels 32g + 8a .. +7
      const uint32_t x0 = window(wa[g], IC<a>{}), x1 = window(wb[g], IC<a>{});
      static_for<0, 4>([&](auto ik) {
        constexpr int k = decltype(ik)::v;         // channel 32g + 8a + 2k + half
        const uint32_t ax = ((k == 0 ? (x0 << 2) : (x0 >> (6 * k - 2))) & 0x1Cu) | hb;
        const uint32_t ay = ((k == 0 ? (x1 << 2) : (x1 >> (6 * k - 2))) & 0x1Cu) | hb;
        x[k] = lds_tabv<(32 * g + 8 * a + 2 * k) * 32>(ax);
        y[k] = lds_tabv<(32 * g + 8 * a + 2 * k + kHalf) * 32>(ay);
      });
    };
    auto consume = [&](auto iv, const uint32_t (&x)[4], const uint32_t (&y)[4]) {
      constexpr int v = decltype(iv)::v;
      static_for<0, 4>([&](auto ik) {
        constexpr int k = decltype(ik)::v;
        constexpr int i = 4 * v + k;               // = 16g + 4a + k
        fhfma_lo(a0, x[k], cs[i]); fhfma_hi(a1, x[k], cs[i]);
        fhfma_lo(b0, y[k], cs[i]); fhfma_hi(b1, y[k], cs[i]);
      });
    };
    issue(IC<0>{}, xs[0], ys[0]);
    static_for<0, 8>([&](auto iv) {
      constexpr int v = decltype(iv)::v;
      if constexpr (v + 1 < 8) issue(IC<v + 1>{}, xs[(v + 1) & 1], ys[(v + 1) & 1]);
      consume(iv, xs[v & 1], ys[v & 1]);
    });
  }
  return (a0 + b0) + (a1 + b1);
}
// pair index of this lane's i-th (cos, sin) register
template <int BITS> __device__ __forceinline__ int k_fast_pair(int i, int half) {
  if constexpr (BITS == 4) return 8 * (i >> 2) + 2 * (i & 3) + half;          // i = 4w + k
  else if constexpr (BITS == 2) return 16 * (i >> 3) + 2 * (i & 7) + half;    // i = 8w + k
  else return 2 * i + half;                                                    // i = 16g + 4a + k -> 32g + 8a + 2k
}

template <int BITS>
__global__ void __launch_bounds__(kKFThreads, 1) k_fast_kernel(const __grid_constant__ CUtensorMap tmap, const KFParams p) {
  using C = KFCfg<BITS>;
  constexpr int W = C::W;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int S = p.n_stages;
  const int h0 = blockIdx.y * p.G;
  const int nh = min(p.G, p.H - h0);
  const uint32_t tab_bytes = (uint32_t)nh * C::kHeadTab;
  const uint32_t tab_span = (uint32_t)p.G * C::kHeadTab;
  unsigned char* s_tab = smem;                                         // [G][128][N] half2
  unsigned char* s_stage = smem + tab_span;                            // [S][4 boxes][W][64] u32
  uint64_t* s_full = reinterpret_cast<uint64_t*>(s_stage + (size_t)S * C::kStage);
  uint64_t* s_empty = s_full + S;
  uint64_t* s_tabbar = s_empty + S;
  int* s_max = reinterpret_cast<int*>(s_tabbar + 1);                    // [G] running max (ordered-int encoding)

  // token range of this CTA (multiple of 32; device-resident length re-derives it)
  int64_t L_eff = p.L;
  int64_t range = p.range;
  if (p.len_dev != nullptr) {
    const int64_t l = *p.len_dev + p.len_add - p.t0;
    L_eff = l < 0 ? 0 : (l < p.L ? l : p.L);
    const int64_t r = (L_eff + gridDim.x - 1) / gridDim.x;
    range = (r + 31) & ~(int64_t)31;
  }
  const int64_t t_begin = p.t0 + (int64_t)blockIdx.x * range;
  const int64_t t_limit = p.t0 + min(L_eff, ((int64_t)blockIdx.x + 1) * range);
  if (t_begin >= t_limit) return;
  const int ncols = (int)((t_limit - t_begin + kKFColTok - 1) / kKFColTok);      // 16-token warp columns
  const int nrounds = (ncols + kKFWarps - 1) / kKFWarps;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(&s_full[s], 1); mbar_init(&s_empty[s], kKFWarps); }
    mbar_init(s_tabbar, 1);
    mbar_fence_init();
  }
  if (tid < p.G) s_max[tid] = (int)(0xFF800000u ^ 0x7FFFFFFFu);   // -inf in the ordered-int encoding
  __syncthreads();

  if (warp == kKFWarps) {
    // ---------------- producer warp: table, then the slab ring ------------------------------------------------------
    if (lane == 0) {
      prefetch_tensormap(&tmap);
      mbar_expect_tx(s_tabbar, tab_bytes);
      const unsigned char* src = reinterpret_cast<const unsigned char*>(p.qtab) + (size_t)h0 * C::kHeadTab;
      for (uint32_t o = 0; o < tab_bytes; o += 16384u)
        bulk_load_1d(s_tab + o, src + o, min(16384u, tab_bytes - o), s_tabbar);
      int s = 0;
      uint32_t ph = 1;   // parity of the previous use of stage s (first pass: nothing to wait for)
      bool wrapped = false;
      for (int r = 0; r < nrounds; ++r) {
        const int nlive = min(kKFWarps, ncols - r * kKFWarps);
        const int nbox = (nlive + C::kBoxWarps - 1) / C::kBoxWarps;    // the last box may reach past the range: read-only
        const int x0 = (int)(t_begin + (int64_t)r * kKFWarps * kKFColTok);
        for (int hl = 0; hl < nh; ++hl) {
          if (wrapped) mbar_wait(&s_empty[s], ph);
          mbar_expect_tx(&s_full[s], (uint32_t)nbox * C::kBox);
          unsigned char* dst = s_stage + (size_t)s * C::kStage;
          for (int b = 0; b < nbox; ++b)
            tma_load_2d(dst + (size_t)b * C::kBox, &tmap, &s_full[s], x0 + kKFColTok * C::kBoxWarps * b, (h0 + hl) * W);
          if (++s == S) { s = 0; ph ^= 1u; wrapped = true; }
        }
      }
    }
    return;
  }

  // ---------------- consumer warps: lane = half * 16 + token ---------------------------------------------------------
  const uint64_t pol_keep = policy_evict_last();
  const uint32_t tab0 = smem_u32(s_tab);
  const int tl = lane & 15;
  KFHalf hs;
  hs.half = (uint32_t)lane >> 4;
  hs.rot = hs.half ? 30u : 2u;
  hs.bias = hs.half * (BITS == 4 ? 0x40404040u : (BITS == 2 ? 0x10101010u : 0x20u));
  // this lane's token column inside the slab: box warp/4, token (warp%4)*16 + tl; rows are kKFRow bytes apart
  const uint32_t stage0 = smem_u32(s_stage) + (uint32_t)(warp / C::kBoxWarps) * C::kBox +
                          (uint32_t)((warp % C::kBoxWarps) * kKFColTok + tl) * 4u;
  mbar_wait(s_tabbar, 0);
  int s = 0;
  uint32_t ph = 0;
  for (int r = 0; r < nrounds; ++r) {
    const int col = r * kKFWarps + warp;
    const bool live = col < ncols;                       // warp-uniform
    const int64_t t = t_begin + (int64_t)col * kKFColTok + tl;
    const bool mine = live && t < t_limit;
    uint32_t cs[32];
    if (live) {
      const uint32_t* rp = p.rope_h + (mine ? (t + p.pos_offset) : 0);
#pragma unroll
      for (int i = 0; i < 32; ++i)
        cs[i] = mine ? ld_keep_u32(rp + (int64_t)k_fast_pair<BITS>(i, (int)hs.half) * p.rope_npos, pol_keep) : 0u;
    }
    for (int hl = 0; hl < nh; ++hl) {
      float* optr = p.out + (int64_t)(h0 + hl) * p.out_stride + t;
      float old = 0.f;
      if (p.accumulate && mine && hs.half == 0) old = __ldcg(optr);
      mbar_wait(&s_full[s], ph);
      if (live) {
        float acc = k_fast_head<BITS>(stage0 + (uint32_t)s * C::kStage, tab0 + (uint32_t)hl * C::kHeadTab, hs, cs);
        acc += __shfl_xor_sync(0xffffffffu, acc, 16);    // even + odd channels
        const float sc = (acc + old) * p.scale;
        if (mine && hs.half == 0) *optr = sc;
        if (p.gmax != nullptr) {
          // warp max in ONE instruction: floats compare like their bit patterns once the negative range is mirrored
          // (REDUX.MAX.S32); s_max keeps the same ordered-int encoding
          const int bits = __float_as_int((mine && hs.half == 0) ? sc : -INFINITY);
          const int key = __reduce_max_sync(0xffffffffu, bits >= 0 ? bits : (bits ^ 0x7FFFFFFF));
          if (lane == 0) atomicMax(&s_max[hl], key);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&s_empty[s]);
      if (++s == S) { s = 0; ph ^= 1u; }
    }
  }
  if (p.gmax != nullptr) {
    asm volatile("bar.sync 1, %0;" ::"n"(kKFWarps * 32) : "memory");
    if (tid < nh) {
      const int key = s_max[tid];
      const float m = __int_as_float(key >= 0 ? key : (key ^ 0x7FFFFFFF));
      if (m > -INFINITY) atomic_max_float(p.gmax + h0 + tid, m);
    }
  }
}

// premultiplied table T[h][c][code] = half2(LUT q_c, s_c LUT q_{c^64}); grid = H, block = 128 (thread = channel)
template <int BITS>
__global__ void k_fast_prep_kernel(const float* __restrict__ q, const float* __restrict__ lut, uint32_t* __restrict__ qtab) {
  constexpr int N = 1 << BITS;
  const int h = blockIdx.x, c = threadIdx.x;
  const float qa = q[h * kHeadDim + c];
  const float qb = q[h * kHeadDim + (c ^ kHalf)];
  const float sg = (c < kHalf) ? 1.f : -1.f;
  const float* l = lut + ((int64_t)h * kHeadDim + c) * N;
  uint32_t* o = qtab + ((int64_t)h * kHeadDim + c) * N;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    const float v = l[i];
    const float t1 = fminf(fmaxf(v * qa, -65504.f), 65504.f);
    const float t2 = fminf(fmaxf(sg * (v * qb), -65504.f), 65504.f);
    const __half2 e = __floats2half2_rn(t1, t2);
    o[i] = *reinterpret_cast<const uint32_t*>(&e);
  }
}

template <int BITS>
static int launch_k_fast(KFParams p, const float* q, const float* lut, uint32_t* qtab, const int32_t* cache,
                         cudaStream_t st) {
  using C = KFCfg<BITS>;
  k_fast_prep_kernel<BITS><<<p.H, kHeadDim, 0, st>>>(q, lut, qtab);
  KVQ_LAUNCH_CHECK();
  const int groups = (p.H + C::GMAX - 1) / C::GMAX;
  p.G = (p.H + groups - 1) / groups;
  const uint32_t tab_span = (uint32_t)p.G * C::kHeadTab;
  const uint32_t fixed = tab_span + 1024u /*align*/ + 8u * 20u + 4u * 64u + 64u;
  int S = (int)((kKFSmemBudget - fixed) / C::kStage);
  if (S > 8) S = 8;
  if (S < 2) return KVQ_E_UNSUPPORTED;
  p.n_stages = S;
  const size_t smem = (size_t)tab_span + (size_t)S * C::kStage + 8u * (2 * S + 1) + 4u * p.G + 1024u;
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(k_fast_kernel<BITS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kKFSmemBudget);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  CUtensorMap tmap;
  int rc = make_cache_tensor_map(&tmap, cache, (uint64_t)p.H * C::W, (uint64_t)p.Lmax, kKFColTok * C::kBoxWarps, C::W, /*swizzle*/ 0);
  if (rc != 0) return rc;
  const int sms = num_sms_cached();
  const int64_t max_splits = sms / groups > 0 ? sms / groups : 1;
  p.range = k_token_range(p.L, max_splits);
  const int64_t splits = (p.L + p.range - 1) / p.range;
  k_fast_kernel<BITS><<<dim3((unsigned)splits, (unsigned)groups), kKFThreads, smem, st>>>(tmap, p);
  KVQ_LAUNCH_CHECK();
  return 0;
}

// dense K scores of the fused attend, fp16-table form.  s.scores holds the (unscaled) outlier partial sums on entry
// when accumulate != 0.
int k_fast_dispatch(const AttendCall& c, const AttendScratch& s, int accumulate) {
  KFParams p{};
  uint32_t* qtab = reinterpret_cast<uint32_t*>(s.qtab);
  p.qtab = qtab;
  p.rope_h = static_cast<const uint32_t*>(c.rope_half);
  p.out = s.scores; p.gmax = s.gmax;
  p.Lmax = c.Lmax; p.L = c.L; p.out_stride = s.stride; p.rope_npos = c.rope_npos;
  p.len_dev = c.len_dev; p.len_add = c.len_add;
  p.H = c.Hq; p.pos_offset = c.pos_offset; p.accumulate = accumulate; p.scale = kAttendScale;
  switch (c.bits) {
    case 4: return launch_k_fast<4>(p, c.q, c.klut, qtab, c.kcache, c.stream);
    case 3: return launch_k_fast<3>(p, c.q, c.klut, qtab, c.kcache, c.stream);
    case 2: return launch_k_fast<2>(p, c.q, c.klut, qtab, c.kcache, c.stream);
    default: return KVQ_E_BITS;
  }
}

}  // namespace kvq
