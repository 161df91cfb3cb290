// kvquant_b200 -- dense Q.K^T decode matvec, PAIR-TABLE form (4-bit and 3-bit).
//
// Replaces (reference deployment/kvquant/quant_cuda_kernel.cu):
//   VecQuant{4,3}MatMulKernelNUQPerChannelTransposedRopeMHABatchedFusedOpt   3040-3209, 3692-4115
//
//   S[h,t] = sum_j  cos(th_j p) * (A q_j + B q_j64)  +  sin(th_j p) * (A q_j64 - B q_j)        p = t + pos_offset
//            A = LUT[h, j, code(h, j, t)],  B = LUT[h, j+64, code(h, j+64, t)],  q_j = q[h, j], q_j64 = q[h, j+64]
//
// which is the reference's per-channel sum with the two channels that share a rotary pair (j, j+64) taken together.
//
// Why: the per-channel form (kvq_kscore.cu) costs one 8-byte shared-memory lookup per ELEMENT and the SM's
// load/store data path (one 128-byte wavefront per clock) is what bounds it.
// Here one lookup serves a PAIR: the table is indexed by both codes,
//   T[h][j][a | b << BITS] = (A q_j + B q_j64,  A q_j64 - B q_j)            256 (4-bit) / 64 (3-bit) entries,
// so an element costs half a lookup, one FFMA and ~1 address op.  The tables of all 64 pairs x 8 heads would
// need 1 MiB (4-bit) / 256 KiB (3-bit), so a CTA walks its token range in P passes over PP pairs each (8 x 8 pairs /
// 2 x 32 pairs), rebuilding the 128 KiB table between passes; the running sum travels through the score buffer
// (the thread that owns column t writes it and reads it back in the next pass: no atomics, deterministic).
//
//   * thread = token, 512-token tiles, G = 8 heads per CTA, grid = (SMs / head groups token ranges) x (H / 8 head groups);
//   * packed words are prefetched one tile ahead into a rotating register buffer (evict-first), the pass's rope
//     values likewise; 3-bit words are loaded exactly once (the 24-bit windows are funnel-shifted out of a carried
//     word) -- the per-channel kernel re-read straddled words;
//   * per 8 pairs: 4 logic ops to interleave the two code streams into (a | b << BITS) units, then per pair
//     SHF + LOP3 (mask | table base) + LDS.64 + 2 FFMA.
#include "kvq_kscore.cuh"

namespace kvq {

template <int BITS> struct PCfg {
  static constexpr int N = 1 << BITS;
  static constexpr int NN = N * N;                       // entries per (head, pair): 256 / 64
  static constexpr int W = Layout<BITS>::kWords;         // 16 / 12
  static constexpr int G = 8;                            // heads per CTA
  static constexpr int PP = (BITS == 4) ? 8 : 32;        // pairs per pass -> table = G*PP*NN*8 = 128 KiB
  static constexpr int P = kHalf / PP;                   // passes: 8 / 2
  static constexpr int kThreads = 512;
  static constexpr int TT = kThreads;                    // tokens per tile
  static constexpr int kAlign = NN * 8;                  // one (head, pair) table; base alignment for the OR trick
  static constexpr size_t kSmem = kAlign + (size_t)G * PP * NN * 8 + (size_t)G * kHeadDim * 4;
};

// 8 pairs of one head: units u_k = a_k | b_k << BITS sit in ce (even k) / co (odd k) at UB-bit spacing.
//   tab = shared address of T[0][0][0] (kAlign-aligned), IMM0 = byte offset of T[hl][first pair of this chunk][0]
template <int BITS, int IMM0>
__device__ __forceinline__ void pair_item(const uint32_t ce, const uint32_t co, const uint32_t tab,
                                          const float2* __restrict__ cs, float2& acc) {
  constexpr int NN = PCfg<BITS>::NN;
  constexpr int UB = 2 * BITS;                 // bits per unit: 8 / 6
  constexpr uint32_t MASK = (NN - 1) * 8;      // 0x7F8 / 0x1F8
  static_for<0, 8>([&](auto ik) {
    constexpr int k = decltype(ik)::v;
    constexpr int m = k >> 1;                  // unit index inside ce / co
    const uint32_t c = (k & 1) ? co : ce;
    const uint32_t sh = (m == 0) ? (c << 3) : (c >> (UB * m - 3));
    const uint32_t addr = (sh & MASK) | tab;
    ffma2(acc, cs[k], lds_f2<IMM0 + k * NN * 8>(addr));
  });
}

template <int BITS, bool FULL>
__global__ void __launch_bounds__(PCfg<BITS>::kThreads, 1) k_pair_kernel(const KParams p) {
  using C = PCfg<BITS>;
  constexpr int N = C::N, NN = C::NN, W = C::W, G = C::G, PP = C::PP, P = C::P, TT = C::TT;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((C::kAlign - (smem_u32(smem_raw) & (C::kAlign - 1))) & (C::kAlign - 1));
  float2* s_tab = reinterpret_cast<float2*>(smem);               // [G][PP][NN]
  float* s_q = reinterpret_cast<float*>(s_tab + G * PP * NN);    // [G][128]

  const int tid = threadIdx.x;
  const uint64_t pol_stream = policy_evict_first(), pol_keep = policy_evict_last();
  const int h0 = blockIdx.y * G;
  const int nh = FULL ? G : min(G, p.H - h0);

  const int64_t tile_first = (int64_t)blockIdx.x * p.tiles_per_cta;
  const int64_t tile_end = min(tile_first + p.tiles_per_cta, (p.L + TT - 1) / TT);
  if (tile_first >= tile_end) return;                 // uniform per CTA
  const int64_t t_limit = min(p.L, tile_end * TT);    // tokens this CTA may touch
  const uint32_t pitch = (uint32_t)p.Lmax * 4u;       // row pitch in bytes (host checks Lmax < 2^30)
  const unsigned char* cb0 = reinterpret_cast<const unsigned char*>(p.cache + (int64_t)h0 * W * p.Lmax);
  const uint32_t tab0 = smem_u32(s_tab);

  for (int i = tid; i < nh * kHeadDim; i += C::kThreads) s_q[i] = p.q[(int64_t)h0 * kHeadDim + i];

  for (int pass = 0; pass < P; ++pass) {
    __syncthreads();   // s_q visible / every lookup of the previous pass has been issued and consumed
    // ---- pair tables of this pass: T[hl][kp][a | b<<BITS] = (A q_j + B q_j64, A q_j64 - B q_j), j = pass*PP + kp ------
    for (int i = tid; i < G * PP * NN; i += C::kThreads) {
      const int idx = i & (NN - 1);
      const int hk = i / NN;
      const int kp = hk % PP, hl = hk / PP;
      float2 e = make_float2(0.f, 0.f);   // heads past nh: zero tables (their items still run, results are dropped)
      if (FULL || hl < nh) {
        const int j = pass * PP + kp;
        const int64_t row = ((int64_t)(h0 + hl) * kHeadDim + j) * N;
        const float A = __ldg(p.lut + row + (idx & (N - 1)));
        const float B = __ldg(p.lut + row + (int64_t)kHalf * N + (idx >> BITS));
        const float qj = s_q[hl * kHeadDim + j], qj64 = s_q[hl * kHeadDim + j + kHalf];
        e = make_float2(A * qj + B * qj64, A * qj64 - B * qj);
      }
      s_tab[i] = e;
    }
    __syncthreads();

    const bool last = (pass == P - 1);
    const bool need_old = (pass != 0) || (p.accumulate != 0);
    const unsigned char* src_cur = cb0 + (tile_first * TT + tid) * 4;
    bool ok_cur = (tile_first * TT + tid) < t_limit;

    // load-item (r, hl): the two packed words (stream A = channels < 64, stream B = their +64 partners) of word-row
    // step r of this pass.  4-bit: r = 0 only (rows pass, pass + 8).  3-bit: r = 0..2 (rows 3*pass + r, 3*(pass+2) + r).
    uint32_t wq[G][2];
#pragma unroll
    for (int g = 0; g < G; ++g) { wq[g][0] = 0; wq[g][1] = 0; }
    const uint32_t rowA = (BITS == 4) ? (uint32_t)pass : (uint32_t)(3 * pass);
    const uint32_t rowB = (BITS == 4) ? (uint32_t)(pass + 8) : (uint32_t)(3 * (pass + 2));
    auto fetch = [&](uint32_t* dst, const unsigned char* base, bool ok, int r, int hl) {
      if (ok && (FULL || hl < nh)) {   // heads past nh do not exist in the cache: never touch them
        dst[0] = ld_stream_u32(reinterpret_cast<const uint32_t*>(base + (uint64_t)((uint32_t)(hl * W + r) + rowA) * pitch), pol_stream);
        dst[1] = ld_stream_u32(reinterpret_cast<const uint32_t*>(base + (uint64_t)((uint32_t)(hl * W + r) + rowB) * pitch), pol_stream);
      }
    };
    // rope values of 8-pair chunk `a8` (pairs 8*a8 .. 8*a8+7) for token t
    auto load_cs = [&](float2* dst, const int64_t t, int a8) {
      if (t < t_limit) {
        const float2* rp = p.rope + (t + p.pos_offset) + (int64_t)(8 * a8) * p.rope_npos;
#pragma unroll
        for (int k = 0; k < 8; ++k) dst[k] = ld_keep_f2(rp + (int64_t)k * p.rope_npos, pol_keep);
      }
    };
    constexpr int CH = PP / 8;   // 8-pair chunks per pass: 1 / 4

    static_for<0, G>([&](auto ig) { constexpr int hl = decltype(ig)::v; fetch(wq[hl], src_cur, ok_cur, 0, hl); });
    float2 cs[8], csn[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { cs[k] = make_float2(0.f, 0.f); csn[k] = make_float2(0.f, 0.f); }
    load_cs(cs, tile_first * TT + tid, pass * CH);

    for (int64_t tile = tile_first; tile < tile_end; ++tile) {
      const int64_t t = tile * TT + tid;
      const bool live = t < p.L;
      const unsigned char* src_nxt = src_cur + TT * 4;
      const bool ok_nxt = (t + TT) < t_limit;
      float old[G];
#pragma unroll
      for (int hl = 0; hl < G; ++hl) {
        old[hl] = 0.f;
        if (need_old && live && (FULL || hl < nh)) old[hl] = p.out[(int64_t)(h0 + hl) * p.out_stride + t];
      }
      float2 acc[G];
#pragma unroll
      for (int g = 0; g < G; ++g) acc[g] = make_float2(0.f, 0.f);

      if constexpr (BITS == 4) {
        load_cs(csn, t + TT, pass);
        static_for<0, G>([&](auto ig) {
          constexpr int hl = decltype(ig)::v;
          const uint32_t w0 = wq[hl][0], w1 = wq[hl][1];
          fetch(wq[hl], src_nxt, ok_nxt, 0, hl);
          // nibble k of w0 = code of channel 8*pass+k, of w1 = its +64 partner
          const uint32_t ce = (w0 & 0x0F0F0F0Fu) | ((w1 << 4) & 0xF0F0F0F0u);   // pairs 0,2,4,6: bytes a | b<<4
          const uint32_t co = ((w0 >> 4) & 0x0F0F0F0Fu) | (w1 & 0xF0F0F0F0u);   // pairs 1,3,5,7
          pair_item<4, hl * PP * NN * 8>(ce, co, tab0, cs, acc[hl]);
        });
#pragma unroll
        for (int k = 0; k < 8; ++k) cs[k] = csn[k];
      } else {
        uint32_t cw[G][2] = {};   // carried word of each stream (the 24-bit windows straddle word boundaries)
        static_for<0, CH>([&](auto ia) {
          constexpr int a = decltype(ia)::v;   // chunk inside the pass: stream bits 24a .. 24a+23
          load_cs(csn, a == CH - 1 ? t + TT : t, pass * CH + ((a + 1) & (CH - 1)));
          static_for<0, G>([&](auto ig) {
            constexpr int hl = decltype(ig)::v;
            uint32_t x0, x1;
            if constexpr (a < 3) {
              const uint32_t n0 = wq[hl][0], n1 = wq[hl][1];
              if constexpr (a < 2) fetch(wq[hl], src_cur, ok_cur, a + 1, hl);
              else fetch(wq[hl], src_nxt, ok_nxt, 0, hl);
              if constexpr (a == 0) { x0 = n0; x1 = n1; }
              else {
                constexpr int sh = (a == 1) ? 24 : 16;
                x0 = __funnelshift_r(cw[hl][0], n0, sh);
                x1 = __funnelshift_r(cw[hl][1], n1, sh);
              }
              cw[hl][0] = n0; cw[hl][1] = n1;
            } else {
              x0 = cw[hl][0] >> 8; x1 = cw[hl][1] >> 8;
            }
            // code k of the window sits at bit 3k; M selects codes 0,2,4,6
            constexpr uint32_t M = 0x001C71C7u;
            const uint32_t ce = (x0 & M) | ((x1 << 3) & ~M);          // units a | b<<3 of pairs 0,2,4,6 at bits 0,6,12,18
            const uint32_t co = ((x0 >> 3) & M) | (x1 & ~M);          // pairs 1,3,5,7
            pair_item<3, (hl * PP + 8 * a) * NN * 8>(ce, co, tab0, cs, acc[hl]);
          });
#pragma unroll
          for (int k = 0; k < 8; ++k) cs[k] = csn[k];
        });
      }

      // ---- write back: this thread owns column t of the score matrix for the CTA's heads ---------------------------
#pragma unroll
      for (int hl = 0; hl < G; ++hl) {
        if (FULL || hl < nh) {
          float s = (acc[hl].x + acc[hl].y) + old[hl];
          if (last) {
            s *= p.scale;
            if (p.gmax != nullptr) {
              const float m = warp_max(live ? s : -INFINITY);
              if ((tid & 31) == 0 && m > -INFINITY) atomic_max_float(p.gmax + h0 + hl, m);
            }
          }
          if (live) p.out[(int64_t)(h0 + hl) * p.out_stride + t] = s;
        }
      }
      src_cur = src_nxt;
      ok_cur = ok_nxt;
    }
  }
}

template <int BITS>
static int launch_k_pair(const KParams& p, cudaStream_t st) {
  using C = PCfg<BITS>;
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(k_pair_kernel<BITS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::kSmem);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(k_pair_kernel<BITS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::kSmem);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  const int n_groups = (p.H + C::G - 1) / C::G;
  const int64_t n_tiles = (p.L + C::TT - 1) / C::TT;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t max_splits = sms / n_groups > 0 ? sms / n_groups : 1;
  KParams q = p;
  q.tiles_per_cta = (int)((n_tiles + max_splits - 1) / max_splits);
  const int64_t splits = (n_tiles + q.tiles_per_cta - 1) / q.tiles_per_cta;
  const dim3 grid((unsigned)splits, (unsigned)n_groups);
  if (p.H % C::G == 0) k_pair_kernel<BITS, true><<<grid, C::kThreads, C::kSmem, st>>>(q);
  else k_pair_kernel<BITS, false><<<grid, C::kThreads, C::kSmem, st>>>(q);
  KVQ_LAUNCH_CHECK();
  return 0;
}

int k_pair_dispatch(int bits, const KParams& p, cudaStream_t st) {
  switch (bits) {
    case 4: return launch_k_pair<4>(p, st);
    case 3: return launch_k_pair<3>(p, st);
    default: return KVQ_E_BITS;
  }
}

}  // namespace kvq
