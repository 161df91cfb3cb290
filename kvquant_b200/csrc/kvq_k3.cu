// kvquant_b200 -- dense Q.K^T decode matvec, 3-bit cache, per-channel 8-byte tables with carried words.
//
// Replaces (reference deployment/kvquant/quant_cuda_kernel.cu):
//   VecQuant3MatMulKernelNUQPerChannelTransposedRopeMHABatchedFusedOpt   3692-4115
//
// The arithmetic of k_scores_kernel (kvq_kscore.cu, 4 and 2 bits): T[h][c][code] = (LUT q_c, s_c LUT q_c^64), one
// LDS.64 + two FFMA per element.  The 96-bit code streams are fed so that:
//   * every packed word is loaded exactly ONCE: the four 24-bit windows of a 32-channel group are funnel-shifted out
//     of the current and the carried word;
//   * G = 8 heads per CTA (64 KiB of tables) -> H/8 head groups x (SMs / groups) token ranges, one CTA per SM;
//   * token ranges are cut at warp granularity and a warp whose 32 tokens lie past the range skips the tile, so the
//     last tile of a range costs only its live warps.
#include "kvq_kscore.cuh"

namespace kvq {

struct K3Cfg {
  static constexpr int N = 8;
  static constexpr int W = 12;
  static constexpr int G = 8;
  static constexpr int kThreads = 512;
  static constexpr int TT = kThreads;
  static constexpr size_t kSmem = 256 + (size_t)G * kHeadDim * N * 8 + (size_t)G * kHeadDim * 4;
};

template <bool FULL>
__global__ void __launch_bounds__(K3Cfg::kThreads, 1) k_scores3_kernel(const KParams p) {
  using C = K3Cfg;
  constexpr int N = C::N, W = C::W, G = C::G, TT = C::TT;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((256u - (smem_u32(smem_raw) & 255u)) & 255u);   // table base 64-byte aligned at least
  float2* s_tab = reinterpret_cast<float2*>(smem);                  // [G][128][N]
  float* s_q = reinterpret_cast<float*>(s_tab + G * kHeadDim * N);   // [G][128]

  const int tid = threadIdx.x;
  const uint64_t pol_stream = policy_evict_first(), pol_keep = policy_evict_last();
  const int h0 = blockIdx.y * G;
  const int nh = FULL ? G : min(G, p.H - h0);

  for (int i = tid; i < nh * kHeadDim; i += C::kThreads) s_q[i] = p.q[(int64_t)h0 * kHeadDim + i];
  __syncthreads();
  for (int i = tid; i < G * kHeadDim * N; i += C::kThreads) {
    float2 e = make_float2(0.f, 0.f);
    if (i < nh * kHeadDim * N) {
      const int hc = i / N;
      const int c = hc & (kHeadDim - 1);
      const float l = p.lut[((int64_t)h0 * kHeadDim) * N + i];
      const float qa = s_q[hc];
      const float qb = s_q[hc ^ kHalf];
      e = make_float2(l * qa, (c < kHalf) ? (l * qb) : -(l * qb));
    }
    s_tab[i] = e;
  }
  __syncthreads();
  const uint32_t tab0 = smem_u32(s_tab);

  // this CTA's token range [t_begin, t_limit): p.range is a multiple of 32
  const int64_t t_begin = (int64_t)blockIdx.x * p.range;
  const int64_t t_limit = min(p.L, t_begin + p.range);
  if (t_begin >= t_limit) return;
  const uint32_t pitch = (uint32_t)p.Lmax * 4u;
  const unsigned char* cb0 = reinterpret_cast<const unsigned char*>(p.cache + (int64_t)h0 * W * p.Lmax);

  const unsigned char* src_cur = cb0 + (t_begin + tid) * 4;
  bool ok_cur = (t_begin + tid) < t_limit;

  // load-item (g, r, hl): word r (0..2) of group g (stream A, channels 32g..32g+31) and of group g+2 (stream B)
  uint32_t wq[G][2];
#pragma unroll
  for (int g = 0; g < G; ++g) { wq[g][0] = 0; wq[g][1] = 0; }
  auto fetch = [&](uint32_t* dst, const unsigned char* base, bool ok, int g, int r, int hl) {
    if (ok && (FULL || hl < nh)) {
      const uint32_t row = (uint32_t)(hl * W + r) + (uint32_t)(3 * g);
      dst[0] = ld_stream_u32(reinterpret_cast<const uint32_t*>(base + (uint64_t)row * pitch), pol_stream);
      dst[1] = ld_stream_u32(reinterpret_cast<const uint32_t*>(base + (uint64_t)(row + 6u) * pitch), pol_stream);
    }
  };
  auto load_cs = [&](float2* dst, const int64_t t, int a8) {
    if (t < t_limit) {
      const float2* rp = p.rope + (t + p.pos_offset) + (int64_t)(8 * a8) * p.rope_npos;
#pragma unroll
      for (int k = 0; k < 8; ++k) dst[k] = ld_keep_f2(rp + (int64_t)k * p.rope_npos, pol_keep);
    }
  };

  static_for<0, G>([&](auto ig) { constexpr int hl = decltype(ig)::v; fetch(wq[hl], src_cur, ok_cur, 0, 0, hl); });
  float2 cs[8], csn[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { cs[k] = make_float2(0.f, 0.f); csn[k] = make_float2(0.f, 0.f); }
  load_cs(cs, t_begin + tid, 0);

  for (int64_t tb = t_begin; tb < t_limit; tb += TT) {
    const int64_t t = tb + tid;
    const unsigned char* src_nxt = src_cur + TT * 4;
    const bool ok_nxt = (t + TT) < t_limit;
    // warp-uniform: a warp whose tokens all lie past the range has nothing to do in this (last) tile
    if (tb + (tid & ~31) < t_limit) {
      const bool live = t < t_limit;
      float2 acc[G];
#pragma unroll
      for (int g = 0; g < G; ++g) acc[g] = make_float2(0.f, 0.f);
      uint32_t cw[G][2] = {};   // carried word of each stream

      for (int g = 0; g < 2; ++g) {
        const uint32_t tabg = tab0 + (uint32_t)g * (32 * N * 8);
        static_for<0, 4>([&](auto ia) {
          constexpr int a = decltype(ia)::v;   // window: stream bits 24a .. 24a+23 = channels 32g + 8a .. +7
          load_cs(csn, (a == 3 && g == 1) ? t + TT : t, ((4 * g + a) + 1) & 7);
          static_for<0, G>([&](auto ig) {
            constexpr int hl = decltype(ig)::v;
            uint32_t x0, x1;
            if constexpr (a < 3) {
              const uint32_t n0 = wq[hl][0], n1 = wq[hl][1];
              if constexpr (a < 2) fetch(wq[hl], src_cur, ok_cur, g, a + 1, hl);
              else fetch(wq[hl], g ? src_nxt : src_cur, g ? ok_nxt : ok_cur, g ^ 1, 0, hl);
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
            constexpr int IMM = (hl * kHeadDim + 8 * a) * N * 8;
            constexpr int HI = kHalf * N * 8;
            static_for<0, 8>([&](auto ik) {
              constexpr int k = decltype(ik)::v;
              const uint32_t a0 = ((k == 0 ? (x0 << 3) : (x0 >> (3 * k - 3))) & 0x38u) | tabg;
              const uint32_t a1 = ((k == 0 ? (x1 << 3) : (x1 >> (3 * k - 3))) & 0x38u) | tabg;
              ffma2(acc[hl], cs[k], lds_f2<IMM + k * N * 8>(a0));
              ffma2(acc[hl], cs[k], lds_f2<IMM + k * N * 8 + HI>(a1));
            });
          });
#pragma unroll
          for (int k = 0; k < 8; ++k) cs[k] = csn[k];
        });
      }

#pragma unroll
      for (int hl = 0; hl < G; ++hl) {
        if (live && (FULL || hl < nh)) {
          float* o = p.out + (int64_t)(h0 + hl) * p.out_stride + t;
          *o = (acc[hl].x + acc[hl].y) + *o;
        }
      }
    }
    src_cur = src_nxt;
    ok_cur = ok_nxt;
  }
}

int k_scores3_dispatch(const KParams& p, cudaStream_t st) {
  using C = K3Cfg;
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(k_scores3_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::kSmem);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(k_scores3_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::kSmem);
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
  if (p.H % C::G == 0) k_scores3_kernel<true><<<grid, C::kThreads, C::kSmem, st>>>(q);
  else k_scores3_kernel<false><<<grid, C::kThreads, C::kSmem, st>>>(q);
  KVQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace kvq
