// kvquant_b200 -- causal attention of a T-token chunk over [sinks | quantised slots 0..L-1 | the chunk itself], read
// straight from the quantised cache: K/V tiles of the slots are dequantised into shared memory (kvq_dequant.cuh, the
// same per-element steps as kvq_dequant_kv, so every operand is the fp16 value that kernel writes) and consumed there
// by mma.sync m16n8k16 (fp16 in, fp32 accumulate) in the FlashAttention-2 style.  Nothing the size of the cache
// touches HBM.  DESIGN.md section 4.8.
//
// CTA (query block qb of kBQ rows, head h, key split s), 8 warps, warp w owns query rows qb*kBQ + 16w .. +15 and keeps
// their fp16 Q fragments in registers.  The CTA walks its key tiles of kBK tokens, a tile never mixing regions:
//   split 0:  sink tiles, then its share of the slot tiles, then the chunk tiles up to the block's last row;
//   split s:  its share of the slot tiles.
// Per tile: (1) producer, all 256 threads: sink tile copied (K transposed from channel-major), chunk tile copied,
// slot tile dequantised from packed words that cp.async brought in while the previous tile was being consumed;
// (2) consumer, each warp: S = Q K^T (fp32), online softmax in fp32 with exp2f and the log2(e)/sqrt(128) scale folded
// in, P rounded to fp16, O += P V (fp32).  The causal mask applies to chunk tiles only.
// One split: the kernel writes out = O / l.  Several: each writes (O, m, l) per row to scratch and chunk_combine_kernel
// merges them in split order.  No global atomics: two identical calls return identical bits.
#include <cuda_fp16.h>

#include "kvq_common.cuh"
#include "kvq_dequant.cuh"

namespace kvq {
namespace chunk {

constexpr int kBQ = 128;             // query rows per CTA (8 warps x 16)
constexpr int kBK = 64;              // key tokens per tile
constexpr int kWarps = 8;
constexpr int kThreads = 32 * kWarps;
constexpr int kKP = kHeadDim + 8;    // fp16 operand row pitch: 272 B, so the 8 row addresses of an ldmatrix hit 32 banks
constexpr int kFP = kHeadDim + 4;    // fp32 dequantisation row pitch (as kvq_dequant.cu's tile)
constexpr int kMaxSplits = 32;
constexpr int kMaxSms = 256;         // SM counts above this are treated as this (bounds the scratch)
constexpr int kPart = kHeadDim + 2;  // floats per (split, row, head) partial: O[128], m, l

template <int BITS>
struct Smem {
  static constexpr int W = Layout<BITS>::kWords;
  static constexpr int kWP = W + 1;                  // token-major word rows, odd pitch (as kvq_dequant.cu)
  static constexpr int kLP = Layout<BITS>::kLevels + 1;
  static constexpr size_t kOp = (size_t)kBK * kKP * 2;               // one fp16 operand tile
  static constexpr size_t kStage = (size_t)kBK * kFP * 4;            // one fp32 dequantisation tile
  static constexpr size_t kWords = (size_t)kBK * kWP * 4;            // one side's words of one tile
  static constexpr size_t oK = 0, oV = oK + kOp, oSK = oV + kOp, oSV = oSK + kStage;
  static constexpr size_t oW = oSV + kStage;                         // [2 buffers][K, V] words
  static constexpr size_t oAff = oW + 4 * kWords;                    // [2 buffers][kBK][2]
  static constexpr size_t oLut = oAff + 2 * kBK * 2 * 4;             // K LUT of the head [128][kLP]
  static constexpr size_t oCent = oLut + (size_t)kHeadDim * kLP * 4;
  static constexpr size_t kBytes = oCent + Layout<BITS>::kLevels * 4;
  static_assert((size_t)kBQ * kKP * 2 <= 2 * kStage, "Q staging reuses the two fp32 tiles");
};

struct Params {
  const float* q;                    // f32 [T, H, 128]
  const __half* ck;                  // f16 [H / grp, T, 128] rotated chunk keys
  const __half* cv;                  // f16 [H / grp, T, 128]
  const int32_t* kcache; const float* klut; const float* kout; const int32_t* kidx;
  const int32_t* vcache; const float* vcent; const float* vaff; const float* vout; const int32_t* vidx;
  const float2* rope; int64_t npos; int64_t pos0;   // pos0: absolute position of slot 0
  const __half* sink_k; const __half* sink_v; int ns;
  float* out;                        // f32 [T, H, 128]
  float* part;                       // [nsplit][T][H][kPart] when nsplit > 1
  int H, n_out, nsplit;              // H: query heads
  int grp;                           // query heads per KV head: query head h reads KV head h / grp
  int64_t Lmax, L, T, tiles_per_split;
  // ragged forms only (chunk_attend_ragged_kernel): rows per KV head of ck / cv, and a paged slot's page-table row
  int64_t cstride;
  const int32_t* pages; int P;
};

// FORM 0: one sequence of a contiguous cache (chunk_attend_kernel); 1: a segment of a contiguous batch, 2: a segment
// of a page pool (chunk_attend_ragged_kernel: Params rebased on the segment, ck / cv rows cstride apart per KV head)
constexpr int kLone = 0, kRagged = 1, kRaggedPaged = 2;

__device__ __forceinline__ void cp_async4(void* dst, const void* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(valid ? 4 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// the tile list of one CTA: [sink tiles | slot tiles s0..s1 | chunk tiles]
struct Tiles {
  int64_t n_sink, s0, n_slot, n_chunk;
  __device__ int64_t count() const { return n_sink + n_slot + n_chunk; }
};

// cp.async the packed K/V words and (sf, off) of slot tile `st` into buffer `b`; rows past L are zero-filled.
// kRaggedPaged: each token's words through its own page (64-token tiles straddle pages of 160 * k tokens)
template <int BITS, int FORM>
__device__ __forceinline__ void prefetch_slot(const Params& p, unsigned char* smem, int64_t st, int b, int h) {
  using S = Smem<BITS>;
  constexpr int W = S::W;
  uint32_t* wk = reinterpret_cast<uint32_t*>(smem + S::oW) + (2 * b) * kBK * S::kWP;
  uint32_t* wv = wk + kBK * S::kWP;
  float* aff = reinterpret_cast<float*>(smem + S::oAff) + b * 2 * kBK;
  const int64_t t0 = st * kBK;
  const int nt = (int)min((int64_t)kBK, p.L - t0);
  if constexpr (FORM == kRaggedPaged) {
    const PageRef pr{p.pages, nullptr, 0, p.P, 0};
    const int t = threadIdx.x % kBK;                // kThreads % kBK == 0: a thread keeps its token
    const bool ok = t < nt;
    const PageCol pc = page_col(pr, (int)(t0 + (ok ? t : 0)));
    const int64_t g0 = ((int64_t)pc.page * (p.H / p.grp) + h) * W * p.P + pc.col;   // pool [page][Hkv][W][P]
    for (int r = threadIdx.x / kBK; r < W; r += kThreads / kBK) {
      cp_async4(wk + t * S::kWP + r, p.kcache + g0 + (int64_t)r * p.P, ok);
      cp_async4(wv + t * S::kWP + r, p.vcache + g0 + (int64_t)r * p.P, ok);
    }
    if (threadIdx.x < 2 * kBK) {
      const int tt = threadIdx.x >> 1;
      const bool oka = tt < nt;
      cp_async4(aff + threadIdx.x, p.vaff + 2 * page_row(pr, (int)(t0 + (oka ? tt : 0))) + (threadIdx.x & 1), oka);
    }
  } else {
    for (int i = threadIdx.x; i < W * kBK; i += kThreads) {
      const int r = i / kBK, t = i % kBK;           // t fastest: coalesced along the sequence
      const bool ok = t < nt;
      const int64_t g = ((int64_t)h * W + r) * p.Lmax + t0 + (ok ? t : 0);
      cp_async4(wk + t * S::kWP + r, p.kcache + g, ok);
      cp_async4(wv + t * S::kWP + r, p.vcache + g, ok);
    }
    if (threadIdx.x < 2 * kBK) {
      const bool ok = (int)threadIdx.x < 2 * nt;
      cp_async4(aff + threadIdx.x, p.vaff + 2 * t0 + (ok ? threadIdx.x : 0), ok);
    }
  }
}

// CTA (query block qb, head h, key split s) of the call (or segment) p; the lone kernel reads them from its grid
template <int BITS, int FORM>
__device__ __forceinline__ void chunk_attend_body(const Params& p, int64_t qb_r, int h_r, int s_r) {
  using S = Smem<BITS>;
  constexpr int W = S::W;
  constexpr int WQ = W / 4;
  constexpr int NL = Layout<BITS>::kLevels;
  extern __shared__ __align__(16) unsigned char smem[];
  __half* Ks = reinterpret_cast<__half*>(smem + S::oK);
  __half* Vs = reinterpret_cast<__half*>(smem + S::oV);
  float* stK = reinterpret_cast<float*>(smem + S::oSK);
  float* stV = reinterpret_cast<float*>(smem + S::oSV);
  float* lut = reinterpret_cast<float*>(smem + S::oLut);
  float* cent = reinterpret_cast<float*>(smem + S::oCent);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t qb = FORM == kLone ? (int64_t)blockIdx.x : qb_r;
  const int h = FORM == kLone ? (int)blockIdx.y : h_r, s = FORM == kLone ? (int)blockIdx.z : s_r, H = p.H;
  const int hk = h / p.grp;                           // the KV head: LUT, words, (sf, off), outliers, sinks, chunk K/V
  const int64_t T = p.T, L = p.L;
  const int64_t row0 = qb * kBQ;                      // first query row of the block

  Tiles tl;
  const int64_t slot_tiles = (L + kBK - 1) / kBK;
  tl.s0 = min((int64_t)s * p.tiles_per_split, slot_tiles);
  tl.n_slot = min(tl.s0 + p.tiles_per_split, slot_tiles) - tl.s0;
  tl.n_sink = s == 0 ? (p.ns + kBK - 1) / kBK : 0;
  tl.n_chunk = s == 0 ? (min(T, row0 + kBQ) + kBK - 1) / kBK : 0;   // chunk tiles wholly after the last row: skipped
  const int64_t n_tiles = tl.count();

  if (tl.n_sink == 0 && tl.n_slot > 0) prefetch_slot<BITS, FORM>(p, smem, tl.s0, 0, hk);
  cp_async_commit();

  // Q of the block, rounded to fp16 once, staged over the fp32 tiles, then held in registers as A fragments
  {
    __half* Qs = reinterpret_cast<__half*>(smem + S::oSK);
    for (int i = tid; i < kBQ * (kHeadDim / 4); i += kThreads) {
      const int r = i / (kHeadDim / 4), c = (i % (kHeadDim / 4)) * 4;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row0 + r < T) x = *reinterpret_cast<const float4*>(p.q + ((row0 + r) * H + h) * kHeadDim + c);
      __half2* d = reinterpret_cast<__half2*>(Qs + r * kKP + c);
      d[0] = __floats2half2_rn(x.x, x.y);
      d[1] = __floats2half2_rn(x.z, x.w);
    }
    for (int i = tid; i < kHeadDim * NL; i += kThreads)
      lut[(i / NL) * S::kLP + i % NL] = p.klut[(int64_t)hk * kHeadDim * NL + i];
    if (tid < NL) cent[tid] = p.vcent[tid];
  }
  __syncthreads();
  uint32_t qf[kHeadDim / 16][4];
  {
    const __half* Qs = reinterpret_cast<const __half*>(smem + S::oSK);
#pragma unroll
    for (int kk = 0; kk < kHeadDim / 16; ++kk)
      ldsm_x4(qf[kk], Qs + (warp * 16 + (lane & 15)) * kKP + kk * 16 + (lane >> 4) * 8);
  }

  constexpr float kScaleLog2 = 1.4426950408889634f * 0.08838834764831845f;   // log2(e) / sqrt(128)
  float o[kHeadDim / 8][4];
#pragma unroll
  for (int i = 0; i < kHeadDim / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const int g = lane >> 2, c2 = (lane & 3) * 2;
  const int64_t wrow = row0 + warp * 16 + g;         // this thread's rows: wrow and wrow + 8

  for (int64_t j = 0; j < n_tiles; ++j) {
    // next slot tile's words on their way while this tile is produced and consumed
    const int64_t jn = j + 1 - tl.n_sink;
    if (jn >= 0 && jn < tl.n_slot) prefetch_slot<BITS, FORM>(p, smem, tl.s0 + jn, (int)(jn & 1), hk);
    cp_async_commit();
    cp_async_wait_1();
    __syncthreads();                                  // words of tile j landed; Ks / Vs free

    int nv;                                           // valid keys of the tile
    int64_t chunk0 = -1;                              // first chunk token of a chunk tile
    if (j < tl.n_sink) {
      const int k0 = (int)j * kBK;
      nv = min(kBK, p.ns - k0);
      for (int i = tid; i < kBK * kHeadDim; i += kThreads) {
        const int t = i % kBK, c = i / kBK;           // sink_k [H, 128, n]: tokens fastest
        Ks[t * kKP + c] = t < nv ? p.sink_k[((int64_t)hk * kHeadDim + c) * p.ns + k0 + t] : __float2half(0.f);
        const int tv = i / kHeadDim, cv = i % kHeadDim;
        Vs[tv * kKP + cv] = tv < nv ? p.sink_v[((int64_t)hk * p.ns + k0 + tv) * kHeadDim + cv] : __float2half(0.f);
      }
    } else if (j < tl.n_sink + tl.n_slot) {
      const int64_t js = j - tl.n_sink;
      const int b = (int)(js & 1);
      const int64_t t0 = (tl.s0 + js) * kBK;
      nv = (int)min((int64_t)kBK, L - t0);
      const uint32_t* wk = reinterpret_cast<const uint32_t*>(smem + S::oW) + (2 * b) * kBK * S::kWP;
      const uint32_t* wv = wk + kBK * S::kWP;
      const float* aff = reinterpret_cast<const float*>(smem + S::oAff) + b * 2 * kBK;
      {
        const int t = tid % kBK, qq = tid / kBK;      // one (token, 32-channel quarter) per thread and side
        uint32_t w[WQ];
#pragma unroll
        for (int k = 0; k < WQ; ++k) w[k] = wk[t * S::kWP + qq * WQ + k];
        dq_quarter<BITS, false>(w, lut + qq * 32 * S::kLP, S::kLP, 0.f, 0.f, stK + t * kFP + qq * 32);
#pragma unroll
        for (int k = 0; k < WQ; ++k) w[k] = wv[t * S::kWP + qq * WQ + k];
        dq_quarter<BITS, true>(w, cent, 0, aff[2 * t], aff[2 * t + 1], stV + t * kFP + qq * 32);
      }
      if (p.kout != nullptr || p.vout != nullptr) {
        __syncthreads();
        const int64_t r0 = t0 * p.n_out;
        if constexpr (FORM == kRaggedPaged) {         // the same, each token's row through its page
          const PageRef pr{p.pages, nullptr, 0, p.P, 0};
          for (int i = tid; i < nv * p.n_out; i += kThreads) {
            const int t = i / p.n_out;
            const int64_t e = page_row(pr, (int)(t0 + t)) * p.n_out + (i - t * p.n_out);
            if (p.kout != nullptr) {
              const int idx = p.kidx[e];
              if ((idx >> 7) == hk) dq_add_outlier(&stK[t * kFP + (idx & 127)], p.kout[e]);
            }
            if (p.vout != nullptr) {
              const int idx = p.vidx[e];
              if ((idx >> 7) == hk) dq_add_outlier(&stV[t * kFP + (idx & 127)], p.vout[e]);
            }
          }
        } else {
          for (int i = tid; i < nv * p.n_out; i += kThreads) {
            const int t = i / p.n_out;
            if (p.kout != nullptr) {
              const int idx = p.kidx[r0 + i];
              if ((idx >> 7) == hk) dq_add_outlier(&stK[t * kFP + (idx & 127)], p.kout[r0 + i]);
            }
            if (p.vout != nullptr) {
              const int idx = p.vidx[r0 + i];
              if ((idx >> 7) == hk) dq_add_outlier(&stV[t * kFP + (idx & 127)], p.vout[r0 + i]);
            }
          }
        }
      }
      __syncthreads();
      for (int i = tid; i < kBK * (kHeadDim / 8); i += kThreads) {
        const int t = i % kBK, c0 = (i / kBK) * 8;    // tokens fastest: the cos/sin reads are coalesced
        uint4 ko = make_uint4(0u, 0u, 0u, 0u), vo = ko;
        if (t < nv) {
          float2 cs[8];
          const float2* rp = p.rope + (int64_t)(c0 & 63) * p.npos + p.pos0 + t0 + t;
#pragma unroll
          for (int k = 0; k < 8; ++k) cs[k] = rp[(int64_t)k * p.npos];
          ko = dq_finish8<true>(stK + t * kFP, c0, cs);
          vo = dq_finish8<false>(stV + t * kFP, c0, nullptr);
        }
        *reinterpret_cast<uint4*>(Ks + t * kKP + c0) = ko;
        *reinterpret_cast<uint4*>(Vs + t * kKP + c0) = vo;
      }
    } else {
      chunk0 = (j - tl.n_sink - tl.n_slot) * kBK;
      nv = (int)min((int64_t)kBK, T - chunk0);
      for (int i = tid; i < kBK * (kHeadDim / 8); i += kThreads) {
        const int t = i / (kHeadDim / 8), c0 = (i % (kHeadDim / 8)) * 8;
        uint4 ko = make_uint4(0u, 0u, 0u, 0u), vo = ko;
        if (t < nv) {
          const int64_t off = ((int64_t)hk * (FORM == kLone ? T : p.cstride) + chunk0 + t) * kHeadDim + c0;
          ko = *reinterpret_cast<const uint4*>(p.ck + off);
          vo = *reinterpret_cast<const uint4*>(p.cv + off);
        }
        *reinterpret_cast<uint4*>(Ks + t * kKP + c0) = ko;
        *reinterpret_cast<uint4*>(Vs + t * kKP + c0) = vo;
      }
    }
    __syncthreads();                                  // tile j complete in Ks / Vs

    // a warp whose rows all precede the chunk tile has nothing to add
    if (chunk0 >= 0 && chunk0 > row0 + warp * 16 + 15) continue;

    float sc[kBK / 8][4];
#pragma unroll
    for (int n = 0; n < kBK / 8; ++n) sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
#pragma unroll
    for (int n = 0; n < kBK / 8; ++n) {
#pragma unroll
      for (int kk = 0; kk < kHeadDim / 32; ++kk) {
        uint32_t b[4];
        ldsm_x4(b, Ks + (n * 8 + (lane & 7)) * kKP + kk * 32 + (lane >> 3) * 8);
        mma16816(sc[n], qf[2 * kk], b[0], b[1]);
        mma16816(sc[n], qf[2 * kk + 1], b[2], b[3]);
      }
    }
    // scale, mask, running max
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < kBK / 8; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = n * 8 + c2 + (e & 1);
        const int64_t row = wrow + (e >> 1) * 8;
        const bool ok = key < nv && (chunk0 < 0 || chunk0 + key <= row);
        sc[n][e] = ok ? sc[n][e] * kScaleLog2 : -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], sc[n][e]);
      }
    }
    float corr[2], base[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      base[r] = m_new == -INFINITY ? 0.f : m_new;     // a row with no valid key yet keeps everything at 0
      corr[r] = exp2f(m_run[r] - base[r]);
      m_run[r] = m_new;
      l_run[r] *= corr[r];
    }
#pragma unroll
    for (int n = 0; n < kHeadDim / 8; ++n) {
      o[n][0] *= corr[0]; o[n][1] *= corr[0];
      o[n][2] *= corr[1]; o[n][3] *= corr[1];
    }
    // P in fp16 (the sums take the rounded weights, so numerator and denominator agree), then O += P V
#pragma unroll
    for (int kv = 0; kv < kBK / 16; ++kv) {
      uint32_t a[4];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int n = 2 * kv + hh;
        const __half2 top = __floats2half2_rn(exp2f(sc[n][0] - base[0]), exp2f(sc[n][1] - base[0]));
        const __half2 bot = __floats2half2_rn(exp2f(sc[n][2] - base[1]), exp2f(sc[n][3] - base[1]));
        const float2 tf = __half22float2(top), bf = __half22float2(bot);
        l_run[0] += tf.x + tf.y;
        l_run[1] += bf.x + bf.y;
        a[2 * hh] = *reinterpret_cast<const uint32_t*>(&top);
        a[2 * hh + 1] = *reinterpret_cast<const uint32_t*>(&bot);
      }
#pragma unroll
      for (int dp = 0; dp < kHeadDim / 16; ++dp) {
        uint32_t b[4];
        ldsm_x4_t(b, Vs + (kv * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * kKP + dp * 16 + (lane >> 4) * 8);
        mma16816(o[2 * dp], a, b[0], b[1]);
        mma16816(o[2 * dp + 1], a, b[2], b[3]);
      }
    }
  }

  // the row sums are spread over the 4 threads of a quad
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int64_t row = wrow + r * 8;
    if (row >= T) continue;
    if (p.nsplit == 1) {
      float* dst = p.out + (row * H + h) * kHeadDim + c2;
      const float inv = 1.f / l_run[r];
#pragma unroll
      for (int n = 0; n < kHeadDim / 8; ++n)
        *reinterpret_cast<float2*>(dst + n * 8) = make_float2(o[n][2 * r] * inv, o[n][2 * r + 1] * inv);
    } else {
      float* dst = p.part + (((int64_t)s * T + row) * H + h) * kPart;
#pragma unroll
      for (int n = 0; n < kHeadDim / 8; ++n)
        *reinterpret_cast<float2*>(dst + n * 8 + c2) = make_float2(o[n][2 * r], o[n][2 * r + 1]);
      if (c2 == 0) { dst[kHeadDim] = m_run[r]; dst[kHeadDim + 1] = l_run[r]; }
    }
  }
}

template <int BITS>
__global__ void __launch_bounds__(kThreads, 1) chunk_attend_kernel(const Params p) {
  chunk_attend_body<BITS, kLone>(p, 0, 0, 0);
}

// out[row, h] = sum_s 2^(m_s - M) O_s / sum_s 2^(m_s - M) l_s, splits taken in order; (row, head) rh, channel d
__device__ __forceinline__ void combine_row(const float* __restrict__ part, float* __restrict__ out, int64_t TH,
                                            int nsplit, int64_t rh, int d) {
  float M = -INFINITY;
  for (int s = 0; s < nsplit; ++s) M = fmaxf(M, part[(s * TH + rh) * kPart + kHeadDim]);
  float num = 0.f, den = 0.f;
  for (int s = 0; s < nsplit; ++s) {
    const float* ps = part + (s * TH + rh) * kPart;
    const float w = exp2f(ps[kHeadDim] - M);
    num = fmaf(w, ps[d], num);
    den = fmaf(w, ps[kHeadDim + 1], den);
  }
  out[rh * kHeadDim + d] = num / den;
}

__global__ void __launch_bounds__(kHeadDim) chunk_combine_kernel(const float* __restrict__ part, float* __restrict__ out,
                                                                 int64_t TH, int nsplit) {
  combine_row(part, out, TH, nsplit, blockIdx.x, threadIdx.x);
}

// ---- ragged chunk attend (kvq_attend_chunk_ragged[_paged], DESIGN.md section 4.15) ------------------------------------
// Several slots' chunks in one launch: segment i attends its T rows over slot b's sinks, its first L (= s0) quantised
// slots and its own rows, with the split count the lone call would choose for (T, L).  Grid (sum of the segments'
// query blocks x splits, H): segment i owns x in [cta0[i], cta0[i + 1]), x - cta0[i] = split * blocks + query block.
struct RagChunkSeg {
  int64_t L, part, tiles_per_split;   // cached slots attended, first float of its partials in scratch, slot tiles per split
  int b, T, row0, nsplit;
};
struct RaggedChunk {
  Params base;                        // the call; q, out, ck, cv at row 0, the cache and sinks at slot 0
  int n_seg, Hkv, max_pages;
  int cta0[kMaxSeg + 1];              // first CTA of each segment (cta0[n_seg]: the grid's x extent)
  int comb0[kMaxSeg + 1];             // first combine block of each segment (none unless it splits)
  RagChunkSeg seg[kMaxSeg];
};

// The CTA's segment view of the call is built once in shared memory and the body reads it there: its pointers and
// sizes stay out of the registers of a kernel that holds 240+ of them.
template <int BITS, bool PAGED>
__global__ void __launch_bounds__(kThreads, 1) chunk_attend_ragged_kernel(const __grid_constant__ RaggedChunk rg) {
  __shared__ Params sp;
  __shared__ int64_t s_qb;
  __shared__ int s_split;
  if (threadIdx.x == 0) {
    const int i = find_segment(rg.cta0, rg.n_seg, (int)blockIdx.x);
    const RagChunkSeg sg = rg.seg[i];
    const int nqb = (sg.T + kBQ - 1) / kBQ;
    const int local = (int)blockIdx.x - rg.cta0[i];
    Params p = rg.base;
    const int64_t rowq = (int64_t)sg.row0 * p.H * kHeadDim;
    p.q += rowq;
    p.out += rowq;
    p.ck += (int64_t)sg.row0 * kHeadDim;
    p.cv += (int64_t)sg.row0 * kHeadDim;
    p.part += sg.part;
    p.L = sg.L; p.T = sg.T; p.nsplit = sg.nsplit; p.tiles_per_split = sg.tiles_per_split;
    const int64_t b = sg.b;
    if (p.ns > 0) {
      p.sink_k += b * rg.Hkv * kHeadDim * p.ns;
      p.sink_v += b * rg.Hkv * kHeadDim * p.ns;
    }
    if constexpr (PAGED) {
      p.pages += b * rg.max_pages;
    } else {
      const int64_t words = (int64_t)rg.Hkv * Layout<BITS>::kWords * p.Lmax, rows = p.Lmax * p.n_out;
      p.kcache += b * words; p.vcache += b * words;
      p.vaff += b * p.Lmax * 2;
      if (p.kout != nullptr) { p.kout += b * rows; p.kidx += b * rows; }
      if (p.vout != nullptr) { p.vout += b * rows; p.vidx += b * rows; }
    }
    sp = p;
    s_qb = local % nqb;
    s_split = local / nqb;
  }
  __syncthreads();
  chunk_attend_body<BITS, PAGED ? kRaggedPaged : kRagged>(sp, s_qb, blockIdx.y, s_split);
}

// the lone combine of every segment that split, one block per (row, head) of those segments
__global__ void __launch_bounds__(kHeadDim) chunk_combine_ragged_kernel(const __grid_constant__ RaggedChunk rg) {
  const int i = find_segment(rg.comb0, rg.n_seg, (int)blockIdx.x);
  const RagChunkSeg& sg = rg.seg[i];
  combine_row(rg.base.part + sg.part, rg.base.out + (int64_t)sg.row0 * rg.base.H * kHeadDim,
              (int64_t)sg.T * rg.base.H, sg.nsplit, (int)blockIdx.x - rg.comb0[i], threadIdx.x);
}

// key splits: only when the (query block, head) CTAs fill at most half the SMs; one split per slot tile at most
__host__ __device__ inline int n_splits(int64_t T, int H, int64_t L, int sms) {
  const int64_t base = (T + kBQ - 1) / kBQ * H;
  const int64_t slot_tiles = (L + kBK - 1) / kBK;
  sms = min(sms, kMaxSms);
  if (slot_tiles < 2 || 2 * base > sms) return 1;
  const int64_t n = min(min((int64_t)sms / base, slot_tiles), (int64_t)kMaxSplits);
  const int64_t per = (slot_tiles + n - 1) / n;
  return (int)((slot_tiles + per - 1) / per);   // every split gets at least one slot tile
}

template <int BITS>
int launch(Params& p, cudaStream_t st) {
  auto kern = chunk_attend_kernel<BITS>;
  const size_t smem = Smem<BITS>::kBytes;
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return (int)e;
  p.nsplit = n_splits(p.T, p.H, p.L, sms);
  const int64_t slot_tiles = (p.L + kBK - 1) / kBK;
  p.tiles_per_split = p.nsplit > 1 ? (slot_tiles + p.nsplit - 1) / p.nsplit : max(slot_tiles, (int64_t)1);
  const dim3 grid((unsigned)((p.T + kBQ - 1) / kBQ), (unsigned)p.H, (unsigned)p.nsplit);
  kern<<<grid, kThreads, smem, st>>>(p);
  KVQ_LAUNCH_CHECK();
  if (p.nsplit > 1) {
    chunk_combine_kernel<<<(unsigned)(p.T * p.H), kHeadDim, 0, st>>>(p.part, p.out, p.T * p.H, p.nsplit);
    KVQ_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace chunk
}  // namespace kvq

using namespace kvq;

extern "C" int64_t kvq_attend_chunk_scratch_bytes(int H, int64_t T, int64_t L) {
  // partials of nsplit x T x H rows; nsplit > 1 only when nsplit x ceil(T/kBQ) x H <= the SM count (<= kMaxSms)
  if (H <= 0 || T <= 0 || L < 0) return 0;
  const int64_t slot_tiles = max((L + chunk::kBK - 1) / chunk::kBK, (int64_t)1);
  const int64_t row = (int64_t)chunk::kPart * sizeof(float);
  const int64_t by_shape = min(slot_tiles, (int64_t)chunk::kMaxSplits) * T * H * row;
  return min(by_shape, (int64_t)chunk::kMaxSms * chunk::kBQ * row);
}

// H query heads over an Hkv-head cache (Hkv == H: one KV head per query head)
static int attend_chunk_impl(int bits, int H, int Hkv, int64_t Lmax, int64_t L, int64_t T, const float* q,
                             const void* chunk_k, const void* chunk_v, const int32_t* kcache, const float* klut,
                             const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                             const float* v_cent, const float* v_aff, const float* v_outliers,
                             const int32_t* v_outlier_idx, int n_out, const float* rope_cos_sin, int64_t rope_npos,
                             int pos_offset, const void* sink_k, const void* sink_v, int n_sink, float* out,
                             void* scratch, void* stream) {
  if (bits < 2 || bits > 4) return KVQ_E_BITS;
  if (H <= 0 || (H & 3) != 0 || H > 64 || Lmax <= 0 || L < 0 || L > Lmax || T < 0) return KVQ_E_SHAPE;
  if (Hkv <= 0 || ((Hkv & 3) != 0 && Hkv > 2) || H % Hkv != 0) return KVQ_E_SHAPE;
  if (n_out < 0 || (n_out & 1) != 0 || n_out > kMaxOutDq) return KVQ_E_SHAPE;
  if (n_sink < 0 || pos_offset < 0 || rope_npos < (int64_t)pos_offset + L) return KVQ_E_SHAPE;
  if (T == 0) return 0;   // nothing to attend: no launch
  if (!q || !chunk_k || !chunk_v || !out || !scratch) return KVQ_E_NULL;
  if (!kcache || !klut || !vcache || !v_cent || !v_aff || !rope_cos_sin) return KVQ_E_NULL;
  if ((k_outliers == nullptr) != (k_outlier_idx == nullptr) || (v_outliers == nullptr) != (v_outlier_idx == nullptr))
    return KVQ_E_NULL;
  if ((k_outliers || v_outliers) && n_out == 0) return KVQ_E_SHAPE;
  if (n_sink > 0 && (!sink_k || !sink_v)) return KVQ_E_NULL;
  if ((reinterpret_cast<uintptr_t>(q) & 15) != 0 || (reinterpret_cast<uintptr_t>(chunk_k) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(chunk_v) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 7) != 0 ||
      (reinterpret_cast<uintptr_t>(scratch) & 7) != 0)
    return KVQ_E_ALIGN;

  chunk::Params p{};
  p.q = q;
  p.ck = static_cast<const __half*>(chunk_k);
  p.cv = static_cast<const __half*>(chunk_v);
  p.kcache = kcache; p.klut = klut; p.kout = k_outliers; p.kidx = k_outlier_idx;
  p.vcache = vcache; p.vcent = v_cent; p.vaff = v_aff; p.vout = v_outliers; p.vidx = v_outlier_idx;
  p.rope = reinterpret_cast<const float2*>(rope_cos_sin); p.npos = rope_npos; p.pos0 = pos_offset;
  p.sink_k = static_cast<const __half*>(sink_k); p.sink_v = static_cast<const __half*>(sink_v);
  p.ns = n_sink;
  p.out = out;
  p.part = static_cast<float*>(scratch);
  p.H = H; p.grp = H / Hkv; p.n_out = n_out; p.Lmax = Lmax; p.L = L; p.T = T;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (bits) {
    case 4: return chunk::launch<4>(p, st);
    case 3: return chunk::launch<3>(p, st);
    default: return chunk::launch<2>(p, st);
  }
}

extern "C" int kvq_attend_chunk(int bits, int H, int64_t Lmax, int64_t L, int64_t T, const float* q,
                                const void* chunk_k, const void* chunk_v, const int32_t* kcache, const float* klut,
                                const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                                const float* v_cent, const float* v_aff, const float* v_outliers,
                                const int32_t* v_outlier_idx, int n_out, const float* rope_cos_sin, int64_t rope_npos,
                                int pos_offset, const void* sink_k, const void* sink_v, int n_sink, float* out,
                                void* scratch, void* stream) {
  return attend_chunk_impl(bits, H, H, Lmax, L, T, q, chunk_k, chunk_v, kcache, klut, k_outliers, k_outlier_idx, vcache,
                           v_cent, v_aff, v_outliers, v_outlier_idx, n_out, rope_cos_sin, rope_npos, pos_offset, sink_k,
                           sink_v, n_sink, out, scratch, stream);
}

extern "C" int kvq_attend_chunk_gqa(int bits, int Hq, int Hkv, int64_t Lmax, int64_t L, int64_t T, const float* q,
                                    const void* chunk_k, const void* chunk_v, const int32_t* kcache, const float* klut,
                                    const float* k_outliers, const int32_t* k_outlier_idx, const int32_t* vcache,
                                    const float* v_cent, const float* v_aff, const float* v_outliers,
                                    const int32_t* v_outlier_idx, int n_out, const float* rope_cos_sin, int64_t rope_npos,
                                    int pos_offset, const void* sink_k, const void* sink_v, int n_sink, float* out,
                                    void* scratch, void* stream) {
  return attend_chunk_impl(bits, Hq, Hkv, Lmax, L, T, q, chunk_k, chunk_v, kcache, klut, k_outliers, k_outlier_idx,
                           vcache, v_cent, v_aff, v_outliers, v_outlier_idx, n_out, rope_cos_sin, rope_npos, pos_offset,
                           sink_k, sink_v, n_sink, out, scratch, stream);
}

// ---- ragged entry points ------------------------------------------------------------------------------------------
namespace kvq {
namespace chunk {

// segments checked; segment i's partials start at the sum of the earlier segments' kvq_attend_chunk_scratch_bytes
template <int BITS>
int launch_ragged(RaggedChunk& rg, const int64_t* segs, cudaStream_t st, bool paged) {
  const size_t smem = Smem<BITS>::kBytes;
  static PerDeviceOnce attr_once[2];
  bool& attr_done = attr_once[paged].cur();
  if (!attr_done) {
    cudaError_t e = paged ? cudaFuncSetAttribute(chunk_attend_ragged_kernel<BITS, true>,
                                                 cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                          : cudaFuncSetAttribute(chunk_attend_ragged_kernel<BITS, false>,
                                                 cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return (int)e;
  const int H = rg.base.H;
  int64_t ctas = 0, combs = 0, part = 0;
  for (int i = 0; i < rg.n_seg; ++i) {
    RagChunkSeg& sg = rg.seg[i];
    sg.b = (int)segs[4 * i]; sg.L = segs[4 * i + 1]; sg.T = (int)segs[4 * i + 2]; sg.row0 = (int)segs[4 * i + 3];
    sg.nsplit = sg.T > 0 ? n_splits(sg.T, H, sg.L, sms) : 1;   // the lone call's rule for (T, L)
    const int64_t slot_tiles = (sg.L + kBK - 1) / kBK;
    sg.tiles_per_split = sg.nsplit > 1 ? (slot_tiles + sg.nsplit - 1) / sg.nsplit : max(slot_tiles, (int64_t)1);
    sg.part = part;
    rg.cta0[i] = (int)ctas;
    rg.comb0[i] = (int)combs;
    ctas += (int64_t)(sg.T + kBQ - 1) / kBQ * sg.nsplit;
    if (sg.nsplit > 1) combs += (int64_t)sg.T * H;
    if (sg.T > 0) part += kvq_attend_chunk_scratch_bytes(H, sg.T, sg.L) / (int64_t)sizeof(float);
  }
  rg.cta0[rg.n_seg] = (int)ctas;
  rg.comb0[rg.n_seg] = (int)combs;
  const dim3 grid((unsigned)ctas, (unsigned)H);
  if (paged) chunk_attend_ragged_kernel<BITS, true><<<grid, kThreads, smem, st>>>(rg);
  else chunk_attend_ragged_kernel<BITS, false><<<grid, kThreads, smem, st>>>(rg);
  KVQ_LAUNCH_CHECK();
  if (combs > 0) {
    chunk_combine_ragged_kernel<<<(unsigned)combs, kHeadDim, 0, st>>>(rg);
    KVQ_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace chunk
}  // namespace kvq

extern "C" int64_t kvq_attend_chunk_ragged_scratch_bytes(int Hq, int n_seg, const int64_t* segs) {
  if (Hq <= 0 || n_seg < 0 || n_seg > kMaxSeg || (n_seg > 0 && segs == nullptr)) return 0;
  int64_t total = 0;
  for (int i = 0; i < n_seg; ++i) {
    const int64_t L = segs[4 * i + 1], T = segs[4 * i + 2];
    if (L < 0 || T < 0) return 0;
    if (T > 0) total += kvq_attend_chunk_scratch_bytes(Hq, T, L);
  }
  return total;
}

// the ragged chunk attend over a contiguous batch (pg == nullptr) or a page pool (n_mapped: host, one per segment):
// attend_chunk_impl's checks in its order, with the segment table's after its size checks and rope_npos checked against
// the largest s0, then one launch (two when a segment splits)
static int attend_chunk_ragged_impl(int bits, int B, int Hq, int Hkv, int64_t Lmax, int n_seg, const int64_t* segs,
                                    int64_t N, const float* q, const void* chunk_k, const void* chunk_v,
                                    const int32_t* kcache, const float* klut, const float* k_outliers,
                                    const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent,
                                    const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx, int n_out,
                                    const float* rope_cos_sin, int64_t rope_npos, int pos_offset, const void* sink_k,
                                    const void* sink_v, int n_sink, float* out, void* scratch, void* stream,
                                    const PageRef* pg, const int32_t* n_mapped) {
  if (bits < 2 || bits > 4) return KVQ_E_BITS;
  if (Hq <= 0 || (Hq & 3) != 0 || Hq > 64 || Lmax <= 0) return KVQ_E_SHAPE;
  if (B < 1 || B > kMaxSeg || n_seg < 0 || n_seg > B || N < 0) return KVQ_E_SHAPE;
  if (Hkv <= 0 || ((Hkv & 3) != 0 && Hkv > 2) || Hq % Hkv != 0) return KVQ_E_SHAPE;
  if (n_out < 0 || (n_out & 1) != 0 || n_out > kMaxOutDq) return KVQ_E_SHAPE;
  if (n_sink < 0 || pos_offset < 0) return KVQ_E_SHAPE;
  if (n_seg > 0 && (segs == nullptr || (pg != nullptr && n_mapped == nullptr))) return KVQ_E_NULL;
  int64_t max_s0 = 0;
  const int rc = check_segments(B, n_seg, segs, N, Lmax, pg != nullptr ? n_mapped : nullptr,
                                pg != nullptr ? pg->max_pages : 0, pg != nullptr ? pg->P : 0, false, &max_s0);
  if (rc) return rc;
  if (rope_npos < (int64_t)pos_offset + max_s0) return KVQ_E_SHAPE;
  if (N == 0) return 0;   // nothing to attend: no launch
  if (!q || !chunk_k || !chunk_v || !out || !scratch) return KVQ_E_NULL;
  if (!kcache || !klut || !vcache || !v_cent || !v_aff || !rope_cos_sin) return KVQ_E_NULL;
  if ((k_outliers == nullptr) != (k_outlier_idx == nullptr) || (v_outliers == nullptr) != (v_outlier_idx == nullptr))
    return KVQ_E_NULL;
  if ((k_outliers || v_outliers) && n_out == 0) return KVQ_E_SHAPE;
  if (n_sink > 0 && (!sink_k || !sink_v)) return KVQ_E_NULL;
  if (pg != nullptr && pg->table == nullptr) return KVQ_E_NULL;
  if ((reinterpret_cast<uintptr_t>(q) & 15) != 0 || (reinterpret_cast<uintptr_t>(chunk_k) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(chunk_v) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 7) != 0 ||
      (reinterpret_cast<uintptr_t>(scratch) & 7) != 0)
    return KVQ_E_ALIGN;

  chunk::RaggedChunk rg{};        // ~12 KB, passed to the kernels by value
  chunk::Params& p = rg.base;
  p.q = q;
  p.ck = static_cast<const __half*>(chunk_k);
  p.cv = static_cast<const __half*>(chunk_v);
  p.kcache = kcache; p.klut = klut; p.kout = k_outliers; p.kidx = k_outlier_idx;
  p.vcache = vcache; p.vcent = v_cent; p.vaff = v_aff; p.vout = v_outliers; p.vidx = v_outlier_idx;
  p.rope = reinterpret_cast<const float2*>(rope_cos_sin); p.npos = rope_npos; p.pos0 = pos_offset;
  p.sink_k = static_cast<const __half*>(sink_k); p.sink_v = static_cast<const __half*>(sink_v);
  p.ns = n_sink;
  p.out = out;
  p.part = static_cast<float*>(scratch);
  p.H = Hq; p.grp = Hq / Hkv; p.n_out = n_out; p.Lmax = pg != nullptr ? pg->P : Lmax;
  p.cstride = N;
  p.pages = pg != nullptr ? pg->table : nullptr; p.P = pg != nullptr ? pg->P : 0;
  rg.n_seg = n_seg; rg.Hkv = Hkv; rg.max_pages = pg != nullptr ? pg->max_pages : 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (bits) {
    case 4: return chunk::launch_ragged<4>(rg, segs, st, pg != nullptr);
    case 3: return chunk::launch_ragged<3>(rg, segs, st, pg != nullptr);
    default: return chunk::launch_ragged<2>(rg, segs, st, pg != nullptr);
  }
}

extern "C" int kvq_attend_chunk_ragged(int bits, int B, int Hq, int Hkv, int64_t Lmax, int n_seg, const int64_t* segs,
                                       int64_t N, const float* q, const void* chunk_k, const void* chunk_v,
                                       const int32_t* kcache, const float* klut, const float* k_outliers,
                                       const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent,
                                       const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx,
                                       int n_out, const float* rope_cos_sin, int64_t rope_npos, int pos_offset,
                                       const void* sink_k, const void* sink_v, int n_sink, float* out, void* scratch,
                                       void* stream) {
  return attend_chunk_ragged_impl(bits, B, Hq, Hkv, Lmax, n_seg, segs, N, q, chunk_k, chunk_v, kcache, klut, k_outliers,
                                  k_outlier_idx, vcache, v_cent, v_aff, v_outliers, v_outlier_idx, n_out, rope_cos_sin,
                                  rope_npos, pos_offset, sink_k, sink_v, n_sink, out, scratch, stream, nullptr, nullptr);
}

extern "C" int kvq_attend_chunk_ragged_paged(int bits, int B, int Hq, int Hkv, int n_pool, int n_seg,
                                             const int64_t* segs, int64_t N, const float* q, const void* chunk_k,
                                             const void* chunk_v, const int32_t* kcache, const float* klut,
                                             const float* k_outliers, const int32_t* k_outlier_idx,
                                             const int32_t* vcache, const float* v_cent, const float* v_aff,
                                             const float* v_outliers, const int32_t* v_outlier_idx, int n_out,
                                             const float* rope_cos_sin, int64_t rope_npos, int pos_offset,
                                             const void* sink_k, const void* sink_v, int n_sink, float* out,
                                             void* scratch, void* stream, const int32_t* page_table, int max_pages,
                                             const int32_t* n_mapped, int P) {
  if (bits < 2 || bits > 4) return KVQ_E_BITS;
  if (Hkv <= 0 || ((Hkv & 3) != 0 && Hkv > 2)) return KVQ_E_SHAPE;
  const int rc = check_pages(n_pool, max_pages, P, (int64_t)Hkv * kHeadDim * bits / 32);
  if (rc) return rc;
  const PageRef pg{page_table, nullptr, max_pages, P, n_pool};
  return attend_chunk_ragged_impl(bits, B, Hq, Hkv, (int64_t)max_pages * P, n_seg, segs, N, q, chunk_k, chunk_v, kcache,
                                  klut, k_outliers, k_outlier_idx, vcache, v_cent, v_aff, v_outliers, v_outlier_idx,
                                  n_out, rope_cos_sin, rope_npos, pos_offset, sink_k, sink_v, n_sink, out, scratch,
                                  stream, &pg, n_mapped);
}
