// kvquant_b200 -- declarations shared by the K-score kernels (kvq_kscore.cu, kvq_kpair.cu).
#pragma once
#include "kvq_common.cuh"

namespace kvq {

struct KParams {
  const float* q;            // [H,128]
  const uint32_t* cache;     // [H*W, Lmax]
  float* out;                // [H, out_stride]
  const float* lut;          // [H*128, N]
  const float* outliers;     // [>=L, n_out] or null (consumed by k_outlier_kernel, not by the dense kernel)
  const int32_t* outlier_idx;
  const float2* rope;        // [64, rope_npos]
  float* gmax;               // [H] or null (fused mode: running max of scaled scores)
  int64_t Lmax, L, out_stride, rope_npos;
  int64_t range;             // tokens per CTA (multiple of 32), set by the launcher
  const int64_t* len_dev;    // device-resident length (optional): L = min(*len_dev + len_add, L); L is then a cap
  int64_t len_add;
  int H, n_out, pos_offset, tiles_per_cta;
  float theta;               // rope base (outlier scatter evaluates cos/sin of theta_j * pos directly)
  float scale;               // applied before the store (fused mode: 1/sqrt(128)); 1 for legacy
  int accumulate;            // 1: out = (out + S)*scale, 0: out = S*scale
  const float* opart;        // fused path: outlier partial sums, TOKEN-major [L][opart_stride] (null: none / in `out`)
  int opart_stride;          // floats per token row (H rounded up to 32: one 128-byte line per 32 heads)
  const uint32_t* rope_h;    // optional half2 copy of the rope table (fp16 mode of the fused attend: the outlier scatter
                             // gathers 4-byte entries from the table the dense kernel streams anyway)
};

// compile-time loop (immediate LDS offsets and PRMT selectors need constant expressions)
template <int K> struct IC { static constexpr int v = K; };
template <int B, int E, class F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (B < E) { f(IC<B>{}); static_for<B + 1, E>(f); }
}
// 8-byte shared load at [addr + IMM] (addr is a 32-bit shared-window address)
template <int IMM>
__device__ __forceinline__ float2 lds_f2(uint32_t addr) {
  float2 v;
  asm("ld.shared.v2.f32 {%0,%1}, [%2+%3];" : "=f"(v.x), "=f"(v.y) : "r"(addr), "n"(IMM));
  return v;
}
// acc.xy += a.xy * b.xy, each lane one fused, round-to-nearest fp32 FMA (sm_90 has no packed FFMA2: two FFMA)
__device__ __forceinline__ void ffma2(float2& acc, const float2 a, const float2 b) {
  acc.x = __fmaf_rn(a.x, b.x, acc.x);
  acc.y = __fmaf_rn(a.y, b.y, acc.y);
}
// effective length / per-CTA range of a launch whose length lives on the device (CUDA-graph replays with a growing
// cache): the grid was sized for the cap p.L, the kernel re-derives its split from the current length
__device__ __forceinline__ int64_t k_eff_len(const KParams& p) {
  if (p.len_dev == nullptr) return p.L;
  const int64_t l = *p.len_dev + p.len_add;
  return l < 0 ? 0 : (l < p.L ? l : p.L);
}
__device__ __forceinline__ int64_t k_eff_range(const KParams& p, int64_t L) {
  if (p.len_dev == nullptr) return p.range;
  const int64_t r = (L + gridDim.x - 1) / gridDim.x;
  return (r + 31) & ~(int64_t)31;
}
// tokens per CTA when L tokens are cut into at most `splits` ranges: warp granularity, >= 32
inline int64_t k_token_range(int64_t L, int64_t splits) {
  const int64_t r = (L + splits - 1) / splits;
  return (r + 31) & ~(int64_t)31;
}
// dense K-score kernel, pair-table form (kvq_kpair.cu); bits 4 and 3
int k_pair_dispatch(int bits, const KParams& p, cudaStream_t st);
// dense K-score kernel, 3-bit, carried words (kvq_k3.cu)
int k_scores3_dispatch(const KParams& p, cudaStream_t st);
// dense K-score kernel of the fused attend, exact fp32 ratio form (kvq_kratio.cu)
int k_ratio_dispatch(int bits, const float* q, const int32_t* cache, float* scores, int64_t score_stride, const float* lut,
                     int H, int64_t Lmax, int64_t L, const float* rope, int64_t rope_npos, int pos_offset, float* gmax,
                     float scale, int accumulate, const int64_t* len_dev, int64_t len_add, void* qtab, int64_t t0,
                     int run_prep, cudaStream_t st);
// dense K-score kernel of the fused attend, fp16-table form (kvq_kfast.cu)
int k_fast_dispatch(int bits, const float* q, const int32_t* cache, float* scores, int64_t score_stride, const float* lut,
                    int H, int64_t Lmax, int64_t L, const void* rope_half, int64_t rope_npos, int pos_offset, float* gmax,
                    float scale, int accumulate, const int64_t* len_dev, int64_t len_add, void* qtab, int64_t t0,
                     int run_prep, cudaStream_t st);

}  // namespace kvq
