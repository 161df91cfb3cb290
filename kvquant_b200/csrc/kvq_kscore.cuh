// kvquant_b200 -- declarations shared by the K-score kernels (kvq_kscore.cu, kvq_k3.cu).
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
  int64_t Lmax, L, out_stride, rope_npos;
  int64_t range;             // tokens per CTA (multiple of 32), set by the launcher
  const int64_t* len_dev;    // device-resident length of the outlier pass (optional): L = min(*len_dev + len_add, L), L a cap
  int64_t len_add;
  int H, n_out, pos_offset;
  float theta;               // rope base (outlier scatter evaluates cos/sin of theta_j * pos directly)
  const uint32_t* rope_h;    // optional half2 copy of the rope table (fp16 mode of the fused attend: the outlier scatter
                             // gathers 4-byte entries from the table the dense kernel streams anyway)
  int grp;                   // query heads per KV head (H counts query heads; the fused attend's outlier pass only)
  bool freq;                 // scaled rotary frequencies: the outlier pass computes cos / sin of rope_freq[j] * pos,
  const float* rope_freq;    // times attn, instead of using theta (the fused attend's outlier pass only)
  float attn;
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
// tokens per CTA when L tokens are cut into at most `splits` ranges: warp granularity, >= 32
inline int64_t k_token_range(int64_t L, int64_t splits) {
  const int64_t r = (L + splits - 1) / splits;
  return (r + 31) & ~(int64_t)31;
}
// dense K-score kernel, 3-bit, carried words (kvq_k3.cu)
int k_scores3_dispatch(const KParams& p, cudaStream_t st);

}  // namespace kvq
