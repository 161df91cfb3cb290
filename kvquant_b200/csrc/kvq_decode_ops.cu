// kvquant_b200 -- small fused element-wise kernels of the LLaMA decode harness (kvquant_b200/decode.py).
// NOT part of the reference's quant_cuda surface: these replace ~25 tiny torch launches per layer around the hot
// path (RMSNorm = 7 torch kernels, HF rotate-half RoPE on Q + fp32 split of q/k/v = 9, SwiGLU = 3) so that the
// decode-step graph is dominated by the KV-cache kernels and the cuBLAS GEMVs.
#include "kvq_common.cuh"
#include <cuda_fp16.h>

namespace kvq {

// y = (x.float() * rsqrt(mean(x^2) + eps)).half() * w          (HF LlamaRMSNorm semantics, fp16 in/out)
__global__ void __launch_bounds__(1024) dec_rmsnorm_kernel(const __half* __restrict__ x, const __half* __restrict__ w,
                                                           __half* __restrict__ y, int n, float eps) {
  __shared__ float s_red[32];
  float ss = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { const float v = __half2float(x[i]); ss = fmaf(v, v, ss); }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? s_red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) s_red[0] = rsqrtf(v / (float)n + eps);
  }
  __syncthreads();
  const float r = s_red[0];
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    y[i] = __hmul(__float2half(__half2float(x[i]) * r), w[i]);
}

// Row b = blockIdx.y of qkv fp16 [B][hidden + 2*kv_hidden] -> q (HF rotate-half RoPE at `pos`, modeling_llama.py:
// 1851-1859) f32 [B][hidden], k, v f32 [B][kv_hidden] (kv_hidden < hidden: grouped-query attention).  pos = pos_add,
// plus pos_dev[b] when given (device-resident positions: graph replays with a growing cache).  Row b turns at
// inv_freq[b * f_stride + j] (f_stride 64: length-dependent frequencies, one vector per row; 0: one shared vector), and
// cos / sin are times attn -- HF's attention_factor, applied to the query as to the keys (rope_table_kernel); attn = 1
// for theta, where the product is exact.
__global__ void dec_rope_split_kernel(const __half* __restrict__ qkv, const float* __restrict__ inv_freq, int f_stride,
                                      float attn, float pos_add, const int64_t* __restrict__ pos_dev,
                                      float* __restrict__ q, float* __restrict__ k, float* __restrict__ v, int hidden,
                                      int kv_hidden) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hidden) return;
  const int64_t r = blockIdx.y;
  inv_freq += r * f_stride;
  qkv += r * (hidden + 2 * kv_hidden);
  q += r * hidden; k += r * kv_hidden; v += r * kv_hidden;
  const float pos = pos_dev != nullptr ? pos_add + (float)pos_dev[r] : pos_add;
  const int c = i & (kHeadDim - 1), j = c & (kHalf - 1);
  const float ang = inv_freq[j] * pos;
  float sn, cs;
  sincosf(ang, &sn, &cs);
  cs *= attn;
  sn *= attn;
  const float a = __half2float(qkv[i]);
  const float b = __half2float(qkv[i ^ kHalf]);
  q[i] = a * cs + ((c < kHalf) ? -b : b) * sn;
  if (i < kv_hidden) {
    k[i] = __half2float(qkv[hidden + i]);
    v[i] = __half2float(qkv[hidden + kv_hidden + i]);
  }
}

// act = silu(gate) * up, gu fp16 [2*n] -> fp16 [n]
__global__ void dec_silu_mul_kernel(const __half* __restrict__ gu, __half* __restrict__ act, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float g = __half2float(gu[i]);
  const __half s = __float2half(g / (1.f + __expf(-g)));
  act[i] = __hmul(s, gu[n + i]);
}

__global__ void dec_counter_add_kernel(int64_t* c, int64_t d) { *c += d; }

// counter[b] += delta for every b with active[b] != 0 (active == null: every b)
__global__ void dec_counter_add_batch_kernel(int64_t* c, const int32_t* __restrict__ active, int64_t d, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B && (active == nullptr || active[b] != 0)) c[b] += d;
}

__global__ void dec_f32_to_f16_kernel(const float* __restrict__ a, __half* __restrict__ b, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) b[i] = __float2half(a[i]);
}

}  // namespace kvq

using namespace kvq;

extern "C" {

int kvq_dec_rmsnorm(const void* x_f16, const void* w_f16, void* y_f16, int n, float eps, void* stream) {
  if (!x_f16 || !w_f16 || !y_f16) return KVQ_E_NULL;
  if (n <= 0) return KVQ_E_SHAPE;
  dec_rmsnorm_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(x_f16), static_cast<const __half*>(w_f16), static_cast<__half*>(y_f16), n, eps);
  KVQ_LAUNCH_CHECK();
  return 0;
}

static int check_split_gqa(int Hq, int Hkv) {
  return (Hq <= 0 || Hkv <= 0 || Hq % Hkv != 0) ? KVQ_E_SHAPE : 0;
}

// the launch every kvq_dec_rope_split* entry point makes once its arguments are checked: B rows of Hq query heads
static int dec_rope_split(const void* qkv_f16, const float* inv_freq, int f_stride, float attn, float pos_add,
                          const int64_t* pos_dev, float* q, float* k, float* v, int Hq, int Hkv, int B, void* stream) {
  const int hidden = Hq * kHeadDim;
  dec_rope_split_kernel<<<dim3((hidden + 255) / 256, B), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(qkv_f16), inv_freq, f_stride, attn, pos_add, pos_dev, q, k, v, hidden, Hkv * kHeadDim);
  KVQ_LAUNCH_CHECK();
  return 0;
}

int kvq_dec_rope_split(const void* qkv_f16, const float* inv_freq, float pos, float* q, float* k, float* v, int hidden,
                       void* stream) {
  if (!qkv_f16 || !inv_freq || !q || !k || !v) return KVQ_E_NULL;
  if (hidden <= 0 || (hidden % kHeadDim) != 0) return KVQ_E_SHAPE;
  return dec_rope_split(qkv_f16, inv_freq, 0, 1.f, pos, nullptr, q, k, v, hidden / kHeadDim, hidden / kHeadDim, 1, stream);
}

int kvq_dec_rope_split_dyn(const void* qkv_f16, const float* inv_freq, const int64_t* pos_dev, int64_t pos_add,
                           float* q, float* k, float* v, int hidden, void* stream) {
  if (!qkv_f16 || !inv_freq || !pos_dev || !q || !k || !v) return KVQ_E_NULL;
  if (hidden <= 0 || (hidden % kHeadDim) != 0) return KVQ_E_SHAPE;
  return dec_rope_split(qkv_f16, inv_freq, 0, 1.f, (float)pos_add, pos_dev, q, k, v, hidden / kHeadDim, hidden / kHeadDim, 1,
                        stream);
}

int kvq_dec_rope_split_gqa(const void* qkv_f16, const float* inv_freq, float pos, float* q, float* k, float* v, int Hq,
                           int Hkv, void* stream) {
  if (!qkv_f16 || !inv_freq || !q || !k || !v) return KVQ_E_NULL;
  if (check_split_gqa(Hq, Hkv)) return KVQ_E_SHAPE;
  return dec_rope_split(qkv_f16, inv_freq, 0, 1.f, pos, nullptr, q, k, v, Hq, Hkv, 1, stream);
}

int kvq_dec_rope_split_gqa_dyn(const void* qkv_f16, const float* inv_freq, const int64_t* pos_dev, int64_t pos_add,
                               float* q, float* k, float* v, int Hq, int Hkv, void* stream) {
  if (!qkv_f16 || !inv_freq || !pos_dev || !q || !k || !v) return KVQ_E_NULL;
  if (check_split_gqa(Hq, Hkv)) return KVQ_E_SHAPE;
  return dec_rope_split(qkv_f16, inv_freq, 0, 1.f, (float)pos_add, pos_dev, q, k, v, Hq, Hkv, 1, stream);
}

int kvq_dec_counter_add(int64_t* counter, int64_t delta, void* stream) {
  if (!counter) return KVQ_E_NULL;
  dec_counter_add_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(counter, delta);
  KVQ_LAUNCH_CHECK();
  return 0;
}

int kvq_dec_rope_split_batch(const void* qkv_f16, const float* inv_freq, const int64_t* pos_dev, int64_t pos_add,
                             float* q, float* k, float* v, int Hq, int Hkv, int B, void* stream) {
  if (!qkv_f16 || !inv_freq || !pos_dev || !q || !k || !v) return KVQ_E_NULL;
  if (check_split_gqa(Hq, Hkv) || B < 1 || B > 65535) return KVQ_E_SHAPE;
  return dec_rope_split(qkv_f16, inv_freq, 0, 1.f, (float)pos_add, pos_dev, q, k, v, Hq, Hkv, B, stream);
}

int kvq_dec_rope_split_freq(const void* qkv_f16, const float* inv_freq, float attn_factor, const int64_t* pos_dev,
                            int64_t pos_add, float* q, float* k, float* v, int Hq, int Hkv, int B, void* stream) {
  if (!qkv_f16 || !inv_freq || !q || !k || !v) return KVQ_E_NULL;
  if (check_split_gqa(Hq, Hkv) || B < 1 || B > 65535) return KVQ_E_SHAPE;
  if (!(attn_factor > 0.f && attn_factor < INFINITY)) return KVQ_E_SHAPE;
  return dec_rope_split(qkv_f16, inv_freq, 0, attn_factor, (float)pos_add, pos_dev, q, k, v, Hq, Hkv, B, stream);
}

int kvq_dec_rope_split_freq_seq(const void* qkv_f16, const float* inv_freq, float attn_factor, const int64_t* pos_dev,
                                int64_t pos_add, float* q, float* k, float* v, int Hq, int Hkv, int B, void* stream) {
  if (!qkv_f16 || !inv_freq || !q || !k || !v) return KVQ_E_NULL;
  if (check_split_gqa(Hq, Hkv) || B < 1 || B > 65535) return KVQ_E_SHAPE;
  if (!(attn_factor > 0.f && attn_factor < INFINITY)) return KVQ_E_SHAPE;
  return dec_rope_split(qkv_f16, inv_freq, kHalf, attn_factor, (float)pos_add, pos_dev, q, k, v, Hq, Hkv, B, stream);
}

int kvq_dec_counter_add_batch(int64_t* counter, const int32_t* active, int64_t delta, int B, void* stream) {
  if (!counter) return KVQ_E_NULL;
  if (B < 1) return KVQ_E_SHAPE;
  dec_counter_add_batch_kernel<<<(B + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(counter, active, delta, B);
  KVQ_LAUNCH_CHECK();
  return 0;
}

int kvq_dec_silu_mul(const void* gu_f16, void* act_f16, int n, void* stream) {
  if (!gu_f16 || !act_f16) return KVQ_E_NULL;
  if (n <= 0) return KVQ_E_SHAPE;
  dec_silu_mul_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(gu_f16), static_cast<__half*>(act_f16), n);
  KVQ_LAUNCH_CHECK();
  return 0;
}

int kvq_dec_f32_to_f16(const float* a, void* b_f16, int n, void* stream) {
  if (!a || !b_f16) return KVQ_E_NULL;
  if (n <= 0) return KVQ_E_SHAPE;
  dec_f32_to_f16_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(a, static_cast<__half*>(b_f16), n);
  KVQ_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
