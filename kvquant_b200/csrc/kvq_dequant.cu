// kvquant_b200 -- dequantisation of a slot range of a layer cache to fp16 K (pre-RoPE or rotated) and V.
//
// One kernel per side, persistent CTAs: CTA (x, y) owns head group y (kGroup heads) and walks the token tiles
// x, x + gridDim.x, ...  Per tile of kTile tokens:
//   1. the group's packed words are read coalesced along the sequence axis into shared memory, token-major
//      (so code_of<BITS> reads one token's words contiguously); K also stages the tile's cos/sin, V its (sf, off);
//   2. one thread per (head, token, 32-channel group) dequantises into an fp32 tile [kGroup][kTile][128 + 4]: the group's
//      words in registers, code_of<BITS> at compile-time channel offsets (K: the group's LUT, staged once per CTA as
//      [channel][2^BITS + 1], so the 32 tokens of a warp, one channel, meet distinct codes in distinct banks; V:
//      v_cent[code]*sf + off as one fma); padded rows keep the warp's 16-byte tile stores conflict-free;
//   3. the tile's outlier entries that fall in the group are added (shared-memory atomics: a V row may repeat
//      channel 0 as a pad, whose value 0 is skipped);
//   4. each thread converts 8 consecutive channels of one token to fp16 and writes them as one 16-byte store --
//      for rotated K after combining with the partner channels c ^ 64, which step 3 has already completed.
#include <cuda_fp16.h>

#include "kvq_common.cuh"

namespace kvq {

constexpr int kTile = 32;       // tokens per tile
constexpr int kGroup = 2;       // heads per CTA (every accepted H is a multiple of 4)
constexpr int kThreads = 256;
constexpr int kMaxOutDq = 128;  // outlier row width bound (2 * n_each, n_each <= 64)
constexpr int kRopePitch = 65;  // float2 per staged cos/sin row (one token); odd pitch spreads the transposing writes
constexpr int kTP = kHeadDim + 4;  // fp32 tile row pitch (one token of one head)

struct DqParams {
  const int32_t* cache;
  const float* klut;        // K: [H*128, 2^BITS]
  const float* v_cent;      // V: [2^BITS]
  const float* v_aff;       // V: [Lmax, 2] = (sf, off)
  const float* outliers;    // [Lmax, n_out] or NULL
  const int32_t* outlier_idx;
  const float2* rope;       // K: [64, rope_npos] (cos, sin) or NULL
  int64_t rope_npos;
  int64_t pos_offset;
  __half* out;
  int64_t head_stride;
  int64_t Lmax, start, stop;
  int n_out;
};

template <int BITS>
struct DqLayout {
  static constexpr int W = Layout<BITS>::kWords;
  static constexpr int kWPitch = W + 1;  // odd pitch: the transposing word stores of a warp hit distinct banks
  static constexpr int kWordsSmem = kGroup * kTile * kWPitch;
  static constexpr int kTileSmem = kGroup * kTile * kTP;
  static constexpr int kLP = Layout<BITS>::kLevels + 1;   // K LUT pitch per channel
};

template <int BITS>
__host__ __device__ constexpr size_t dq_smem_bytes(bool is_v, bool rope) {
  using D = DqLayout<BITS>;
  return sizeof(float) * (D::kTileSmem + D::kWordsSmem) +
         (is_v ? sizeof(float) * (Layout<BITS>::kLevels + 2 * kTile)
               : sizeof(float) * DqLayout<BITS>::kLP * kGroup * kHeadDim + (rope ? sizeof(float2) * kTile * kRopePitch : 0));
}

// IS_V: V side (affine centroids) else K side (per-channel LUT, optional rotation)
template <int BITS, bool IS_V, bool ROPE>
__global__ void __launch_bounds__(kThreads, 3) dequant_kernel(const DqParams p) {
  using D = DqLayout<BITS>;
  constexpr int W = D::W;
  constexpr int NL = Layout<BITS>::kLevels;
  extern __shared__ __align__(16) float smem[];
  float* tile = smem;                                                       // [kGroup][kTile][kTP]
  uint32_t* words = reinterpret_cast<uint32_t*>(tile + D::kTileSmem);       // [kGroup][kTile][kWPitch]
  float* tab = reinterpret_cast<float*>(words + D::kWordsSmem);             // K: LUT [kGroup*128][kLP]; V: cent[NL], aff[kTile][2]
  float2* cs = reinterpret_cast<float2*>(tab + D::kLP * kGroup * kHeadDim); // K + ROPE: [kTile][kRopePitch]
  float* aff = tab + NL;

  const int tid = threadIdx.x;
  const int h0 = blockIdx.y * kGroup;
  if constexpr (IS_V) {
    if (tid < NL) tab[tid] = p.v_cent[tid];
  } else {
    for (int i = tid; i < kGroup * kHeadDim * NL; i += kThreads)
      tab[(i / NL) * D::kLP + i % NL] = p.klut[(int64_t)h0 * kHeadDim * NL + i];
  }

  const int64_t n = p.stop - p.start;
  const int64_t n_tiles = (n + kTile - 1) / kTile;
  for (int64_t tl = blockIdx.x; tl < n_tiles; tl += gridDim.x) {
    const int64_t t0 = p.start + tl * kTile;                  // first slot of the tile
    const int nt = (int)min((int64_t)kTile, p.stop - t0);
    __syncthreads();                                          // previous tile fully written out
    for (int i = tid; i < kGroup * W * kTile; i += kThreads) {
      const int r = i / kTile, t = i % kTile;                 // r: word row within the group, t fastest (coalesced)
      uint32_t w = 0;
      if (t < nt) w = static_cast<uint32_t>(p.cache[((int64_t)h0 * W + r) * p.Lmax + t0 + t]);
      words[((r / W) * kTile + t) * D::kWPitch + (r % W)] = w;
    }
    if constexpr (IS_V) {
      if (tid < 2 * kTile) aff[tid] = tid < 2 * nt ? p.v_aff[2 * t0 + tid] : 0.f;
    } else if constexpr (ROPE) {
      for (int i = tid; i < 64 * kTile; i += kThreads) {
        const int j = i / kTile, t = i % kTile;                // position-fastest table: t fastest is coalesced
        cs[t * kRopePitch + j] = t < nt ? p.rope[(int64_t)j * p.rope_npos + p.pos_offset + t0 + t] : make_float2(0.f, 0.f);
      }
    }
    __syncthreads();
    for (int i = tid; i < kGroup * kTile * 4; i += kThreads) {
      const int t = i % kTile, q = (i / kTile) % 4, g = i / (4 * kTile);   // lanes: 32 tokens of one channel group
      constexpr int WQ = W / 4;                                // words of 32 channels: 4 / 3 / 2
      uint32_t w[WQ];
#pragma unroll
      for (int k = 0; k < WQ; ++k) w[k] = words[(g * kTile + t) * D::kWPitch + q * WQ + k];
      float* dst = tile + (g * kTile + t) * kTP + q * 32;
      const float* lut = tab + (g * kHeadDim + q * 32) * D::kLP;
      float sf = 0.f, off = 0.f;
      if constexpr (IS_V) { sf = aff[2 * t]; off = aff[2 * t + 1]; }
#pragma unroll
      for (int l = 0; l < 32; l += 4) {
        float x[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t code = code_of<BITS>(w, l + k);
          if constexpr (IS_V) x[k] = fmaf(tab[code], sf, off);
          else x[k] = lut[(l + k) * D::kLP + code];
        }
        *reinterpret_cast<float4*>(dst + l) = make_float4(x[0], x[1], x[2], x[3]);
      }
    }
    if (p.outliers != nullptr) {
      __syncthreads();
      const int64_t row0 = t0 * p.n_out;
      for (int i = tid; i < nt * p.n_out; i += kThreads) {
        const int idx = p.outlier_idx[row0 + i];
        const int g = (idx >> 7) - h0;
        if (g >= 0 && g < kGroup) {
          const float v = p.outliers[row0 + i];
          if (v != 0.f) atomicAdd(&tile[(g * kTile + i / p.n_out) * kTP + (idx & 127)], v);
        }
      }
    }
    __syncthreads();
    for (int i = tid; i < kGroup * kTile * (kHeadDim / 8); i += kThreads) {
      const int q = i % (kHeadDim / 8), gt = i / (kHeadDim / 8);
      const int t = gt % kTile, g = gt / kTile;
      if (t >= nt) continue;
      const int c0 = q * 8;
      const float* src = tile + gt * kTP;
      const float4 a = *reinterpret_cast<const float4*>(src + c0);
      const float4 b = *reinterpret_cast<const float4*>(src + c0 + 4);
      float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      if constexpr (!IS_V && ROPE) {
        // k'[c] = cos*k[c] - sin*k[c+64] (c < 64), cos*k[c] + sin*k[c-64] (c >= 64); j = c mod 64
        const float4 pa = *reinterpret_cast<const float4*>(src + (c0 ^ 64));
        const float4 pb = *reinterpret_cast<const float4*>(src + (c0 ^ 64) + 4);
        const float pv[8] = {pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w};
        const float sgn = c0 < 64 ? -1.f : 1.f;
        const float2* row = cs + t * kRopePitch + (c0 & 63);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float2 r = row[k];
          v[k] = r.x * v[k] + sgn * (r.y * pv[k]);
        }
      }
      uint4 o;
      __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int k = 0; k < 4; ++k) oh[k] = __floats2half2_rn(v[2 * k], v[2 * k + 1]);
      __half* dst = p.out + (int64_t)(h0 + g) * p.head_stride + (t0 - p.start + t) * kHeadDim + c0;
      *reinterpret_cast<uint4*>(dst) = o;
    }
  }
}

template <int BITS, bool IS_V, bool ROPE>
int launch_dequant(const DqParams& p, int H, cudaStream_t st) {
  auto kern = dequant_kernel<BITS, IS_V, ROPE>;
  const size_t smem = dq_smem_bytes<BITS>(IS_V, ROPE);
  static PerDeviceOnce attr_once;
  bool& attr_done = attr_once.cur();
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_done = true;
  }
  int dev = 0, sms = 0, per_sm = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem);
  if (e != cudaSuccess) return (int)e;
  // one wave of resident CTAs: the head groups side by side (they read the same tile's outlier rows and cos/sin at
  // about the same time), the token tiles split evenly over the rest
  const int groups = H / kGroup;
  const int64_t n_tiles = (p.stop - p.start + kTile - 1) / kTile;
  const int64_t per_group = max(1, sms * max(per_sm, 1) / groups);
  const dim3 grid((unsigned)min(n_tiles, per_group), (unsigned)groups);
  kern<<<grid, kThreads, smem, st>>>(p);
  KVQ_LAUNCH_CHECK();
  return 0;
}

template <int BITS>
int dequant_bits(const DqParams& pk, const DqParams& pv, int H, cudaStream_t st) {
  int rc = 0;
  if (pk.out) rc = pk.rope ? launch_dequant<BITS, false, true>(pk, H, st) : launch_dequant<BITS, false, false>(pk, H, st);
  if (rc == 0 && pv.out) rc = launch_dequant<BITS, true, false>(pv, H, st);
  return rc;
}

}  // namespace kvq

using namespace kvq;

extern "C" int kvq_dequant_kv(int bits, int H, int64_t Lmax, int64_t start, int64_t stop,
                              const int32_t* kcache, const float* klut, const float* k_outliers,
                              const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent,
                              const float* v_aff, const float* v_outliers, const int32_t* v_outlier_idx, int n_out,
                              const float* rope_cos_sin, int64_t rope_npos, int pos_offset, void* out_k, void* out_v,
                              int64_t head_stride, void* stream) {
  if (bits < 2 || bits > 4) return KVQ_E_BITS;
  if (H <= 0 || (H & 3) != 0 || H > 64 || Lmax <= 0 || start < 0 || start > stop || stop > Lmax) return KVQ_E_SHAPE;
  if (n_out < 0 || (n_out & 1) != 0 || n_out > kMaxOutDq) return KVQ_E_SHAPE;
  if (head_stride < (stop - start) * kHeadDim) return KVQ_E_SHAPE;
  if (start == stop) return 0;   // nothing to write: outputs of zero elements may well be NULL
  if (!out_k && !out_v) return KVQ_E_NULL;
  if (out_k && (!kcache || !klut)) return KVQ_E_NULL;
  if (out_v && (!vcache || !v_cent || !v_aff)) return KVQ_E_NULL;
  if ((k_outliers == nullptr) != (k_outlier_idx == nullptr) || (v_outliers == nullptr) != (v_outlier_idx == nullptr))
    return KVQ_E_NULL;
  if ((k_outliers || v_outliers) && n_out == 0) return KVQ_E_SHAPE;
  if (out_k && rope_cos_sin && (pos_offset < 0 || rope_npos < (int64_t)pos_offset + stop)) return KVQ_E_SHAPE;
  if ((head_stride & 7) != 0 || (reinterpret_cast<uintptr_t>(out_k) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(out_v) & 15) != 0)
    return KVQ_E_ALIGN;

  DqParams pk{}, pv{};
  pk.Lmax = pv.Lmax = Lmax;
  pk.start = pv.start = start;
  pk.stop = pv.stop = stop;
  pk.head_stride = pv.head_stride = head_stride;
  pk.n_out = pv.n_out = n_out;
  pk.cache = kcache; pk.klut = klut; pk.outliers = k_outliers; pk.outlier_idx = k_outlier_idx;
  pk.rope = reinterpret_cast<const float2*>(rope_cos_sin); pk.rope_npos = rope_npos; pk.pos_offset = pos_offset;
  pk.out = static_cast<__half*>(out_k);
  pv.cache = vcache; pv.v_cent = v_cent; pv.v_aff = v_aff; pv.outliers = v_outliers; pv.outlier_idx = v_outlier_idx;
  pv.out = static_cast<__half*>(out_v);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (bits) {
    case 4: return dequant_bits<4>(pk, pv, H, st);
    case 3: return dequant_bits<3>(pk, pv, H, st);
    default: return dequant_bits<2>(pk, pv, H, st);
  }
}
