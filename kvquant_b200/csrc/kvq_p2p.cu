// kvquant_b200 -- sequence-sharded decode: exchange of the per-GPU partial attention results over NVLink peer memory,
// fused with their merge.  Validated against NCCL all_gather + kvq_attend_merge (bit-identical over
// 200 rounds, tests/test_zz_p2p_exchange.py).  It is the default
// of the sequence-sharded decode (bench.py --sp-exchange p2p).
//
// No counterpart in the reference (it never shards a layer's cache).  What it replaces here is
//     dist.all_gather_into_tensor(parts) ; kvq_attend_merge(parts)            (kvquant_b200/decode.py)
// i.e. a collective launch in front of a tiny merge kernel, once per layer and token.
//
// Every rank owns one buffer, allocated with cudaMalloc and opened by its peers through CUDA IPC:
//     float  data [2][world][H*129]     slot [b][r] = rank r's (out[H][128], lse[H]) of an exchange with parity b
//     int64  flags[2][world][H]         = sequence number of the exchange whose slot [b][r], head h is complete
// One kernel per exchange, grid = H CTAs x 128 threads; CTA h
//   1. PUSHES head h of this rank's partial straight into slot [b][rank] of every peer's buffer (plain stores over
//      NVLink), fences at system scope, and releases flag [b][rank][h] = seq on every peer;
//   2. WAITS (acquire loads on its OWN buffer) until flags [b][r][h] >= seq for every r;
//   3. MERGES head h from its own buffer:  out = sum_r exp(lse_r - M) out_r / sum_r exp(lse_r - M).
// No rank waits before it has pushed, so there is no circular wait; two parities suffice because a rank can only start
// exchange n+1 after it has seen every peer's flags of exchange n, i.e. after every peer has left exchange n-1.
// seq comes from a device counter (one graph replay = the next exchange numbers); a spin limit turns a lost peer into
// an error flag instead of a hung GPU.
#include "kvq_common.cuh"
#include <string.h>

namespace kvq {

constexpr long long kP2PSpinLimit = 4000000000LL;   // ~2 s of SM clocks

__device__ __forceinline__ void st_release_sys(int64_t* p, int64_t v) {
  asm volatile("st.release.sys.global.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ int64_t ld_acquire_sys(const int64_t* p) {
  int64_t v;
  asm volatile("ld.acquire.sys.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float ld_volatile_f32(const float* p) {
  float v;
  asm volatile("ld.volatile.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(kHeadDim) attend_exchange_merge_kernel(
    const float* __restrict__ part, float* const* __restrict__ peers, int world, int rank, int H,
    const int64_t* __restrict__ seq_dev, float* __restrict__ out, int32_t* __restrict__ err) {
  __shared__ float s_w[64];
  __shared__ int s_fail;
  const int h = blockIdx.x, c = threadIdx.x;
  const int64_t seq = *seq_dev + 1;
  const int b = (int)(seq & 1);
  const int64_t slot = (int64_t)H * (kHeadDim + 1);            // floats per (parity, rank) slot
  const int64_t data_floats = 2 * (int64_t)world * slot;
  if (c == 0) s_fail = 0;
  // ---- 1. push ---------------------------------------------------------------------------------------------------
  const float v = part[h * kHeadDim + c];
  const float lse = part[H * kHeadDim + h];
  for (int r = 0; r < world; ++r) {
    float* dst = peers[r] + ((int64_t)b * world + rank) * slot;
    dst[h * kHeadDim + c] = v;
    if (c == 0) dst[H * kHeadDim + h] = lse;
  }
  __threadfence_system();
  __syncthreads();
  if (c < world) {
    int64_t* fl = reinterpret_cast<int64_t*>(peers[c] + data_floats) + ((int64_t)b * world + rank) * H + h;
    st_release_sys(fl, seq);
  }
  // ---- 2. wait ---------------------------------------------------------------------------------------------------
  const float* mine = peers[rank];
  if (c < world) {
    const int64_t* fl = reinterpret_cast<const int64_t*>(mine + data_floats) + ((int64_t)b * world + c) * H + h;
    const long long t0 = clock64();
    while (ld_acquire_sys(fl) < seq) {
      if (clock64() - t0 > kP2PSpinLimit) { s_fail = 1; break; }
      __nanosleep(64);
    }
  }
  __syncthreads();
  if (s_fail) {
    if (c == 0) atomicExch(err, 1);
    out[h * kHeadDim + c] = __int_as_float(0x7fc00000);       // NaN: never a silently wrong result
    return;
  }
  // ---- 3. merge --------------------------------------------------------------------------------------------------
  if (c < world) s_w[c] = ld_volatile_f32(mine + ((int64_t)b * world + c) * slot + H * kHeadDim + h);
  __syncthreads();
  float m = -INFINITY;
  for (int r = 0; r < world; ++r) m = fmaxf(m, s_w[r]);
  float o = 0.f, l = 0.f;
  for (int r = 0; r < world; ++r) {
    const float w = __expf(s_w[r] - m);
    o = fmaf(w, ld_volatile_f32(mine + ((int64_t)b * world + r) * slot + h * kHeadDim + c), o);
    l += w;
  }
  out[h * kHeadDim + c] = o / l;
}

__global__ void p2p_counter_add_kernel(int64_t* c) { *c += 1; }

}  // namespace kvq

using namespace kvq;

extern "C" {

int64_t kvq_p2p_buffer_bytes(int world, int H) {
  if (world <= 0 || H <= 0) return 0;
  return 2 * (int64_t)world * H * (kHeadDim + 1) * 4 + 2 * (int64_t)world * H * 8;
}

int kvq_p2p_alloc(void** ptr, int64_t bytes, void* ipc_handle_64) {
  if (!ptr || !ipc_handle_64) return KVQ_E_NULL;
  if (bytes <= 0) return KVQ_E_SHAPE;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaError_t e = cudaMalloc(ptr, (size_t)bytes);
  if (e != cudaSuccess) return (int)e;
  e = cudaMemset(*ptr, 0, (size_t)bytes);
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(static_cast<cudaIpcMemHandle_t*>(ipc_handle_64), *ptr);
  if (e != cudaSuccess) { cudaFree(*ptr); *ptr = nullptr; return (int)e; }
  return 0;
}

int kvq_p2p_open(const void* ipc_handle_64, void** ptr) {
  if (!ptr || !ipc_handle_64) return KVQ_E_NULL;
  cudaIpcMemHandle_t h;
  memcpy(&h, ipc_handle_64, sizeof(h));
  const cudaError_t e = cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
  return e == cudaSuccess ? 0 : (int)e;
}

int kvq_p2p_close(void* ptr) {
  if (!ptr) return KVQ_E_NULL;
  const cudaError_t e = cudaIpcCloseMemHandle(ptr);
  return e == cudaSuccess ? 0 : (int)e;
}

int kvq_p2p_free(void* ptr) {
  if (!ptr) return KVQ_E_NULL;
  const cudaError_t e = cudaFree(ptr);
  return e == cudaSuccess ? 0 : (int)e;
}

int kvq_attend_exchange_merge(const float* part, void* const* peers_dev, int world, int rank, int H,
                              int64_t* seq_dev, float* out, int32_t* err_flag, void* stream) {
  if (!part || !peers_dev || !seq_dev || !out || !err_flag) return KVQ_E_NULL;
  if (world <= 0 || world > 64 || rank < 0 || rank >= world || H <= 0) return KVQ_E_SHAPE;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  attend_exchange_merge_kernel<<<H, kHeadDim, 0, st>>>(part, reinterpret_cast<float* const*>(peers_dev), world, rank, H,
                                                       seq_dev, out, err_flag);
  KVQ_LAUNCH_CHECK();
  p2p_counter_add_kernel<<<1, 1, 0, st>>>(seq_dev);
  KVQ_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
