/*
 * kvquant_b200 -- C ABI of the H100-native KVQuant deployment hot path.
 *
 * This header is the drop-in boundary (SURVEY.md section 8b).  Every entry point takes plain device pointers,
 * sizes and a CUDA stream; nothing here mentions torch.  The reference binds the same operations through
 * pybind11 in deployment/kvquant/quant_cuda.cpp (34 free functions, m.def list at quant_cuda.cpp:401-436);
 * the Python shim kvquant_b200/quant_cuda.py re-exports those 34 names on top of this ABI (see INTEGRATION.md).
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host;
 *   - cache:   int32 [H, W, Lmax], W = 128*bits/32, sequence fastest (reference layout, modeling_llama.py:392,1012;
 *              packing rules quant_cuda_kernel.cu:1240-1243 (4b), 1395-1424 (3b), 1601-1604 (2b));
 *   - head_dim is 128 (every reference kernel assumes it, quant_cuda_kernel.cu:3107-3108,3120);
 *   - offsets are 64-bit (the reference's 32-bit `fullwidth*row+col` overflows at Lmax > 4.19M);
 *   - return value: 0 on success, a positive cudaError_t for CUDA failures, a negative KVQ_E_* for bad arguments.
 *     (The reference aborts the process on shape mismatch via device-side assert -- quant_cuda_kernel.cu:1184-1187.)
 *   - `stream` is a cudaStream_t passed as void*; NULL = legacy default stream (what the reference always uses).
 */
#ifndef KVQUANT_B200_H
#define KVQUANT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KVQ_ABI_VERSION 2

#if defined(__GNUC__)
#define KVQ_API __attribute__((visibility("default")))
#else
#define KVQ_API
#endif

#define KVQ_E_BITS      (-1) /* bits not in {2,3,4} */
#define KVQ_E_SHAPE     (-2) /* inconsistent sizes (H<=0, slot>=Lmax, L>Lmax, n_out odd, ...) */
#define KVQ_E_NULL      (-3) /* required pointer is NULL */
#define KVQ_E_ALIGN     (-4) /* pointer / Lmax alignment requirement violated */
#define KVQ_E_UNSUPPORTED (-5)

KVQ_API int kvq_abi_version(void);
KVQ_API const char* kvq_error_string(int code);
/* number of kernels launched by this library in this process (bench.py's gpu_launches evidence) */
KVQ_API uint64_t kvq_launch_count(void);

/* ---------------------------------------------------------------------------------------------------------------
 * Append (quantise + pack), one token.  Replaces vecquant{4,3,2}appendvecK   (quant_cuda.cpp:5-33;  kernel
 * quant_cuda_kernel.cu:1202-1245,1357-1425,1563-1606) and vecquant{4,3,2}appendvecV (quant_cuda.cpp:96-126;
 * kernel 1280-1320).  code = argmin_i |lut[i]-x|, first minimum wins; the packed word is ADDED to the cache word
 * (reference atomicAdd semantics: the slot must be zero for a meaningful result).
 *   lut (K): f32 [H*128, 2^bits] per channel.      lut_tok (V): f32 [Lmax, 2^bits], row `slot` is used.
 * ------------------------------------------------------------------------------------------------------------- */
KVQ_API int kvq_append_k(int bits, int32_t* cache, const float* lut, const float* newvec,
                 int H, int64_t Lmax, int64_t slot, void* stream);
KVQ_API int kvq_append_v(int bits, int32_t* cache, const float* lut_tok, const float* newvec,
                 int H, int64_t Lmax, int64_t slot, void* stream);

/* vecquant{4,3,2}appendvecKsparse (quant_cuda.cpp:35-93; kernel 1725-1781): dense code as above plus
 * outliers_rescaled[j] = (x_j - (up_j+lo_j)/2) / ((up_j-lo_j)/2)  (f32 [H*128], written). */
KVQ_API int kvq_append_k_sparse(int bits, int32_t* cache, const float* lut, const float* newvec,
                        float* outliers_rescaled, const float* thr_lower, const float* thr_upper,
                        int H, int64_t Lmax, int64_t slot, void* stream);
/* vecquant{4,3,2}appendvecVsparse (quant_cuda.cpp:128-175; kernel 2049-2102): x<lo or x>hi -> zero-point code
 * 7/3/1, else nearest entry of lut_tok[slot].  `zeropoint` is accepted and unused, as in the reference. */
KVQ_API int kvq_append_v_sparse(int bits, int32_t* cache, const float* lut_tok, const float* newvec,
                        float zeropoint, float thr_lower, float thr_upper,
                        int H, int64_t Lmax, int64_t slot, void* stream);

/* Prefill packers.  vecquant{4,3,2}appendvecKsparseParallel (kernel 1829-1898) / ...VsparseParallel (1944-2009).
 * newvec, outliers_rescaled: f32 [H,128,T] (token fastest); tokens go to slots 0..T-1; words are ADDED.
 * V: lut_tok f32 [Lmax,2^bits] row t for token t; thr_lower/upper f32 [T].
 * (The reference's 3-bit V variant indexes the LUT by channel for entries 1..7 -- quant_cuda_kernel.cu:2574-2579,
 * a defect; this library implements the single-token semantics for all bit widths, see DESIGN.md.) */
KVQ_API int kvq_append_k_sparse_parallel(int bits, int32_t* cache, const float* lut, const float* newvec,
                                 float* outliers_rescaled, const float* thr_lower, const float* thr_upper,
                                 int H, int64_t Lmax, int64_t T, void* stream);
KVQ_API int kvq_append_v_sparse_parallel(int bits, int32_t* cache, const float* lut_tok, const float* newvec,
                                 const float* thr_lower, const float* thr_upper,
                                 int H, int64_t Lmax, int64_t T, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * RoPE table.  rope[j*n_pos + p] = (cosf(th_j*p), sinf(th_j*p)), th_j = powf(theta, (-2*j)/128), j<64 --
 * exactly the expressions of quant_cuda_kernel.cu:3081,3123-3126 evaluated once per (j,p) instead of once per
 * (head, channel, token).  float2 [64, n_pos]. */
KVQ_API int kvq_rope_table_build(float* rope_cos_sin, float theta, int64_t n_pos, void* stream);
/* The same table rounded once to fp16: half2 [64, n_pos] = (cos, sin) -- read by the fp16 mode of kvq_attend. */
KVQ_API int kvq_rope_table_build_half(void* rope_half, float theta, int64_t n_pos, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Legacy decode matvecs (results are ADDED to `mul`, which the caller pre-zeroes -- modeling_llama.py:782,1209).
 *
 * kvq_k_matvec replaces vecquant{4,3,2}matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt
 * (quant_cuda.cpp:188-198; kernel 3040-3209) and, with outliers != NULL, ..._opt2 (quant_cuda.cpp:200-212; dense
 * kernel + SPMV_ATOMIC_ROPE_BALANCED 472-521) in ONE call (outlier scatter + dense kernel on `stream`):
 *   mul[b,h,t] += sum_c (LUT[h,c,code] (+) outlier) * (cos(th_c*p)*q[b,h,c] + s_c*sin(th_c*p)*q[b,h,(c+64)%128])
 *   p = t + pos_offset.   q f32 [B,H,128]; mul f32 [B,H,L]; lut f32 [H*128,2^bits];
 *   outliers f32 [>=L, n_out], outlier_idx i32 [>=L, n_out] (flat channel index), B must be 1 when given;
 *   rope: table from kvq_rope_table_build(theta) covering positions [0, pos_offset+L), with row length rope_npos
 *   (used by the dense kernel and by the outlier scatter); theta: the rope base the table was built with (kept in the
 *   signature for callers that build the table lazily; the kernels take every cos/sin from the table).
 * kvq_v_matvec replaces ..._transposed_mha_batched_fused_opt (quant_cuda.cpp:214-224; kernel 3211-3433) and ..._opt2
 * (quant_cuda.cpp:226-238; + SPMV_ATOMIC_BALANCED 436-470):
 *   mul[b,h,c] += sum_t (LUT[t,code] (+) outlier) * score[b,h,t].   score f32 [B,H,L]; mul f32 [B,H,128].
 * Requires Lmax % 4 == 0 and a 16-byte aligned cache (TMA row pitch).
 * ------------------------------------------------------------------------------------------------------------- */
KVQ_API int kvq_k_matvec(int bits, const float* q, const int32_t* cache, float* mul, const float* lut,
                 int B, int H, int64_t Lmax, int64_t L,
                 const float* outliers, const int32_t* outlier_idx, int n_out,
                 const float* rope_cos_sin, int64_t rope_npos, float theta, int pos_offset, void* stream);
KVQ_API int kvq_v_matvec(int bits, const float* score, const int32_t* cache, float* mul, const float* lut_tok,
                 int B, int H, int64_t Lmax, int64_t L,
                 const float* outliers, const int32_t* outlier_idx, int n_out, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Fused decode attention (native op; no single counterpart in the reference -- it is the chain
 * modeling_llama.py:1928-1995: K op -> /sqrt(128) -> [cat sink scores] -> softmax -> V op [+ sink output]).
 *   out[h,:] = softmax_t( S[h,t]/sqrt(128) ) . V      over the L quantised slots and n_sink fp16 sink tokens.
 * V side: either the reference's materialised per-token LUT (vlut_tok f32 [Lmax,2^bits]) or -- faster -- the
 * sorted centroids v_cent f32 [2^bits] plus the per-token affine map v_aff f32 [Lmax,2] = (sf_t, off_t) with
 * LUT_t[i] = v_cent[i]*sf_t + off_t (what kvq_append_kv_fused writes); when both are given the affine form is used.
 * scratch: device buffer of kvq_attend_scratch_bytes(H, L) bytes.
 * sink_k: f16 [H,128,n_sink] post-RoPE keys, sink_v: f16 [H,n_sink,128] (modeling_llama.py:1464-1466), or NULL.
 * out: f32 [H,128].  out_lse (optional): f32 [H], log-sum-exp of the scaled scores over this call's tokens.
 * rope_half selects the precision of the K lookup tables:
 *   NULL      exact mode (default of the Python layer): fp32 "ratio" tables T = LUT*q_c with r_c = s_c q_{c^64}/q_c
 *             (one 4-byte lookup per element), results equal to the legacy op chain to ~1e-6;
 *   non-NULL  fp16 mode (north_star: "fp16 LUT"): half2 table from kvq_rope_table_build_half (same theta, same
 *             rope_npos); the K tables (LUT*q_c, s_c*LUT*q_{c^64}) and cos/sin are fp16, every product is exact and
 *             every sum is fp32 (each fp16 product widened exactly to fp32).  ~20 % faster K kernel; output within 1e-3 of the exact
 *             result at a few thousand tokens, 1.4e-3 .. 2e-3 at 128K.
 * V keeps fp32 tables and weights in both modes.
 * ------------------------------------------------------------------------------------------------------------- */
KVQ_API int64_t kvq_attend_scratch_bytes(int H, int64_t L);
KVQ_API int kvq_attend(int bits, const float* q,
               const int32_t* kcache, const float* klut,
               const float* k_outliers, const int32_t* k_outlier_idx,
               const int32_t* vcache, const float* vlut_tok, const float* v_cent, const float* v_aff,
               const float* v_outliers, const int32_t* v_outlier_idx,
               int n_out, int H, int64_t Lmax, int64_t L,
               const float* rope_cos_sin, int64_t rope_npos, float theta, int pos_offset,
               const void* sink_k, const void* sink_v, int n_sink,
               float* out, float* out_lse, void* scratch, const void* rope_half, void* stream);
/* Merge of n_parts partial results of kvq_attend over disjoint token ranges (sequence-sharded decode, SURVEY 8e-2):
 * parts f32 [n_parts, H*128 + H] = (out[H,128], lse[H]) per part, as produced with out_lse != NULL; out f32 [H,128]. */
KVQ_API int kvq_attend_merge(const float* parts, int n_parts, int H, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Device-resident cache length (SURVEY.md 8(f)-2): the same operations with the length read from device memory at
 * run time, so that ONE captured CUDA graph serves a growing cache -- the reference re-reads klen / vlen on the host
 * every step (modeling_llama.py:791, 1215).  len_dev points at an int64 that the caller advances (e.g. with
 * kvq_dec_counter_add at the end of the captured step).
 *   kvq_append_kv_fused_dyn : writes slot  *len_dev + slot_add  (a full cache drops the token)
 *   kvq_attend_dyn          : attends over L = min(*len_dev + len_add, L_cap) slots; grids, scratch
 *                             (kvq_attend_scratch_bytes(H, L_cap)) and the rope table are sized for L_cap.
 *                             Native V form only (v_cent + v_aff); accepts every shape kvq_attend accepts (bits 2-4,
 *                             H <= 64, H % 4 == 0).
 * ------------------------------------------------------------------------------------------------------------- */
KVQ_API int kvq_append_kv_fused_dyn(int bits, int H, int64_t Lmax, const int64_t* len_dev, int64_t slot_add, int n_each,
                            const float* k_new, int32_t* kcache, const float* klut, const float* klut_sub,
                            const float* k_thr_lower, const float* k_thr_upper, float* k_outliers,
                            int32_t* k_outlier_idx, const float* v_new, int32_t* vcache, const float* v_cent,
                            const float* v_cent_deq, float* vlut_tok, float* v_aff, float* v_outliers,
                            int32_t* v_outlier_idx, void* stream);
KVQ_API int kvq_attend_dyn(int bits, const float* q, const int32_t* kcache, const float* klut, const float* k_outliers,
                   const int32_t* k_outlier_idx, const int32_t* vcache, const float* v_cent, const float* v_aff,
                   const float* v_outliers, const int32_t* v_outlier_idx, int n_out, int H, int64_t Lmax, int64_t L_cap,
                   const int64_t* len_dev, int64_t len_add, const float* rope_cos_sin, int64_t rope_npos, float theta,
                   int pos_offset, const void* sink_k, const void* sink_v, int n_sink, float* out, float* out_lse,
                   void* scratch, const void* rope_half, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Fused device-side append (native op): replaces the whole host round trip of
 * QuantK/QuantV.forward_fused_sparse (modeling_llama.py:664-751, 1803-1820, 1091-1176): append kernel +
 * .cpu() + torch.topk + gather/mask/sort + row writes, for K and V of one token, in one launch, no host sync.
 *   k_new, v_new: f32 [H*128].  n_each = int(((1-t)/2)*hidden)+1 (21 for 7B): K keeps the n_each largest /
 *   smallest normalised values, V thresholds are the (n_each+1)-th order statistics.  n_each <= 64.
 *   Ties: K values equal at the n_each boundary are taken lowest channel first.  The V outliers are the elements
 *   strictly beyond the thresholds (those packed as the zero-point code); when values equal to a threshold leave
 *   fewer than n_each on a side, the side is padded with (value 0.0, channel 0), and the row is sorted by channel.
 *   (The reference's topk row keeps tied elements instead, which then count twice: their dense code is their
 *   nearest entry, not the zero point -- DESIGN.md section 2.)
 *   klut_sub: LUT used for the K end-entry subtraction (lookup_table2 under Q-Norm), may equal klut.
 *   v_cent: f32 [2^bits] sorted centroids; vlut_tok row `slot` is WRITTEN; v_aff (optional, f32 [Lmax,2]) row
 *   `slot` receives (sf, off); v_cent_deq (optional): Q-Norm centroids cent*normscale+normoffset -- the outlier
 *   residual is taken against LUT2_t[zp] = v_cent_deq[zp]*sf+off (modeling_llama.py:1115-1118,1149-1152).
 *   Cache words at `slot` are OVERWRITTEN (not added).  Outlier rows (f32/i32 [Lmax, 2*n_each]) row `slot` written.
 *   k_outliers / k_outlier_idx (and likewise the V pair) may be NULL: that cache is then dense-only -- the reference's
 *   include_sparse=False branch (modeling_llama.py:753-779, 1178-1201): every K value keeps its nearest code, the V
 *   range is the min / max of the vector (compute_lut, modeling_llama.py:318-349).  BASELINE configs[3] (dense-only)
 *   and configs[4] (K outliers only) use this.
 * ------------------------------------------------------------------------------------------------------------- */
KVQ_API int kvq_append_kv_fused(int bits, int H, int64_t Lmax, int64_t slot, int n_each,
                        const float* k_new, int32_t* kcache, const float* klut, const float* klut_sub,
                        const float* k_thr_lower, const float* k_thr_upper,
                        float* k_outliers, int32_t* k_outlier_idx,
                        const float* v_new, int32_t* vcache, const float* v_cent, const float* v_cent_deq,
                        float* vlut_tok, float* v_aff,
                        float* v_outliers, int32_t* v_outlier_idx,
                        void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Dequantise slots [start, stop) of a layer cache to fp16 (native op: the cache read back as dense K / V, for
 * multi-token attention, other attention kernels, or checking the cache on the device).
 *   out_k / out_v: __half, element (h, t, c) at  h*head_stride + (t-start)*128 + c  (either may be NULL, not both);
 *   head_stride >= (stop-start)*128 and a multiple of 8; outputs 16-byte aligned (so a slice of a bigger [H, S, 128]
 *   buffer can be written in place).
 *   K: klut = the dequantisation table (LUT2 under Q-Norm, as kvq_attend takes it); value = LUT[h,c,code] + the K
 *      outlier residual of (slot, channel) if present, one fp32 add, then one rounding to fp16.
 *      rope_cos_sin == NULL -> written pre-RoPE; otherwise rotated at position p = pos_offset + t with the
 *      kvq_rope_table_build table (rotate-half: k'[c] = cos*k[c] - sin*k[c+64] (c<64), cos*k[c] + sin*k[c-64]
 *      (c>=64)), so that for a query already rotated at its own position, q . k'[t] is the score kvq_attend computes
 *      for slot t; the table must cover positions [0, pos_offset + stop).
 *   V: value = v_cent[code]*sf_t + off_t (one fma; v_cent = the Q-Norm-shifted centroids when V Q-Norm is on, (sf_t,
 *      off_t) = v_aff row t) + the V outlier residual.  Native V form only (like kvq_attend_dyn).
 *   k_outliers / v_outliers pairs may be NULL (dense-only cache, or K outliers only); n_out <= 128, even.
 *   start == stop returns 0 once the sizes are valid, whatever the pointers (an empty output may be NULL), and
 *   launches nothing.  All offsets are 64-bit.  Two launches (K, V) on `stream`.
 * ------------------------------------------------------------------------------------------------------------- */
KVQ_API int kvq_dequant_kv(int bits, int H, int64_t Lmax, int64_t start, int64_t stop,
                   const int32_t* kcache, const float* klut, const float* k_outliers, const int32_t* k_outlier_idx,
                   const int32_t* vcache, const float* v_cent, const float* v_aff,
                   const float* v_outliers, const int32_t* v_outlier_idx, int n_out,
                   const float* rope_cos_sin, int64_t rope_npos, int pos_offset,
                   void* out_k, void* out_v, int64_t head_stride, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Uncapped "orig" sparse path, 4-bit only (quant_cuda.cpp:347-399).
 * SpMV halves of ..._opt2_orig: balanced CSR (K; rows = tokens) quant_cuda_kernel.cu:523-614 and CSC (V; cols =
 * tokens) 616-689; the dense half is kvq_k_matvec / kvq_v_matvec with outliers == NULL.
 * rows (K) / cols (V) are the CSR / CSC pointer arrays (num_rows + 1 entries); start_rows / start_cols / num_threads are
 * the reference's work-split metadata: accepted for signature parity, not used (one warp per token here).  K takes the
 * rope table of kvq_rope_table_build covering positions [0, pos_offset + num_rows).
 * ------------------------------------------------------------------------------------------------------------- */
KVQ_API int kvq_k_spmv_csr(const int32_t* rows, const int32_t* cols, const int32_t* start_rows, const float* vals,
                   const float* q, float* mul, int H, int64_t L, int num_rows, int num_threads, int nnz,
                   const float* rope_cos_sin, int64_t rope_npos, int pos_offset, void* stream);
KVQ_API int kvq_v_spmv_csc(const int32_t* rows, const int32_t* cols, const int32_t* start_cols, const float* vals,
                   const float* score, float* mul, int H, int64_t L, int num_cols, int num_threads, int nnz,
                   void* stream);
/* First half of vecquant4appendvec{K,V}sparseorig (quant_cuda_kernel.cu:691-1163): pack one token and emit its
 * threshold-crossing elements compacted in channel order: out_cols i32[H*128], out_vals f32[H*128] (value minus
 * zeropoint), *out_count = number of outliers.  K: per-channel thresholds/zeropoint arrays; V: scalars. */
KVQ_API int kvq_append_k_orig(int32_t* cache, const float* lut, const float* newvec, const float* zeropoint,
                      const float* thr_lower, const float* thr_upper, int32_t* out_cols, float* out_vals,
                      int32_t* out_count, int H, int64_t Lmax, int64_t slot, void* stream);
KVQ_API int kvq_append_v_orig(int32_t* cache, const float* lut_tok, const float* newvec, float zeropoint,
                      float thr_lower, float thr_upper, int32_t* out_rows, float* out_vals,
                      int32_t* out_count, int H, int64_t Lmax, int64_t slot, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Exchange of the per-GPU partial attention results over NVLink peer memory, fused with their merge (sequence-sharded
 * decode; validated against NCCL all_gather + kvq_attend_merge at 2 / 4 / 8 GPUs, tests/test_zz_p2p_exchange.py).
 *   kvq_p2p_buffer_bytes(world, H)          size of one rank's exchange buffer
 *   kvq_p2p_alloc / kvq_p2p_free            cudaMalloc'ed, zeroed buffer + its 64-byte CUDA IPC handle
 *   kvq_p2p_open / kvq_p2p_close            map a peer's buffer from its handle
 *   kvq_attend_exchange_merge               part = this rank's (out[H,128], lse[H]) from kvq_attend(out, out_lse);
 *                                           peers_dev = DEVICE array of `world` buffer base pointers (own buffer at
 *                                           index rank); seq_dev = device counter, advanced by one per call (all ranks
 *                                           call in lockstep); out = merged [H,128]; *err_flag is set (and out is NaN)
 *                                           if a peer did not arrive within ~2 s.
 * ------------------------------------------------------------------------------------------------------------- */
KVQ_API int64_t kvq_p2p_buffer_bytes(int world, int H);
KVQ_API int kvq_p2p_alloc(void** ptr, int64_t bytes, void* ipc_handle_64);
KVQ_API int kvq_p2p_open(const void* ipc_handle_64, void** ptr);
KVQ_API int kvq_p2p_close(void* ptr);
KVQ_API int kvq_p2p_free(void* ptr);
KVQ_API int kvq_attend_exchange_merge(const float* part, void* const* peers_dev, int world, int rank, int H,
                              int64_t* seq_dev, float* out, int32_t* err_flag, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Decode-harness helpers (kvquant_b200/decode.py; NOT part of the reference's quant_cuda surface): fused fp16
 * element-wise kernels around the hot path -- HF LlamaRMSNorm, rotate-half RoPE on Q + fp32 split of q/k/v
 * (modeling_llama.py:1851-1859), SwiGLU activation, fp32->fp16 cast.  Pointers named *_f16 are __half*.
 * ------------------------------------------------------------------------------------------------------------- */
KVQ_API int kvq_dec_rmsnorm(const void* x_f16, const void* w_f16, void* y_f16, int n, float eps, void* stream);
KVQ_API int kvq_dec_rope_split(const void* qkv_f16, const float* inv_freq, float pos, float* q, float* k, float* v,
                               int hidden, void* stream);
/* q RoPE position = *pos_dev + pos_add (device-resident, see kvq_attend_dyn) */
KVQ_API int kvq_dec_rope_split_dyn(const void* qkv_f16, const float* inv_freq, const int64_t* pos_dev, int64_t pos_add,
                                   float* q, float* k, float* v, int hidden, void* stream);
/* *counter += delta on the stream (advances the device-resident length / position inside a captured step) */
KVQ_API int kvq_dec_counter_add(int64_t* counter, int64_t delta, void* stream);
KVQ_API int kvq_dec_silu_mul(const void* gu_f16, void* act_f16, int n, void* stream);
KVQ_API int kvq_dec_f32_to_f16(const float* a, void* b_f16, int n, void* stream);
/* Batch-1 GEMV with its element-wise neighbours fused (replaces nn.Linear at q_len = 1, modeling_llama.py:1811-1813,
 * 2004, and the norm / activation launch in front of it):  y[r] = residual[r] + sum_k W[r,k] * f(x)[k],
 * W fp16 [N,K] row-major (16-byte aligned, K % 256 == 0, K <= 14336), fp32 accumulation.
 * x_kind: 0 = fp16 [K]; 1 = f32 [K] (rounded through fp16 first); 2 = fp16 [2K] gate|up -> silu(gate)*up;
 * 3 = fp16 [K] + HF LlamaRMSNorm with norm_w_f16 and eps.  residual_f16 may be NULL and may alias y; x must not.
 * y is fp16 [N], or f32 [N] when y_f32 != 0. */
KVQ_API int kvq_dec_gemv(const void* w_f16, int N, int K, const void* x, int x_kind, const void* norm_w_f16, float eps,
                         const void* residual_f16, void* y, int y_f32, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KVQUANT_B200_H */
