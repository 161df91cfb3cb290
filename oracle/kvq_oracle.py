"""CPU oracle for the KVQuant deployment hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module; the product package (kvquant_b200/) never does and fails loudly without its CUDA library.

This is a plain numpy restatement of the reference algorithm (SqueezeAILab/KVQuant @ 57a2383), each
function citing the reference file:line it follows.  Shorthand (relative to the reference checkout):
  DK.cu = deployment/kvquant/quant_cuda_kernel.cu
  ML.py = deployment/transformers/src/transformers/models/llama/modeling_llama.py
  SQ.py = quant/kvquant/simquant_module_quantizer.py

Parity pinning (SURVEY.md section 8c): the reference ships NO golden vectors / KATs for this path.  The oracle
is pinned two ways instead:
  (1) the simulated-quant functions at the bottom of this file are checked against the reference's own
      Python (`quant_fn_nuq_recon`, `get_outliers`, `get_outliers_dynamic`, imported from the reference
      checkout) through committed fixtures: tests/golden/simquant_*.npz, generator
      tests/golden/gen_simquant_golden.py;
  (2) the kernel-semantics functions are checked against the reference's own CUDA kernels, compiled
      unmodified by oracle/build_ref.py: tests/golden/refcuda_*.npz, generator
      tests/golden/gen_refcuda_golden.py, plus stored reference results for the ours-vs-reference tests
      (tests/golden/ref_*.npz, tests/_refgold.py).

Arithmetic notes
  * all "kernel" arithmetic is fp32 in the reference; codes/packing are integer and must be BIT-EXACT;
  * dot products are accumulated here in float64 (the reference accumulates fp32 with atomics in a
    non-deterministic order, so its own run-to-run noise is ~1e-6 relative);
  * RoPE: the reference evaluates cosf/sinf(fl32(theta_c * pos)) with theta_c = powf(base, -2*(c%64)/128)
    (DK.cu:3081,3120-3129).  We reproduce the fp32 rounding of theta_c*pos exactly; theta_c itself is
    float64 pow rounded to fp32, which can differ from CUDA's powf by 1 ulp (angle error <= 6e-8*theta*pos).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32

HEAD_DIM = 128  # every reference kernel assumes head_dim == 128 (DK.cu:3107-3108,3120)


# --------------------------------------------------------------------------------------------------
# packed-code layout (SURVEY 2.3)
# --------------------------------------------------------------------------------------------------
def words_per_head(bits: int) -> int:
    """int32 words per head per token: D*b/32 = 16/12/8 (BLOCKHEIGHT{4,3,2}, DK.cu:43-46)."""
    return HEAD_DIM * bits // 32


def zero_point_code(bits: int) -> int:
    """V zero-point code for outliers: 7/3/1 (DK.cu:2083-2084, 2441-2442, 3019-3020)."""
    return {4: 7, 3: 3, 2: 1}[bits]


def pack_codes(codes: np.ndarray, bits: int) -> np.ndarray:
    """codes uint [hidden, T] -> words int32 [hidden*bits/32, T].

    4-bit: row j//8, shift 4*(j%8)            (DK.cu:1240-1243)
    2-bit: row j//16, shift 2*(j%16)          (DK.cu:1601-1604)
    3-bit: GPTQ 32-in-3-words                 (DK.cu:1395-1424): loc=j%32, base row (j//32)*3;
           loc<10 -> row+0 << 3*loc; loc==10 -> (code<<30) into row+0 and (code>>2) into row+1;
           11..20 -> row+1 << (3*loc)%32; loc==21 -> (code<<31) into row+1, (code>>1) into row+2;
           22..31 -> row+2 << (3*loc)%32.
    Packing is additive into a zero-initialised cache (atomicAdd / +=); fields never overlap so the
    result equals a bitwise OR; int32 wrap-around of `code << 30/31` keeps only the low bits.
    """
    codes = np.asarray(codes)
    if codes.ndim == 1:
        codes = codes[:, None]
    hidden, T = codes.shape
    c = codes.astype(np.uint32)
    nwords = hidden * bits // 32
    out = np.zeros((nwords, T), dtype=np.uint32)
    j = np.arange(hidden)
    if bits == 4:
        np.add.at(out, j // 8, c << ((j % 8) * 4).astype(np.uint32)[:, None])
    elif bits == 2:
        np.add.at(out, j // 16, c << ((j % 16) * 2).astype(np.uint32)[:, None])
    elif bits == 3:
        for l in range(32):              # every channel at position l of its 32-group, all groups at once
            js = j[l::32]
            b = (js // 32) * 3
            v = c[js]
            if l == 10:
                out[b] += (v << np.uint32(30))
                out[b + 1] += (v >> np.uint32(2))
            elif l == 21:
                out[b + 1] += (v << np.uint32(31))
                out[b + 2] += (v >> np.uint32(1))
            else:
                out[b + l // 11] += (v << np.uint32((3 * l) % 32))
    else:
        raise ValueError(bits)
    return out.view(np.int32)


def unpack_codes(words: np.ndarray, bits: int) -> np.ndarray:
    """words int32 [hidden*bits/32, T] -> codes uint8 [hidden, T] (inverse of pack_codes;
    unpack order DK.cu:3122-3192 (4b), 3775-4103 (3b), 4747-4996 (2b))."""
    w = np.ascontiguousarray(words).view(np.uint32)
    if w.ndim == 1:
        w = w[:, None]
    nwords, T = w.shape
    hidden = nwords * 32 // bits
    j = np.arange(hidden)
    if bits == 4:
        return ((w[j // 8] >> ((j % 8) * 4).astype(np.uint32)[:, None]) & 0xF).astype(np.uint8)
    if bits == 2:
        return ((w[j // 16] >> ((j % 16) * 2).astype(np.uint32)[:, None]) & 0x3).astype(np.uint8)
    if bits == 3:
        out = np.zeros((hidden, T), dtype=np.uint8)
        for l in range(32):
            js = j[l::32]
            b = (js // 32) * 3
            if l == 10:
                v = ((w[b] >> np.uint32(30)) & 0x3) | ((w[b + 1] & 0x1) << np.uint32(2))
            elif l == 21:
                v = ((w[b + 1] >> np.uint32(31)) & 0x1) | ((w[b + 2] & 0x3) << np.uint32(1))
            else:
                v = (w[b + l // 11] >> np.uint32((3 * l) % 32)) & 0x7
            out[js] = v.astype(np.uint8)
        return out
    raise ValueError(bits)


# --------------------------------------------------------------------------------------------------
# LUT construction
# --------------------------------------------------------------------------------------------------
def build_k_lut(upper, lower, centroids, normscale=None, normoffset=None):
    """QuantK.load_lookup_table (ML.py:437-501).

    upper/lower: per-channel thresholds [hidden] (pickle entries [0],[1]); rounded fp32->fp16 (ML.py:447-448);
    offset=(max+min)/2, range=(max-min)/2 computed IN fp16 (ML.py:461-462); centroids sorted ascending
    (ML.py:449-450,483); LUT[j,:] = cent*range_j + offset_j in fp32, two roundings (ML.py:490).
    Returns dict(lut[hidden,n] f32, lut2 or None, thr_upper f32, thr_lower f32, zeropoint f32).
    """
    up16 = np.asarray(upper, dtype=np.float32).astype(np.float16).ravel()
    lo16 = np.asarray(lower, dtype=np.float32).astype(np.float16).ravel()
    cent = np.sort(np.asarray(centroids, dtype=np.float32).ravel())
    offset16 = ((up16 + lo16) / np.float16(2)).astype(np.float16)
    range16 = ((up16 - lo16) / np.float16(2)).astype(np.float16)
    sf = range16.astype(np.float32)[:, None]
    off = offset16.astype(np.float32)[:, None]
    lut = (cent[None, :] * sf).astype(np.float32) + off
    lut = lut.astype(np.float32)
    lut2 = None
    if normscale is not None:
        c2 = (cent * F32(normscale)).astype(np.float32) + F32(normoffset)
        lut2 = ((c2.astype(np.float32)[None, :] * sf).astype(np.float32) + off).astype(np.float32)
    return dict(
        lut=lut, lut2=lut2, cent=cent,
        thr_upper=up16.astype(np.float32), thr_lower=lo16.astype(np.float32),
        zeropoint=offset16.astype(np.float32),  # ML.py:497-498 (computed in fp16, then .float())
    )


def v_token_affine(hi, lo):
    """(sf, off) = ((hi-lo)/2, (hi+lo)/2) in fp32 (ML.py:1097-1098)."""
    hi = F32(hi)
    lo = F32(lo)
    return F32(F32(hi - lo) / F32(2)), F32(F32(hi + lo) / F32(2))


def v_token_lut(cent_sorted, hi, lo):
    """Per-token V LUT (ML.py:1097-1114): sf=(hi-lo)/2, off=(hi+lo)/2 in fp32; LUT = cent*sf + off."""
    sf, off = v_token_affine(hi, lo)
    cent = np.asarray(cent_sorted, dtype=np.float32)
    return ((cent * sf).astype(np.float32) + off).astype(np.float32)


# --------------------------------------------------------------------------------------------------
# quantise (nearest LUT entry, first minimum wins)
# --------------------------------------------------------------------------------------------------
def nearest_code(x, lut):
    """argmin_i |lut[..., i] - x| in fp32, strict '<' scan from i=0 => first minimum wins
    (DK.cu:1219-1235, 1767-1773).  x [...], lut [..., n] -> uint8 [...].
    NaN input: every comparison is false in the reference -> code 0; np.argmin over all-NaN row gives 0 too."""
    x = np.asarray(x, dtype=np.float32)
    lut = np.asarray(lut, dtype=np.float32)
    d = np.abs((lut - x[..., None]).astype(np.float32))
    return np.argmin(d, axis=-1).astype(np.uint8)


def append_k_codes(k, lut):
    """vecquant{4,3,2}appendvecK[sparse] dense codes (DK.cu:1202-1245 / 1725-1781).  k [hidden] or [hidden,T];
    lut [hidden, n].  K outliers are NOT special-cased in the dense code (nearest entry = LUT end)."""
    k = np.asarray(k, dtype=np.float32)
    if k.ndim == 1:
        return nearest_code(k, lut)
    return nearest_code(k, lut[:, None, :])


def k_outliers_rescaled(k, thr_lower, thr_upper):
    """outliers_rescaled = (k - zp)/range, zp=(up+lo)/2, range=(up-lo)/2 recomputed in fp32 inside the
    kernel (DK.cu:1759-1764)."""
    k = np.asarray(k, dtype=np.float32)
    up = np.asarray(thr_upper, dtype=np.float32)
    lo = np.asarray(thr_lower, dtype=np.float32)
    rg = ((up - lo).astype(np.float32) / F32(2)).astype(np.float32)
    zp = ((up + lo).astype(np.float32) / F32(2)).astype(np.float32)
    if k.ndim == 2:
        rg, zp = rg[:, None], zp[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        return ((k - zp).astype(np.float32) / rg).astype(np.float32)


def _topk_idx(x, k, largest=True):
    """indices of the k largest / smallest entries, equal values lowest index first (stable sort).

    torch.topk, which the reference calls, leaves the order of equal values unspecified.  Lowest index first is the
    fused append's K rule (kvq_append_kv_fused: among equal normalised values at the n_each boundary the lowest channel
    is taken), so K rows here are exact with ties.  For V the choice only matters under v_ties="reference": which of
    several values equal to a threshold land in the row (see v_outlier_row_strict for the fused append's V rule).
    fp16-valued activations -- what a decode step feeds the append -- produce such ties in a few % of V tokens."""
    x = np.asarray(x)
    order = np.argsort(-x if largest else x, kind="stable")
    return order[:k]


def n_out_each(hidden, sparsity_threshold=0.99):
    """threshold_k = int(((1-t)/2)*hidden) + 1  (= 21 for 7B at t=0.99; ML.py:707)."""
    return int(((1 - sparsity_threshold) / 2) * hidden) + 1


def k_outlier_row(k, rescaled, lut_sub, n_each):
    """Host-side outlier-row build of QuantK.forward_fused_sparse (ML.py:706-751).

    k [hidden] fp32 new key; rescaled [hidden] from the append kernel; lut_sub [hidden,n] = LUT used for the
    end-entry subtraction (lookup_table2 under Q-Norm, else lookup_table; ML.py:724-727).
    Returns (vals f32[2*n_each], idx i32[2*n_each]) sorted by idx ascending; pads are 0 with real indices."""
    k = np.asarray(k, dtype=np.float32)
    r = np.asarray(rescaled, dtype=np.float32)
    n = lut_sub.shape[-1]
    ui = _topk_idx(r, n_each, True)
    li = _topk_idx(r, n_each, False)
    uv = (k[ui] - lut_sub[ui, n - 1]).astype(np.float32)
    lv = (k[li] - lut_sub[li, 0]).astype(np.float32)
    uz = r[ui] <= 1
    lz = r[li] >= -1
    vals = np.concatenate([uv, lv])
    idx = np.concatenate([ui, li]).astype(np.int64)
    zer = np.concatenate([uz, lz])
    order = np.argsort(idx, kind="stable")
    vals = vals[order].copy()
    vals[zer[order]] = 0
    return vals.astype(np.float32), idx[order].astype(np.int32)


def v_thresholds(v, n_each):
    """V per-token thresholds: topk(n_each+1) largest / smallest; the LAST of each is the threshold
    (hi = 22nd largest, lo = 22nd smallest), the first n_each are the outliers (ML.py:1814-1816,1091-1096).
    Returns hi, lo, upper_idx[n_each], lower_idx[n_each]."""
    v = np.asarray(v, dtype=np.float32)
    ui = _topk_idx(v, n_each + 1, True)
    li = _topk_idx(v, n_each + 1, False)
    return F32(v[ui[-1]]), F32(v[li[-1]]), ui[:-1], li[:-1]


def append_v_codes(v, lut_t, bits, thr_lower=None, thr_upper=None):
    """vecquant{4,3,2}appendvecV (DK.cu:1280-1320) / ...Vsparse (DK.cu:2049-2102): per-token LUT nearest code;
    sparse: v<lo or v>hi -> zero-point code."""
    v = np.asarray(v, dtype=np.float32)
    codes = nearest_code(v, np.broadcast_to(lut_t, v.shape + (lut_t.shape[-1],)))
    if thr_lower is not None:
        out = (v < F32(thr_lower)) | (v > F32(thr_upper))
        codes = np.where(out, np.uint8(zero_point_code(bits)), codes)
    return codes.astype(np.uint8)


def v_outlier_row(v, upper_idx, lower_idx, zeropoint_val):
    """QuantV outlier row (ML.py:1168-1176): vals = cat(v[upper], v[lower]) - LUT_t[zp]; sorted by index."""
    v = np.asarray(v, dtype=np.float32)
    idx = np.concatenate([upper_idx, lower_idx]).astype(np.int64)
    vals = (v[idx] - F32(zeropoint_val)).astype(np.float32)
    order = np.argsort(idx, kind="stable")
    return vals[order], idx[order].astype(np.int32)


def v_outlier_row_strict(v, hi, lo, n_each, zeropoint_val):
    """V outlier row of the fused append (kvq_append_kv_fused), the rule for ties at the thresholds.

    The outliers are the elements strictly beyond the (n_each+1)-th order statistics: v > hi and v < lo -- exactly the
    elements whose dense code is the zero-point code (append_v_codes), so each element is represented once.  When
    values equal to a threshold leave fewer than n_each on a side, that side is padded with (0.0, channel 0).
    Sorted by channel; entries of one channel keep the order upper outliers, upper pads, lower outliers, lower pads.

    The reference (v_outlier_row, v_ties="reference") instead keeps n_each topk indices per side, some of them equal
    to the threshold.  Such an element's dense code is its nearest LUT entry (the sparse append compares strictly),
    so it dequantises to LUT_t[code] + (v - LUT_t[zp]): its value is counted twice."""
    v = np.asarray(v, dtype=np.float32)
    up = np.nonzero(v > F32(hi))[0]
    lw = np.nonzero(v < F32(lo))[0]
    assert len(up) <= n_each and len(lw) <= n_each

    def side(ix):
        vals = np.zeros(n_each, dtype=np.float32)
        vals[:len(ix)] = (v[ix] - F32(zeropoint_val)).astype(np.float32)
        idx = np.zeros(n_each, dtype=np.int64)
        idx[:len(ix)] = ix
        return vals, idx
    uv, ui = side(up)
    lv, li = side(lw)
    vals = np.concatenate([uv, lv])
    idx = np.concatenate([ui, li])
    order = np.argsort(idx, kind="stable")
    return vals[order], idx[order].astype(np.int32)


# --------------------------------------------------------------------------------------------------
# RoPE helpers
# --------------------------------------------------------------------------------------------------
def rope_theta_vec(rope_theta, head_dim=HEAD_DIM):
    """theta_c = powf(rope_theta, (-2*float(c % 64)) / float(128)), c in [0,128)  (DK.cu:3081).
    float64 pow rounded to fp32 (CUDA powf may differ by 1 ulp; theta_0 == 1 exactly)."""
    c = np.arange(head_dim)
    expo = ((F32(-2) * (c % (head_dim // 2)).astype(np.float32)) / F32(head_dim)).astype(np.float32)
    return np.power(np.float64(F32(rope_theta)), expo.astype(np.float64)).astype(np.float32)


def rope_cos_sin(theta_vec, positions):
    """cos/sin of fl32(theta_c * float(pos)) (DK.cu:3123-3126).  Returns float64 [len(pos), 128] x2
    (accurate cos/sin of the fp32-rounded argument)."""
    pos = np.asarray(positions).astype(np.float32)
    arg = (theta_vec[None, :].astype(np.float32) * pos[:, None]).astype(np.float32)
    a64 = arg.astype(np.float64)
    return np.cos(a64), np.sin(a64)


def rope_rotate_q(q, position, rope_theta, head_dim=HEAD_DIM):
    """HF-style rotate-half RoPE applied to q [H,128] at `position` (what the caller does to Q before the K
    matvec; ML.py:1851-1859).  fp64 math, fp32 result.  Used to synthesise realistic queries."""
    th = rope_theta_vec(rope_theta, head_dim).astype(np.float64)
    ang = th * float(position)
    cos, sin = np.cos(ang), np.sin(ang)
    q = np.asarray(q, dtype=np.float64)
    half = head_dim // 2
    rot = np.concatenate([-q[..., half:], q[..., :half]], axis=-1)
    return (q * cos + rot * sin).astype(np.float32)


# --------------------------------------------------------------------------------------------------
# decode matvecs (kernel semantics)
# --------------------------------------------------------------------------------------------------
def k_dequant(words, lut, bits):
    """words int32 [H*W, L] -> K values f32 [hidden, L] with per-channel LUT [hidden, n]."""
    codes = unpack_codes(words, bits)
    return np.take_along_axis(lut, codes.astype(np.int64), axis=1)


def k_scores_dense(q, words, lut, bits, L, rope_theta, pos_offset, num_heads):
    """vecquantNmatmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt (DK.cu:3040-3209):
    S[h,t] = sum_c LUT[h,c,code] * (cos(th_c*p)*q[h,c] + s_c*sin(th_c*p)*q[h,(c+64)%128]), p = t+pos_offset,
    s_c = +1 (c<64) else -1.  q f32 [H,128]; words [H*W, >=L]; returns float64 [H, L] (to be ADDED to mul)."""
    q = np.asarray(q, dtype=np.float32).reshape(num_heads, HEAD_DIM).astype(np.float64)
    kv = k_dequant(np.asarray(words)[:, :L], lut, bits).astype(np.float64).reshape(num_heads, HEAD_DIM, L)
    th = rope_theta_vec(rope_theta)
    cos, sin = rope_cos_sin(th, np.arange(L) + pos_offset)  # [L,128]
    sign = np.where(np.arange(HEAD_DIM) < 64, 1.0, -1.0)
    q2 = q[:, (np.arange(HEAD_DIM) + 64) % HEAD_DIM]
    # rotated query per token: rq[h,c,t]
    rq = q[:, :, None] * cos.T[None] + (sign[None, :, None] * q2[:, :, None]) * sin.T[None]
    return np.einsum("hct,hct->ht", kv, rq)


def k_scores_outliers(q, outliers, outlier_idx, L, rope_theta, pos_offset, num_heads):
    """SPMV_ATOMIC_ROPE_BALANCED (DK.cu:472-521): for token row t and each of its n_out (val, col) pairs:
    mul[head(col), t] += val*(cos*q[col] + sign*sin*q[col2]).  Padded zeros contribute 0.  float64 [H,L]."""
    qf = np.asarray(q, dtype=np.float64).ravel()
    vals = np.asarray(outliers, dtype=np.float64)[:L]
    idx = np.asarray(outlier_idx, dtype=np.int64)[:L]
    out = np.zeros((num_heads, L), dtype=np.float64)
    th = rope_theta_vec(rope_theta)
    cos, sin = rope_cos_sin(th, np.arange(L) + pos_offset)
    ch = idx % HEAD_DIM
    head = idx // HEAD_DIM
    col2 = ((ch + 64) % HEAD_DIM) + head * HEAD_DIM
    sign = np.where(ch < 64, 1.0, -1.0)
    rows = np.arange(L)[:, None]
    contrib = vals * (cos[rows, ch] * qf[idx] + sign * sin[rows, ch] * qf[col2])
    np.add.at(out, (head, np.broadcast_to(rows, head.shape)), contrib)
    return out


def v_dequant(words, lut_tok, bits):
    """words int32 [H*W, L], per-token LUT [L, n] -> V values f32 [hidden, L]."""
    codes = unpack_codes(words, bits).astype(np.int64)  # [hidden, L]
    L = codes.shape[1]
    return lut_tok[np.arange(L)[None, :], codes]


def v_out_dense(score, words, lut_tok, bits, L, num_heads):
    """vecquantNmatmul_nuq_perchannel_transposed_mha_batched_fused_opt (DK.cu:3211-3433):
    O[h,c] = sum_t LUT[t, code(h,c,t)] * score[h,t].  score f32 [H,L]; returns float64 [H,128]."""
    sc = np.asarray(score, dtype=np.float32).reshape(num_heads, -1)[:, :L].astype(np.float64)
    vv = v_dequant(np.asarray(words)[:, :L], np.asarray(lut_tok)[:L], bits).astype(np.float64)
    vv = vv.reshape(num_heads, HEAD_DIM, L)
    return np.einsum("hct,ht->hc", vv, sc)


def v_out_outliers(score, outliers, outlier_idx, L, num_heads):
    """SPMV_ATOMIC_BALANCED (DK.cu:436-470): mul[row] += val * score[row//128, t].  float64 [H,128]."""
    sc = np.asarray(score, dtype=np.float64).reshape(num_heads, -1)[:, :L]
    vals = np.asarray(outliers, dtype=np.float64)[:L]
    idx = np.asarray(outlier_idx, dtype=np.int64)[:L]
    out = np.zeros(num_heads * HEAD_DIM, dtype=np.float64)
    head = idx // HEAD_DIM
    t = np.broadcast_to(np.arange(L)[:, None], idx.shape)
    np.add.at(out, idx, vals * sc[head, t])
    return out.reshape(num_heads, HEAD_DIM)


# --------------------------------------------------------------------------------------------------
# uncapped "orig" CSR / CSC path (DK.cu:691-1163, 523-689, 5506-5668)
# --------------------------------------------------------------------------------------------------
def orig_k_token_outliers(k, thr_lower, thr_upper, zeropoint):
    """vecquant4appendvecKsparseorig, per token: every element with k<lo or k>up is an outlier, stored as
    (k - zeropoint_j) and its dense code is computed on ... see append_k_orig_codes.  Returns (cols, vals)
    in ascending channel order (DK.cu:846-931: serial per-block compaction keeps channel order)."""
    k = np.asarray(k, dtype=np.float32)
    m = (k < thr_lower) | (k > thr_upper)
    cols = np.nonzero(m)[0].astype(np.int32)
    vals = (k[cols] - np.asarray(zeropoint, dtype=np.float32)[cols]).astype(np.float32)
    return cols, vals


def csr_grow(ptr, idx, val, start, new_idx, new_val, cachelen):
    """Host side of vecquant4appendvec{K,V}sparseorig (DK.cu:765-823): append one token's `count` outliers to the
    growing CSR (K: rows = tokens) / CSC (V: cols = tokens) arrays.  The SpMV is balanced at 10 nonzeros per thread;
    `start[k]` = the token at which thread k's first nonzero was appended (new threads start at the current token).
    Plain Python lists in, lists out: (ptr, idx, val, start, num_threads)."""
    count = len(new_idx)
    if len(ptr) == 0:                                   # DK.cu:768-786
        ptr2 = [0, count]
        idx2, val2 = list(new_idx), list(new_val)
        nthreads = (count + 9) // 10
        start2 = [int(cachelen)] * nthreads
    else:                                               # DK.cu:788-820
        ptr2 = list(ptr) + [len(idx) + count]
        prevmax = len(start)
        if count > 0:
            idx2, val2 = list(idx) + list(new_idx), list(val) + list(new_val)
            nthreads = (len(idx2) + 9) // 10
            new_alloc = nthreads - prevmax
            start2 = list(start) + [int(cachelen)] * new_alloc if new_alloc > 0 else list(start)
        else:
            idx2, val2, start2 = list(idx), list(val), list(start)
            nthreads = (len(idx2) + 9) // 10
    return ptr2, idx2, val2, start2, nthreads


def csr_k_scores(q, rows_ptr_tokens, cols, vals, L, rope_theta, pos_offset, num_heads):
    """SPMV_ATOMIC_CSR_ROPE_BALANCED semantics (DK.cu:523-614), token-major CSR given as per-token
    (start,end) pointer array rows_ptr_tokens [L+1]."""
    qf = np.asarray(q, dtype=np.float64).ravel()
    out = np.zeros((num_heads, L), dtype=np.float64)
    th = rope_theta_vec(rope_theta)
    cos, sin = rope_cos_sin(th, np.arange(L) + pos_offset)
    for t in range(L):
        s, e = int(rows_ptr_tokens[t]), int(rows_ptr_tokens[t + 1])
        for i in range(s, e):
            col = int(cols[i]); ch = col % HEAD_DIM; h = col // HEAD_DIM
            col2 = ((ch + 64) % HEAD_DIM) + h * HEAD_DIM
            sg = 1.0 if ch < 64 else -1.0
            out[h, t] += float(vals[i]) * (cos[t, ch] * qf[col] + sg * sin[t, ch] * qf[col2])
    return out


def csc_v_out(score, cols_ptr_tokens, rows, vals, L, num_heads):
    """SPMV_ATOMIC_CSC_BALANCED semantics (DK.cu:616-689): token-major CSC; out[row] += val*score[row//128,t]."""
    sc = np.asarray(score, dtype=np.float64).reshape(num_heads, -1)
    out = np.zeros(num_heads * HEAD_DIM, dtype=np.float64)
    for t in range(L):
        s, e = int(cols_ptr_tokens[t]), int(cols_ptr_tokens[t + 1])
        for i in range(s, e):
            r = int(rows[i])
            out[r] += float(vals[i]) * sc[r // HEAD_DIM, t]
    return out.reshape(num_heads, HEAD_DIM)


# --------------------------------------------------------------------------------------------------
# whole decode-step attention with the reference's dtype round trips (ML.py:1928-1995, 873-874, 1291)
# --------------------------------------------------------------------------------------------------
def softmax_f32(x):
    x = np.asarray(x, dtype=np.float32)
    m = x.max(axis=-1, keepdims=True)
    e = np.exp((x - m).astype(np.float32)).astype(np.float32)
    return (e / e.sum(axis=-1, keepdims=True, dtype=np.float32)).astype(np.float32)


def attend_reference(scores_kernel_f64, v_fn, num_heads, sink_scores_f16=None, head_dim=HEAD_DIM):
    """The reference's post-processing chain around the two matvec ops:
      K op result fp32 -> .half() (ML.py:873-874) -> / sqrt(128) in fp16 (ML.py:1959/1973) ->
      cat sink scores in front (ML.py:1962) -> softmax in fp32 -> cast fp16 (ML.py:1976) ->
      V op consumes P[:, n_sink:].float() (ML.py:1083) -> result fp32 -> .half() (ML.py:1291).
    `v_fn(P_f32[H,L]) -> float64 [H,128]`.  Returns (P_f16 [H, n_sink+L], out_f16 [H,128])."""
    s16 = np.asarray(scores_kernel_f64).astype(np.float32).astype(np.float16)
    s16 = (s16 / np.float16(np.sqrt(head_dim))).astype(np.float16)  # fp16 tensor / python float -> fp16
    if sink_scores_f16 is not None:
        s16 = np.concatenate([np.asarray(sink_scores_f16, dtype=np.float16), s16], axis=-1)
    p16 = softmax_f32(s16.astype(np.float32)).astype(np.float16)
    n_sink = 0 if sink_scores_f16 is None else sink_scores_f16.shape[-1]
    o = v_fn(p16[:, n_sink:].astype(np.float32))
    return p16, np.asarray(o).astype(np.float32).astype(np.float16)


def attend_ideal(scores_kernel_f64, v_fn, head_dim=HEAD_DIM, sink_scores=None):
    """Same chain with no fp16 round trips (float64 softmax) -- what a fused kernel approximates."""
    s = np.asarray(scores_kernel_f64, dtype=np.float64) / np.sqrt(head_dim)
    if sink_scores is not None:
        s = np.concatenate([np.asarray(sink_scores, dtype=np.float64), s], axis=-1)
    m = s.max(axis=-1, keepdims=True)
    e = np.exp(s - m)
    p = e / e.sum(axis=-1, keepdims=True)
    n_sink = 0 if sink_scores is None else sink_scores.shape[-1]
    return p, np.asarray(v_fn(p[:, n_sink:]))


# --------------------------------------------------------------------------------------------------
# a whole quantised cache built token by token with the reference decode semantics
# --------------------------------------------------------------------------------------------------
def attend_partial(scores_kernel_f64, v_fn, head_dim=HEAD_DIM):
    """Partial attention over one contiguous token shard (sequence-sharded decode, SURVEY.md 8e-2): the shard's own
    softmax-normalised output and the log-sum-exp of its scaled scores.  float64: (out [H,128], lse [H])."""
    s = np.asarray(scores_kernel_f64, dtype=np.float64) / np.sqrt(head_dim)
    m = s.max(axis=-1, keepdims=True)
    e = np.exp(s - m)
    l = e.sum(axis=-1, keepdims=True)
    return v_fn(e / l), (m + np.log(l))[:, 0]


def merge_partials(outs, lses):
    """Exact merge of per-shard (out, lse) pairs: out = sum_r exp(lse_r - M) out_r / sum_r exp(lse_r - M), M = max lse
    (what kvq_attend_merge computes on the device).  outs [R,H,128], lses [R,H] -> [H,128] float64."""
    outs = np.asarray(outs, dtype=np.float64)
    lses = np.asarray(lses, dtype=np.float64)
    w = np.exp(lses - lses.max(axis=0, keepdims=True))          # [R,H]
    return (w[:, :, None] * outs).sum(axis=0) / w.sum(axis=0)[:, None]


class OracleCache:
    """QuantK + QuantV state for one layer, filled token by token exactly as
    QuantK/QuantV.forward_fused_sparse do (ML.py:653-751, 1069-1176)."""

    def __init__(self, bits, num_heads, max_len, klut, v_cent, include_sparse=True, sparsity_threshold=0.99,
                 v_norm=None, sparse_v=None, v_ties="reference"):
        """v_norm = (normscale, normoffset) enables Q-Norm on V (ML.py:1054-1066,1115-1118); K Q-Norm is enabled by
        klut['lut2'] (ML.py:485-488): packing uses LUT, dequantisation and outlier subtraction use LUT2.
        v_ties: which V outlier row a token with values equal to a threshold gets -- "reference" (the reference's topk
        row, v_outlier_row) or "strict" (the fused append's row, v_outlier_row_strict).  Without such ties both agree."""
        if v_ties not in ("reference", "strict"):
            raise ValueError(v_ties)
        self.v_ties = v_ties
        self.bits = bits
        self.H = num_heads
        self.hidden = num_heads * HEAD_DIM
        self.Lmax = max_len
        self.klut = klut  # dict from build_k_lut
        self.v_cent = np.sort(np.asarray(v_cent, dtype=np.float32).ravel())
        self.sparse = include_sparse
        # sparse_v=False with include_sparse=True: capped K outliers only (BASELINE configs[4]); V then takes the
        # reference's dense-only branch (ML.py:1101-1108, 1178-1201)
        self.sparse_v = include_sparse if sparse_v is None else (bool(sparse_v) and include_sparse)
        self.n_each = n_out_each(self.hidden, sparsity_threshold)
        W = self.hidden * bits // 32
        self.kwords = np.zeros((W, max_len), dtype=np.int32)
        self.vwords = np.zeros((W, max_len), dtype=np.int32)
        self.vlut = np.zeros((max_len, 2 ** bits), dtype=np.float32)
        self.vaff = np.zeros((max_len, 2), dtype=np.float32)   # (sf_t, off_t) of each row of vlut
        self.v_norm = v_norm
        self.v_cent2 = None if v_norm is None else ((self.v_cent * F32(v_norm[0])).astype(np.float32) + F32(v_norm[1])).astype(np.float32)
        self.vlut2 = np.zeros((max_len, 2 ** bits), dtype=np.float32) if v_norm is not None else None
        n_out = 2 * self.n_each
        self.k_out = np.zeros((max_len, n_out), dtype=np.float32)
        self.k_idx = np.zeros((max_len, n_out), dtype=np.int32)
        self.v_out = np.zeros((max_len, n_out), dtype=np.float32)
        self.v_idx = np.zeros((max_len, n_out), dtype=np.int32)
        self.len = 0

    def append(self, k, v):
        t = self.len
        lut = self.klut["lut"]
        self.kwords[:, t] = pack_codes(append_k_codes(k, lut), self.bits)[:, 0]
        if self.sparse:
            r = k_outliers_rescaled(k, self.klut["thr_lower"], self.klut["thr_upper"])
            sub = self.klut["lut2"] if self.klut.get("lut2") is not None else lut
            self.k_out[t], self.k_idx[t] = k_outlier_row(k, r, sub, self.n_each)
        if self.sparse_v:
            hi, lo, ui, li = v_thresholds(v, self.n_each)
            self.vaff[t] = v_token_affine(hi, lo)
            self.vlut[t] = v_token_lut(self.v_cent, hi, lo)
            codes = append_v_codes(v, self.vlut[t], self.bits, lo, hi)
            zrow = self.vlut[t]
            if self.v_norm is not None:   # ML.py:1115-1118, 1149-1152: zero-point taken from the Q-Norm table
                self.vlut2[t] = v_token_lut(self.v_cent2, hi, lo)
                zrow = self.vlut2[t]
            zp = zrow[zero_point_code(self.bits)]
            if self.v_ties == "strict":
                self.v_out[t], self.v_idx[t] = v_outlier_row_strict(v, hi, lo, self.n_each, zp)
            else:
                self.v_out[t], self.v_idx[t] = v_outlier_row(v, ui, li, zp)
        else:
            v = np.asarray(v, dtype=np.float32)
            self.vaff[t] = v_token_affine(v.max(), v.min())
            self.vlut[t] = v_token_lut(self.v_cent, v.max(), v.min())  # compute_lut (ML.py:318-349)
            codes = append_v_codes(v, self.vlut[t], self.bits)
        self.vwords[:, t] = pack_codes(codes, self.bits)[:, 0]
        self.len += 1

    def k_scores(self, q, rope_theta=10000.0, pos_offset=0):
        deq = self.klut["lut2"] if self.klut.get("lut2") is not None else self.klut["lut"]
        s = k_scores_dense(q, self.kwords, deq, self.bits, self.len, rope_theta, pos_offset, self.H)
        if self.sparse:
            s = s + k_scores_outliers(q, self.k_out, self.k_idx, self.len, rope_theta, pos_offset, self.H)
        return s

    def v_output(self, p):
        o = v_out_dense(p, self.vwords, self.vlut2 if self.v_norm is not None else self.vlut, self.bits, self.len, self.H)
        if self.sparse_v:
            o = o + v_out_outliers(p, self.v_out, self.v_idx, self.len, self.H)
        return o

    def k_recon(self):
        """dequantised K incl. outliers, [hidden, L]."""
        kk = k_dequant(self.kwords[:, :self.len], self.klut["lut"], self.bits).astype(np.float64)
        if self.sparse:
            t = np.broadcast_to(np.arange(self.len)[:, None], self.k_idx[:self.len].shape)
            np.add.at(kk, (self.k_idx[:self.len].astype(np.int64), t), self.k_out[:self.len].astype(np.float64))
        return kk

    def v_recon(self):
        vv = v_dequant(self.vwords[:, :self.len], self.vlut[:self.len], self.bits).astype(np.float64)
        if self.sparse_v:
            t = np.broadcast_to(np.arange(self.len)[:, None], self.v_idx[:self.len].shape)
            np.add.at(vv, (self.v_idx[:self.len].astype(np.int64), t), self.v_out[:self.len].astype(np.float64))
        return vv


# --------------------------------------------------------------------------------------------------
# simulated-quant path (the reference's CPU-runnable oracle, config 1) -- SQ.py
# --------------------------------------------------------------------------------------------------
def sim_round_to_nearest_pole(w, poles):
    """round_to_nearest_pole_sim (SQ.py:10-28): nearest pole, first minimum (torch argmin)."""
    w = np.asarray(w, dtype=np.float32)
    poles = np.asarray(poles, dtype=np.float32).ravel()
    d = np.abs((w[None, ...] - poles.reshape((-1,) + (1,) * w.ndim)).astype(np.float32))
    idx = np.argmin(d, axis=0)
    return poles[idx]


def sim_get_outliers(w, channel, thr_upper, thr_lower, cap_outliers=-1, first_few_fp16=-1):
    """get_outliers (SQ.py:30-78).  w [T, hidden]; static thresholds broadcast along `channel`."""
    w = np.asarray(w, dtype=np.float32)
    up = np.expand_dims(np.asarray(thr_upper, dtype=np.float32), channel)
    lo = np.expand_dims(np.asarray(thr_lower, dtype=np.float32), channel)
    mask = (w < lo) | (w > up)
    if cap_outliers > -1:
        zp = ((up + lo) / F32(2)).astype(np.float32)
        dist = ((up - lo) / F32(2)).astype(np.float32)
        values = np.zeros_like(w)
        nv = ((w - zp) / dist).astype(np.float32)
        values[mask] = nv[mask]
        ui = np.argsort(-values, axis=-1, kind="stable")[..., :21]
        li = np.argsort(values, axis=-1, kind="stable")[..., :21]
        idx = np.concatenate([ui, li], axis=-1)
        val = np.take_along_axis(values, idx, axis=-1)
        v2 = np.zeros_like(w)
        np.put_along_axis(v2, idx, val, axis=-1)
        mask = v2 != 0
    if first_few_fp16 > -1:
        mask[:first_few_fp16, :] = True
    return mask


def _torch_quantile_f32(w, q, axis):
    """torch.quantile(..., interpolation='linear') in fp32: rank = q*(n-1); lerp(lo, hi, frac)."""
    w = np.sort(np.asarray(w, dtype=np.float32), axis=axis)
    n = w.shape[axis]
    rank = np.float32(q) * np.float32(n - 1)
    lo_i = int(np.floor(rank))
    hi_i = int(np.ceil(rank))
    frac = np.float32(rank - np.float32(lo_i))
    lo = np.take(w, lo_i, axis=axis)
    hi = np.take(w, hi_i, axis=axis)
    return (lo + (hi - lo) * frac).astype(np.float32)


def sim_get_outliers_dynamic(w, channel=-1, thresh=0.999, first_few_fp16=-1):
    """get_outliers_dynamic (SQ.py:80-113): per-token quantile thresholds, >= / <= compares."""
    t = 1 - ((1 - thresh) / 2)
    w = np.asarray(w, dtype=np.float32)
    up = np.expand_dims(_torch_quantile_f32(w, t, channel), channel)
    lo = np.expand_dims(_torch_quantile_f32(w, 1 - t, channel), channel)
    mask = (w <= lo) | (w >= up)
    if first_few_fp16 > -1:
        mask[:first_few_fp16, :] = True
    return mask


def sim_quant_fn_nuq_recon(inp, qchannel, lut, dynamicquantization=False, include_sparse=False,
                           outlier_mask=None, maxval=None, minval=None, norm=False, normscale=None,
                           normoffset=None, first_few_fp16=-1):
    """quant_fn_nuq_recon (SQ.py:265-361).  inp [T, hidden]; qchannel=0 -> per-channel (K), -1 -> per-token (V)."""
    inp = np.asarray(inp, dtype=np.float32)
    orig = inp
    if dynamicquantization:
        if include_sparse:
            outliers = (inp * outlier_mask).astype(np.float32)
            srt = np.sort(inp, axis=qchannel)
            n = inp.shape[qchannel]
            median = np.expand_dims(np.take(srt, (n - 1) // 2, axis=qchannel), qchannel)  # torch.median: lower middle
            median_mask = (median * outlier_mask).astype(np.float32)
            tmp = ((inp - outliers).astype(np.float32) + median_mask).astype(np.float32)
            maxval = tmp.max(axis=qchannel)
            minval = tmp.min(axis=qchannel)
        else:
            maxval = inp.max(axis=qchannel)
            minval = inp.min(axis=qchannel)
    maxval = np.asarray(maxval, dtype=np.float32)
    minval = np.asarray(minval, dtype=np.float32)
    offset = np.expand_dims(((maxval + minval) / F32(2)).astype(np.float32), qchannel)
    rangeval = np.expand_dims(((maxval - minval) / F32(2)).astype(np.float32), qchannel)
    x = (inp - offset).astype(np.float32)
    if include_sparse:
        outliers = (x * outlier_mask).astype(np.float32)
        x = (x - outliers).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        xs = (x / rangeval).astype(np.float32)
    poles = np.asarray(lut, dtype=np.float32).ravel()  # NOT sorted by the reference here (SQ.py:330)
    q = sim_round_to_nearest_pole(xs.ravel(), poles).reshape(x.shape).astype(np.float32)
    if norm:
        q = (q * F32(normscale) + F32(normoffset)).astype(np.float32)
    q = (q * rangeval).astype(np.float32)
    if include_sparse:
        q[outlier_mask] = 0
        q = (q + outliers).astype(np.float32)
    q = (q + offset).astype(np.float32)
    q = np.nan_to_num(q, nan=0.0, posinf=0.0, neginf=0.0)
    if first_few_fp16 > -1:
        q[:first_few_fp16, :] = orig[:first_few_fp16, :]
    return q.astype(np.float32)
