"""Drop-in replacement for the reference's `quant_cuda` torch extension.

Exports the 34 operator names of the reference's deployment/kvquant/quant_cuda.cpp:401-436 with the same
positional arguments, dtypes (fp32 / int32), shapes and in-place semantics, implemented on top of the C ABI in
include/kvquant_b200.h (hand-written sm_90a kernels).  `import quant_cuda` in the reference's
modeling_llama.py:53 resolves to this module through the top-level `quant_cuda.py` shim at the repo root.

Differences a caller can observe (all documented in INTEGRATION.md):
  * kernels run on the CURRENT torch stream (the reference always uses the legacy default stream);
  * wrong dtype / device / contiguity raises TypeError/ValueError instead of aborting the process on a
    device-side assert (reference quant_cuda_kernel.cu:1184-1187) or reading garbage;
  * `..._opt2` (dense + sparse) is ONE launch instead of two;
  * RoPE cos/sin come from a per-(device, theta) table built once with the reference's own powf/cosf/sinf
    expressions (bit-identical values), instead of being re-evaluated 4096 times per token.
"""
from __future__ import annotations

import torch

from . import _lib
from .rope import RotarySpec

_HEAD_DIM = 128
_rope_tables = {}  # (device index, theta or RotarySpec.key) -> (f32 [64, npos, 2], half2 [64, npos] as int32, npos, build event)
_rope_freqs = {}   # (device index, RotarySpec.key) -> f32 [64] inv_freq on the device (read by the freq table builders)
_rope_retired = []  # superseded tables stay allocated (graphs / other streams may still read them)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _chk(t, dtype, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor" % name)
    if t.dtype != dtype:
        raise TypeError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError("%s must be contiguous" % name)
    return t.data_ptr()


def _f32(t, name):
    return _chk(t, torch.float32, name)


def _i32(t, name):
    return _chk(t, torch.int32, name)


def _cache_dims(mat, bits):
    if mat.dim() != 3:
        raise ValueError("cache must be [H, 128*bits/32, Lmax]")
    H, W, Lmax = mat.shape
    if W != _HEAD_DIM * bits // 32:
        raise ValueError("cache dim 1 is %d, expected %d for %d-bit" % (W, _HEAD_DIM * bits // 32, bits))
    return H, Lmax


def rope_freq(device, spec):
    """HF's inv_freq of a scaled RotarySpec as a device f32 [64] tensor (one per device and spec, never freed: the
    attend entry points and captured graphs hold its pointer)."""
    dev = device.index if device.index is not None else torch.cuda.current_device()
    f = _rope_freqs.get((dev, spec.key))
    if f is None:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("rope frequencies of %r must be on the device before graph capture" % (spec,))
        f = spec.inv_freq.to(torch.device("cuda", dev))
        _rope_freqs[(dev, spec.key)] = f
    return f


def rope_tables(device, theta, min_npos: int):
    """(f32 table [64, npos, 2], half2 table [64, npos] as int32, npos) with npos >= min_npos; grown geometrically.

    theta: the rope base (float), or a scaled kvquant_b200.rope.RotarySpec, whose tables are built from its frequency
    vector and attention factor (kvq_rope_table_build_freq[_half]).
    Superseded tables are never freed: a captured CUDA graph (or a kernel still in flight on another stream) may hold
    their raw pointers.  Both tables are built on the current stream; an event recorded after the build is waited on
    by every later caller's stream, so a consumer on another stream never reads a half-built table."""
    dev = device.index if device.index is not None else torch.cuda.current_device()
    spec = theta if isinstance(theta, RotarySpec) else None
    if spec is not None and not spec.scaled:
        spec, theta = None, spec.theta
    key = (dev, spec.key) if spec is not None else (dev, float(theta))
    cur = _rope_tables.get(key)
    if cur is None or cur[2] < min_npos:
        npos = max(int(min_npos), 2 * cur[2] if cur else 0, 4096)
        npos = (npos + 255) // 256 * 256
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("rope table for %s must cover %d positions before graph capture "
                               "(call rope_tables() once outside the capture)"
                               % (spec if spec is not None else "theta=%g" % theta, min_npos))
        t = torch.empty((64, npos, 2), dtype=torch.float32, device=device)
        th = torch.empty((64, npos), dtype=torch.int32, device=device)
        lib = _lib.load()
        with torch.cuda.device(device):
            if spec is not None:
                f, a = rope_freq(device, spec).data_ptr(), float(spec.attention_factor)
                _lib.check(lib.kvq_rope_table_build_freq(t.data_ptr(), f, a, npos, _stream()),
                           "kvq_rope_table_build_freq")
                _lib.check(lib.kvq_rope_table_build_freq_half(th.data_ptr(), f, a, npos, _stream()),
                           "kvq_rope_table_build_freq_half")
            else:
                _lib.check(lib.kvq_rope_table_build(t.data_ptr(), float(theta), npos, _stream()), "kvq_rope_table_build")
                _lib.check(lib.kvq_rope_table_build_half(th.data_ptr(), float(theta), npos, _stream()),
                           "kvq_rope_table_build_half")
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
        if cur is not None:
            _rope_retired.append(cur)
        cur = (t, th, npos, ev)
        _rope_tables[key] = cur
    # (event queries are illegal while a stream is capturing; the eager warm-up that precedes a capture has already
    # ordered this stream behind the build)
    if not torch.cuda.is_current_stream_capturing() and not cur[3].query():
        torch.cuda.current_stream(device).wait_event(cur[3])
    return cur[0], cur[1], cur[2]


def rope_table(device, theta: float, min_npos: int):
    """(f32 tensor, npos) -- the table the legacy K ops read."""
    t, _, npos = rope_tables(device, theta, min_npos)
    return t, npos


# ---------------------------------------------------------------------------------------------------------------
# appends
# ---------------------------------------------------------------------------------------------------------------
def _append_k(bits, mat, lookup_table, newvec, kcachelen):
    lib = _lib.load()
    H, Lmax = _cache_dims(mat, bits)
    with torch.cuda.device(mat.device):
        _lib.check(lib.kvq_append_k(bits, _i32(mat, "mat"), _f32(lookup_table, "lookup_table"),
                                    _f32(newvec, "newvec"), H, Lmax, int(kcachelen), _stream()), "appendvecK")


def _append_v(bits, mat, lookup_table, newvec, vcachelen):
    lib = _lib.load()
    H, Lmax = _cache_dims(mat, bits)
    with torch.cuda.device(mat.device):
        _lib.check(lib.kvq_append_v(bits, _i32(mat, "mat"), _f32(lookup_table, "lookup_table"),
                                    _f32(newvec, "newvec"), H, Lmax, int(vcachelen), _stream()), "appendvecV")


def _append_k_sparse(bits, mat, lookup_table, newvec, outliers_rescaled, thr_lower, thr_upper, kcachelen):
    lib = _lib.load()
    H, Lmax = _cache_dims(mat, bits)
    with torch.cuda.device(mat.device):
        _lib.check(lib.kvq_append_k_sparse(
            bits, _i32(mat, "mat"), _f32(lookup_table, "lookup_table"), _f32(newvec, "newvec"),
            _f32(outliers_rescaled, "outliers_rescaled"), _f32(thr_lower, "outlier_threshold_lower"),
            _f32(thr_upper, "outlier_threshold_upper"), H, Lmax, int(kcachelen), _stream()), "appendvecKsparse")


def _append_k_sparse_parallel(bits, mat, lookup_table, newvec, outliers_rescaled, thr_lower, thr_upper):
    lib = _lib.load()
    H, Lmax = _cache_dims(mat, bits)
    if newvec.dim() != 3 or newvec.shape[0] != H or newvec.shape[1] != _HEAD_DIM:
        raise ValueError("newvec must be [H,128,T]")
    T = newvec.shape[2]
    with torch.cuda.device(mat.device):
        _lib.check(lib.kvq_append_k_sparse_parallel(
            bits, _i32(mat, "mat"), _f32(lookup_table, "lookup_table"), _f32(newvec, "newvec"),
            _f32(outliers_rescaled, "outliers_rescaled"), _f32(thr_lower, "outlier_threshold_lower"),
            _f32(thr_upper, "outlier_threshold_upper"), H, Lmax, T, _stream()), "appendvecKsparseParallel")


def _append_v_sparse(bits, mat, lookup_table, newvec, zeropoint, thr_lower, thr_upper, vcachelen):
    lib = _lib.load()
    H, Lmax = _cache_dims(mat, bits)
    with torch.cuda.device(mat.device):
        # float(...) on a 0-dim CUDA tensor synchronises, exactly like pybind11's float conversion in the reference
        _lib.check(lib.kvq_append_v_sparse(
            bits, _i32(mat, "mat"), _f32(lookup_table, "lookup_table"), _f32(newvec, "newvec"),
            float(zeropoint), float(thr_lower), float(thr_upper), H, Lmax, int(vcachelen), _stream()),
            "appendvecVsparse")


def _append_v_sparse_parallel(bits, mat, lookup_table, newvec, thr_lower, thr_upper):
    lib = _lib.load()
    H, Lmax = _cache_dims(mat, bits)
    if newvec.dim() != 3 or newvec.shape[0] != H or newvec.shape[1] != _HEAD_DIM:
        raise ValueError("newvec must be [H,128,T]")
    T = newvec.shape[2]
    with torch.cuda.device(mat.device):
        _lib.check(lib.kvq_append_v_sparse_parallel(
            bits, _i32(mat, "mat"), _f32(lookup_table, "lookup_table"), _f32(newvec, "newvec"),
            _f32(thr_lower, "outlier_threshold_lower"), _f32(thr_upper, "outlier_threshold_upper"),
            H, Lmax, T, _stream()), "appendvecVsparseParallel")


# ---------------------------------------------------------------------------------------------------------------
# matvecs
# ---------------------------------------------------------------------------------------------------------------
def _k_matvec(bits, vec, mat, mul, lookup_table, kcachelen, outliers, outlier_indices, theta, pos_offset):
    lib = _lib.load()
    H, Lmax = _cache_dims(mat, bits)
    L = int(kcachelen)
    if vec.dim() != 3 or vec.shape[1] != H or vec.shape[2] != _HEAD_DIM:
        raise ValueError("vec must be [B,H,128]")
    B = vec.shape[0]
    if tuple(mul.shape) != (B, H, L):
        raise ValueError("mul must be [B,H,kcachelen]")
    n_out = 0
    po = pi = None
    if outliers is not None:
        if outliers.dim() != 2 or outliers.shape != outlier_indices.shape or outliers.shape[0] < L:
            raise ValueError("outliers / outlier_indices must be [>=kcachelen, n_out]")
        n_out = outliers.shape[1]
        po, pi = _f32(outliers, "outliers"), _i32(outlier_indices, "outlier_indices")
    with torch.cuda.device(mat.device):
        rope, npos = rope_table(mat.device, theta, L + int(pos_offset))
        _lib.check(lib.kvq_k_matvec(bits, _f32(vec, "vec"), _i32(mat, "mat"), _f32(mul, "mul"),
                                    _f32(lookup_table, "lookup_table"), B, H, Lmax, L, po, pi, n_out,
                                    rope.data_ptr(), npos, float(theta), int(pos_offset), _stream()), "matmul K")


def _v_matvec(bits, vec, mat, mul, lookup_table, vcachelen, outliers, outlier_indices):
    lib = _lib.load()
    H, Lmax = _cache_dims(mat, bits)
    L = int(vcachelen)
    if vec.dim() != 3 or vec.shape[1] != H or vec.shape[2] != L:
        raise ValueError("vec must be [B,H,vcachelen]")
    B = vec.shape[0]
    if tuple(mul.shape) != (B, H, _HEAD_DIM):
        raise ValueError("mul must be [B,H,128]")
    n_out = 0
    po = pi = None
    if outliers is not None:
        if outliers.dim() != 2 or outliers.shape != outlier_indices.shape or outliers.shape[0] < L:
            raise ValueError("outliers / outlier_indices must be [>=vcachelen, n_out]")
        n_out = outliers.shape[1]
        po, pi = _f32(outliers, "outliers"), _i32(outlier_indices, "outlier_indices")
    with torch.cuda.device(mat.device):
        _lib.check(lib.kvq_v_matvec(bits, _f32(vec, "vec"), _i32(mat, "mat"), _f32(mul, "mul"),
                                    _f32(lookup_table, "lookup_table"), B, H, Lmax, L, po, pi, n_out, _stream()),
                   "matmul V")


def _make_ops():
    g = globals()
    for b in (4, 3, 2):
        def mk(bits):
            def appendvecK(mat, lookup_table, newvec, kcachelen):
                _append_k(bits, mat, lookup_table, newvec, kcachelen)

            def appendvecV(mat, lookup_table, newvec, vcachelen):
                _append_v(bits, mat, lookup_table, newvec, vcachelen)

            def appendvecKsparse(mat, lookup_table, newvec, outliers_rescaled, outlier_threshold_lower,
                                 outlier_threshold_upper, kcachelen):
                _append_k_sparse(bits, mat, lookup_table, newvec, outliers_rescaled, outlier_threshold_lower,
                                 outlier_threshold_upper, kcachelen)

            def appendvecKsparseParallel(mat, lookup_table, newvec, outliers_rescaled, outlier_threshold_lower,
                                         outlier_threshold_upper):
                _append_k_sparse_parallel(bits, mat, lookup_table, newvec, outliers_rescaled,
                                          outlier_threshold_lower, outlier_threshold_upper)

            def appendvecVsparse(mat, lookup_table, newvec, zeropoint, outlier_threshold_lower,
                                 outlier_threshold_upper, vcachelen):
                _append_v_sparse(bits, mat, lookup_table, newvec, zeropoint, outlier_threshold_lower,
                                 outlier_threshold_upper, vcachelen)

            def appendvecVsparseParallel(mat, lookup_table, newvec, outlier_threshold_lower,
                                         outlier_threshold_upper):
                _append_v_sparse_parallel(bits, mat, lookup_table, newvec, outlier_threshold_lower,
                                          outlier_threshold_upper)

            def k_opt(vec, mat, mul, lookup_table, kcachelen, theta, pos_offset):
                _k_matvec(bits, vec, mat, mul, lookup_table, kcachelen, None, None, theta, pos_offset)

            def k_opt2(vec, mat, mul, lookup_table, kcachelen, outliers, outlier_indices, theta, pos_offset):
                _k_matvec(bits, vec, mat, mul, lookup_table, kcachelen, outliers, outlier_indices, theta, pos_offset)

            def v_opt(vec, mat, mul, lookup_table, vcachelen):
                _v_matvec(bits, vec, mat, mul, lookup_table, vcachelen, None, None)

            def v_opt2(vec, mat, mul, lookup_table, vcachelen, outliers, outlier_indices):
                _v_matvec(bits, vec, mat, mul, lookup_table, vcachelen, outliers, outlier_indices)

            return {
                "vecquant%dappendvecK" % bits: appendvecK,
                "vecquant%dappendvecV" % bits: appendvecV,
                "vecquant%dappendvecKsparse" % bits: appendvecKsparse,
                "vecquant%dappendvecKsparseParallel" % bits: appendvecKsparseParallel,
                "vecquant%dappendvecVsparse" % bits: appendvecVsparse,
                "vecquant%dappendvecVsparseParallel" % bits: appendvecVsparseParallel,
                "vecquant%dmatmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt" % bits: k_opt,
                "vecquant%dmatmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2" % bits: k_opt2,
                "vecquant%dmatmul_nuq_perchannel_transposed_mha_batched_fused_opt" % bits: v_opt,
                "vecquant%dmatmul_nuq_perchannel_transposed_mha_batched_fused_opt2" % bits: v_opt2,
            }
        for name, fn in mk(b).items():
            fn.__name__ = name
            fn.__qualname__ = name
            g[name] = fn


_make_ops()


# ---------------------------------------------------------------------------------------------------------------
# uncapped "orig" ops (4-bit only, quant_cuda.cpp:347-399)
# ---------------------------------------------------------------------------------------------------------------
def vecquant4matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2_orig(
        vec, mat, mul, lookup_table, kcachelen, rows, cols, startrows, spmat, num_rows, num_threads, nnz,
        rope_theta, pos_offset):
    """dense K matvec + balanced CSR SpMV (quant_cuda_kernel.cu:5506-5596)."""
    _k_matvec(4, vec, mat, mul, lookup_table, kcachelen, None, None, rope_theta, pos_offset)
    lib = _lib.load()
    H, _ = _cache_dims(mat, 4)
    with torch.cuda.device(mat.device):
        rope, npos = rope_table(mat.device, rope_theta, int(kcachelen) + int(pos_offset))
        _lib.check(lib.kvq_k_spmv_csr(_i32(rows, "rows"), _i32(cols, "cols"), _i32(startrows, "startrows"),
                                      _f32(spmat, "spmat"), _f32(vec, "vec"), _f32(mul, "mul"), H, int(kcachelen),
                                      int(num_rows), int(num_threads), int(nnz), rope.data_ptr(), npos, int(pos_offset),
                                      _stream()), "spmv csr")


def vecquant4matmul_nuq_perchannel_transposed_mha_batched_fused_opt2_orig(
        vec, mat, mul, lookup_table, vcachelen, rows, cols, startcols, spmat, num_rows, num_threads, nnz):
    """dense V matvec + balanced CSC SpMV (quant_cuda_kernel.cu:5599-5668).  `num_rows` is the column (token) count."""
    _v_matvec(4, vec, mat, mul, lookup_table, vcachelen, None, None)
    lib = _lib.load()
    H, _ = _cache_dims(mat, 4)
    with torch.cuda.device(mat.device):
        _lib.check(lib.kvq_v_spmv_csc(_i32(rows, "rows"), _i32(cols, "cols"), _i32(startcols, "startcols"),
                                      _f32(spmat, "spmat"), _f32(vec, "vec"), _f32(mul, "mul"), H, int(vcachelen),
                                      int(num_rows), int(num_threads), int(nnz), _stream()), "spmv csc")


def _grow_csr(ptr, idx, val, start, new_idx, new_val, count, cachelen, device):
    """Host glue of vecquant4appendvec{K,V}sparseorig (quant_cuda_kernel.cu:773-829): append one token's outliers
    to the growing CSR/CSC arrays; 10 nonzeros per SpMV thread; new threads start at the current token."""
    i32 = dict(dtype=torch.int32, device=device)
    if ptr.numel() == 0:
        ptr2 = torch.tensor([0, count], **i32)
        idx2, val2 = new_idx, new_val
        nthreads = (count + 9) // 10
        start2 = torch.full((nthreads,), int(cachelen), **i32)
    else:
        ptr2 = torch.cat([ptr, torch.full((1,), idx.shape[0] + count, **i32)], 0)
        prevmax = start.shape[0]
        if count > 0:
            idx2 = torch.cat([idx, new_idx], 0)
            val2 = torch.cat([val, new_val], 0)
            nthreads = (idx2.shape[0] + 9) // 10
            new_alloc = nthreads - prevmax
            start2 = torch.cat([start, torch.full((new_alloc,), int(cachelen), **i32)], 0) if new_alloc > 0 else start
        else:
            idx2, val2, start2 = idx, val, start
            nthreads = (idx2.shape[0] + 9) // 10
    return ptr2, idx2, val2, start2, nthreads


def vecquant4appendvecKsparseorig(mat, lookup_table, newvec, zeropoint, row, col, val, start_rows,
                                  outlier_threshold_lower, outlier_threshold_upper, kcachelen):
    """-> [rows, cols, vals, start_rows, num_threads (cpu int32[1]), outlier_count (cuda int32[1])]."""
    lib = _lib.load()
    H, Lmax = _cache_dims(mat, 4)
    dev = mat.device
    hidden = H * _HEAD_DIM
    with torch.cuda.device(dev):
        oi = torch.empty(hidden, dtype=torch.int32, device=dev)
        ov = torch.empty(hidden, dtype=torch.float32, device=dev)
        oc = torch.zeros(1, dtype=torch.int32, device=dev)
        _lib.check(lib.kvq_append_k_orig(_i32(mat, "mat"), _f32(lookup_table, "lookup_table"), _f32(newvec, "newvec"),
                                         _f32(zeropoint, "zeropoint"), _f32(outlier_threshold_lower, "thr_lower"),
                                         _f32(outlier_threshold_upper, "thr_upper"), oi.data_ptr(), ov.data_ptr(),
                                         oc.data_ptr(), H, Lmax, int(kcachelen), _stream()), "appendvecKsparseorig")
        count = int(oc.item())  # the reference blocks on the same D2H read (quant_cuda_kernel.cu:745-747)
        row2, col2, val2, start2, nthreads = _grow_csr(row, col, val, start_rows, oi[:count].clone(),
                                                       ov[:count].clone(), count, kcachelen, dev)
    return [row2, col2, val2, start2, torch.tensor([nthreads], dtype=torch.int32), oc]


def vecquant4appendvecVsparseorig(mat, lookup_table, newvec, zeropoint, row, col, val, start_cols,
                                  outlier_threshold_lower, outlier_threshold_upper, vcachelen):
    """V twin: CSC with cols = tokens.  Returns [rows, cols(ptr), vals, start_cols, num_threads, outlier_count]."""
    lib = _lib.load()
    H, Lmax = _cache_dims(mat, 4)
    dev = mat.device
    hidden = H * _HEAD_DIM
    with torch.cuda.device(dev):
        oi = torch.empty(hidden, dtype=torch.int32, device=dev)
        ov = torch.empty(hidden, dtype=torch.float32, device=dev)
        oc = torch.zeros(1, dtype=torch.int32, device=dev)
        _lib.check(lib.kvq_append_v_orig(_i32(mat, "mat"), _f32(lookup_table, "lookup_table"), _f32(newvec, "newvec"),
                                         float(zeropoint), float(outlier_threshold_lower),
                                         float(outlier_threshold_upper), oi.data_ptr(), ov.data_ptr(), oc.data_ptr(),
                                         H, Lmax, int(vcachelen), _stream()), "appendvecVsparseorig")
        count = int(oc.item())
        col2, row2, val2, start2, nthreads = _grow_csr(col, row, val, start_cols, oi[:count].clone(),
                                                       ov[:count].clone(), count, vcachelen, dev)
    return [row2, col2, val2, start2, torch.tensor([nthreads], dtype=torch.int32), oc]


OP_NAMES = sorted(n for n in globals() if n.startswith("vecquant"))
assert len(OP_NAMES) == 34, len(OP_NAMES)
__all__ = list(OP_NAMES) + ["rope_table"]
