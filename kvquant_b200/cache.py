"""KV-cache managers.

* `QuantK` / `QuantV` mirror the reference's cache-manager classes
  (deployment/transformers/src/transformers/models/llama/modeling_llama.py:352-975 and 978-1385): same constructor
  arguments, attributes (kcache / lookup_table / outliers / outlier_indices / klen ...), methods and return values,
  so the reference's LlamaAttention code drives them unchanged.  They call the legacy 34-op surface
  (kvquant_b200.quant_cuda) and keep the reference's host-side top-K glue, but on the GPU (torch.topk on device
  instead of a .cpu() round trip -- same result, no blocking D2H).
* `LayerCache` is the native path: one fused device-side append (`kvq_append_kv_fused`) and one fused decode
  attention (`kvq_attend`) per layer per token, no host synchronisation, CUDA-graph capturable.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib
from . import quant_cuda as qc

HEAD_DIM = 128


def n_outliers_each(hidden_size: int, sparsity_threshold: float) -> int:
    """threshold_k of the reference (modeling_llama.py:707): 21 for hidden 4096 at 0.99."""
    return int(((1 - sparsity_threshold) / 2) * hidden_size) + 1


def build_k_lookup_table(upper, lower, centroids, num_heads, normscale=None, normoffset=None, device="cuda"):
    """Per-channel K LUT exactly as QuantK.load_lookup_table builds it (modeling_llama.py:447-501): thresholds are
    rounded through fp16, offset/range are computed in fp16, LUT = cent*range + offset in fp32 (two roundings).
    Vectorised (the reference loops 4096 times in Python).  Returns dict of CUDA tensors."""
    up16 = torch.as_tensor(np.asarray(upper, dtype=np.float32)).to(device).half().flatten()
    lo16 = torch.as_tensor(np.asarray(lower, dtype=np.float32)).to(device).half().flatten()
    cent = torch.as_tensor(np.asarray(centroids, dtype=np.float32)).to(device).flatten().sort().values
    offset = (up16 + lo16) / 2
    rangeval = (up16 - lo16) / 2
    sf = rangeval.float()[:, None]
    off = offset.float()[:, None]
    lut = (cent[None, :] * sf + off).contiguous()
    out = dict(lut=lut.view(num_heads, HEAD_DIM, -1), cent=cent, thr_upper=up16.float(), thr_lower=lo16.float(),
               zeropoint=offset.float(), lut2=None)
    if normscale is not None:
        c2 = cent * float(normscale) + float(normoffset)
        out["lut2"] = (c2[None, :] * sf + off).contiguous().view(num_heads, HEAD_DIM, -1)
    return out


def _on_cache_device(fn):
    """Run a LayerCache method with the cache's device current (the C ABI launches on the current device; one
    process may hold caches on several GPUs, as the reference's set_devices mode does)."""
    import functools

    @functools.wraps(fn)
    def wrapped(self, *a, **kw):
        if torch.cuda.current_device() == self.device.index:
            return fn(self, *a, **kw)
        with torch.cuda.device(self.device):
            return fn(self, *a, **kw)
    return wrapped


class LayerCache:
    """Native quantised K+V cache of one layer (reference-compatible tensor layouts, see DESIGN.md section 3)."""

    def __init__(self, bits, num_heads, max_len, klut, klut_sub, thr_lower, thr_upper, v_cent, device,
                 include_sparse=True, sparsity_threshold=0.99, n_sink=0, v_norm=None, sparse_v=None):
        self.lib = _lib.load()
        self.bits, self.H, self.Lmax = int(bits), int(num_heads), int(max_len)
        if self.Lmax % 4:
            raise ValueError("max_len must be a multiple of 4 (TMA row pitch)")
        self.hidden = self.H * HEAD_DIM
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        # include_sparse: outlier rows for K (and for V unless sparse_v=False: BASELINE configs[4] keeps capped K
        # outliers only); include_sparse=False is the reference's dense-only branch (configs[3])
        self.include_sparse = bool(include_sparse)
        self.sparse_k = self.include_sparse
        self.sparse_v = self.include_sparse if sparse_v is None else (bool(sparse_v) and self.include_sparse)
        self.n_each = n_outliers_each(self.hidden, sparsity_threshold)
        self.n_out = 2 * self.n_each
        W = HEAD_DIM * bits // 32
        dev = self.device
        self.kcache = torch.zeros((self.H, W, self.Lmax), dtype=torch.int32, device=dev)
        self.vcache = torch.zeros((self.H, W, self.Lmax), dtype=torch.int32, device=dev)
        self.klut = klut.contiguous()
        # Q-Norm (ML.py:485-488): codes are chosen against LUT, dequantisation and the outlier end-entry subtraction
        # use LUT2 = (cent*normscale+normoffset)*range + zp
        self.klut_sub = (klut_sub if klut_sub is not None else klut).contiguous()
        self.klut_deq = self.klut_sub
        self.thr_lower, self.thr_upper = thr_lower.contiguous(), thr_upper.contiguous()
        self.v_cent = v_cent.contiguous()
        # V Q-Norm (ML.py:1115-1118): LUT2_t = (cent*ns+no)*sf_t + off_t -> same affine form with shifted centroids
        self.v_cent_deq = self.v_cent if v_norm is None else (self.v_cent * float(v_norm[0]) + float(v_norm[1])).contiguous()
        self.v_norm = v_norm
        self.vlut = torch.zeros((self.Lmax, 2 ** bits), dtype=torch.float32, device=dev)
        # per-token affine map (sf_t, off_t): LUT_t = v_cent*sf_t + off_t  -- what the native V kernel consumes
        self.vaff = torch.zeros((self.Lmax, 2), dtype=torch.float32, device=dev)
        self.use_native_v = True
        def rows(on):   # a dense-only cache allocates no outlier rows (1M-token configs: 2 x 0.4 GB per layer saved)
            n = self.Lmax if on else 1
            return (torch.zeros((n, self.n_out), dtype=torch.float32, device=dev),
                    torch.zeros((n, self.n_out), dtype=torch.int32, device=dev))
        self.k_outliers, self.k_outlier_idx = rows(self.sparse_k)
        self.v_outliers, self.v_outlier_idx = rows(self.sparse_v)
        self.len = 0          # tokens in the quantised cache
        self.n_sink = int(n_sink)
        self.pos_base = 0     # absolute position of slot 0 minus n_sink (non-zero for a sequence shard)
        self.sink_k = self.sink_v = None
        self._scratch = None
        self._retired = []   # superseded scratch buffers (a captured graph may still point at them)
        self._out = torch.empty((self.H, HEAD_DIM), dtype=torch.float32, device=dev)
        # lookup-table precision of the K side of the fused attend:
        #   "fp32" (default) exact: the one-wavefront "ratio" tables of kvq_kratio.cu, equal to the legacy op chain to ~1e-6;
        #   "fp16"           north_star's fp16 LUT (kvq_kfast.cu): ~20 % faster K kernel, output within 1e-3 of the exact
        #                    result at test sizes and 1.4e-3 .. 2e-3 at 128K tokens (measured; DESIGN.md section 5).
        # KVQ_FP16_TABLES=1 makes fp16 the default.
        import os
        self.precision = "fp16" if os.environ.get("KVQ_FP16_TABLES", "0") not in ("", "0") else "fp32"

    @classmethod
    def from_luts(cls, bits, num_heads, max_len, klut, v_cent, device="cuda", include_sparse=True,
                  sparsity_threshold=0.99, n_sink=0, v_norm=None, sparse_v=None):
        """klut: mapping with 'lut' [hidden, n] (and optional 'lut2'), 'thr_lower', 'thr_upper' (numpy or torch)."""
        def t(x):
            return torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).to(device).float().contiguous()
        lut = t(klut["lut"]).view(num_heads * HEAD_DIM, -1)
        lut2 = t(klut["lut2"]).view(num_heads * HEAD_DIM, -1) if klut.get("lut2") is not None else None
        return cls(bits, num_heads, max_len, lut, lut2, t(klut["thr_lower"]), t(klut["thr_upper"]),
                   t(np.sort(np.asarray(v_cent.cpu() if torch.is_tensor(v_cent) else v_cent).ravel())), device,
                   include_sparse, sparsity_threshold, n_sink, v_norm, sparse_v)

    def reset(self):
        self.len = 0
        for x in (self.kcache, self.vcache, self.vlut, self.vaff, self.k_outliers, self.k_outlier_idx,
                  self.v_outliers, self.v_outlier_idx):
            x.zero_()

    def set_sinks(self, sink_k, sink_v):
        """fp16 attention-sink side caches (modeling_llama.py:1464-1466): sink_k [H,128,n] post-RoPE, sink_v [H,n,128]."""
        assert sink_k.dtype == torch.float16 and sink_v.dtype == torch.float16
        assert tuple(sink_k.shape) == (self.H, HEAD_DIM, self.n_sink) and tuple(sink_v.shape) == (self.H, self.n_sink, HEAD_DIM)
        self.sink_k, self.sink_v = sink_k.contiguous(), sink_v.contiguous()

    def load_state(self, src):
        """Copy a pre-built cache (any object exposing kwords/vwords/vlut/k_out/k_idx/v_out/v_idx/len as arrays)."""
        def put(dst, a):
            dst.copy_(torch.as_tensor(np.ascontiguousarray(a)).view(dst.shape) if not torch.is_tensor(a) else a.view(dst.shape))
        put(self.kcache, src.kwords); put(self.vcache, src.vwords); put(self.vlut, src.vlut)
        if self.sparse_k:
            put(self.k_outliers, src.k_out); put(self.k_outlier_idx, src.k_idx)
        if self.sparse_v:
            put(self.v_outliers, src.v_out); put(self.v_outlier_idx, src.v_idx)
        self.len = int(src.len)
        self.derive_vaff()

    def derive_vaff(self):
        """Recover (sf_t, off_t) from materialised LUT rows (caches filled through the legacy per-token-LUT path):
        sf = (LUT[n-1]-LUT[0])/(cent[n-1]-cent[0]), off = LUT[0]-cent[0]*sf  (agrees with the stored row to ~1 ulp)."""
        c0, c1 = self.v_cent[0], self.v_cent[-1]
        sf = (self.vlut[:, -1] - self.vlut[:, 0]) / (c1 - c0)
        self.vaff[:, 0] = sf
        self.vaff[:, 1] = self.vlut[:, 0] - c0 * sf

    def _vec(self, t, n, name, dtype=torch.float32):
        """Device pointer of a caller tensor after the checks the C ABI cannot make: dtype, contiguity, this cache's
        device, at least n elements (a short or foreign tensor would be read / written out of bounds)."""
        qc._chk(t, dtype, name)
        if t.device != self.device:
            raise ValueError("%s is on %s, the cache lives on %s" % (name, t.device, self.device))
        if t.numel() < n:
            raise ValueError("%s has %d elements, %d needed" % (name, t.numel(), n))
        return t.data_ptr()

    def _out_ptrs(self, which):
        """(values, indices) device pointers of a cache's outlier rows, or (None, None) when that cache is dense-only."""
        if which == "k":
            return (self.k_outliers.data_ptr(), self.k_outlier_idx.data_ptr()) if self.sparse_k else (None, None)
        return (self.v_outliers.data_ptr(), self.v_outlier_idx.data_ptr()) if self.sparse_v else (None, None)

    _shared_scratch = {}     # device index -> one attend scratch shared by every cache that opted in (share_scratch)
    share_scratch = False    # True: the caches of a device attend one after another on one stream (the decode harness);
                             # at 1M tokens a private scratch per layer would cost 0.3 GB x layers

    def _ensure_scratch(self, need, slack):
        """Attend scratch, grown on demand.  A superseded buffer is kept alive (never handed back to the allocator):
        a captured CUDA graph bakes the raw pointer in, and growing must not happen inside a capture."""
        cur = LayerCache._shared_scratch.get(self.device.index) if self.share_scratch else self._scratch
        if cur is None or cur.numel() < need:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("attend scratch must be sized before graph capture (run one eager attend / "
                                   "attend_dyn with the same L_cap first)")
            if cur is not None:
                self._retired.append(cur)
            cur = torch.empty(int(need * slack) + 1024, dtype=torch.uint8, device=self.device)
            if self.share_scratch:
                LayerCache._shared_scratch[self.device.index] = cur
        self._scratch = cur

    @_on_cache_device
    def append(self, k_new, v_new):
        """Quantise + pack + outlier split of one token's K and V, entirely on the device (one launch)."""
        if self.len >= self.Lmax:
            raise IndexError("cache full")
        s = torch.cuda.current_stream().cuda_stream
        _lib.check(self.lib.kvq_append_kv_fused(
            self.bits, self.H, self.Lmax, self.len, self.n_each,
            self._vec(k_new, self.hidden, "k_new"), self.kcache.data_ptr(), self.klut.data_ptr(), self.klut_sub.data_ptr(),
            self.thr_lower.data_ptr(), self.thr_upper.data_ptr(), *self._out_ptrs("k"),
            self._vec(v_new, self.hidden, "v_new"), self.vcache.data_ptr(), self.v_cent.data_ptr(),
            self.v_cent_deq.data_ptr() if self.v_norm is not None else None, self.vlut.data_ptr(), self.vaff.data_ptr(),
            *self._out_ptrs("v"), s), "kvq_append_kv_fused")
        self.len += 1

    @_on_cache_device
    def append_chunk(self, k, v):
        """append() of T tokens in one launch (kvq_append_kv_fused_chunk): k, v f32 [T, hidden] pre-RoPE keys and
        values, the layout attend_chunk() takes.  Token t goes to slot len + t and len advances by T; the cache is left
        bit for bit as T append() calls would leave it.  T == 0 does nothing.  Allocates nothing and does not
        synchronise, so it can be captured in a CUDA graph."""
        if k.dim() != 2 or tuple(k.shape) != tuple(v.shape) or k.shape[1] != self.hidden:
            raise ValueError("k and v must both be [T, %d], got %s and %s" % (self.hidden, tuple(k.shape), tuple(v.shape)))
        T = k.shape[0]
        kp, vp = self._vec(k, T * self.hidden, "k"), self._vec(v, T * self.hidden, "v")
        if self.len + T > self.Lmax:
            raise IndexError("chunk of %d tokens does not fit: %d of %d slots used" % (T, self.len, self.Lmax))
        if T == 0:
            return
        _lib.check(self.lib.kvq_append_kv_fused_chunk(
            self.bits, self.H, self.Lmax, self.len, T, self.n_each,
            kp, self.kcache.data_ptr(), self.klut.data_ptr(), self.klut_sub.data_ptr(),
            self.thr_lower.data_ptr(), self.thr_upper.data_ptr(), *self._out_ptrs("k"),
            vp, self.vcache.data_ptr(), self.v_cent.data_ptr(),
            self.v_cent_deq.data_ptr() if self.v_norm is not None else None, self.vlut.data_ptr(), self.vaff.data_ptr(),
            *self._out_ptrs("v"), torch.cuda.current_stream().cuda_stream), "kvq_append_kv_fused_chunk")
        self.len += T

    @_on_cache_device
    def attend(self, q, rope_theta=10000.0, out=None, lse=None):
        """softmax(q.K^T/sqrt(128)).V over sinks + quantised slots.  q: f32 [H,128] already rotated at its own
        position.  Returns f32 [H,128].  lse (optional f32 [H]) receives the log-sum-exp of the scaled scores, which
        lets partial results over disjoint token ranges be merged exactly (sequence-sharded decode)."""
        L = self.len
        if self.v_norm is not None and not self.use_native_v:
            # the per-token LUT rows hold the un-normed centroids while the outlier residuals were taken against the
            # Q-Norm table: the legacy-LUT V kernel would mix the two
            raise NotImplementedError("V Q-Norm needs the native V form (use_native_v=True)")
        self._ensure_scratch(self.lib.kvq_attend_scratch_bytes(self.H, max(L, 1)), 1.25)
        pos_offset = self.n_sink + self.pos_base
        rope, rope_h, npos = qc.rope_tables(self.device, rope_theta, L + pos_offset + 1)
        fast = self.precision == "fp16" and self.use_native_v
        out = self._out if out is None else out
        ns = self.n_sink if self.sink_k is not None else 0
        _lib.check(self.lib.kvq_attend(
            self.bits, self._vec(q, self.hidden, "q"), self.kcache.data_ptr(), self.klut_deq.data_ptr(), *self._out_ptrs("k"),
            self.vcache.data_ptr(), self.vlut.data_ptr(),
            self.v_cent_deq.data_ptr() if self.use_native_v else None, self.vaff.data_ptr() if self.use_native_v else None,
            *self._out_ptrs("v"),
            self.n_out, self.H, self.Lmax, L, rope.data_ptr(), npos, float(rope_theta), pos_offset,
            self.sink_k.data_ptr() if ns else None, self.sink_v.data_ptr() if ns else None, ns,
            self._vec(out, self.hidden, "out"), self._vec(lse, self.H, "lse") if lse is not None else None, self._scratch.data_ptr(),
            rope_h.data_ptr() if fast else None, torch.cuda.current_stream().cuda_stream), "kvq_attend")
        return out

    # -- device-resident length (one captured CUDA graph serves a growing cache; SURVEY.md 8(f)-2) ----------------------
    @_on_cache_device
    def append_dyn(self, k_new, v_new, len_dev, slot_add=0):
        """append() at slot `len_dev[0] + slot_add`, the length read on the device.  The host-side `len` is NOT
        advanced: the caller owns the device counter (kvq_dec_counter_add) and re-syncs `len` when it leaves the graph."""
        s = torch.cuda.current_stream().cuda_stream
        _lib.check(self.lib.kvq_append_kv_fused_dyn(
            self.bits, self.H, self.Lmax, self._vec(len_dev, 1, "len_dev", torch.int64), int(slot_add), self.n_each,
            self._vec(k_new, self.hidden, "k_new"), self.kcache.data_ptr(), self.klut.data_ptr(), self.klut_sub.data_ptr(),
            self.thr_lower.data_ptr(), self.thr_upper.data_ptr(), *self._out_ptrs("k"),
            self._vec(v_new, self.hidden, "v_new"), self.vcache.data_ptr(), self.v_cent.data_ptr(),
            self.v_cent_deq.data_ptr() if self.v_norm is not None else None, self.vlut.data_ptr(), self.vaff.data_ptr(),
            *self._out_ptrs("v"), s), "kvq_append_kv_fused_dyn")

    @_on_cache_device
    def attend_dyn(self, q, len_dev, len_add=0, rope_theta=10000.0, out=None, lse=None, L_cap=None):
        """attend() over `min(len_dev[0] + len_add, L_cap)` slots, the length read on the device; grids, scratch and
        the rope table are sized for L_cap (default: the whole allocation)."""
        if not self.use_native_v:
            raise NotImplementedError("device-resident length needs the native V form")
        L_cap = self.Lmax if L_cap is None else int(L_cap)
        self._ensure_scratch(self.lib.kvq_attend_scratch_bytes(self.H, max(L_cap, 1)), 1.0)
        pos_offset = self.n_sink + self.pos_base
        rope, rope_h, npos = qc.rope_tables(self.device, rope_theta, L_cap + pos_offset + 1)
        fast = self.precision == "fp16"
        out = self._out if out is None else out
        ns = self.n_sink if self.sink_k is not None else 0
        _lib.check(self.lib.kvq_attend_dyn(
            self.bits, self._vec(q, self.hidden, "q"), self.kcache.data_ptr(), self.klut_deq.data_ptr(), *self._out_ptrs("k"),
            self.vcache.data_ptr(), self.v_cent_deq.data_ptr(), self.vaff.data_ptr(), *self._out_ptrs("v"),
            self.n_out, self.H, self.Lmax, L_cap, self._vec(len_dev, 1, "len_dev", torch.int64), int(len_add), rope.data_ptr(), npos,
            float(rope_theta), pos_offset, self.sink_k.data_ptr() if ns else None,
            self.sink_v.data_ptr() if ns else None, ns, self._vec(out, self.hidden, "out"),
            self._vec(lse, self.H, "lse") if lse is not None else None, self._scratch.data_ptr(),
            rope_h.data_ptr() if fast else None, torch.cuda.current_stream().cuda_stream), "kvq_attend_dyn")
        return out

    def _kv_out(self, t, n, name):
        """Caller-supplied fp16 [H, n, 128] output, possibly a view into a larger [H, S, 128] buffer: tokens and
        channels packed (stride (S*128, 128, 1)), on this cache's device, 16-byte aligned.  Returns the head stride."""
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a torch.Tensor" % name)
        if t.dtype != torch.float16:
            raise TypeError("%s must be torch.float16, got %s" % (name, t.dtype))
        if t.device != self.device:
            raise ValueError("%s is on %s, the cache lives on %s" % (name, t.device, self.device))
        if tuple(t.shape) != (self.H, n, HEAD_DIM):
            raise ValueError("%s has shape %s, expected %s" % (name, tuple(t.shape), (self.H, n, HEAD_DIM)))
        if t.stride(2) != 1 or t.stride(1) != HEAD_DIM or t.stride(0) < n * HEAD_DIM:
            raise ValueError("%s must have strides (S*128, 128, 1) with S >= %d, got %s" % (name, n, t.stride()))
        if t.data_ptr() % 16 or t.stride(0) % 8:
            raise ValueError("%s must be 16-byte aligned with a head stride that is a multiple of 8" % name)
        return t.stride(0)

    @_on_cache_device
    def dequantize(self, start=0, stop=None, rope_theta=None, out_k=None, out_v=None):
        """Slots [start, stop) of the cache as fp16 K and V, each [H, stop-start, 128] (one device pass, kvq_dequant_kv).

        K is the dequantised value (dequantisation table plus outlier residual); with rope_theta=None it is pre-RoPE,
        otherwise rotated at the absolute positions n_sink + pos_base + t -- the positions attend() uses -- so that
        q . k[t] for a query rotated at its own position is the score attend() computes for slot t.  V is
        v_cent[code]*sf_t + off_t plus its outlier residual.  out_k / out_v may be views into larger [H, S, 128]
        buffers (stride (S*128, 128, 1)), each with its own S; an output not given is allocated.  An empty range
        returns empty outputs.  With both outputs given, and a rope table that already covers the range, the call
        allocates nothing and can be captured in a CUDA graph."""
        if not self.use_native_v:
            raise NotImplementedError("dequantize reads the native V form (use_native_v=True)")
        stop = self.len if stop is None else int(stop)
        start = int(start)
        if not 0 <= start <= stop:
            raise ValueError("need 0 <= start <= stop, got start=%d stop=%d" % (start, stop))
        if stop > self.len:
            raise ValueError("stop=%d is past the %d cached tokens" % (stop, self.len))
        n = stop - start
        if out_k is None:
            out_k = torch.empty((self.H, n, HEAD_DIM), dtype=torch.float16, device=self.device)
        if out_v is None:
            out_v = torch.empty((self.H, n, HEAD_DIM), dtype=torch.float16, device=self.device)
        sk, sv = self._kv_out(out_k, n, "out_k"), self._kv_out(out_v, n, "out_v")
        if n == 0:
            return out_k, out_v
        pos_offset = self.n_sink + self.pos_base
        rope, npos = None, 0
        if rope_theta is not None:
            rope, _, npos = qc.rope_tables(self.device, rope_theta, stop + pos_offset)

        def run(ok, ov, stride):
            _lib.check(self.lib.kvq_dequant_kv(
                self.bits, self.H, self.Lmax, start, stop,
                self.kcache.data_ptr(), self.klut_deq.data_ptr(), *self._out_ptrs("k"),
                self.vcache.data_ptr(), self.v_cent_deq.data_ptr(), self.vaff.data_ptr(), *self._out_ptrs("v"),
                self.n_out, rope.data_ptr() if rope is not None else None, npos, pos_offset,
                ok, ov, stride, torch.cuda.current_stream().cuda_stream), "kvq_dequant_kv")
        # one head stride per call: outputs with different strides are written by one call each (K and V are separate
        # launches either way)
        if sk == sv:
            run(out_k.data_ptr(), out_v.data_ptr(), sk)
        else:
            run(out_k.data_ptr(), None, sk)
            run(None, out_v.data_ptr(), sv)
        return out_k, out_v

    def _chunk_check(self, q, k, v):
        """The argument checks of attend_chunk / attend_chunk_fused; returns T."""
        if q.dim() != 3 or q.shape[1:] != (self.H, HEAD_DIM) or q.shape[0] < 1:
            raise ValueError("q must be [T, %d, %d] with T >= 1, got %s" % (self.H, HEAD_DIM, tuple(q.shape)))
        T = q.shape[0]
        for t, name in ((q, "q"), (k, "k"), (v, "v")):
            self._vec(t, T * self.hidden, name)
        if tuple(k.shape) != (T, self.hidden) or tuple(v.shape) != (T, self.hidden):
            raise ValueError("k and v must be [%d, %d]" % (T, self.hidden))
        return T

    def _chunk_kv16(self, k, v, rope_theta, p0, out_k, out_v):
        """The chunk's keys rotated at positions p0 + i and its values, written as fp16 into out_k / out_v [H, T, 128]
        (views allowed): the chunk operands both chunk attentions use.  Returns the f32 rope table, covering
        p0 + T positions."""
        T = k.shape[0]
        rope, _, _ = qc.rope_tables(self.device, rope_theta, p0 + T)
        cos, sin = rope[:, p0:p0 + T, 0].t()[:, None, :], rope[:, p0:p0 + T, 1].t()[:, None, :]   # [T, 1, 64]
        kc = k.view(T, self.H, HEAD_DIM)
        lo, hi = kc[..., :HEAD_DIM // 2], kc[..., HEAD_DIM // 2:]
        out_k[:, :, :HEAD_DIM // 2] = (cos * lo - sin * hi).transpose(0, 1)
        out_k[:, :, HEAD_DIM // 2:] = (cos * hi + sin * lo).transpose(0, 1)
        out_v[:] = v.view(T, self.H, HEAD_DIM).transpose(0, 1)
        return rope

    @_on_cache_device
    def attend_chunk(self, q, k, v, rope_theta=10000.0):
        """Causal attention of a T-token chunk placed right after the cached tokens (a follow-up prompt).

        q: f32 [T, H, 128], token i already rotated at position P0 + i, P0 = n_sink + pos_base + len.
        k: f32 [T, hidden] pre-RoPE keys and v: f32 [T, hidden] values of the chunk, as append() takes them.
        Chunk token i attends over the fp16 sinks (when set), all `len` quantised slots (dequantised and rotated) and
        chunk tokens 0..i; the chunk's keys are rotated with the same table, and its keys and values rounded to fp16,
        as a prefill runs attention on the prompt's fp16 K/V.  Scale 1/sqrt(128).  Returns f32 [T, H, 128].

        The cache is NOT modified: append the chunk's tokens afterwards with append_chunk(k, v) (one launch, as
        DecoderStage.prefill does).  The call materialises K and V for every
        position, 2*H*(n_sink + len + T)*128 fp16 values (2 GiB for 32 heads at 128K tokens), and hands them to
        torch.nn.functional.scaled_dot_product_attention.  attend_chunk_fused computes the same attention without
        materialising the cache."""
        T = self._chunk_check(q, k, v)
        L = self.len
        ns = self.n_sink if self.sink_k is not None else 0
        S = ns + L + T
        p0 = self.n_sink + self.pos_base + L
        kbuf = torch.empty((1, self.H, S, HEAD_DIM), dtype=torch.float16, device=self.device)
        vbuf = torch.empty_like(kbuf)
        if ns:
            kbuf[0, :, :ns] = self.sink_k.transpose(1, 2)
            vbuf[0, :, :ns] = self.sink_v
        if L:
            self.dequantize(0, L, rope_theta, out_k=kbuf[0, :, ns:ns + L], out_v=vbuf[0, :, ns:ns + L])
        self._chunk_kv16(k, v, rope_theta, p0, kbuf[0, :, ns + L:], vbuf[0, :, ns + L:])
        mask = torch.arange(S, device=self.device)[None, :] <= (ns + L + torch.arange(T, device=self.device))[:, None]
        out = torch.nn.functional.scaled_dot_product_attention(
            q.transpose(0, 1)[None].half(), kbuf, vbuf, attn_mask=mask, scale=1.0 / math.sqrt(HEAD_DIM))
        return out[0].transpose(0, 1).float().contiguous()

    @_on_cache_device
    def attend_chunk_fused(self, q, k, v, rope_theta=10000.0):
        """attend_chunk() read straight from the quantised cache (kvq_attend_chunk): same arguments, checks, result
        (f32 [T, H, 128]) and semantics, and the cache is likewise left untouched.

        One tensor-core kernel dequantises each K/V tile of the cached slots into shared memory -- the same fp16
        values dequantize() writes -- and attends the chunk over it, FlashAttention-2 style.  Extra device memory per
        call is the chunk's fp16 rotated K and V (2*H*T*128*2 bytes) plus kvq_attend_chunk_scratch_bytes(H, T, len),
        whatever `len` is: at 1M cached tokens the materialising attend_chunk would need 2*H*1M*128*2 bytes more."""
        if not self.use_native_v:
            raise NotImplementedError("attend_chunk_fused reads the native V form (use_native_v=True)")
        T = self._chunk_check(q, k, v)
        L = self.len
        ns = self.n_sink if self.sink_k is not None else 0
        pos_offset = self.n_sink + self.pos_base
        kc = torch.empty((self.H, T, HEAD_DIM), dtype=torch.float16, device=self.device)
        vc = torch.empty_like(kc)
        rope = self._chunk_kv16(k, v, rope_theta, pos_offset + L, kc, vc)
        scratch = torch.empty(max(self.lib.kvq_attend_chunk_scratch_bytes(self.H, T, L), 16), dtype=torch.uint8,
                              device=self.device)
        out = torch.empty((T, self.H, HEAD_DIM), dtype=torch.float32, device=self.device)
        _lib.check(self.lib.kvq_attend_chunk(
            self.bits, self.H, self.Lmax, L, T, q.data_ptr(), kc.data_ptr(), vc.data_ptr(),
            self.kcache.data_ptr(), self.klut_deq.data_ptr(), *self._out_ptrs("k"),
            self.vcache.data_ptr(), self.v_cent_deq.data_ptr(), self.vaff.data_ptr(), *self._out_ptrs("v"),
            self.n_out, rope.data_ptr(), rope.shape[1], pos_offset,
            self.sink_k.data_ptr() if ns else None, self.sink_v.data_ptr() if ns else None, ns,
            out.data_ptr(), scratch.data_ptr(), torch.cuda.current_stream().cuda_stream), "kvq_attend_chunk")
        return out

    def bytes_per_token(self):
        """Algorithmic HBM bytes one decode step reads per cached token (SURVEY.md 8d formula)."""
        b = 2 * self.H * HEAD_DIM * self.bits // 8 + 4 * 2 ** self.bits
        b += (int(self.sparse_k) + int(self.sparse_v)) * self.n_out * 8
        return b


# -----------------------------------------------------------------------------------------------------------------
# reference-interface mirrors
# -----------------------------------------------------------------------------------------------------------------
class QuantK(torch.nn.Module):
    """Mirror of the reference's QuantK (modeling_llama.py:352-975)."""

    def __init__(self, bits=2, hidden_size=4096, num_heads=32, max_position_embeddings=-1, include_sparse=False,
                 sparsity_threshold=0.99, rope_theta=10000, use_orig_sparse=False, first_few_fp16=0):
        super().__init__()
        self.hidden_size, self.num_heads = hidden_size, num_heads
        self.head_dim = hidden_size // num_heads
        self.bits = bits
        self.lut = None
        self.lookup_table = None
        self.zeropoint = None
        self.sparsity_threshold = sparsity_threshold
        self.include_sparse = include_sparse
        self.outlier_threshold_upper = self.outlier_threshold_lower = None
        self.max_len = max_position_embeddings
        self.klen = 0
        self.kcache = torch.zeros((num_heads, (self.head_dim // 32) * bits, self.max_len), dtype=torch.int).cuda()
        self.n_out = 2 * n_outliers_each(hidden_size, sparsity_threshold)  # reference hard-codes 42 (ML.py:396)
        if include_sparse:
            self.outliers = torch.zeros((self.max_len, self.n_out), dtype=torch.float).cuda()
            self.outlier_indices = torch.zeros((self.max_len, self.n_out), dtype=torch.int).cuda()
        self.rope_theta = rope_theta
        self.rows = torch.tensor([]).cuda(); self.cols = torch.tensor([]).cuda()
        self.vals = torch.tensor([]).cuda(); self.start_rows = torch.tensor([]).cuda()
        self.num_threads = -1
        self.use_orig_sparse = use_orig_sparse
        self.first_few_fp16 = first_few_fp16
        self.norm = False
        self.lookup_table2 = None

    def reset(self):
        self.klen = 0
        self.kcache.zero_()
        if self.include_sparse:
            if self.use_orig_sparse:
                self.rows = torch.tensor([]).cuda(); self.cols = torch.tensor([]).cuda()
                self.vals = torch.tensor([]).cuda(); self.start_rows = torch.tensor([]).cuda()
                self.num_threads = -1
            else:
                self.outliers.zero_()
                self.outlier_indices.zero_()

    def load_lookup_table(self, quantizer, include_sparse=True, sparsity_threshold=0.99, norm=False):
        """quantizer: one `quantizers.pickle` entry (upper, lower, [centroids], [normscale, normoffset])."""
        self.include_sparse, self.sparsity_threshold, self.norm = include_sparse, sparsity_threshold, norm
        ns = no = None
        if norm:
            ns, no = float(quantizer[3]), float(quantizer[4])
            self.normscale, self.normoffset = quantizer[3], quantizer[4]
        t = build_k_lookup_table(quantizer[0], quantizer[1], quantizer[2][0], self.num_heads, ns, no,
                                 device=self.kcache.device)
        self.lut = t["cent"]
        self.lookup_table = t["lut"]
        self.lookup_table2 = t["lut2"]
        self.zeropoint = t["zeropoint"]
        self.outlier_threshold_upper, self.outlier_threshold_lower = t["thr_upper"], t["thr_lower"]

    def _op(self, fmt):
        return getattr(qc, fmt % self.bits)

    def _outlier_rows(self, k_tok, rescaled_tok):
        """k_tok, rescaled_tok: [T, hidden].  Device version of modeling_llama.py:706-751 / 934-971."""
        n_each = n_outliers_each(self.hidden_size, self.sparsity_threshold)
        up_r, up_i = torch.topk(rescaled_tok, n_each, dim=-1)
        lo_r, lo_i = torch.topk(rescaled_tok, n_each, dim=-1, largest=False)
        numvals = 2 ** self.bits
        lut = (self.lookup_table2 if self.norm else self.lookup_table).reshape(-1, numvals)
        up_v = torch.gather(k_tok, 1, up_i) - lut[up_i, numvals - 1]
        lo_v = torch.gather(k_tok, 1, lo_i) - lut[lo_i, 0]
        zer = torch.cat((up_r <= 1, lo_r >= -1), dim=-1)
        vals = torch.cat((up_v, lo_v), dim=-1)
        idx = torch.cat((up_i, lo_i), dim=-1)
        idx, order = idx.sort(dim=-1)
        vals = torch.gather(vals, 1, order)
        vals[torch.gather(zer, 1, order)] = 0
        return vals, idx.int()

    def forward_fused_sparse(self, q, k):
        """Append the new pre-RoPE key and return q.K^T over the compressed cache: fp16 [num_heads, B, klen]."""
        k = k.flatten().float()
        q = q.float().transpose(0, 1).contiguous()
        slot = self.klen - self.first_few_fp16
        if self.include_sparse:
            resc = k.clone()
            self._op("vecquant%dappendvecKsparse")(self.kcache, self.lookup_table, k, resc,
                                                    self.outlier_threshold_lower, self.outlier_threshold_upper, slot)
            vals, idx = self._outlier_rows(k[None], resc[None])
            self.outliers[slot] = vals[0]
            self.outlier_indices[slot] = idx[0]
        else:
            self._op("vecquant%dappendvecK")(self.kcache, self.lookup_table, k, slot)
        self.klen += 1
        L = self.klen - self.first_few_fp16
        mul = torch.zeros((q.shape[0], q.shape[1], L), dtype=torch.float, device=q.device)
        # (deliberate: the reference switches to lookup_table2 only in its 2-bit branch, modeling_llama.py:812-815; Q-Norm
        # checkpoints exist for 2 bits only, and dequantising with the table the outlier residuals were taken against
        # is the consistent choice at every width)
        lut = self.lookup_table2 if (self.norm and self.lookup_table2 is not None) else self.lookup_table
        if self.include_sparse:
            self._op("vecquant%dmatmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2")(
                q, self.kcache, mul, lut, L, self.outliers, self.outlier_indices, self.rope_theta, self.first_few_fp16)
        else:
            self._op("vecquant%dmatmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt")(
                q, self.kcache, mul, lut, L, self.rope_theta, self.first_few_fp16)
        return mul.transpose(0, 1).contiguous().half()

    def parallel_pack(self, k):
        """Prefill: k [H,128,T] pre-RoPE keys -> slots 0..T-1 (modeling_llama.py:879-975)."""
        assert self.include_sparse
        k = k.float().contiguous()
        T = k.shape[-1]
        self.klen += T
        resc = k.clone()
        self._op("vecquant%dappendvecKsparseParallel")(self.kcache, self.lookup_table, k, resc,
                                                        self.outlier_threshold_lower, self.outlier_threshold_upper)
        vals, idx = self._outlier_rows(k.reshape(-1, T).t().contiguous(), resc.reshape(-1, T).t().contiguous())
        self.outliers[:self.klen] = vals
        self.outlier_indices[:self.klen] = idx


class QuantV(torch.nn.Module):
    """Mirror of the reference's QuantV (modeling_llama.py:978-1385)."""

    def __init__(self, bits=2, hidden_size=4096, num_heads=32, max_position_embeddings=-1, include_sparse=False,
                 sparsity_threshold=0.99, first_few_fp16=0):
        super().__init__()
        self.hidden_size, self.num_heads = hidden_size, num_heads
        self.head_dim = hidden_size // num_heads
        self.bits = bits
        self.lut = None
        self.include_sparse, self.sparsity_threshold = include_sparse, sparsity_threshold
        self.max_len = max_position_embeddings
        self.vlen = 0
        self.vcache = torch.zeros((num_heads, (self.head_dim // 32) * bits, self.max_len), dtype=torch.int).cuda()
        self.lookup_table = torch.zeros((self.max_len, 2 ** bits), dtype=torch.float).cuda()
        self.n_out = 2 * n_outliers_each(hidden_size, sparsity_threshold)
        if include_sparse:
            self.outliers = torch.zeros((self.max_len, self.n_out), dtype=torch.float).cuda()
            self.outlier_indices = torch.zeros((self.max_len, self.n_out), dtype=torch.int).cuda()
        self.first_few_fp16 = first_few_fp16
        self.norm = False

    def reset(self):
        self.vlen = 0
        self.vcache.zero_()
        self.lookup_table.zero_()
        if self.include_sparse:
            self.outliers.zero_()
            self.outlier_indices.zero_()

    def load_lookup_table(self, quantizer, include_sparse=True, sparsity_threshold=0.99, norm=False):
        """Only the sorted centroids are kept (modeling_llama.py:1054-1055); the per-token LUT is built on append."""
        if norm:
            # the reference dequantises 2-bit V through a second per-token table under Q-Norm (modeling_llama.py:1115-1118,
            # 1151, 1235); this mirror does not carry it -- LayerCache(v_norm=...) is the Q-Norm path of this library
            raise NotImplementedError("QuantV mirror: Q-Norm is served by LayerCache(v_norm=(normscale, normoffset))")
        self.lut = torch.as_tensor(np.asarray(quantizer[2][0], dtype=np.float32)).flatten().sort().values.to(self.vcache.device)
        self.include_sparse, self.sparsity_threshold, self.norm = include_sparse, sparsity_threshold, norm

    def _op(self, fmt):
        return getattr(qc, fmt % self.bits)

    def topk_thresholds(self, v):
        """Device version of modeling_llama.py:1803-1820: (upper_vals, upper_idx, lower_vals, lower_idx), k = n_each+1."""
        kk = n_outliers_each(self.hidden_size, self.sparsity_threshold) + 1
        uv, ui = torch.topk(v, kk, dim=-1)
        lv, li = torch.topk(v, kk, dim=-1, largest=False)
        return uv, ui, lv, li

    def forward_fused_sparse(self, score, v, upper_outlier_vals=None, upper_outlier_indices=None,
                             lower_outlier_vals=None, lower_outlier_indices=None):
        """Append the new value vector and return score.V: fp16 [num_heads, B, 128]."""
        score = score.float()
        v = v.flatten().float()
        slot = self.vlen - self.first_few_fp16
        zp_idx = {4: 7, 3: 3, 2: 1}[self.bits]
        if self.include_sparse:
            if upper_outlier_vals is None:
                upper_outlier_vals, upper_outlier_indices, lower_outlier_vals, lower_outlier_indices = self.topk_thresholds(v)
            maxval, minval = upper_outlier_vals[-1], lower_outlier_vals[-1]
            uv, lv = upper_outlier_vals[:-1], lower_outlier_vals[:-1]
            ui, li = upper_outlier_indices[:-1], lower_outlier_indices[:-1]
            offset = (maxval + minval) / 2
            sf = (maxval - minval) / 2
        else:
            maxval, minval = v.max(), v.min()
            offset = (maxval + minval) / 2
            sf = (maxval - minval) / 2
        lut_t = self.lut.float() * sf.float() + offset.float()   # device math (the reference calls .item() three times here)
        self.lookup_table[slot] = lut_t
        score = score.transpose(0, 1).contiguous()
        if self.include_sparse:
            zeropoint = lut_t[zp_idx]
            self._op("vecquant%dappendvecVsparse")(self.vcache, self.lookup_table, v, zeropoint, minval, maxval, slot)
            vals = torch.cat((uv, lv), dim=-1) - zeropoint
            idx = torch.cat((ui, li), dim=-1)
            idx, order = idx.sort()
            self.outliers[slot] = vals[order]
            self.outlier_indices[slot] = idx.int()
        else:
            self._op("vecquant%dappendvecV")(self.vcache, self.lookup_table, v, slot)
        self.vlen += 1
        L = self.vlen - self.first_few_fp16
        mul = torch.zeros((score.shape[0], score.shape[1], self.head_dim), dtype=torch.float, device=score.device)
        if self.include_sparse:
            self._op("vecquant%dmatmul_nuq_perchannel_transposed_mha_batched_fused_opt2")(
                score, self.vcache, mul, self.lookup_table, L, self.outliers, self.outlier_indices)
        else:
            self._op("vecquant%dmatmul_nuq_perchannel_transposed_mha_batched_fused_opt")(
                score, self.vcache, mul, self.lookup_table, L)
        return mul.transpose(0, 1).contiguous().half()

    def parallel_pack(self, v, upper_outlier_vals, upper_outlier_indices, lower_outlier_vals, lower_outlier_indices):
        """Prefill: v [H,128,T]; top-k tensors [T, n_each+1] (modeling_llama.py:1294-1385)."""
        assert self.include_sparse
        v = v.float().contiguous()
        T = v.shape[-1]
        zp_idx = {4: 7, 3: 3, 2: 1}[self.bits]
        maxval, minval = upper_outlier_vals[:, -1], lower_outlier_vals[:, -1]
        offset = ((maxval + minval) / 2)[:, None]
        sf = ((maxval - minval) / 2)[:, None]
        lut = self.lut.float()[None, :] * sf + offset
        self.lookup_table[self.vlen:self.vlen + T] = lut
        self._op("vecquant%dappendvecVsparseParallel")(self.vcache, self.lookup_table, v, minval.contiguous(),
                                                        maxval.contiguous())
        vals = torch.cat((upper_outlier_vals[:, :-1], lower_outlier_vals[:, :-1]), dim=-1) - lut[:, zp_idx:zp_idx + 1]
        idx = torch.cat((upper_outlier_indices[:, :-1], lower_outlier_indices[:, :-1]), dim=-1)
        idx, order = idx.sort(dim=-1)
        self.outliers[self.vlen:self.vlen + T] = torch.gather(vals, 1, order)
        self.outlier_indices[self.vlen:self.vlen + T] = idx.int()
        self.vlen += T


def attention_decode_reference_chain(kcache: QuantK, vcache: QuantV, q, k, v, head_dim=HEAD_DIM):
    """The reference's decode attention chain around the two managers (modeling_llama.py:1963-1999, no sinks):
    scores.half()/sqrt(d) -> fp32 softmax -> .half() -> V."""
    s = kcache.forward_fused_sparse(q, k)               # [H,1,L] fp16
    s = s.unsqueeze(0) / math.sqrt(head_dim)
    p = torch.nn.functional.softmax(s, dim=-1, dtype=torch.float32).to(torch.float16).squeeze(0)
    return vcache.forward_fused_sparse(p, v)            # [H,1,128] fp16
