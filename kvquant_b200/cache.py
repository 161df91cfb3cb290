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

import ctypes
import math

import numpy as np
import torch

from . import _lib
from . import quant_cuda as qc
from .rope import LengthDependentRotary, RotarySpec, resolve as _resolve_rope

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


def _rope_call(device, rope):
    """(entry point suffix, rotary arguments) of a fused attend over tables for `rope` (a float theta, a scaled
    RotarySpec or a prepared RopeLenState): the theta entry points take theta, their *_freq siblings the device
    frequency vector and the attention factor in its place, and the batched *_freq_seq ones a vector and a table per
    sequence (a RopeLenState of several sequences)."""
    if isinstance(rope, RopeLenState):
        return "_freq_seq" if rope.B > 1 else "_freq", (rope.f_cur.data_ptr(), float(rope.spec.attention_factor))
    if isinstance(rope, RotarySpec):
        return "_freq", (qc.rope_freq(device, rope).data_ptr(), float(rope.attention_factor))
    return "", (float(rope),)


class RopeLenState:
    """The device rotation state of B sequences under a LengthDependentRotary (kvq_rope_len_update, DESIGN.md section
    4.14): the current frequencies f_cur f32 [B, 64], a table float2 [B, 64, npos] in the rope table layout, and a key
    per sequence saying which frequencies its table holds.  update() prepares it for a call's s; the attend, dequantise
    and chunk-attend methods take a prepared state as `rope=` and use it as is, so the layers of a decode step share
    one state and prepare it once.  Its contents are a function of s alone: a sequence retired, refilled or forked
    needs no reset."""

    def __init__(self, spec, B, npos, device):
        if not isinstance(spec, LengthDependentRotary):
            raise TypeError("RopeLenState needs a LengthDependentRotary, got %r" % (type(spec).__name__,))
        self.spec, self.B, self.device = spec, int(B), torch.device(device)
        self.npos = (max(int(npos), 256) + 255) // 256 * 256
        self.lib = _lib.load()
        lo, hi = spec.base_vectors()
        self.f_lo = lo.to(self.device)
        self.f_hi = hi.to(self.device) if hi is not None else None
        self.mode, params, self.m_pos = spec.device_params()
        self._params = np.asarray(params, dtype=np.float64)      # read on the host by the call
        self.f_cur = torch.empty((self.B, HEAD_DIM // 2), dtype=torch.float32, device=self.device)
        self.state = torch.full((self.B, 2), -1, dtype=torch.int64, device=self.device)
        self.table = torch.empty((self.B, HEAD_DIM // 2, self.npos, 2), dtype=torch.float32, device=self.device)

    def fits(self, spec, B, npos):
        return self.spec == spec and self.B == B and self.npos >= npos

    def update(self, s=None, len_dev=None, len_add=0, L_cap=0, pos_offset=0):
        """Prepare for one call: s (one sequence), or per sequence pos_offset + min(max(len_dev[b] + len_add, 0),
        L_cap).  Two launches on the current stream, no allocation: can be captured."""
        _lib.check(self.lib.kvq_rope_len_update(
            self.mode, self._params.ctypes.data, self.m_pos, self.f_lo.data_ptr(),
            self.f_hi.data_ptr() if self.f_hi is not None else None, float(self.spec.attention_factor),
            int(s) if s is not None else 0, len_dev.data_ptr() if len_dev is not None else None, int(len_add),
            int(L_cap), int(pos_offset), self.B, self.f_cur.data_ptr(), self.state.data_ptr(), self.table.data_ptr(),
            self.npos, torch.cuda.current_stream().cuda_stream), "kvq_rope_len_update")
        return self

    def slot(self, b):
        """Sequence b's state as a one-sequence state over the same memory."""
        v = RopeLenState.__new__(RopeLenState)
        v.__dict__.update(self.__dict__)
        v.B = 1
        v.f_cur, v.state, v.table = self.f_cur[b:b + 1], self.state[b:b + 1], self.table[b:b + 1]
        return v


def _resolve(rope, rope_theta):
    """rope.resolve, with a prepared RopeLenState passed through as it is."""
    return rope if isinstance(rope, RopeLenState) else _resolve_rope(rope, rope_theta)


def _len_refusals(cache, spec):
    """What a length-dependent rotation cannot serve (DESIGN.md section 4.14)."""
    if cache.n_sink:
        raise NotImplementedError("attention sinks with length-dependent rotary frequencies: the sink keys are stored "
                                  "post-RoPE in fp16 and cannot be rotated again at another length's frequencies")
    if getattr(cache, "precision", "fp32") == "fp16":
        raise NotImplementedError("length-dependent rotary frequencies use the exact fp32 tables (precision='fp32')")


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
    """Native quantised K+V cache of one layer (reference-compatible tensor layouts, see DESIGN.md section 3).

    Grouped-query attention: `num_heads` is the number of KV heads the cache stores (H); `q_heads` (default H) the
    number of query heads that attend over it, q_heads = g * H, query head h reading KV head h // g (HF repeat_kv).
    Everything that writes or reads the cache itself (append, append_chunk, dequantize, the outlier budget from the
    KV hidden size, sinks [H, ...]) is that of an H-head cache; attend / attend_dyn take q [q_heads, 128] and the chunk
    attends q [T, q_heads, 128].  With q_heads > H: exact tables and the native V form only (DESIGN.md section 4.9)."""

    def __init__(self, bits, num_heads, max_len, klut, klut_sub, thr_lower, thr_upper, v_cent, device,
                 include_sparse=True, sparsity_threshold=0.99, n_sink=0, v_norm=None, sparse_v=None, q_heads=None,
                 storage=None):
        """storage (optional): a mapping with the cache tensors to wrap instead of allocating them -- kcache, vcache,
        vlut, vaff and (for each sparse side) k_outliers / k_outlier_idx, v_outliers / v_outlier_idx, in the shapes
        this constructor would allocate (a sequence slice of a BatchedLayerCache)."""
        self.lib = _lib.load()
        self.bits, self.H, self.Lmax = int(bits), int(num_heads), int(max_len)
        if self.Lmax % 4:
            raise ValueError("max_len must be a multiple of 4 (TMA row pitch)")
        self.Hq = self.H if q_heads is None else int(q_heads)
        if self.Hq != self.H and (self.H <= 0 or (self.H % 4 and self.H > 2) or self.Hq % 4 or self.Hq > 64
                                  or self.Hq % self.H):
            raise ValueError("grouped-query attention needs q_heads <= 64, q_heads %% 4 == 0, KV heads %% 4 == 0 or "
                             "KV heads in {1, 2}, and q_heads a multiple of the KV heads; got q_heads=%d, KV heads=%d"
                             % (self.Hq, self.H))
        self.group = self.Hq // self.H       # query heads per KV head (1: one KV head per query head)
        self.hidden = self.H * HEAD_DIM
        self.q_hidden = self.Hq * HEAD_DIM
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
        st = storage or {}
        if storage:
            want = {"kcache": ((self.H, W, self.Lmax), torch.int32), "vcache": ((self.H, W, self.Lmax), torch.int32),
                    "vlut": ((self.Lmax, 2 ** bits), torch.float32), "vaff": ((self.Lmax, 2), torch.float32)}
            n_out = 2 * n_outliers_each(self.hidden, sparsity_threshold)
            for side, on in (("k", self.sparse_k), ("v", self.sparse_v)):
                if on:
                    want[side + "_outliers"] = ((self.Lmax, n_out), torch.float32)
                    want[side + "_outlier_idx"] = ((self.Lmax, n_out), torch.int32)
            for name, (shape, dtype) in want.items():
                t = st.get(name)
                if (not isinstance(t, torch.Tensor) or tuple(t.shape) != shape or t.dtype != dtype
                        or t.device != dev or not t.is_contiguous()):
                    raise ValueError("storage[%r] must be a contiguous %s tensor of shape %s on %s" % (name, dtype, shape, dev))
        self.kcache = st["kcache"] if storage else torch.zeros((self.H, W, self.Lmax), dtype=torch.int32, device=dev)
        self.vcache = st["vcache"] if storage else torch.zeros((self.H, W, self.Lmax), dtype=torch.int32, device=dev)
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
        self.vlut = st["vlut"] if storage else torch.zeros((self.Lmax, 2 ** bits), dtype=torch.float32, device=dev)
        # per-token affine map (sf_t, off_t): LUT_t = v_cent*sf_t + off_t  -- what the native V kernel consumes
        self.vaff = st["vaff"] if storage else torch.zeros((self.Lmax, 2), dtype=torch.float32, device=dev)
        self.use_native_v = True
        def rows(on, which):   # a dense-only cache allocates no outlier rows (1M-token configs: 2 x 0.4 GB per layer saved)
            if storage and on:
                return st[which + "_outliers"], st[which + "_outlier_idx"]
            n = self.Lmax if on else 1
            return (torch.zeros((n, self.n_out), dtype=torch.float32, device=dev),
                    torch.zeros((n, self.n_out), dtype=torch.int32, device=dev))
        self.k_outliers, self.k_outlier_idx = rows(self.sparse_k, "k")
        self.v_outliers, self.v_outlier_idx = rows(self.sparse_v, "v")
        self.len = 0          # tokens in the quantised cache
        self.n_sink = int(n_sink)
        self.pos_base = 0     # absolute position of slot 0 minus n_sink (non-zero for a sequence shard)
        self.sink_k = self.sink_v = None
        self._scratch = None
        self._retired = []   # superseded scratch buffers (a captured graph may still point at them)
        self._out = torch.empty((self.Hq, HEAD_DIM), dtype=torch.float32, device=dev)
        # RopeLenState under a LengthDependentRotary: created on first use, or set to share one (DecoderStage)
        self.rope_len_state = None
        # lookup-table precision of the K side of the fused attend:
        #   "fp32" (default) exact: the one-wavefront "ratio" tables of kvq_kratio.cu, equal to the legacy op chain to ~1e-6;
        #   "fp16"           north_star's fp16 LUT (kvq_kfast.cu): ~20 % faster K kernel, output within 1e-3 of the exact
        #                    result at test sizes and 1.4e-3 .. 2e-3 at 128K tokens (measured; DESIGN.md section 5).
        # KVQ_FP16_TABLES=1 makes fp16 the default.
        import os
        self.precision = "fp16" if os.environ.get("KVQ_FP16_TABLES", "0") not in ("", "0") else "fp32"

    @classmethod
    def from_luts(cls, bits, num_heads, max_len, klut, v_cent, device="cuda", include_sparse=True,
                  sparsity_threshold=0.99, n_sink=0, v_norm=None, sparse_v=None, q_heads=None):
        """klut: mapping with 'lut' [hidden, n] (and optional 'lut2'), 'thr_lower', 'thr_upper' (numpy or torch);
        hidden = num_heads * 128 is the KV hidden size.  q_heads: query heads (grouped-query attention), default
        num_heads."""
        def t(x):
            return torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).to(device).float().contiguous()
        lut = t(klut["lut"]).view(num_heads * HEAD_DIM, -1)
        lut2 = t(klut["lut2"]).view(num_heads * HEAD_DIM, -1) if klut.get("lut2") is not None else None
        return cls(bits, num_heads, max_len, lut, lut2, t(klut["thr_lower"]), t(klut["thr_upper"]),
                   t(np.sort(np.asarray(v_cent.cpu() if torch.is_tensor(v_cent) else v_cent).ravel())), device,
                   include_sparse, sparsity_threshold, n_sink, v_norm, sparse_v, q_heads)

    def _gqa_check(self):
        """The grouped-query readers cover the exact tables and the native V form only."""
        if self.precision == "fp16":
            raise NotImplementedError("grouped-query attention uses the exact fp32 K tables (precision='fp32')")
        if not self.use_native_v:
            raise NotImplementedError("grouped-query attention reads the native V form (use_native_v=True)")

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

    def _len_rope(self, rope, **where):
        """A float theta / RotarySpec as is; a LengthDependentRotary becomes this cache's RopeLenState prepared at
        `where` (RopeLenState.update's arguments); a RopeLenState is used as the caller prepared it."""
        if isinstance(rope, RopeLenState):
            _len_refusals(self, rope.spec)
            return rope
        if not isinstance(rope, LengthDependentRotary):
            return rope
        _len_refusals(self, rope)
        npos = self.Lmax + self.n_sink + self.pos_base + 1
        st = self.rope_len_state
        if st is None or not st.fits(rope, 1, npos):
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("the rotation state must be allocated before graph capture")
            st = self.rope_len_state = RopeLenState(rope, 1, npos, self.device)
        return st.update(**where)

    @staticmethod
    def _table(rope):
        """(f32 table [64, npos, 2], npos) of a prepared one-sequence RopeLenState."""
        return rope.table[0], rope.npos

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
    def attend(self, q, rope_theta=10000.0, out=None, lse=None, rope=None):
        """softmax(q.K^T/sqrt(128)).V over sinks + quantised slots.  q: f32 [H,128] already rotated at its own
        position.  Returns f32 [H,128].  lse (optional f32 [H]) receives the log-sum-exp of the scaled scores, which
        lets partial results over disjoint token ranges be merged exactly (sequence-sharded decode).
        Grouped-query cache: q, out f32 [q_heads, 128], lse [q_heads] (kvq_attend_gqa).
        rope (optional RotarySpec): the keys' rotary frequencies in place of rope_theta (scaled RoPE: the
        kvq_attend_gqa_freq entry points); q must be rotated with the same spec."""
        if self.group > 1:
            self._gqa_check()
        elif self.v_norm is not None and not self.use_native_v:
            # the per-token LUT rows hold the un-normed centroids while the outlier residuals were taken against the
            # Q-Norm table: the legacy-LUT V kernel would mix the two
            raise NotImplementedError("V Q-Norm needs the native V form (use_native_v=True)")
        rope_theta = self._len_rope(_resolve(rope, rope_theta), s=self.n_sink + self.pos_base + self.len)
        return self._attend(q, None, 0, rope_theta, out, lse, self.len)

    def _attend(self, q, len_dev, len_add, rope_theta, out, lse, L):
        """attend over L slots (len_dev None: kvq_attend_gqa) or attend_dyn with the cap L (kvq_attend_gqa_dyn).  With
        one KV head per query head the C entry points are kvq_attend / kvq_attend_dyn themselves."""
        native, mha = self.use_native_v, self.group == 1
        self._ensure_scratch(self.lib.kvq_attend_scratch_bytes(self.Hq, max(L, 1)), 1.25 if len_dev is None else 1.0)
        pos_offset = self.n_sink + self.pos_base
        if isinstance(rope_theta, RopeLenState):
            (rope, npos), rope_h = self._table(rope_theta), None
        else:
            rope, rope_h, npos = qc.rope_tables(self.device, rope_theta, L + pos_offset + 1)
        fast = self.precision == "fp16" and native and mha
        out = self._out if out is None else out
        ns = self.n_sink if self.sink_k is not None else 0
        head = (self.bits, self._vec(q, self.q_hidden, "q"), self.kcache.data_ptr(), self.klut_deq.data_ptr(),
                *self._out_ptrs("k"), self.vcache.data_ptr())
        vpart = (self.v_cent_deq.data_ptr() if native else None, self.vaff.data_ptr() if native else None,
                 *self._out_ptrs("v"), self.n_out, self.Hq, self.H, self.Lmax, L)
        sfx, rargs = _rope_call(self.device, rope_theta)
        tail = (rope.data_ptr(), npos, *rargs, pos_offset, self.sink_k.data_ptr() if ns else None,
                self.sink_v.data_ptr() if ns else None, ns, self._vec(out, self.q_hidden, "out"),
                self._vec(lse, self.Hq, "lse") if lse is not None else None, self._scratch.data_ptr(),
                rope_h.data_ptr() if fast else None, torch.cuda.current_stream().cuda_stream)
        if len_dev is None:
            vlut = self.vlut.data_ptr() if mha else None
            _lib.check(getattr(self.lib, "kvq_attend_gqa" + sfx)(*head, vlut, *vpart, *tail), "kvq_attend_gqa" + sfx)
        else:
            _lib.check(getattr(self.lib, "kvq_attend_gqa_dyn" + sfx)(
                *head, *vpart, self._vec(len_dev, 1, "len_dev", torch.int64), int(len_add), *tail),
                "kvq_attend_gqa_dyn" + sfx)
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
    def attend_dyn(self, q, len_dev, len_add=0, rope_theta=10000.0, out=None, lse=None, L_cap=None, rope=None):
        """attend() over `min(len_dev[0] + len_add, L_cap)` slots, the length read on the device; grids, scratch and
        the rope table are sized for L_cap (default: the whole allocation).  rope: as attend()."""
        if self.group > 1:
            self._gqa_check()
        elif not self.use_native_v:
            raise NotImplementedError("device-resident length needs the native V form")
        L_cap = self.Lmax if L_cap is None else int(L_cap)
        rope_theta = self._len_rope(_resolve(rope, rope_theta), len_dev=self._check_len_dev(len_dev),
                                    len_add=len_add, L_cap=L_cap, pos_offset=self.n_sink + self.pos_base)
        return self._attend(q, len_dev, len_add, rope_theta, out, lse, L_cap)

    def _check_len_dev(self, len_dev):
        self._vec(len_dev, 1, "len_dev", torch.int64)
        return len_dev

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
    def dequantize(self, start=0, stop=None, rope_theta=None, out_k=None, out_v=None, rope=None):
        """Slots [start, stop) of the cache as fp16 K and V, each [H, stop-start, 128] (one device pass, kvq_dequant_kv).

        K is the dequantised value (dequantisation table plus outlier residual); with rope_theta=None it is pre-RoPE,
        otherwise rotated at the absolute positions n_sink + pos_base + t -- the positions attend() uses -- so that
        q . k[t] for a query rotated at its own position is the score attend() computes for slot t.  V is
        v_cent[code]*sf_t + off_t plus its outlier residual.  out_k / out_v may be views into larger [H, S, 128]
        buffers (stride (S*128, 128, 1)), each with its own S; an output not given is allocated.  An empty range
        returns empty outputs.  With both outputs given, and a rope table that already covers the range, the call
        allocates nothing and can be captured in a CUDA graph.  rope (optional RotarySpec): rotate K with the spec's
        table (scaled RoPE) in place of rope_theta's."""
        def call(start, stop, ok, ov, stride, rope, npos, pos_offset):
            _lib.check(self.lib.kvq_dequant_kv(
                self.bits, self.H, self.Lmax, start, stop,
                self.kcache.data_ptr(), self.klut_deq.data_ptr(), *self._out_ptrs("k"),
                self.vcache.data_ptr(), self.v_cent_deq.data_ptr(), self.vaff.data_ptr(), *self._out_ptrs("v"),
                self.n_out, rope.data_ptr() if rope is not None else None, npos, pos_offset,
                ok, ov, stride, torch.cuda.current_stream().cuda_stream), "kvq_dequant_kv")
        rope_theta = _resolve(rope, rope_theta)
        if isinstance(rope_theta, (LengthDependentRotary, RopeLenState)) and (stop if stop is not None else self.len) > start:
            rope_theta = self._len_rope(rope_theta, s=self.n_sink + self.pos_base + self.len)
        return self._dequantize(start, stop, self.len, self.pos_base, rope_theta, out_k, out_v, call)

    def _dequantize(self, start, stop, n_cached, pos_base, rope_theta, out_k, out_v, call):
        """The body of dequantize for a cache of this one's shape holding n_cached tokens (this cache, or a slot of a
        PagedLayerCache): the range and output checks, the outputs, the rope table, then call(start, stop, out_k ptr,
        out_v ptr, head stride, rope, npos, pos_offset) -- the C entry point -- once per distinct head stride."""
        if not self.use_native_v:
            raise NotImplementedError("dequantize reads the native V form (use_native_v=True)")
        stop = n_cached if stop is None else int(stop)
        start = int(start)
        if not 0 <= start <= stop:
            raise ValueError("need 0 <= start <= stop, got start=%d stop=%d" % (start, stop))
        if stop > n_cached:
            raise ValueError("stop=%d is past the %d cached tokens" % (stop, n_cached))
        n = stop - start
        if out_k is None:
            out_k = torch.empty((self.H, n, HEAD_DIM), dtype=torch.float16, device=self.device)
        if out_v is None:
            out_v = torch.empty((self.H, n, HEAD_DIM), dtype=torch.float16, device=self.device)
        sk, sv = self._kv_out(out_k, n, "out_k"), self._kv_out(out_v, n, "out_v")
        if n == 0:
            return out_k, out_v
        pos_offset = self.n_sink + pos_base
        rope, npos = None, 0
        if isinstance(rope_theta, RopeLenState):
            rope, npos = self._table(rope_theta)
        elif rope_theta is not None:
            rope, _, npos = qc.rope_tables(self.device, rope_theta, stop + pos_offset)

        def run(ok, ov, stride):
            call(start, stop, ok, ov, stride, rope, npos, pos_offset)
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
        if q.dim() != 3 or q.shape[1:] != (self.Hq, HEAD_DIM) or q.shape[0] < 1:
            raise ValueError("q must be [T, %d, %d] with T >= 1, got %s" % (self.Hq, HEAD_DIM, tuple(q.shape)))
        T = q.shape[0]
        for t, name, n in ((q, "q", self.q_hidden), (k, "k", self.hidden), (v, "v", self.hidden)):
            self._vec(t, T * n, name)
        if tuple(k.shape) != (T, self.hidden) or tuple(v.shape) != (T, self.hidden):
            raise ValueError("k and v must be [%d, %d]" % (T, self.hidden))
        return T

    def _chunk_kv16(self, k, v, rope_theta, p0, out_k, out_v, npos=None):
        """The chunk's keys rotated at positions p0 + i and its values, written as fp16 into out_k / out_v [H, T, 128]
        (views allowed): the chunk operands both chunk attentions use.  Returns the f32 rope table, covering
        p0 + T positions.  p0 may instead be an int64 device tensor [T] of per-row positions, all below npos (the rows
        of several slots' chunks, _BatchCommon.attend_chunks); row i is then rotated at p0[i], with the same values."""
        T = k.shape[0]
        rows = isinstance(p0, torch.Tensor)
        if isinstance(rope_theta, RopeLenState):
            rope, _ = self._table(rope_theta)
        else:
            rope, _, _ = qc.rope_tables(self.device, rope_theta, npos if rows else p0 + T)
        tab = rope[:, p0] if rows else rope[:, p0:p0 + T]                                          # [64, T, 2]
        cos, sin = tab[..., 0].t()[:, None, :], tab[..., 1].t()[:, None, :]                         # [T, 1, 64]
        kc = k.view(T, self.H, HEAD_DIM)
        lo, hi = kc[..., :HEAD_DIM // 2], kc[..., HEAD_DIM // 2:]
        out_k[:, :, :HEAD_DIM // 2] = (cos * lo - sin * hi).transpose(0, 1)
        out_k[:, :, HEAD_DIM // 2:] = (cos * hi + sin * lo).transpose(0, 1)
        out_v[:] = v.view(T, self.H, HEAD_DIM).transpose(0, 1)
        return rope

    @_on_cache_device
    def attend_chunk(self, q, k, v, rope_theta=10000.0, rope=None):
        """Causal attention of a T-token chunk placed right after the cached tokens (a follow-up prompt).

        q: f32 [T, q_heads, 128], token i already rotated at position P0 + i, P0 = n_sink + pos_base + len.
        k: f32 [T, hidden] pre-RoPE keys and v: f32 [T, hidden] values of the chunk, as append() takes them.
        Chunk token i attends over the fp16 sinks (when set), all `len` quantised slots (dequantised and rotated) and
        chunk tokens 0..i; the chunk's keys are rotated with the same table, and its keys and values rounded to fp16,
        as a prefill runs attention on the prompt's fp16 K/V.  Scale 1/sqrt(128).  Returns f32 [T, H, 128].

        The cache is NOT modified: append the chunk's tokens afterwards with append_chunk(k, v) (one launch, as
        DecoderStage.prefill does).  The call materialises K and V for every
        position, 2*H*(n_sink + len + T)*128 fp16 values (2 GiB for 32 heads at 128K tokens), and hands them to
        torch.nn.functional.scaled_dot_product_attention.  attend_chunk_fused computes the same attention without
        materialising the cache.  A grouped-query cache hands the same H-head buffers to SDPA with enable_gqa=True
        (nothing is repeated in memory).  rope (optional RotarySpec): the cached and the chunk's keys are rotated with
        the spec's table in place of rope_theta's; q must be rotated with the same spec."""
        if self.group > 1:
            self._gqa_check()
        T = self._chunk_check(q, k, v)
        rope_theta = self._len_rope(_resolve(rope, rope_theta), s=self.n_sink + self.pos_base + self.len + T)
        sinks = (self.sink_k, self.sink_v) if self.sink_k is not None else None
        return self._attend_chunk_sdpa(q, k, v, rope_theta, self.len, self.pos_base, sinks,
                                       lambda ok, ov: self.dequantize(0, self.len, rope_theta, out_k=ok, out_v=ov))

    def _attend_chunk_sdpa(self, q, k, v, rope_theta, L, pos_base, sinks, dequant):
        """The body of attend_chunk for a cache of this one's shape holding L tokens (this cache, or a slot of a
        PagedLayerCache), arguments checked: one fp16 [1, H, S, 128] K and one V buffer of the sinks ((sink_k, sink_v)
        or None), the L cached slots -- dequant(out_k, out_v) writes them, K rotated, into two [H, L, 128] views -- and
        the chunk, then SDPA with the causal-offset mask.  Slot t sits at position n_sink + pos_base + t."""
        T = q.shape[0]
        ns = self.n_sink if sinks is not None else 0
        S = ns + L + T
        p0 = self.n_sink + pos_base + L
        kbuf = torch.empty((1, self.H, S, HEAD_DIM), dtype=torch.float16, device=self.device)
        vbuf = torch.empty_like(kbuf)
        if ns:
            kbuf[0, :, :ns] = sinks[0].transpose(1, 2)
            vbuf[0, :, :ns] = sinks[1]
        if L:
            dequant(kbuf[0, :, ns:ns + L], vbuf[0, :, ns:ns + L])
        self._chunk_kv16(k, v, rope_theta, p0, kbuf[0, :, ns + L:], vbuf[0, :, ns + L:])
        mask = torch.arange(S, device=self.device)[None, :] <= (ns + L + torch.arange(T, device=self.device))[:, None]
        gqa = dict(enable_gqa=True) if self.group > 1 else {}
        out = torch.nn.functional.scaled_dot_product_attention(
            q.transpose(0, 1)[None].half(), kbuf, vbuf, attn_mask=mask, scale=1.0 / math.sqrt(HEAD_DIM), **gqa)
        return out[0].transpose(0, 1).float().contiguous()

    @_on_cache_device
    def attend_chunk_fused(self, q, k, v, rope_theta=10000.0, rope=None):
        """attend_chunk() read straight from the quantised cache (kvq_attend_chunk): same arguments, checks, result
        (f32 [T, H, 128]) and semantics, and the cache is likewise left untouched.

        One tensor-core kernel dequantises each K/V tile of the cached slots into shared memory -- the same fp16
        values dequantize() writes -- and attends the chunk over it, FlashAttention-2 style.  Extra device memory per
        call is the chunk's fp16 rotated K and V (2*H*T*128*2 bytes) plus kvq_attend_chunk_scratch_bytes(H, T, len),
        whatever `len` is: at 1M cached tokens the materialising attend_chunk would need 2*H*1M*128*2 bytes more.
        A grouped-query cache calls kvq_attend_chunk_gqa (query head h reads KV head h // group).  rope: as
        attend_chunk()."""
        if self.group > 1:
            self._gqa_check()
        if not self.use_native_v:
            raise NotImplementedError("attend_chunk_fused reads the native V form (use_native_v=True)")
        T = self._chunk_check(q, k, v)
        rope_theta = self._len_rope(_resolve(rope, rope_theta), s=self.n_sink + self.pos_base + self.len + T)
        L = self.len
        ns = self.n_sink if self.sink_k is not None else 0
        pos_offset = self.n_sink + self.pos_base
        kc = torch.empty((self.H, T, HEAD_DIM), dtype=torch.float16, device=self.device)
        vc = torch.empty_like(kc)
        rope = self._chunk_kv16(k, v, rope_theta, pos_offset + L, kc, vc)
        scratch = torch.empty(max(self.lib.kvq_attend_chunk_scratch_bytes(self.Hq, T, L), 16), dtype=torch.uint8,
                              device=self.device)
        out = torch.empty((T, self.Hq, HEAD_DIM), dtype=torch.float32, device=self.device)
        fn, heads, name = ((self.lib.kvq_attend_chunk_gqa, (self.Hq, self.H), "kvq_attend_chunk_gqa") if self.group > 1
                           else (self.lib.kvq_attend_chunk, (self.H,), "kvq_attend_chunk"))
        _lib.check(fn(
            self.bits, *heads, self.Lmax, L, T, q.data_ptr(), kc.data_ptr(), vc.data_ptr(),
            self.kcache.data_ptr(), self.klut_deq.data_ptr(), *self._out_ptrs("k"),
            self.vcache.data_ptr(), self.v_cent_deq.data_ptr(), self.vaff.data_ptr(), *self._out_ptrs("v"),
            self.n_out, rope.data_ptr(), rope.shape[1], pos_offset,
            self.sink_k.data_ptr() if ns else None, self.sink_v.data_ptr() if ns else None, ns,
            out.data_ptr(), scratch.data_ptr(), torch.cuda.current_stream().cuda_stream), name)
        return out

    def bytes_per_token(self):
        """Algorithmic HBM bytes one decode step reads per cached token (SURVEY.md 8d formula)."""
        b = 2 * self.H * HEAD_DIM * self.bits // 8 + 4 * 2 ** self.bits
        b += (int(self.sparse_k) + int(self.sparse_v)) * self.n_out * 8
        return b


class _BatchCommon:
    """What the contiguous and the paged batched caches share: the calibration of a template LayerCache, the caller
    tensor checks, sinks, the device-length advance, scratch sizing and the append / attend calls, which differ only
    in the cache extent argument (Lmax or n_pool) and the page-table arguments appended to the paged entry points."""

    def _init_common(self, B, dev, c, lens):
        self.B, self.device = B, dev
        self.lib = c.lib
        self._tmpl = c
        self.bits, self.H, self.Hq, self.group = c.bits, c.H, c.Hq, c.group
        self.hidden, self.q_hidden, self.n_each, self.n_out, self.n_sink = c.hidden, c.q_hidden, c.n_each, c.n_out, c.n_sink
        self.sparse_k, self.sparse_v = c.sparse_k, c.sparse_v
        if lens is not None and (not isinstance(lens, torch.Tensor) or lens.dtype != torch.int64
                                 or tuple(lens.shape) != (B,) or lens.device != dev):
            raise ValueError("lens must be an int64 tensor of shape (%d,) on %s" % (B, dev))
        self.sink_k = self.sink_v = None
        self._scratch = None
        self._retired = []
        self._out = torch.empty((B, self.Hq, HEAD_DIM), dtype=torch.float32, device=dev)
        # RopeLenState of the B slots under a LengthDependentRotary: created on first use, or set to share one
        # (BatchedDecoderStage)
        self.rope_len_state = None

    def _len_state(self, spec):
        """The slots' RopeLenState for `spec` (allocated outside a capture; a sequence view of a contiguous batch
        then rotates with its slot of it)."""
        _len_refusals(self._tmpl, spec)
        st = self.rope_len_state
        if st is None or not st.fits(spec, self.B, self.Lmax + self.n_sink + 1):
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("the rotation state must be allocated before graph capture")
            st = self.rope_len_state = RopeLenState(spec, self.B, self.Lmax + self.n_sink + 1, self.device)
            for b, v in enumerate(getattr(self, "_views", ())):
                v.rope_len_state = st.slot(b)
        return st

    def _len_slot(self, b, rope, s):
        """Slot b's one-sequence state prepared at s, for a LengthDependentRotary; other rotations as they are."""
        if isinstance(rope, LengthDependentRotary):
            return self._len_state(rope).slot(b).update(s=s)
        return rope

    @staticmethod
    def _check_batch(batch):
        B = int(batch)
        if not 1 <= B <= 256:
            raise ValueError("batch must be in [1, 256], got %d" % B)
        return B

    @staticmethod
    def _device(device):
        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        return dev

    def set_sinks(self, sink_k, sink_v):
        """fp16 sinks of every sequence: sink_k [B, H, 128, n_sink] post-RoPE, sink_v [B, H, n_sink, 128]."""
        shp_k, shp_v = (self.B, self.H, HEAD_DIM, self.n_sink), (self.B, self.H, self.n_sink, HEAD_DIM)
        for t, name, shp in ((sink_k, "sink_k", shp_k), (sink_v, "sink_v", shp_v)):
            if not isinstance(t, torch.Tensor) or t.dtype != torch.float16 or tuple(t.shape) != shp:
                raise ValueError("%s must be a float16 tensor of shape %s" % (name, shp))
            if t.device != self.device:
                raise ValueError("%s is on %s, the cache lives on %s" % (name, t.device, self.device))
        self.sink_k, self.sink_v = sink_k.contiguous(), sink_v.contiguous()

    def _rows(self, t, n, name, dtype=torch.float32):
        """Pointer of a caller [B, n] tensor after the checks the C ABI cannot make."""
        if not isinstance(t, torch.Tensor):
            raise ValueError("%s must be a torch.Tensor" % name)
        if t.dtype != dtype:
            raise ValueError("%s must be %s, got %s" % (name, dtype, t.dtype))
        if t.device != self.device:
            raise ValueError("%s is on %s, the cache lives on %s" % (name, t.device, self.device))
        if not t.is_contiguous() or t.numel() != self.B * n or t.shape[0] != self.B:
            raise ValueError("%s must be a contiguous [%d, ...] tensor of %d elements, got %s"
                             % (name, self.B, self.B * n, tuple(t.shape)))
        return t.data_ptr()

    def _ptrs(self, which):
        o, i = (self.k_outliers, self.k_outlier_idx) if which == "k" else (self.v_outliers, self.v_outlier_idx)
        return (o.data_ptr(), i.data_ptr()) if o is not None else (None, None)

    # the entry points and their extra arguments (overridden by the paged cache)
    _append_fn, _attend_fn = "kvq_append_kv_fused_batch", "kvq_attend_batch"
    _append_chunks_fn, _attend_chunks_fn = "kvq_append_kv_fused_chunk_ragged", "kvq_attend_chunk_ragged"

    def _page_args(self):
        return ()

    @_on_cache_device
    def append_dyn(self, k, v, active=None, slot_add=0):
        """One token per sequence, one launch: k, v f32 [B, hidden]; sequence b writes slot lens[b] + slot_add (a
        full sequence drops its token); active (int32 [B], or None = all) == 0 writes nothing.  Lengths are NOT
        advanced (advance() does that on the device); graph-capturable."""
        c = self._tmpl
        args = (self.bits, self.B, self.H, self._extent, self.lens.data_ptr(), int(slot_add),
                self._rows(active, 1, "active", torch.int32) if active is not None else None, self.n_each,
                self._rows(k, self.hidden, "k"), self.kcache.data_ptr(), c.klut.data_ptr(), c.klut_sub.data_ptr(),
                c.thr_lower.data_ptr(), c.thr_upper.data_ptr(), *self._ptrs("k"),
                self._rows(v, self.hidden, "v"), self.vcache.data_ptr(), c.v_cent.data_ptr(),
                c.v_cent_deq.data_ptr() if c.v_norm is not None else None, self.vlut.data_ptr(), self.vaff.data_ptr(),
                *self._ptrs("v"), torch.cuda.current_stream().cuda_stream) + self._page_args()
        _lib.check(getattr(self.lib, self._append_fn)(*args), self._append_fn)

    @_on_cache_device
    def advance(self, active=None, delta=1):
        """lens[b] += delta on the device for every active sequence (graph-capturable)."""
        _lib.check(self.lib.kvq_dec_counter_add_batch(
            self.lens.data_ptr(), self._rows(active, 1, "active", torch.int32) if active is not None else None,
            int(delta), self.B, torch.cuda.current_stream().cuda_stream), "kvq_dec_counter_add_batch")

    @_on_cache_device
    def attend(self, q, out=None, lse=None, L_cap=None, len_add=0, rope_theta=10000.0, rope=None):
        """Decode attention of every sequence (kvq_attend_batch / kvq_attend_paged): q f32 [B, q_heads, 128], row b
        rotated at its own position; sequence b attends over its sinks and min(lens[b] + len_add, L_cap) slots (L_cap
        default: the per-sequence cap; grids, scratch and the rope table are sized for it).  Returns f32 [B, q_heads,
        128]; lse (optional f32 [B, q_heads]) receives the log-sum-exp.  An idle slot (no slot, no sink) gives 0 and
        -inf.  There is no active mask: with len_add > 0 a sequence that did not append this step attends one slot
        past its length, so its output is meaningless and must be ignored.  rope (optional RotarySpec): the keys'
        rotary frequencies in place of rope_theta (kvq_attend_batch_freq / kvq_attend_paged_freq)."""
        c = self._tmpl
        rope_theta = _resolve(rope, rope_theta)
        if c.precision == "fp16":
            raise NotImplementedError("the batched attend uses the exact fp32 K tables (precision='fp32')")
        L_cap = self.Lmax if L_cap is None else int(L_cap)
        if not 1 <= L_cap <= self.Lmax:
            raise ValueError("L_cap must be in [1, %d], got %d" % (self.Lmax, L_cap))
        if isinstance(rope_theta, LengthDependentRotary):
            rope_theta = self._len_state(rope_theta).update(len_dev=self.lens, len_add=len_add, L_cap=L_cap,
                                                            pos_offset=self.n_sink)
        elif isinstance(rope_theta, RopeLenState):
            _len_refusals(c, rope_theta.spec)
            if rope_theta.B != self.B:
                raise ValueError("a RopeLenState of %d sequences for a batch of %d" % (rope_theta.B, self.B))
        need = self.lib.kvq_attend_batch_scratch_bytes(self.B, self.Hq, L_cap)
        if self._scratch is None or self._scratch.numel() < need:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("attend scratch must be sized before graph capture (run one eager attend with the "
                                   "same L_cap first)")
            if self._scratch is not None:
                self._retired.append(self._scratch)
            self._scratch = torch.empty(need, dtype=torch.uint8, device=self.device)
        pos_offset = self.n_sink
        if isinstance(rope_theta, RopeLenState):   # one table and frequency vector per sequence
            rope, npos = rope_theta.table, rope_theta.npos
        else:
            rope, _, npos = qc.rope_tables(self.device, rope_theta, L_cap + pos_offset + 1)
        out = self._out if out is None else out
        ns = self.n_sink if self.sink_k is not None else 0
        sfx, rargs = _rope_call(self.device, rope_theta)
        args = (self.bits, self.B, self._rows(q, self.q_hidden, "q"), self.kcache.data_ptr(), c.klut_deq.data_ptr(),
                *self._ptrs("k"), self.vcache.data_ptr(), c.v_cent_deq.data_ptr(), self.vaff.data_ptr(), *self._ptrs("v"),
                self.n_out, self.Hq, self.H, self._extent, L_cap, self.lens.data_ptr(), int(len_add), rope.data_ptr(),
                npos, *rargs, pos_offset, self.sink_k.data_ptr() if ns else None,
                self.sink_v.data_ptr() if ns else None, ns, self._rows(out, self.q_hidden, "out"),
                self._rows(lse, self.Hq, "lse") if lse is not None else None, self._scratch.data_ptr(), None,
                torch.cuda.current_stream().cuda_stream) + self._page_args()
        _lib.check(getattr(self.lib, self._attend_fn + sfx)(*args), self._attend_fn + sfx)
        return out

    # -- several slots' chunks in one launch (ragged prefill, DESIGN.md section 4.15) ------------------------------------
    def _segments(self, slots, starts, counts, N):
        """The host segment table int64 [n_seg, 4] of (slot, s0, T, first row) after the checks a caller can fail:
        slots distinct and in range, counts >= 0 summing to N (ValueError), s0 + T within the cap (IndexError)."""
        slots, counts = [int(b) for b in slots], [int(t) for t in counts]
        if len(slots) != len(counts):
            raise ValueError("%d slots but %d counts" % (len(slots), len(counts)))
        if len(set(slots)) != len(slots):
            raise ValueError("slots must be distinct, got %s" % (slots,))
        for b in slots:
            if not 0 <= b < self.B:
                raise IndexError("slot %d out of range [0, %d)" % (b, self.B))
        if any(t < 0 for t in counts) or sum(counts) != N:
            raise ValueError("counts must be >= 0 and sum to the %d rows, got %s" % (N, counts))
        for b, s0, t in zip(slots, starts, counts):
            if s0 + t > self.Lmax:
                raise IndexError("a chunk of %d tokens does not fit slot %d: %d of %d slots used" % (t, b, s0, self.Lmax))
        row0 = np.concatenate(([0], np.cumsum(counts)[:-1])) if counts else np.zeros(0)
        return np.ascontiguousarray(np.stack([np.asarray(slots), np.asarray(starts), np.asarray(counts), row0], axis=1)
                                    .astype(np.int64).reshape(-1, 4))

    def _map_chunks(self, slots, starts, counts):
        """Paged: map the pages the segments' writes need, after checking them all (contiguous: nothing to do)."""

    def _chunks_tail(self, slots):
        """The trailing arguments of the ragged entry points (contiguous: none)."""
        return ()

    @_on_cache_device
    def _append_chunks_at(self, slots, starts, k, v, counts):
        """append_chunks at the given first slots, host lengths untouched."""
        c = self._tmpl
        if k.dim() != 2 or tuple(k.shape) != tuple(v.shape) or k.shape[1] != self.hidden:
            raise ValueError("k and v must both be [N, %d], got %s and %s" % (self.hidden, tuple(k.shape), tuple(v.shape)))
        N = k.shape[0]
        kp, vp = c._vec(k, N * self.hidden, "k"), c._vec(v, N * self.hidden, "v")
        segs = self._segments(slots, starts, counts, N)
        self._map_chunks(segs[:, 0].tolist(), segs[:, 1].tolist(), segs[:, 2].tolist())
        if N == 0:
            return
        tail, fn = self._chunks_tail(segs[:, 0].tolist()), self._append_chunks_fn
        _lib.check(getattr(self.lib, fn)(
            self.bits, self.B, self.H, self._extent, len(segs), segs.ctypes.data, N, self.n_each,
            kp, self.kcache.data_ptr(), c.klut.data_ptr(), c.klut_sub.data_ptr(), c.thr_lower.data_ptr(),
            c.thr_upper.data_ptr(), *self._ptrs("k"), vp, self.vcache.data_ptr(), c.v_cent.data_ptr(),
            c.v_cent_deq.data_ptr() if c.v_norm is not None else None, self.vlut.data_ptr(), self.vaff.data_ptr(),
            *self._ptrs("v"), torch.cuda.current_stream().cuda_stream, *tail), fn)

    def append_chunks(self, slots, k, v, counts):
        """append_chunk of several slots in one launch (kvq_append_kv_fused_chunk_ragged[_paged]): k, v f32 [N, hidden]
        hold counts[i] rows for slots[i], in that order; slot b's rows go to its slots host_len(b) onwards, bit for bit
        as append_chunk of those rows alone.  Slots must be distinct; a count of 0 writes nothing.  Past the cap raises
        IndexError, and (paged) an exhausted pool RuntimeError, before anything is written or reserved for any slot.
        Advances the host lengths; commit(*slots) publishes them to the device."""
        starts = [self._host_len(b) for b in slots]
        self._append_chunks_at(slots, starts, k, v, counts)
        for b, t in zip(slots, counts):
            self._set_host_len(b, self._host_len(b) + int(t))

    @_on_cache_device
    def _attend_chunks_at(self, slots, starts, q, k, v, counts, rope):
        """attend_chunks with the given cached lengths; rope: a resolved rotation (theta or RotarySpec)."""
        c = self._tmpl
        if c.group > 1:
            c._gqa_check()
        if not c.use_native_v:
            raise NotImplementedError("attend_chunks reads the native V form (use_native_v=True)")
        if isinstance(rope, (LengthDependentRotary, RopeLenState)):
            raise NotImplementedError("attend_chunks with length-dependent rotary frequencies: each slot needs its own "
                                      "frequency table; prefill such slots one at a time (prefill_seq)")
        if q.dim() != 3 or q.shape[1:] != (self.Hq, HEAD_DIM):
            raise ValueError("q must be [N, %d, %d], got %s" % (self.Hq, HEAD_DIM, tuple(q.shape)))
        N = q.shape[0]
        for t, name, n in ((q, "q", self.q_hidden), (k, "k", self.hidden), (v, "v", self.hidden)):
            c._vec(t, N * n, name)
        if tuple(k.shape) != (N, self.hidden) or tuple(v.shape) != (N, self.hidden):
            raise ValueError("k and v must be [%d, %d]" % (N, self.hidden))
        segs = self._segments(slots, starts, counts, N)
        out = torch.empty((N, self.Hq, HEAD_DIM), dtype=torch.float32, device=self.device)
        if N == 0:
            return out
        # row j of segment i sits at n_sink + s0_i + j
        pos = np.concatenate([np.arange(s0, s0 + t) for s0, t in zip(segs[:, 1], segs[:, 2])]) + self.n_sink
        kc = torch.empty((self.H, N, HEAD_DIM), dtype=torch.float16, device=self.device)
        vc = torch.empty_like(kc)
        tab = c._chunk_kv16(k, v, rope, torch.from_numpy(pos).to(self.device), kc, vc, npos=int(pos.max()) + 1)
        scratch = torch.empty(max(self.lib.kvq_attend_chunk_ragged_scratch_bytes(self.Hq, len(segs), segs.ctypes.data),
                                  16), dtype=torch.uint8, device=self.device)
        ns = self.n_sink if self.sink_k is not None else 0
        tail, fn = self._chunks_tail(segs[:, 0].tolist()), self._attend_chunks_fn
        _lib.check(getattr(self.lib, fn)(
            self.bits, self.B, self.Hq, self.H, self._extent, len(segs), segs.ctypes.data, N, q.data_ptr(),
            kc.data_ptr(), vc.data_ptr(), self.kcache.data_ptr(), c.klut_deq.data_ptr(), *self._ptrs("k"),
            self.vcache.data_ptr(), c.v_cent_deq.data_ptr(), self.vaff.data_ptr(), *self._ptrs("v"), self.n_out,
            tab.data_ptr(), tab.shape[1], self.n_sink, self.sink_k.data_ptr() if ns else None,
            self.sink_v.data_ptr() if ns else None, ns, out.data_ptr(), scratch.data_ptr(),
            torch.cuda.current_stream().cuda_stream, *tail), fn)
        return out

    def attend_chunks(self, slots, q, k, v, counts, rope_theta=10000.0, rope=None):
        """attend_chunk_fused of several slots in one launch (kvq_attend_chunk_ragged[_paged]): q f32 [N, q_heads, 128]
        and k, v f32 [N, hidden] hold counts[i] rows for slots[i], in that order, row j of slot b's rows rotated at
        n_sink + host_len(b) + j.  Each slot's rows attend over its sinks, its host_len(b) cached tokens and its own rows
        causally, and come out bit for bit as attend_chunk_fused of those rows alone on that slot.  Returns f32
        [N, q_heads, 128]; the cache is not modified.  rope: theta or a static RotarySpec (length-dependent rotary
        raises NotImplementedError), as attend_chunk_fused's."""
        starts = [self._host_len(b) for b in slots]
        return self._attend_chunks_at(slots, starts, q, k, v, counts, _resolve(rope, rope_theta))


class BatchedLayerCache(_BatchCommon):
    """One layer's quantised cache for B sequences (batched decode, DESIGN.md section 4.10).

    The tensors are batch-strided -- kcache / vcache [B, H, W, Lmax], vlut [B, Lmax, 2^bits], vaff [B, Lmax, 2], outlier
    rows [B, Lmax, n_out], sinks [B, ...] -- and sequence b's slice of each has exactly the layout of a LayerCache.
    `seq(b)` is that LayerCache (a view sharing the storage), so every single-sequence operation (append_chunk,
    attend, attend_dyn, dequantize, attend_chunk[_fused]) serves one slot unchanged -- a slot's prompt is prefilled
    through its view.  `append` / `attend` serve all B sequences in one launch (set).  The calibration (K LUTs,
    thresholds, centroids) is shared.

    Lengths: `lens` is the device int64 [B] the batched kernels read (several layers' caches may share one tensor:
    `lens=`); each view's `len` is its host mirror.  After a view's length changed on the host (a prefill of slot b),
    `commit(b)` copies that slot's host length to the device, leaving the other slots' device lengths alone (they may
    have advanced on the device, e.g. in graph replays); after device-side appends, `sync_host()` copies them back."""

    def __init__(self, batch, bits, num_heads, max_len, klut, klut_sub, thr_lower, thr_upper, v_cent, device,
                 include_sparse=True, sparsity_threshold=0.99, n_sink=0, v_norm=None, sparse_v=None, q_heads=None,
                 lens=None):
        B = self._check_batch(batch)
        dev = self._device(device)
        H, Lmax, W = int(num_heads), int(max_len), HEAD_DIM * int(bits) // 32
        n_out = 2 * n_outliers_each(H * HEAD_DIM, sparsity_threshold)
        sk = bool(include_sparse)
        sv = sk if sparse_v is None else (bool(sparse_v) and sk)
        z = lambda shape, dt: torch.zeros((B,) + shape, dtype=dt, device=dev)   # noqa: E731
        self.kcache, self.vcache = z((H, W, Lmax), torch.int32), z((H, W, Lmax), torch.int32)
        self.vlut, self.vaff = z((Lmax, 2 ** int(bits)), torch.float32), z((Lmax, 2), torch.float32)
        self.k_outliers = self.k_outlier_idx = self.v_outliers = self.v_outlier_idx = None
        if sk:
            self.k_outliers, self.k_outlier_idx = z((Lmax, n_out), torch.float32), z((Lmax, n_out), torch.int32)
        if sv:
            self.v_outliers, self.v_outlier_idx = z((Lmax, n_out), torch.float32), z((Lmax, n_out), torch.int32)

        def storage(b):
            st = dict(kcache=self.kcache[b], vcache=self.vcache[b], vlut=self.vlut[b], vaff=self.vaff[b])
            for name in ("k_outliers", "k_outlier_idx", "v_outliers", "v_outlier_idx"):
                if getattr(self, name) is not None:
                    st[name] = getattr(self, name)[b]
            return st
        self._views = [LayerCache(bits, num_heads, max_len, klut, klut_sub, thr_lower, thr_upper, v_cent, dev,
                                  include_sparse, sparsity_threshold, n_sink, v_norm, sparse_v, q_heads,
                                  storage=storage(b)) for b in range(B)]
        self._init_common(B, dev, self._views[0], lens)
        self.Lmax = self._extent = self._views[0].Lmax
        self.lens = torch.zeros(B, dtype=torch.int64, device=dev) if lens is None else lens

    @classmethod
    def from_luts(cls, bits, num_heads, max_len, klut, v_cent, device="cuda", include_sparse=True,
                  sparsity_threshold=0.99, n_sink=0, v_norm=None, sparse_v=None, q_heads=None, batch=1):
        """LayerCache.from_luts with the same options, for `batch` sequences."""
        c = LayerCache.from_luts(bits, num_heads, 4, klut, v_cent, device, False, sparsity_threshold, 0, v_norm,
                                 None, q_heads)   # (tables only: a 4-slot dense cache does the conversions)
        return cls(batch, bits, num_heads, max_len, c.klut, c.klut_sub if c.klut_sub is not c.klut else None,
                   c.thr_lower, c.thr_upper, c.v_cent, c.device, include_sparse, sparsity_threshold, n_sink, v_norm,
                   sparse_v, q_heads)

    def seq(self, b):
        """Sequence b's cache as a LayerCache sharing this batch's storage (its `len` is b's host length)."""
        return self._views[b]

    @property
    def lens_host(self):
        return [v.len for v in self._views]

    def _host_len(self, b):
        return self._views[b].len

    def _set_host_len(self, b, n):
        self._views[b].len = n

    def commit(self, *slots):
        """Copy the host lengths (the views' `len`) of the given slots -- every slot when none is given -- to the
        device lengths.  Slots not named keep their device length."""
        for b in (slots or range(self.B)):
            self.lens[b] = self._views[b].len

    def sync_host(self):
        """Copy the device lengths back to the host mirrors (after device-side appends, e.g. graph replays)."""
        for v, n in zip(self._views, self.lens.tolist()):
            v.len = min(int(n), self.Lmax)

    def reset_seq(self, b):
        """Retire slot b: its length becomes 0 on the host and the device (its tensors are not cleared: nothing past a
        sequence's length is ever read)."""
        self._views[b].len = 0
        self.lens[b] = 0

    def set_sinks(self, sink_k, sink_v):
        """fp16 sinks of every sequence: sink_k [B, H, 128, n_sink] post-RoPE, sink_v [B, H, n_sink, 128]."""
        super().set_sinks(sink_k, sink_v)
        for b, v in enumerate(self._views):
            v.set_sinks(self.sink_k[b], self.sink_v[b])

    def append(self, k, v, active=None):
        """append_dyn + advance, with the host lengths kept in step.  Raises IndexError if an active sequence is full."""
        act = [True] * self.B if active is None else [bool(a) for a in active.tolist()]
        if any(a and n >= self.Lmax for a, n in zip(act, self.lens_host)):
            raise IndexError("cache full")
        self.append_dyn(k, v, active)
        self.advance(active)
        for a, view in zip(act, self._views):
            view.len += int(a)


class _SeqRef(ctypes.Structure):
    """kvq_seq_ref: one side of kvq_page_copy."""
    _fields_ = [("kcache", ctypes.c_void_p), ("vcache", ctypes.c_void_p), ("k_outliers", ctypes.c_void_p),
                ("k_outlier_idx", ctypes.c_void_p), ("v_outliers", ctypes.c_void_p), ("v_outlier_idx", ctypes.c_void_p),
                ("vlut_tok", ctypes.c_void_p), ("v_aff", ctypes.c_void_p), ("Lmax", ctypes.c_int64),
                ("pages", ctypes.c_void_p)]


class PageTable:
    """Page allocator of a paged batch (DESIGN.md section 4.11), one per batch and shared by all its layers' caches.

    It owns the device page table `table` int32 [B, max_pages], the mapped counts `npages` int32 [B], the device
    lengths `lens` int64 [B] with their host mirror `lens_host`, and the host-side free list and reference counts of
    the n_pool page ids: page id p names page p of every layer's pool.  Sequence b's token t lives in page
    table[b][t // P], column t % P.

    Entries are written only here, each checked against n_pool.  A live slot's entries never change -- new ones are
    appended behind them -- so a graph replay in flight never sees a remapped page; the writes are ordered on the
    current stream.  A page shared by several slots (fork) is always full, so no append writes a shared page."""

    def __init__(self, batch, page_size, n_pool, max_pages, device="cuda"):
        self.B = _BatchCommon._check_batch(batch)
        P, n_pool, max_pages = int(page_size), int(n_pool), int(max_pages)
        if P <= 0 or P % 160:
            raise ValueError("page_size must be a positive multiple of 160 (whole K boxes and V tiles), got %d" % P)
        if n_pool < 1:
            raise ValueError("n_pool must be >= 1, got %d" % n_pool)
        if max_pages < 1 or max_pages * P >= 2 ** 30:
            raise ValueError("max_pages must be >= 1 with max_pages * page_size < 2^30, got %d" % max_pages)
        self.P, self.n_pool, self.max_pages = P, n_pool, max_pages
        self.cap = max_pages * P                      # per-sequence token cap
        self.device = _BatchCommon._device(device)
        self.table = torch.zeros((self.B, max_pages), dtype=torch.int32, device=self.device)
        self.npages = torch.zeros(self.B, dtype=torch.int32, device=self.device)
        self.lens = torch.zeros(self.B, dtype=torch.int64, device=self.device)
        self.lens_host = [0] * self.B
        self.refs = [0] * n_pool
        self._free = list(range(n_pool - 1, -1, -1))   # pop() hands out the lowest free id first
        self.pages = [[] for _ in range(self.B)]       # host mirror of each row's mapped entries
        self.caches = []                               # the layer caches over this table (fork copies in each)

    @property
    def n_free(self):
        return len(self._free)

    def _slot(self, b):
        b = int(b)
        if not 0 <= b < self.B:
            raise IndexError("slot %d out of range [0, %d)" % (b, self.B))
        return b

    def _map(self, b, ids):
        """Append page ids to row b (host mirror, then the device row and count, stream-ordered)."""
        if not ids:
            return
        for p in ids:
            if not 0 <= p < self.n_pool:
                raise ValueError("page id %d outside the pool of %d pages" % (p, self.n_pool))
        n0 = len(self.pages[b])
        self.pages[b].extend(ids)
        row = torch.tensor(self.pages[b][n0:], dtype=torch.int32).to(self.device, non_blocking=False)
        self.table[b, n0:len(self.pages[b])].copy_(row)
        self.npages[b] = len(self.pages[b])

    def _take(self, n):
        if n > len(self._free):
            raise RuntimeError("page pool exhausted: %d pages needed, %d of %d free" % (n, len(self._free), self.n_pool))
        ids = [self._free.pop() for _ in range(n)]
        for p in ids:
            self.refs[p] = 1
        return ids

    def reserve(self, b, n_tokens):
        """Map pages so that slot b can hold n_tokens tokens (nothing when it already can).  Raises IndexError past
        the per-sequence cap and RuntimeError when the pool is exhausted -- both before anything is written."""
        b, n = self._slot(b), int(n_tokens)
        if n > self.cap:
            raise IndexError("%d tokens exceed the per-sequence cap of %d (max_pages * page_size)" % (n, self.cap))
        need = -(-n // self.P) - len(self.pages[b])
        if need > 0:
            self._map(b, self._take(need))

    def reset_seq(self, b):
        """Retire slot b: its pages go back to the free list (a shared page when its last holder lets go) and its
        length becomes 0 on the host and the device."""
        b = self._slot(b)
        for p in self.pages[b]:
            if self.refs[p] <= 0:
                raise RuntimeError("page %d released twice" % p)
            self.refs[p] -= 1
            if self.refs[p] == 0:
                self._free.append(p)
        self.pages[b] = []
        self.npages[b] = 0
        self.lens_host[b] = 0
        self.lens[b] = 0

    def fork(self, src, dst):
        """Slot dst becomes a copy of slot src's lens_host[src] tokens: src's full pages are shared (reference count
        + 1) and its partial last page is copied into a fresh page with kvq_page_copy in every layer cache over this
        table.  dst must be empty.  Sets dst's host and device length."""
        src, dst = self._slot(src), self._slot(dst)
        if src == dst or self.pages[dst]:
            raise ValueError("fork needs an empty destination slot other than the source")
        n = self.lens_host[src]
        full, part = divmod(n, self.P)
        fresh = self._take(1) if part else []
        shared = self.pages[src][:full]
        for p in shared:
            self.refs[p] += 1
        self._map(dst, shared + fresh)
        for c in self.caches:
            c._copy_between(src, dst, full * self.P, n)
        self.lens_host[dst] = n
        self.lens[dst] = n


class PagedLayerCache(_BatchCommon):
    """One layer's quantised cache for B sequences in a pool of fixed-size pages (DESIGN.md section 4.11).

    The pool holds n_pool pages of P tokens: kcache / vcache [n_pool, H, W, P], vlut [n_pool*P, 2^bits], vaff
    [n_pool*P, 2], outlier rows [n_pool*P, n_out]; a page is laid out as a LayerCache with Lmax = P.  Which pages a
    sequence holds is the business of a PageTable (`pages`), shared by the caches of all layers of a batch; the
    per-sequence cap (what Lmax is to BatchedLayerCache) is its max_pages * P.  Memory scales with the pages in use,
    not with B x cap.

    The public methods are those of BatchedLayerCache with the same semantics (append_dyn, advance, append, attend,
    set_sinks, reset_seq, commit, sync_host, lens); append_dyn and attend read the page table on the device.  A paged
    slot is not a contiguous LayerCache, so there is no seq(b).  Instead the operations a prompt needs work on slot b
    in place (DESIGN.md section 4.12): append_chunk(b, k, v), dequantize(b, ...) and attend_chunk(b, q, k, v), with
    the contracts of the LayerCache methods of those names, and slot(b), the handle DecoderStage.prefill drives.
    load_seq(b, lc, n) pages a contiguous cache's first n slots in and read_seq(b, lc) pages slot b out into one."""

    _append_fn, _attend_fn = "kvq_append_kv_fused_paged", "kvq_attend_paged"
    _append_chunks_fn, _attend_chunks_fn = "kvq_append_kv_fused_chunk_ragged_paged", "kvq_attend_chunk_ragged_paged"

    def __init__(self, batch, bits, num_heads, klut, klut_sub, thr_lower, thr_upper, v_cent, device,
                 include_sparse=True, sparsity_threshold=0.99, n_sink=0, v_norm=None, sparse_v=None, q_heads=None,
                 page_size=None, n_pool=None, max_pages=None, pages=None):
        """pages: the batch's PageTable (shared by its layers); None builds one from page_size (default 640), n_pool
        and max_pages (default: n_pool pages each).  With a given table, page_size / n_pool / max_pages must be None or agree."""
        B = self._check_batch(batch)
        dev = self._device(device)
        if pages is None:
            if n_pool is None:
                raise ValueError("n_pool is needed when no page table is given")
            pages = PageTable(B, 640 if page_size is None else page_size, n_pool,
                              n_pool if max_pages is None else max_pages, dev)
        else:
            if not isinstance(pages, PageTable) or pages.B != B or pages.device != dev:
                raise ValueError("pages must be a PageTable of batch %d on %s" % (B, dev))
            for name, want, got in (("page_size", pages.P, page_size), ("n_pool", pages.n_pool, n_pool),
                                    ("max_pages", pages.max_pages, max_pages)):
                if got is not None and int(got) != want:
                    raise ValueError("%s=%s disagrees with the page table's %d" % (name, got, want))
        self.pages = pages
        P, N = pages.P, pages.n_pool
        H, W = int(num_heads), HEAD_DIM * int(bits) // 32
        c = LayerCache(bits, num_heads, 4, klut, klut_sub, thr_lower, thr_upper, v_cent, dev, False,
                       sparsity_threshold, n_sink, v_norm, None, q_heads)   # (calibration only)
        if N * H * W >= 2 ** 31:
            raise ValueError("a pool of %d pages of %d word rows exceeds 2^31 rows" % (N, H * W))
        self._init_common(B, dev, c, None)
        self.sparse_k = bool(include_sparse)
        self.sparse_v = self.sparse_k if sparse_v is None else (bool(sparse_v) and self.sparse_k)
        self.P, self.n_pool, self.Lmax, self._extent = P, N, pages.cap, N
        self.lens = pages.lens
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)   # noqa: E731
        self.kcache, self.vcache = z((N, H, W, P), torch.int32), z((N, H, W, P), torch.int32)
        self.vlut, self.vaff = z((N * P, 2 ** int(bits)), torch.float32), z((N * P, 2), torch.float32)
        self.k_outliers = self.k_outlier_idx = self.v_outliers = self.v_outlier_idx = None
        if self.sparse_k:
            self.k_outliers, self.k_outlier_idx = z((N * P, self.n_out), torch.float32), z((N * P, self.n_out), torch.int32)
        if self.sparse_v:
            self.v_outliers, self.v_outlier_idx = z((N * P, self.n_out), torch.float32), z((N * P, self.n_out), torch.int32)
        pages.caches.append(self)

    @classmethod
    def from_luts(cls, bits, num_heads, klut, v_cent, device="cuda", include_sparse=True, sparsity_threshold=0.99,
                  n_sink=0, v_norm=None, sparse_v=None, q_heads=None, batch=1, page_size=None, n_pool=None,
                  max_pages=None, pages=None):
        """LayerCache.from_luts with the same options, for `batch` sequences over a pool of n_pool pages of
        page_size tokens (or over the given shared PageTable `pages`)."""
        c = LayerCache.from_luts(bits, num_heads, 4, klut, v_cent, device, False, sparsity_threshold, 0, v_norm,
                                 None, q_heads)
        return cls(batch, bits, num_heads, c.klut, c.klut_sub if c.klut_sub is not c.klut else None, c.thr_lower,
                   c.thr_upper, c.v_cent, c.device, include_sparse, sparsity_threshold, n_sink, v_norm, sparse_v,
                   q_heads, page_size, n_pool, max_pages, pages)

    def _page_args(self):
        pg = self.pages
        return (pg.table.data_ptr(), pg.max_pages, pg.npages.data_ptr(), pg.P)

    @property
    def lens_host(self):
        return list(self.pages.lens_host)

    def _host_len(self, b):
        return self.pages.lens_host[self.pages._slot(b)]

    def _set_host_len(self, b, n):
        self.pages.lens_host[b] = n

    def _map_chunks(self, slots, starts, counts):
        """Check every segment's write range against the shared-page rule and the pool's free pages, then map them:
        a refusal (RuntimeError) leaves the table as it was for every slot."""
        pg = self.pages
        need = 0
        for b, s0, t in zip(slots, starts, counts):
            if t == 0:
                continue
            shared = [p for p in pg.pages[b][s0 // self.P:-(-(s0 + t) // self.P)] if pg.refs[p] > 1]
            if shared:
                raise RuntimeError("slots [%d, %d) of slot %d lie in shared pages %s" % (s0, s0 + t, b, shared))
            need += max(0, -(-(s0 + t) // self.P) - len(pg.pages[b]))
        if need > pg.n_free:
            raise RuntimeError("page pool exhausted: %d pages needed, %d of %d free" % (need, pg.n_free, self.n_pool))
        for b, s0, t in zip(slots, starts, counts):
            pg.reserve(b, s0 + t)

    def _chunks_tail(self, slots):
        pg = self.pages
        self._n_mapped = np.asarray([len(pg.pages[b]) for b in slots], dtype=np.int32)   # (alive through the call)
        return (pg.table.data_ptr(), pg.max_pages, self._n_mapped.ctypes.data, pg.P)

    def commit(self, *slots):
        """Copy the host lengths of the given slots -- every slot when none is given -- to the device lengths."""
        for b in (slots or range(self.B)):
            self.lens[b] = self.pages.lens_host[b]

    def sync_host(self):
        """Copy the device lengths back to the host mirror (after device-side appends, e.g. graph replays)."""
        for b, n in enumerate(self.lens.tolist()):
            self.pages.lens_host[b] = min(int(n), self.Lmax)

    def reset_seq(self, b):
        """Retire slot b: its pages return to the pool and its length becomes 0 (PageTable.reset_seq; a no-op for
        the other layers of a shared table once one has done it)."""
        self.pages.reset_seq(b)

    def append(self, k, v, active=None):
        """append_dyn + advance, with the host lengths kept in step and pages mapped first.  Raises IndexError if an
        active sequence is at the cap and RuntimeError if the pool cannot hold the step -- before anything is
        launched."""
        act = [True] * self.B if active is None else [bool(a) for a in active.tolist()]
        lens = self.pages.lens_host
        if any(a and n >= self.Lmax for a, n in zip(act, lens)):
            raise IndexError("cache full")
        need = sum(-(-(n + 1) // self.P) - len(self.pages.pages[b]) for b, (a, n) in enumerate(zip(act, lens)) if a)
        if need > self.pages.n_free:
            raise RuntimeError("page pool exhausted: %d pages needed, %d of %d free"
                               % (need, self.pages.n_free, self.n_pool))
        for b, a in enumerate(act):
            if a:
                self.pages.reserve(b, lens[b] + 1)
        self.append_dyn(k, v, active)
        self.advance(active)
        for b, a in enumerate(act):
            lens[b] += int(a)

    # -- paging in and out (kvq_page_copy) --------------------------------------------------------------------------
    def _ref(self, lc=None, b=None):
        """kvq_seq_ref of a contiguous LayerCache lc, or of this pool's sequence b."""
        src = self if lc is None else lc
        o = lambda t, on: t.data_ptr() if on else None   # noqa: E731
        return _SeqRef(src.kcache.data_ptr(), src.vcache.data_ptr(), o(src.k_outliers, src.sparse_k),
                       o(src.k_outlier_idx, src.sparse_k), o(src.v_outliers, src.sparse_v),
                       o(src.v_outlier_idx, src.sparse_v), src.vlut.data_ptr(), src.vaff.data_ptr(),
                       lc.Lmax if lc is not None else 0,
                       None if lc is not None else self.pages.table[b].data_ptr())

    def _same_layout(self, lc):
        if not isinstance(lc, LayerCache):
            raise ValueError("expected a LayerCache")
        if (lc.bits, lc.H, lc.n_out, lc.sparse_k, lc.sparse_v, lc.device) != (
                self.bits, self.H, self.n_out, self.sparse_k, self.sparse_v, self.device):
            raise ValueError("the LayerCache's bits, heads, outlier budget, sparse sides and device must be this "
                             "cache's")

    @_on_cache_device
    def _copy(self, a, d, s0, s1):
        _lib.check(self.lib.kvq_page_copy(self.bits, self.H, self.n_out, self.P, int(s0), int(s1), ctypes.byref(a),
                                          ctypes.byref(d), torch.cuda.current_stream().cuda_stream), "kvq_page_copy")

    def _copy_between(self, src, dst, s0, s1):
        self._copy(self._ref(b=src), self._ref(b=dst), s0, s1)

    def load_seq(self, b, layer_cache, n=None):
        """Page slots [0, n) of a contiguous LayerCache (default n: its len) into slot b, mapping pages first (an
        exhausted pool raises before anything is copied).  Sets b's host length; commit(b) publishes it."""
        self._same_layout(layer_cache)
        n = layer_cache.len if n is None else int(n)
        if not 0 <= n <= layer_cache.Lmax:
            raise ValueError("n=%d outside the LayerCache's %d slots" % (n, layer_cache.Lmax))
        self.pages.reserve(b, n)
        self._copy(self._ref(lc=layer_cache), self._ref(b=b), 0, n)
        self.pages.lens_host[b] = n

    def read_seq(self, b, layer_cache):
        """Page slot b's lens_host[b] tokens out into a contiguous LayerCache (its len is set), so that every
        single-sequence reader (attend, dequantize, attend_chunk, ...) can serve the slot."""
        self._same_layout(layer_cache)
        n = self.pages.lens_host[int(b)]
        if n > layer_cache.Lmax:
            raise ValueError("slot %d holds %d tokens, the LayerCache %d slots" % (b, n, layer_cache.Lmax))
        self._copy(self._ref(b=b), self._ref(lc=layer_cache), 0, n)
        layer_cache.len = n

    def fork(self, src, dst):
        """Slot dst becomes a copy of slot src (PageTable.fork: full pages shared, the partial last page copied)."""
        self.pages.fork(src, dst)

    # -- prompts in place (kvq_append_kv_fused_chunk_paged, kvq_dequant_kv_paged) ---------------------------------------
    def _seq_args(self, b):
        """The trailing arguments of the single-sequence paged entry points: slot b's page-table row, max_pages, its
        mapped entries and P."""
        pg = self.pages
        return (pg.table[b].data_ptr(), pg.max_pages, len(pg.pages[b]), pg.P)

    @_on_cache_device
    def _append_chunk_at(self, b, slot0, k, v):
        """Append k, v f32 [T, hidden] at slots slot0 .. slot0 + T - 1 of slot b in one launch, mapping pages first;
        returns slot0 + T.  Raises before anything is written (IndexError past the cap, RuntimeError when the pool
        is exhausted or a slot in range lies in a page shared with another slot)."""
        c, pg = self._tmpl, self.pages
        b = pg._slot(b)
        if k.dim() != 2 or tuple(k.shape) != tuple(v.shape) or k.shape[1] != self.hidden:
            raise ValueError("k and v must both be [T, %d], got %s and %s" % (self.hidden, tuple(k.shape), tuple(v.shape)))
        T = k.shape[0]
        kp, vp = c._vec(k, T * self.hidden, "k"), c._vec(v, T * self.hidden, "v")
        # fork shares full pages only, so a slot's appends land in pages it owns alone; never write through a shared one
        shared = [p for p in pg.pages[b][slot0 // self.P:-(-(slot0 + T) // self.P)] if pg.refs[p] > 1]
        if T and shared:
            raise RuntimeError("slots [%d, %d) of slot %d lie in shared pages %s" % (slot0, slot0 + T, b, shared))
        pg.reserve(b, slot0 + T)
        if T == 0:
            return slot0
        _lib.check(self.lib.kvq_append_kv_fused_chunk_paged(
            self.bits, self.H, self.n_pool, slot0, T, self.n_each,
            kp, self.kcache.data_ptr(), c.klut.data_ptr(), c.klut_sub.data_ptr(),
            c.thr_lower.data_ptr(), c.thr_upper.data_ptr(), *self._ptrs("k"),
            vp, self.vcache.data_ptr(), c.v_cent.data_ptr(),
            c.v_cent_deq.data_ptr() if c.v_norm is not None else None, self.vlut.data_ptr(), self.vaff.data_ptr(),
            *self._ptrs("v"), torch.cuda.current_stream().cuda_stream, *self._seq_args(b)),
            "kvq_append_kv_fused_chunk_paged")
        return slot0 + T

    def append_chunk(self, b, k, v):
        """LayerCache.append_chunk for slot b: k, v f32 [T, hidden] go to slots lens_host[b] .. + T - 1 in one launch
        (kvq_append_kv_fused_chunk_paged), bit for bit as LayerCache.append_chunk leaves a contiguous cache.  Pages are
        mapped first: past the cap raises IndexError and an exhausted pool RuntimeError, before anything is written.
        Advances lens_host[b] (the table's, shared by its layers); commit(b) publishes it to the device.  Several
        layers over one table take a prompt through slot(b) handles instead, as BatchedDecoderStage.prefill_seq does."""
        pg = self.pages
        b = pg._slot(b)
        pg.lens_host[b] = self._append_chunk_at(b, pg.lens_host[b], k, v)

    @_on_cache_device
    def _dequantize_at(self, b, start, stop, n_cached, rope_theta, out_k, out_v):
        c = self._tmpl

        def call(start, stop, ok, ov, stride, rope, npos, pos_offset):
            _lib.check(self.lib.kvq_dequant_kv_paged(
                self.bits, self.H, self.n_pool, start, stop,
                self.kcache.data_ptr(), c.klut_deq.data_ptr(), *self._ptrs("k"),
                self.vcache.data_ptr(), c.v_cent_deq.data_ptr(), self.vaff.data_ptr(), *self._ptrs("v"),
                self.n_out, rope.data_ptr() if rope is not None else None, npos, pos_offset,
                ok, ov, stride, torch.cuda.current_stream().cuda_stream, *self._seq_args(b)), "kvq_dequant_kv_paged")
        return c._dequantize(start, stop, n_cached, 0, rope_theta, out_k, out_v, call)

    def dequantize(self, b, start=0, stop=None, rope_theta=None, out_k=None, out_v=None, rope=None):
        """LayerCache.dequantize for slot b (kvq_dequant_kv_paged): slots [start, stop) of its lens_host[b] tokens as
        fp16 K and V [H, stop - start, 128], the same values, with the same options (rope= included), outputs and
        checks."""
        b = self.pages._slot(b)
        n = self.pages.lens_host[b]
        rope_theta = self._len_slot(b, _resolve(rope, rope_theta), n + self.n_sink)
        return self._dequantize_at(b, start, stop, n, rope_theta, out_k, out_v)

    @_on_cache_device
    def _attend_chunk_at(self, b, L, q, k, v, rope_theta):
        c = self._tmpl
        if c.group > 1:
            c._gqa_check()
        T = c._chunk_check(q, k, v)
        rope_theta = self._len_slot(b, rope_theta, self.n_sink + L + T)
        sinks = (self.sink_k[b], self.sink_v[b]) if self.sink_k is not None else None
        return c._attend_chunk_sdpa(q, k, v, rope_theta, L, 0, sinks,
                                    lambda ok, ov: self._dequantize_at(b, 0, L, L, rope_theta, ok, ov))

    def attend_chunk(self, b, q, k, v, rope_theta=10000.0, rope=None):
        """LayerCache.attend_chunk for slot b: causal attention of a T-token chunk placed after the slot's lens_host[b]
        tokens over its sinks, those tokens (dequantised in place, kvq_dequant_kv_paged) and the chunk; same arguments
        (rope= included), grouped-query rule and result, bit for bit.  The cache is not modified."""
        b = self.pages._slot(b)
        return self._attend_chunk_at(b, self.pages.lens_host[b], q, k, v, _resolve(rope, rope_theta))

    def slot(self, b):
        """Slot b as the single-sequence cache DecoderStage.prefill(caches=...) drives (PagedSlot)."""
        return PagedSlot(self, b)


class PagedSlot:
    """Slot b of a PagedLayerCache seen as one sequence's cache: what DecoderStage.prefill reads and calls -- len,
    Lmax (the per-sequence cap), n_sink, pos_base (0), attend_chunk(q, k, v, rope_theta, rope) and append_chunk(k, v).

    The layers of a batch share one PageTable and so one host length per slot, while a prompt goes through them one
    layer after the other.  So a handle keeps its own `len`, starting at the slot's lens_host[b]: attend_chunk attends
    over that many tokens and append_chunk writes there, advances it and sets lens_host[b] to it (no commit)."""

    pos_base = 0

    def __init__(self, cache, b):
        self.cache, self.b = cache, cache.pages._slot(b)
        self.len = cache.pages.lens_host[self.b]
        self.Lmax, self.n_sink = cache.Lmax, cache.n_sink

    def attend_chunk(self, q, k, v, rope_theta=10000.0, rope=None):
        return self.cache._attend_chunk_at(self.b, self.len, q, k, v, _resolve(rope, rope_theta))

    def append_chunk(self, k, v):
        self.len = self.cache._append_chunk_at(self.b, self.len, k, v)
        self.cache.pages.lens_host[self.b] = self.len


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
