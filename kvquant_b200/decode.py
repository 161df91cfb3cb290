"""LLaMA-shaped batch-1 decode harness over the quantised KV cache, and its layer-group pipeline.

The reference drives the hot path from deployment/llama.py:72-94 (token-by-token decode loop) through its forked
HF LlamaModel; the forked transformers 4.3x does not import under the installed 5.5.0 and there are no weights
offline, so this is a self-contained decoder with the same per-layer dataflow as
LlamaFlashAttention2.forward at q_len == 1 (modeling_llama.py:1778-2011):

    v/q/k proj -> RoPE on Q only -> append pre-RoPE K and V (quantise + outlier split) -> Q.K^T over the
    compressed cache (+ fp16 sinks) -> softmax -> .V -> o_proj -> MLP

with random-init fp16 weights of the LLaMA architecture.  The dense GEMVs are the library's own fused kernels
(kvq_dec_gemv: RMSNorm / SwiGLU / residual folded in); everything that touches the KV cache goes through the C ABI
(kvq_append_kv_fused, kvq_attend).

Multi-GPU: the reference's only parallelism is naive layer-group model parallelism
(`LlamaModel.set_devices`, modeling_llama.py:2428-2453: len(layers)//n_gpus consecutive layers per device, hidden
state moved with .to(device) at the split points and back to cuda:0 at the end, 2552-2585).  `PipelineDecoder`
is the one-process-per-GPU form of that: rank r owns layers [r*n/N, (r+1)*n/N) with their full-length caches,
the [hidden] fp16 vector hops rank r -> r+1 with NCCL send/recv (NVLink P2P), and the last rank returns it to
rank 0 for norm + lm_head.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from .cache import RopeLenState, BatchedLayerCache, LayerCache, PagedLayerCache, PageTable, HEAD_DIM, _resolve
from .rope import LengthDependentRotary, RotarySpec


@dataclass
class DecodeConfig:
    n_layers: int = 32
    hidden: int = 4096
    n_heads: int = 32
    intermediate: int = 11008
    vocab: int = 32000
    rope_theta: float = 10000.0
    rms_eps: float = 1e-5
    bits: int = 4
    n_sink: int = 0            # first_few_fp16
    sparsity_threshold: float = 0.99
    include_sparse: bool = True
    sparse_v: bool = True      # False: outlier rows for K only (BASELINE configs[4]: capped K outliers)
    max_len: int = 4096        # quantised slots allocated per layer
    n_kv_heads: int = None     # grouped-query attention: KV heads (None: n_heads); query head h reads KV head h // g
    rope_scaling: dict = None  # HF rope_scaling dict ("linear", "llama3", "yarn", "dynamic", "longrope"); None: plain
                               # rope_theta frequencies
    max_position_embeddings: int = None   # HF's config value: the switch length of "dynamic" and LongRoPE's default factor

    @property
    def kv_heads(self):
        return self.n_heads if self.n_kv_heads is None else self.n_kv_heads

    @property
    def kv_hidden(self):
        return self.kv_heads * HEAD_DIM

    @property
    def rotary(self):
        """The scaled RotarySpec of rope_theta + rope_scaling, a LengthDependentRotary for "dynamic" and "longrope",
        or None for the plain-theta frequencies."""
        sc = self.rope_scaling or {}
        if sc.get("rope_type", sc.get("type")) in ("dynamic", "longrope"):
            return LengthDependentRotary(self.rope_theta, sc, self.max_position_embeddings)
        spec = RotarySpec(self.rope_theta, self.rope_scaling)
        return spec if spec.scaled else None

    @staticmethod
    def llama7b(**kw):
        return DecodeConfig(32, 4096, 32, 11008, 32000, **kw)

    @staticmethod
    def llama13b(**kw):
        return DecodeConfig(40, 5120, 40, 13824, 32000, **kw)

    @staticmethod
    def llama3_8b(**kw):
        """LLaMA-3-8B shapes: 32 query heads over 8 KV heads (g = 4), rope base 500000."""
        cfg = dict(n_layers=32, hidden=4096, n_heads=32, intermediate=14336, vocab=128256, rope_theta=500000.0,
                   n_kv_heads=8)
        cfg.update(kw)
        return DecodeConfig(**cfg)

    @staticmethod
    def llama31_8b(**kw):
        """LLaMA-3.1-8B: the llama3_8b shapes with LLaMA-3.1's rotary scaling (rope_type "llama3", factor 8, original
        context 8192)."""
        cfg = dict(rope_scaling={"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                 "original_max_position_embeddings": 8192})
        cfg.update(kw)
        return DecodeConfig.llama3_8b(**cfg)


def partition_layers(n_layers: int, world: int, rank: int):
    """Layer range of `rank` -- the reference's split rule (modeling_llama.py:2442-2453): n_layers // world
    consecutive layers per device, the remainder goes to the last device."""
    per = n_layers // world
    lo = rank * per
    hi = n_layers if rank == world - 1 else lo + per
    return lo, hi


def rmsnorm(x, w, eps):
    xf = x.float()
    return (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype) * w


class DecoderLayer:
    def __init__(self, cfg: DecodeConfig, device, gen, quantizer, with_sinks=True):
        h, it = cfg.hidden, cfg.intermediate
        def w(*shape):
            return (torch.randn(shape, generator=gen, device=device, dtype=torch.float32) * 0.02).half()
        self.wqkv = w(h + 2 * cfg.kv_hidden, h)      # q | k | v rows
        self.wo = w(h, h)
        self.wgu = w(2 * it, h)
        self.wdown = w(h, it)
        self.n1 = torch.ones(h, dtype=torch.float16, device=device)
        self.n2 = torch.ones(h, dtype=torch.float16, device=device)
        self.cache = LayerCache.from_luts(cfg.bits, cfg.kv_heads, cfg.max_len, quantizer["klut"], quantizer["v_cent"],
                                          device=device, include_sparse=cfg.include_sparse,
                                          sparsity_threshold=cfg.sparsity_threshold, n_sink=cfg.n_sink,
                                          sparse_v=cfg.sparse_v, q_heads=cfg.n_heads)
        self.cache.share_scratch = True     # the layers of a stage attend one after another on one stream
        if cfg.n_sink and with_sinks:
            sk = (torch.randn((cfg.kv_heads, HEAD_DIM, cfg.n_sink), generator=gen, device=device)).half()
            sv = (torch.randn((cfg.kv_heads, cfg.n_sink, HEAD_DIM), generator=gen, device=device)).half()
            self.cache.set_sinks(sk, sv)


class DecoderStage:
    """Layers [lo, hi) of the model on one device, plus (first stage) the embedding and (rank 0) norm + lm_head."""

    def __init__(self, cfg: DecodeConfig, lo: int, hi: int, device, quantizer, seed=0, with_head=True, sp=None):
        """sp = (rank, world) switches to SEQUENCE-sharded attention (SURVEY 8e-2 / 8f-1): every rank holds all layers'
        weights and a contiguous 1/world slice of every layer's cache; per layer the partial (out, lse) results are
        all-gathered (H*129 floats per rank over NVLink) and merged.  The new token is appended on the last rank.
        Grouped-query models (cfg.n_kv_heads) run unsharded only."""
        if sp is not None and cfg.kv_heads != cfg.n_heads:
            raise NotImplementedError("sequence-sharded attention of a grouped-query model")
        self.rotary = cfg.rotary   # scaled RotarySpec, or None: rope_theta's frequencies
        if sp is not None and self.rotary is not None:
            raise NotImplementedError("sequence-sharded attention with scaled rotary frequencies")
        self.cfg, self.lo, self.hi = cfg, lo, hi
        self.device = torch.device(device)
        self.sp = sp
        self.global_pos = None   # sp: absolute position of the new token (set by the driver)
        self.dyn = None          # device-resident length / position counters (enable_device_length)
        self.xchg = None         # sp: kvquant_b200.p2p.PeerExchange (peer-memory exchange) instead of NCCL all_gather
        gen = torch.Generator(device=self.device)
        gen.manual_seed(seed * 1000 + lo)
        self.layers = [DecoderLayer(cfg, self.device, gen, quantizer, with_sinks=(sp is None or sp[0] == 0))
                       for _ in range(lo, hi)]
        self.with_head = with_head
        if with_head:
            self.embed = (torch.randn((cfg.vocab, cfg.hidden), generator=gen, device=self.device) * 0.02).half()
            self.norm = torch.ones(cfg.hidden, dtype=torch.float16, device=self.device)
            self.lm_head = (torch.randn((cfg.vocab, cfg.hidden), generator=gen, device=self.device) * 0.02).half()
        half = HEAD_DIM // 2
        self.rope_state = None
        if self.rotary is None:
            self.inv_freq = 1.0 / (cfg.rope_theta ** (torch.arange(0, HEAD_DIM, 2, device=self.device).float() / HEAD_DIM))
        elif isinstance(self.rotary, LengthDependentRotary):
            # one rotation state for every layer, prepared once per decode step (the host paths use inv_freq_at)
            self.inv_freq = None
            c0 = self.layers[0].cache
            self.rope_state = RopeLenState(self.rotary, 1, c0.Lmax + c0.n_sink + c0.pos_base + 1, self.device)
            for ly in self.layers:
                ly.cache.rope_len_state = self.rope_state
        else:   # HF's inv_freq, the vector the caches' tables are built from
            self.inv_freq = self.rotary.inv_freq.to(self.device)
        self._half = half

    # -- pieces -------------------------------------------------------------------------------------------------
    def embed_token(self, tok):
        return self.embed[tok].view(-1)

    def head(self, x):
        if x.is_cuda:
            return self._gemv(self.lm_head, x, 3, self._buffers()["logits"], norm_w=self.norm)
        return self.lm_head @ rmsnorm(x, self.norm, self.cfg.rms_eps)

    def _inv_freq(self, s):
        """The frequencies of a call whose last query sits at position s - 1."""
        if isinstance(self.rotary, LengthDependentRotary):
            return self.rotary.inv_freq_at(s).to(self.device)
        return self.inv_freq

    def _rope_q(self, q, pos):
        """HF rotate-half RoPE on the query only (modeling_llama.py:1851-1859); q f32 [H,128]."""
        ang = self._inv_freq(int(pos) + 1) * float(pos)
        cos = torch.cat((ang.cos(), ang.cos()))
        sin = torch.cat((ang.sin(), ang.sin()))
        if self.rotary is not None:     # HF multiplies cos and sin by the attention factor (YaRN)
            cos, sin = cos * self.rotary.attention_factor, sin * self.rotary.attention_factor
        rot = torch.cat((-q[:, self._half:], q[:, :self._half]), dim=-1)
        return q * cos + rot * sin

    def _buffers(self):
        if getattr(self, "_buf", None) is None:
            cfg, dev = self.cfg, self.device
            f16 = dict(dtype=torch.float16, device=dev)
            f32 = dict(dtype=torch.float32, device=dev)
            self._buf = dict(h=torch.empty(cfg.hidden, **f16), qkv=torch.empty(cfg.hidden + 2 * cfg.kv_hidden, **f16),
                             q=torch.empty(cfg.hidden, **f32), k=torch.empty(cfg.kv_hidden, **f32),
                             v=torch.empty(cfg.kv_hidden, **f32), o16=torch.empty(cfg.hidden, **f16),
                             gu=torch.empty(2 * cfg.intermediate, **f16), act=torch.empty(cfg.intermediate, **f16),
                             x0=torch.empty(cfg.hidden, **f16), x1=torch.empty(cfg.hidden, **f16),
                             logits=torch.empty(cfg.vocab, **f16))
            if self.sp is not None:
                n = cfg.hidden + cfg.n_heads
                self._buf["part"] = torch.empty(n, **f32)
                self._buf["gath"] = torch.empty(self.sp[1] * n, **f32)
                self._buf["om"] = torch.empty(cfg.hidden, **f32)
        return self._buf

    def _gemv(self, w, x, kind, y, norm_w=None, residual=None):
        """y = residual + w @ f(x) through the library's fused GEMV (kvq_dec_gemv); kind: 0 fp16, 1 f32, 2 gate|up
        -> silu(gate)*up, 3 fp16 + RMSNorm(norm_w)."""
        from . import _lib
        lib = _lib.load()
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.kvq_dec_gemv(w.data_ptr(), w.shape[0], w.shape[1], x.data_ptr(), kind,
                                    norm_w.data_ptr() if norm_w is not None else None, self.cfg.rms_eps,
                                    residual.data_ptr() if residual is not None else None, y.data_ptr(), 0, st))
        return y

    def forward(self, x):
        """x: fp16 [hidden] -> fp16 [hidden] after this stage's layers; appends one token to every layer cache.
        Four launches per layer outside the KV cache: GEMV(+RMSNorm) -> RoPE/split -> [append, attend] ->
        GEMV(+residual) -> GEMV(+RMSNorm) -> GEMV(SwiGLU input, +residual); everything touching the KV cache is
        kvq_append_kv_fused + kvq_attend."""
        from . import _lib
        cfg = self.cfg
        lib = _lib.load()
        b = self._buffers()
        H, hid = cfg.n_heads, cfg.hidden
        st = torch.cuda.current_stream().cuda_stream
        xs = (b["x0"], b["x1"])     # ping-pong residual stream (the caller's x is never written)
        flip = 0
        rot, freq = self.rotary, self.inv_freq
        if self.rope_state is not None:   # length-dependent: f(s) and the table, once for every layer of the step
            c0 = self.layers[0].cache
            if self.dyn is not None:
                rot = self.rope_state.update(len_dev=self.dyn["len"], len_add=1, L_cap=c0.Lmax,
                                             pos_offset=c0.n_sink + c0.pos_base)
            else:
                rot = self.rope_state.update(s=c0.n_sink + c0.pos_base + c0.len + 1)
            freq = rot.f_cur
        attn = self.rotary.attention_factor if self.rotary is not None else 1.0   # theta: 1, an exact product
        for ly in self.layers:
            c = ly.cache
            dyn = self.dyn          # device-resident length / position (one graph for a growing cache) or None
            self._gemv(ly.wqkv, x, 3, b["qkv"], norm_w=ly.n1)
            # the new token's absolute position: *pos_dev, or the host position
            if dyn is not None:
                pos = (dyn["pos"].data_ptr(), 0)
            else:
                pos = (None, self.global_pos if self.sp is not None else c.n_sink + c.pos_base + c.len)
            _lib.check(lib.kvq_dec_rope_split_freq(b["qkv"].data_ptr(), freq.data_ptr(), attn, *pos, b["q"].data_ptr(),
                                                   b["k"].data_ptr(), b["v"].data_ptr(), H, cfg.kv_heads, 1, st),
                       "kvq_dec_rope_split_freq")
            qh = b["q"].view(H, HEAD_DIM)
            if self.sp is None:
                if dyn is None:
                    c.append(b["k"], b["v"])             # pre-RoPE K, per-token V: quantise + outlier split
                    o = c.attend(qh, rope_theta=cfg.rope_theta, rope=rot)   # f32 [H,128]
                else:
                    c.append_dyn(b["k"], b["v"], dyn["len"])
                    o = c.attend_dyn(qh, dyn["len"], 1, rope_theta=cfg.rope_theta, rope=rot)
            else:
                import torch.distributed as dist
                rank, world = self.sp
                part = b["part"]
                owner = rank == world - 1                # the newest token lives on the last shard
                if dyn is None:
                    if owner:
                        c.append(b["k"], b["v"])
                    c.attend(qh, rope_theta=cfg.rope_theta, out=part[:hid].view(H, HEAD_DIM), lse=part[hid:])
                else:
                    if owner:
                        c.append_dyn(b["k"], b["v"], dyn["len"])
                    c.attend_dyn(qh, dyn["len"], 1 if owner else 0, rope_theta=cfg.rope_theta,
                                 out=part[:hid].view(H, HEAD_DIM), lse=part[hid:])
                o = b["om"]
                if self.xchg is not None:                         # peer-memory exchange fused with the merge (one kernel per layer)
                    self.xchg.exchange_merge(part, o)
                else:
                    dist.all_gather_into_tensor(b["gath"], part)  # H*129 floats per rank over NVLink
                    _lib.check(lib.kvq_attend_merge(b["gath"].data_ptr(), world, H, o.data_ptr(), st))
            x = self._gemv(ly.wo, o, 1, xs[flip], residual=x)
            flip ^= 1
            self._gemv(ly.wgu, x, 3, b["gu"], norm_w=ly.n2)
            x = self._gemv(ly.wdown, b["gu"], 2, xs[flip], residual=x)
            flip ^= 1
        if self.dyn is not None:                          # advance the device counters inside the step
            if self.sp is None or self.sp[0] == self.sp[1] - 1:
                _lib.check(lib.kvq_dec_counter_add(self.dyn["len"].data_ptr(), 1, st))
            if self.dyn["pos"].data_ptr() != self.dyn["len"].data_ptr():
                _lib.check(lib.kvq_dec_counter_add(self.dyn["pos"].data_ptr(), 1, st))
        return x

    def enable_device_length(self, L, pos):
        """Switch the stage to the device-resident length: every layer cache holds L tokens, the next token sits at
        absolute position `pos`.  Returns the counters (int64[1] each; the same tensor when pos tracks len)."""
        ln = torch.full((1,), int(L), dtype=torch.int64, device=self.device)
        ps = torch.full((1,), int(pos), dtype=torch.int64, device=self.device)
        self.dyn = dict(len=ln, pos=ps)
        return self.dyn

    def set_device_length(self, L, pos):
        self.dyn["len"].fill_(int(L))
        self.dyn["pos"].fill_(int(pos))

    def forward_torch(self, x):
        """Same dataflow with plain torch element-wise ops (reference for the helper kernels; used by tests)."""
        cfg = self.cfg
        H = cfg.n_heads
        for ly in self.layers:
            c = ly.cache
            pos = c.n_sink + c.len
            qkv = ly.wqkv @ rmsnorm(x, ly.n1, cfg.rms_eps)
            q, k, v = qkv.float().split((cfg.hidden, cfg.kv_hidden, cfg.kv_hidden))
            q = self._rope_q(q.view(H, HEAD_DIM), pos).contiguous()
            c.append(k.contiguous(), v.contiguous())
            o = c.attend(q, rope_theta=cfg.rope_theta, rope=self.rotary)
            x = x + ly.wo @ o.half().view(-1)
            gu = ly.wgu @ rmsnorm(x, ly.n2, cfg.rms_eps)
            g, u = gu.split(cfg.intermediate)
            x = x + ly.wdown @ (torch.nn.functional.silu(g) * u)
        return x

    def prefill(self, x, chunk=2048, caches=None):
        """Run a T-token prompt through this stage's layers and append its K / V to every layer cache.
        x: fp16 [T, hidden] (the first stage: embed[tokens]); returns fp16 [T, hidden] after the stage's layers, and
        every layer cache holds T more tokens.

        The prompt goes through in chunks of at most `chunk` tokens.  Per chunk and layer: RMSNorm + QKV projection
        (one fp16 matmul), rotate-half RoPE of q at positions n_sink + pos_base + len + i (the convention of
        kvq_dec_rope_split), LayerCache.attend_chunk, LayerCache.append_chunk, then o_proj + residual and the MLP with
        the math of forward_torch.  A chunk attends to the earlier chunks through the quantised cache and to itself in
        fp16; with chunk >= T the whole prompt attends in fp16 and is quantised afterwards, as a prefill over
        full-precision K / V does.  Memory per chunk is that of attend_chunk: 2*H*S*128 fp16 values and a chunk x S
        boolean mask, S = n_sink + len + chunk.  Decoding continues from the prompt with forward() or a GraphedStage at
        L = the caches' new length.  Host-length caches of an unsharded stage only.  caches (optional): one cache per
        layer to prefill instead of the layers' own -- a LayerCache, or anything with its len, Lmax, n_sink, pos_base,
        attend_chunk and append_chunk (BatchedDecoderStage.prefill_seq passes a slot's views or PagedSlot handles)."""
        if self.sp is not None:
            raise NotImplementedError("prefill of a sequence-sharded stage")
        if self.dyn is not None:
            raise NotImplementedError("prefill while the device-resident length is enabled")
        cfg = self.cfg
        H, hid = cfg.n_heads, cfg.hidden
        if x.dtype != torch.float16 or x.dim() != 2 or x.shape[1] != hid:
            raise ValueError("x must be fp16 [T, %d], got %s %s" % (hid, x.dtype, tuple(x.shape)))
        if x.device != self.device:
            raise ValueError("x is on %s, the stage lives on %s" % (x.device, self.device))
        chunk = int(chunk)
        if chunk < 1:
            raise ValueError("chunk must be >= 1")
        T = x.shape[0]
        caches = [ly.cache for ly in self.layers] if caches is None else list(caches)
        for c in caches:
            if c.len + T > c.Lmax:
                raise IndexError("a prompt of %d tokens does not fit: %d of %d slots used" % (T, c.len, c.Lmax))
        outs = []
        for s0 in range(0, T, chunk):
            h = x[s0:s0 + chunk]
            n = h.shape[0]
            for ly, c in zip(self.layers, caches):
                q, k, v = self._prefill_qkv(ly, h)
                pos = c.n_sink + c.pos_base + c.len + torch.arange(n, device=self.device)
                q = self._rope_rows(q.reshape(n, H, HEAD_DIM), pos).contiguous()
                o = c.attend_chunk(q, k, v, rope_theta=cfg.rope_theta, rope=self.rotary)
                c.append_chunk(k, v)
                h = self._prefill_out(ly, h, o)
            outs.append(h)
        return torch.cat(outs) if outs else x.clone()

    def _prefill_qkv(self, ly, h):
        """RMSNorm + the QKV projection of prompt rows h fp16 [n, hidden] (one fp16 matmul): q f32 [n, hidden] and the
        contiguous pre-RoPE k, v f32 [n, kv_hidden].  Shared by prefill and BatchedDecoderStage.prefill_seqs."""
        cfg = self.cfg
        qkv = rmsnorm(h, ly.n1, cfg.rms_eps) @ ly.wqkv.t()
        q, k, v = qkv.float().split((cfg.hidden, cfg.kv_hidden, cfg.kv_hidden), dim=-1)
        return q, k.contiguous(), v.contiguous()

    def _prefill_out(self, ly, h, o):
        """o_proj of the attention output o f32 [n, q_heads, 128] + residual, then the MLP + residual (the math of
        forward_torch): h fp16 [n, hidden] after the layer.  Shared by prefill and BatchedDecoderStage.prefill_seqs."""
        cfg = self.cfg
        h = h + o.half().view(h.shape[0], cfg.hidden) @ ly.wo.t()
        gu = rmsnorm(h, ly.n2, cfg.rms_eps) @ ly.wgu.t()
        g, u = gu.split(cfg.intermediate, dim=-1)
        return h + (torch.nn.functional.silu(g) * u) @ ly.wdown.t()

    def _rope_rows(self, q, pos):
        """_rope_q of every row: q f32 [n, H, 128] rotated at positions pos [n]."""
        ang = pos.float()[:, None] * self._inv_freq(int(pos[-1]) + 1)[None, :]
        cos = torch.cat((ang.cos(), ang.cos()), dim=-1)[:, None, :]
        sin = torch.cat((ang.sin(), ang.sin()), dim=-1)[:, None, :]
        if self.rotary is not None:
            cos, sin = cos * self.rotary.attention_factor, sin * self.rotary.attention_factor
        rot = torch.cat((-q[..., self._half:], q[..., :self._half]), dim=-1)
        return q * cos + rot * sin

    def set_len(self, L):
        for ly in self.layers:
            ly.cache.len = L

    def weight_bytes(self):
        n = sum(t.numel() * 2 for ly in self.layers for t in (ly.wqkv, ly.wo, ly.wgu, ly.wdown))
        if self.with_head:
            n += self.lm_head.numel() * 2
        return n


class GraphedStage:
    """One decode step of a stage captured in a CUDA graph (the reference's host syncs make that impossible;
    here nothing in the step touches the host).

    dynamic=False: the captured step appends at slot L and attends over L+1 slots; replaying it re-runs exactly that
    step (the fused append overwrites its slot, so replays are idempotent).
    dynamic=True : the cache length and the token position live in device memory and are advanced inside the step, so
    every replay of the SAME graph is the next decode step of a growing cache (slot L, L+1, ...)."""

    def __init__(self, stage: DecoderStage, L: int, first: bool, last_to_logits: bool, dynamic: bool = False,
                 pos: int = None, pp=None):
        """pp = (rank, world): layer-group pipeline (the reference's multi-GPU scheme, modeling_llama.py:2428-2453, 2552-2585).
        The hop of the [hidden] fp16 vector is PART of the captured step: rank r's graph is
        `recv from r-1 -> its layers -> send to (r+1) % world`, rank 0 additionally owns a second graph
        `recv from world-1 -> norm + lm_head`.  NCCL send/recv kernels inside the graph cost microseconds per hop; issued
        from the host every hop pays the launch latency of a host-issued collective."""
        if pp is not None and pp[1] > 1 and stage.rotary is not None:
            raise NotImplementedError("a layer-pipelined step with scaled rotary frequencies")
        self.stage = stage
        self.pp = pp
        dev = stage.device
        cfg = stage.cfg
        self.tok = torch.zeros(1, dtype=torch.long, device=dev)
        self.x_in = torch.zeros(cfg.hidden, dtype=torch.float16, device=dev)
        self.first, self.last_to_logits = first, last_to_logits
        self.dynamic, self.L0, self.steps = dynamic, L, 0
        c0 = stage.layers[0].cache
        self.pos0 = (c0.n_sink + c0.pos_base + L) if pos is None else pos
        if dynamic:
            stage.enable_device_length(L, self.pos0)

        self.head_in = None
        self.head_graph = None
        if pp is not None and pp[1] > 1:
            import torch.distributed as dist
            prank, pworld = pp
            if prank == 0:
                self.head_in = torch.zeros(cfg.hidden, dtype=torch.float16, device=dev)

        def body():
            if pp is not None and pp[1] > 1 and pp[0] > 0:
                dist.recv(self.x_in, src=pp[0] - 1)
            x = stage.embed_token(self.tok) if first else self.x_in
            if not dynamic:
                stage.set_len(L)
            y = stage.forward(x)
            if pp is not None and pp[1] > 1:
                dist.send(y, dst=(pp[0] + 1) % pp[1])
            return y

        def head_body():     # rank 0 of a pipeline: the last stage's output comes back for norm + lm_head
            dist.recv(self.head_in, src=pp[1] - 1)
            return stage.head(self.head_in)

        if pp is not None and pp[1] > 1:   # eager pipeline steps first: NCCL creates its P2P channels on first use
            for _ in range(2):
                body()
                if pp[0] == 0:
                    head_body()
            torch.cuda.synchronize(dev)
            dist.barrier()

        if stage.sp is not None:   # a few eager steps first so that NCCL is fully initialised before the capture
            for _ in range(2):
                body()
            torch.cuda.synchronize(dev)

        # warm-up on a side stream (allocates scratch, sets func attributes, builds rope tables)
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            for _ in range(2):
                y = body()
                if self.head_in is not None:
                    head_body()
        torch.cuda.current_stream(dev).wait_stream(s)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.y = body()
            if last_to_logits and stage.with_head:
                self.logits = stage.head(self.y)
        if self.head_in is not None:
            self.head_graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.head_graph):
                self.logits = head_body()
        if dynamic:
            # the eager warm-up steps advanced the counters (and wrote slots >= L that later steps overwrite)
            stage.set_device_length(L, self.pos0)
            stage.set_len(L)
        elif stage.sp is None or stage.sp[0] == stage.sp[1] - 1:
            stage.set_len(L + 1)          # (sp: only the last shard appended a token)

    def replay(self):
        self.graph.replay()
        if self.head_graph is not None:
            self.head_graph.replay()
        if self.dynamic:
            self.steps += 1
            sp = self.stage.sp
            if sp is None or sp[0] == sp[1] - 1:       # host mirror of the device counter (on the rank that appends)
                self.stage.set_len(self.L0 + self.steps)


class BatchedDecoderStage:
    """The layers of a whole-model DecoderStage (same weights) run over B sequences at once (DESIGN.md section 4.10).

    Each layer gets a BatchedLayerCache (the stage's calibration and sinks, one per slot) and every layer shares one
    device length tensor `lens` [B].  A step reads x fp16 [B, hidden]: RMSNorm + the fused QKV projection as one fp16
    matmul, kvq_dec_rope_split_freq (row b at position n_sink + lens[b]), the batched append and attend, o_proj +
    residual and the MLP with the math of DecoderStage.forward_torch / prefill (torch matmuls), then lens += 1 for the
    active slots -- nothing touches the host, so the step can be captured (BatchedGraphedStep).  A slot is filled with
    prefill_seq(b, x) through its sequence views, and retired with reset_seq(b).  The attend of a slot that is not
    active in a step (`active[b] == 0`) still runs, over a slot it did not write: its output row is meaningless.

    Paged (page_size given, DESIGN.md section 4.11): every layer gets a PagedLayerCache over one shared PageTable of
    n_pool pages (default: enough for B full slots); a slot holds pages for the tokens it has, up to the stage's
    max_len rounded up to whole pages.  Change activity with set_active: the graph step keeps a host mirror of the
    mask and the lengths to map pages ahead of each replay without a device synchronisation."""

    def __init__(self, stage: DecoderStage, batch: int, page_size: int = None, n_pool: int = None):
        cfg = stage.cfg
        if stage.sp is not None:
            raise NotImplementedError("a sequence-sharded stage serves one sequence (batch > 1 is not supported)")
        if stage.lo != 0 or stage.hi != cfg.n_layers or not stage.with_head:
            raise NotImplementedError("a layer-pipelined stage serves one sequence (batch > 1 needs the whole model)")
        self.stage, self.cfg, self.B, self.device = stage, cfg, int(batch), stage.device
        self.paged = page_size is not None
        self.pages = None
        if self.paged:
            P = int(page_size)
            max_pages = max(1, -(-stage.layers[0].cache.Lmax // P)) if P > 0 else 1
            self.pages = PageTable(self.B, P, self.B * max_pages if n_pool is None else n_pool, max_pages, self.device)
            self.lens = self.pages.lens
        elif n_pool is not None:
            raise ValueError("n_pool needs a page_size")
        else:
            self.lens = torch.zeros(self.B, dtype=torch.int64, device=self.device)
        self.active = torch.ones(self.B, dtype=torch.int32, device=self.device)
        self.active_host = [True] * self.B
        self.caches = []
        for ly in stage.layers:
            c = ly.cache
            ksub = c.klut_sub if c.klut_sub is not c.klut else None
            if self.paged:
                bc = PagedLayerCache(self.B, c.bits, c.H, c.klut, ksub, c.thr_lower, c.thr_upper, c.v_cent, self.device,
                                     cfg.include_sparse, cfg.sparsity_threshold, c.n_sink, c.v_norm, cfg.sparse_v, c.Hq,
                                     pages=self.pages)
            else:
                bc = BatchedLayerCache(self.B, c.bits, c.H, c.Lmax, c.klut, ksub, c.thr_lower, c.thr_upper, c.v_cent,
                                       self.device, cfg.include_sparse, cfg.sparsity_threshold, c.n_sink, c.v_norm,
                                       cfg.sparse_v, c.Hq, lens=self.lens)
            if c.sink_k is not None:
                bc.set_sinks(c.sink_k[None].expand(self.B, -1, -1, -1).contiguous(),
                             c.sink_v[None].expand(self.B, -1, -1, -1).contiguous())
            self.caches.append(bc)
        self.rope_state = None
        if isinstance(stage.rotary, LengthDependentRotary):   # one state per slot, shared by the layers
            self.rope_state = self.caches[0]._len_state(stage.rotary)
            for bc in self.caches[1:]:
                bc.rope_len_state = self.rope_state
                for b, v in enumerate(getattr(bc, "_views", ())):
                    v.rope_len_state = self.rope_state.slot(b)
        # the layers attend one after another on one stream: one scratch serves them all
        scratch = torch.empty(self.caches[0].lib.kvq_attend_batch_scratch_bytes(self.B, cfg.n_heads, self.caches[0].Lmax),
                              dtype=torch.uint8, device=self.device)
        for bc in self.caches:
            bc._scratch = scratch
        f16, f32 = dict(dtype=torch.float16, device=self.device), dict(dtype=torch.float32, device=self.device)
        B = self.B
        self._q = torch.empty((B, cfg.n_heads, HEAD_DIM), **f32)
        self._k = torch.empty((B, cfg.kv_hidden), **f32)
        self._v = torch.empty((B, cfg.kv_hidden), **f32)
        self._o = torch.empty((B, cfg.n_heads, HEAD_DIM), **f32)

    def reset_seq(self, b):
        """Retire slot b in every layer (length 0 on the host and the device; a paged slot's pages are freed)."""
        for bc in self.caches:
            bc.reset_seq(b)

    def set_active(self, b, on):
        """Slot b takes part in the next steps (appends and advances) or not: device mask and host mirror."""
        self.active[b] = int(bool(on))
        self.active_host[b] = bool(on)

    def prefill_seq(self, b, x, chunk=2048):
        """Run a prompt x fp16 [T, hidden] through the layers into slot b (DecoderStage.prefill on the slot's views),
        then set slot b's device length; the other slots are untouched.  Returns fp16 [T, hidden].
        Paged (DESIGN.md section 4.12): the prompt continues slot b's sequence at its host length -- an empty slot, a
        follow-up turn after graph replays (BatchedGraphedStep keeps the host lengths), or a fork_seq destination --
        and goes through DecoderStage.prefill on the slots' handles (PagedLayerCache.slot), written in place in the
        slot's pages.  The prompt's pages are mapped first, so a prompt past the cap (IndexError) or an exhausted pool
        (RuntimeError) raises before any layer runs.  No recapture is needed."""
        if not self.paged:
            y = self.stage.prefill(x, chunk, caches=[bc.seq(b) for bc in self.caches])
            self.caches[0].commit(b)        # (one shared length tensor)
            return y
        pg = self.pages
        pg.reserve(b, pg.lens_host[pg._slot(b)] + x.shape[0])
        y = self.stage.prefill(x, chunk, caches=[bc.slot(b) for bc in self.caches])
        self.caches[0].commit(b)            # (one shared page table and length tensor)
        return y

    def prefill_seqs(self, prompts, chunk=2048, max_tokens=8192):
        """prefill_seq of several prompts at once (DESIGN.md section 4.15): prompts {slot: fp16 [T_b, hidden]} ->
        {slot: fp16 [T_b, hidden]}, every slot committed.  Each prompt continues its slot at the slot's host length --
        an empty slot, a follow-up turn after graph replays, a fork_seq destination -- and is cut into chunks exactly
        as prefill_seq(b, x, chunk) cuts it.  A round packs the next chunk of as many prompts as fit in max_tokens rows
        (in the mapping's order); per layer and round one RMSNorm + QKV matmul over the packed rows, the per-row query
        rotation, one attend_chunks, one append_chunks, then one o_proj + MLP (DecoderStage._prefill_qkv / _prefill_out).
        So every layer reads its weights once per round instead of once per prompt and chunk.

        The chunks attend through the fused ragged chunk attend, which reads the cache directly; prefill_seq attends
        through attend_chunk (SDPA over a dequantised copy), so the two agree to fp16 rounding, not bit for bit.  A
        prompt past the cap (IndexError), an exhausted pool or a write into a shared page (RuntimeError) raises before
        anything is written or reserved for any slot.  Other slots are untouched and no recapture is needed.
        Length-dependent rotary and the legacy per-token-LUT V form raise NotImplementedError: use prefill_seq."""
        stage, cfg = self.stage, self.cfg
        if isinstance(stage.rotary, LengthDependentRotary):
            raise NotImplementedError("prefill_seqs with length-dependent rotary frequencies needs a frequency table per "
                                      "slot; prefill such prompts one at a time with prefill_seq")
        if not self.caches[0]._tmpl.use_native_v:
            raise NotImplementedError("prefill_seqs reads the native V form; use prefill_seq for the per-token-LUT form")
        chunk, max_tokens = int(chunk), int(max_tokens)
        if chunk < 1 or chunk > max_tokens:
            raise ValueError("need 1 <= chunk <= max_tokens, got chunk=%d, max_tokens=%d" % (chunk, max_tokens))
        H, hid = cfg.n_heads, cfg.hidden
        items = []
        for b, x in prompts.items():
            b = int(b)
            if not 0 <= b < self.B:
                raise IndexError("slot %d out of range [0, %d)" % (b, self.B))
            if x.dtype != torch.float16 or x.dim() != 2 or x.shape[1] != hid:
                raise ValueError("prompt of slot %d must be fp16 [T, %d], got %s %s" % (b, hid, x.dtype, tuple(x.shape)))
            if x.device != self.device:
                raise ValueError("prompt of slot %d is on %s, the stage lives on %s" % (b, x.device, self.device))
            items.append((b, x))
        if len({b for b, _ in items}) != len(items):
            raise ValueError("prompts must name distinct slots")
        bc0 = self.caches[0]
        start = {b: bc0._host_len(b) for b, _ in items}
        for b, x in items:
            if start[b] + x.shape[0] > bc0.Lmax:
                raise IndexError("a prompt of %d tokens does not fit slot %d: %d of %d slots used"
                                 % (x.shape[0], b, start[b], bc0.Lmax))
        if self.paged:    # every page of every prompt, checked together and then mapped, before any layer runs
            bc0._map_chunks([b for b, _ in items], [start[b] for b, _ in items], [x.shape[0] for _, x in items])
        todo = {b: list(range(0, x.shape[0], chunk)) for b, x in items}
        outs = {b: [] for b, _ in items}
        xs = dict(items)
        while any(todo.values()):
            rnd, rows = [], 0
            for b, _ in items:              # the next chunk of every prompt that still fits in this round
                if todo[b]:
                    n = min(chunk, xs[b].shape[0] - todo[b][0])
                    if rows + n <= max_tokens:
                        rnd.append((b, todo[b].pop(0), n))
                        rows += n
            slots, counts = [b for b, _, _ in rnd], [n for _, _, n in rnd]
            starts = [bc0._host_len(b) for b in slots]
            h = torch.cat([xs[b][s0:s0 + n] for b, s0, n in rnd])
            pos = torch.cat([bc0.n_sink + s + torch.arange(n, device=self.device) for s, n in zip(starts, counts)])
            rope = _resolve(stage.rotary, cfg.rope_theta)
            for ly, bc in zip(stage.layers, self.caches):
                q, k, v = stage._prefill_qkv(ly, h)
                q = stage._rope_rows(q.reshape(rows, H, HEAD_DIM), pos).contiguous()
                o = bc._attend_chunks_at(slots, starts, q, k, v, counts, rope)
                bc._append_chunks_at(slots, starts, k, v, counts)
                h = stage._prefill_out(ly, h, o)
            for b, s, n in zip(slots, starts, counts):
                for bc in (self.caches if not self.paged else self.caches[:1]):   # (paged: one shared table)
                    bc._set_host_len(b, s + n)
            for (b, _, _), y in zip(rnd, h.split(counts)):
                outs[b].append(y)
        for b, x in items:
            self.caches[0].commit(b)        # (one shared length tensor)
        return {b: torch.cat(outs[b]) if outs[b] else x.clone() for b, x in items}

    def fork_seq(self, src, dst):
        """Paged: slot dst continues from slot src's current tokens, sharing its full pages in every layer and
        copying its partial last page (PageTable.fork).  dst must be empty; prefill_seq(dst, suffix) then continues
        it (one shared prompt prefix, several suffixes)."""
        if not self.paged:
            raise NotImplementedError("fork_seq shares pages: it needs a paged stage")
        self.pages.fork(src, dst)

    def map_next(self):
        """Paged: map the pages every active slot needs for its next token, from the host mirror of the lengths (no
        device synchronisation); before a step or graph replay."""
        pg = self.pages
        for b in range(self.B):
            if self.active_host[b]:
                pg.reserve(b, min(pg.lens_host[b] + 1, pg.cap))

    def advance_host(self):
        """Paged: the host mirror of one step's lens += active (a slot at the cap stays there)."""
        pg = self.pages
        for b in range(self.B):
            if self.active_host[b]:
                pg.lens_host[b] = min(pg.lens_host[b] + 1, pg.cap)

    def forward(self, x):
        """x fp16 [B, hidden] -> fp16 [B, hidden]; appends one token to every active slot of every layer."""
        from . import _lib
        cfg, B = self.cfg, self.B
        lib = _lib.load()
        st = torch.cuda.current_stream().cuda_stream
        hid = cfg.hidden
        rot = self.stage.rotary
        if self.rope_state is not None:   # every slot's f(s) and table, once for every layer of the step
            bc0 = self.caches[0]
            rot = self.rope_state.update(len_dev=self.lens, len_add=1, L_cap=bc0.Lmax, pos_offset=bc0.n_sink)
        for ly, bc in zip(self.stage.layers, self.caches):
            qkv = (rmsnorm(x, ly.n1, cfg.rms_eps) @ ly.wqkv.t()).contiguous()
            if isinstance(rot, RopeLenState):   # row b at its own frequencies
                fn, freq, attn = "kvq_dec_rope_split_freq_seq", rot.f_cur, rot.spec.attention_factor
            else:
                fn, freq = "kvq_dec_rope_split_freq", self.stage.inv_freq
                attn = rot.attention_factor if rot is not None else 1.0
            _lib.check(getattr(lib, fn)(qkv.data_ptr(), freq.data_ptr(), attn, self.lens.data_ptr(), bc.n_sink,
                                        self._q.data_ptr(), self._k.data_ptr(), self._v.data_ptr(), cfg.n_heads,
                                        cfg.kv_heads, B, st), fn)
            bc.append_dyn(self._k, self._v, active=self.active)
            o = bc.attend(self._q, out=self._o, len_add=1, rope_theta=cfg.rope_theta, rope=rot)
            x = x + o.half().view(B, hid) @ ly.wo.t()
            gu = rmsnorm(x, ly.n2, cfg.rms_eps) @ ly.wgu.t()
            g, u = gu.split(cfg.intermediate, dim=-1)
            x = x + (torch.nn.functional.silu(g) * u) @ ly.wdown.t()
        self.caches[0].advance(active=self.active)
        return x

    def logits(self, x):
        """fp16 [B, vocab] = lm_head(RMSNorm(x)) of every row."""
        return rmsnorm(x, self.stage.norm, self.cfg.rms_eps) @ self.stage.lm_head.t()


class BatchedGraphedStep:
    """One batched decode step captured in a CUDA graph: tokens `tok` [B] -> `logits` [B, vocab].  Every replay is
    the next step of every active slot (lengths advance on the device).  Between replays the host may retire a slot
    and prefill a new prompt into it (BatchedDecoderStage.reset_seq / prefill_seq); the next replay decodes it from
    its prompt, with no recapture."""

    def __init__(self, bstage: BatchedDecoderStage):
        """Paged stage: each replay first maps the pages every active slot needs for its next token (map_next, from
        the host mirror of the lengths, advanced per replay), so slots cross page boundaries without a recapture."""
        self.bstage = bstage
        st = bstage.stage
        self.tok = torch.zeros(bstage.B, dtype=torch.long, device=bstage.device)

        def body():
            return bstage.logits(bstage.forward(st.embed[self.tok]))
        if bstage.paged:
            bstage.map_next()      # (the warm-up step writes the next slot of every active sequence)
        lens = bstage.lens.clone()
        s = torch.cuda.Stream(device=bstage.device)     # warm-up: scratch, rope tables, cuBLAS handles
        s.wait_stream(torch.cuda.current_stream(bstage.device))
        with torch.cuda.stream(s):
            body()
        torch.cuda.current_stream(bstage.device).wait_stream(s)
        torch.cuda.synchronize(bstage.device)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.logits = body()
        bstage.lens.copy_(lens)      # the warm-up step wrote slots that the first replay overwrites

    def replay(self):
        if self.bstage.paged:
            self.bstage.map_next()
        self.graph.replay()
        if self.bstage.paged:
            self.bstage.advance_host()


def layer_step_bytes(cfg: DecodeConfig, L: int):
    """Algorithmic HBM bytes of one layer's fused attend at cache length L (SURVEY.md 8d); the cache holds the KV
    heads (grouped-query models: cfg.kv_hidden < cfg.hidden)."""
    n_out = 2 * (int(((1 - cfg.sparsity_threshold) / 2) * cfg.kv_hidden) + 1)
    n_sparse = (2 if cfg.sparse_v else 1) if cfg.include_sparse else 0
    per_tok = 2 * cfg.kv_hidden * cfg.bits // 8 + 4 * 2 ** cfg.bits + 8 * n_out * n_sparse
    return L * per_tok


class PipelineDecoder:
    """Layer-group pipeline over torch.distributed (one process per GPU; NCCL P2P of the hidden vector).
    Works with world_size == 1 (no communication) and, for host-logic tests, on the gloo backend with CPU
    tensors when `stage_fn` is supplied instead of a CUDA stage."""

    def __init__(self, rank, world, hidden, dtype, device, stage_fn, head_fn=None, embed_fn=None, group=None):
        self.rank, self.world = rank, world
        self.stage_fn, self.head_fn, self.embed_fn = stage_fn, head_fn, embed_fn
        self.buf = torch.zeros(hidden, dtype=dtype, device=device)
        self.group = group

    def step(self, tok):
        """One decode step.  rank 0: embeds `tok`, runs its layers, sends on; rank r: recv, layers, send;
        the last rank sends the final hidden state back to rank 0, which applies norm + lm_head.
        Returns logits on rank 0, None elsewhere."""
        import torch.distributed as dist
        w, r = self.world, self.rank
        if r == 0:
            x = self.embed_fn(tok)
        else:
            dist.recv(self.buf, src=r - 1, group=self.group)
            x = self.buf
        y = self.stage_fn(x)
        if w > 1:
            dist.send(y.contiguous(), dst=(r + 1) % w, group=self.group)
            if r == 0:
                dist.recv(self.buf, src=w - 1, group=self.group)
                y = self.buf
        return self.head_fn(y) if r == 0 else None
