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

from .cache import LayerCache, HEAD_DIM


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

    @staticmethod
    def llama7b(**kw):
        return DecodeConfig(32, 4096, 32, 11008, 32000, **kw)

    @staticmethod
    def llama13b(**kw):
        return DecodeConfig(40, 5120, 40, 13824, 32000, **kw)


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
        self.wqkv = w(3 * h, h)
        self.wo = w(h, h)
        self.wgu = w(2 * it, h)
        self.wdown = w(h, it)
        self.n1 = torch.ones(h, dtype=torch.float16, device=device)
        self.n2 = torch.ones(h, dtype=torch.float16, device=device)
        self.cache = LayerCache.from_luts(cfg.bits, cfg.n_heads, cfg.max_len, quantizer["klut"], quantizer["v_cent"],
                                          device=device, include_sparse=cfg.include_sparse,
                                          sparsity_threshold=cfg.sparsity_threshold, n_sink=cfg.n_sink,
                                          sparse_v=cfg.sparse_v)
        self.cache.share_scratch = True     # the layers of a stage attend one after another on one stream
        if cfg.n_sink and with_sinks:
            sk = (torch.randn((cfg.n_heads, HEAD_DIM, cfg.n_sink), generator=gen, device=device)).half()
            sv = (torch.randn((cfg.n_heads, cfg.n_sink, HEAD_DIM), generator=gen, device=device)).half()
            self.cache.set_sinks(sk, sv)


class DecoderStage:
    """Layers [lo, hi) of the model on one device, plus (first stage) the embedding and (rank 0) norm + lm_head."""

    def __init__(self, cfg: DecodeConfig, lo: int, hi: int, device, quantizer, seed=0, with_head=True, sp=None):
        """sp = (rank, world) switches to SEQUENCE-sharded attention (SURVEY 8e-2 / 8f-1): every rank holds all layers'
        weights and a contiguous 1/world slice of every layer's cache; per layer the partial (out, lse) results are
        all-gathered (H*129 floats per rank over NVLink) and merged.  The new token is appended on the last rank."""
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
        self.inv_freq = 1.0 / (cfg.rope_theta ** (torch.arange(0, HEAD_DIM, 2, device=self.device).float() / HEAD_DIM))
        self._half = half

    # -- pieces -------------------------------------------------------------------------------------------------
    def embed_token(self, tok):
        return self.embed[tok].view(-1)

    def head(self, x):
        if x.is_cuda:
            return self._gemv(self.lm_head, x, 3, self._buffers()["logits"], norm_w=self.norm)
        return self.lm_head @ rmsnorm(x, self.norm, self.cfg.rms_eps)

    def _rope_q(self, q, pos):
        """HF rotate-half RoPE on the query only (modeling_llama.py:1851-1859); q f32 [H,128]."""
        ang = self.inv_freq * float(pos)
        cos = torch.cat((ang.cos(), ang.cos()))
        sin = torch.cat((ang.sin(), ang.sin()))
        rot = torch.cat((-q[:, self._half:], q[:, :self._half]), dim=-1)
        return q * cos + rot * sin

    def _buffers(self):
        if getattr(self, "_buf", None) is None:
            cfg, dev = self.cfg, self.device
            f16 = dict(dtype=torch.float16, device=dev)
            f32 = dict(dtype=torch.float32, device=dev)
            self._buf = dict(h=torch.empty(cfg.hidden, **f16), qkv=torch.empty(3 * cfg.hidden, **f16),
                             q=torch.empty(cfg.hidden, **f32), k=torch.empty(cfg.hidden, **f32),
                             v=torch.empty(cfg.hidden, **f32), o16=torch.empty(cfg.hidden, **f16),
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
        for ly in self.layers:
            c = ly.cache
            dyn = self.dyn          # device-resident length / position (one graph for a growing cache) or None
            self._gemv(ly.wqkv, x, 3, b["qkv"], norm_w=ly.n1)
            if dyn is None:
                # absolute position of the new token
                pos = self.global_pos if self.sp is not None else c.n_sink + c.pos_base + c.len
                _lib.check(lib.kvq_dec_rope_split(b["qkv"].data_ptr(), self.inv_freq.data_ptr(), float(pos),
                                                  b["q"].data_ptr(), b["k"].data_ptr(), b["v"].data_ptr(), hid, st))
            else:
                _lib.check(lib.kvq_dec_rope_split_dyn(b["qkv"].data_ptr(), self.inv_freq.data_ptr(),
                                                      dyn["pos"].data_ptr(), 0, b["q"].data_ptr(), b["k"].data_ptr(),
                                                      b["v"].data_ptr(), hid, st))
            qh = b["q"].view(H, HEAD_DIM)
            if self.sp is None:
                if dyn is None:
                    c.append(b["k"], b["v"])             # pre-RoPE K, per-token V: quantise + outlier split
                    o = c.attend(qh, rope_theta=cfg.rope_theta)   # f32 [H,128]
                else:
                    c.append_dyn(b["k"], b["v"], dyn["len"])
                    o = c.attend_dyn(qh, dyn["len"], 1, rope_theta=cfg.rope_theta)
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
            q, k, v = qkv.float().split(cfg.hidden)
            q = self._rope_q(q.view(H, HEAD_DIM), pos).contiguous()
            c.append(k.contiguous(), v.contiguous())
            o = c.attend(q, rope_theta=cfg.rope_theta)
            x = x + ly.wo @ o.half().view(-1)
            gu = ly.wgu @ rmsnorm(x, ly.n2, cfg.rms_eps)
            g, u = gu.split(cfg.intermediate)
            x = x + ly.wdown @ (torch.nn.functional.silu(g) * u)
        return x

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


def layer_step_bytes(cfg: DecodeConfig, L: int):
    """Algorithmic HBM bytes of one layer's fused attend at cache length L (SURVEY.md 8d)."""
    n_out = 2 * (int(((1 - cfg.sparsity_threshold) / 2) * cfg.hidden) + 1)
    n_sparse = (2 if cfg.sparse_v else 1) if cfg.include_sparse else 0
    per_tok = 2 * cfg.hidden * cfg.bits // 8 + 4 * 2 ** cfg.bits + 8 * n_out * n_sparse
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
