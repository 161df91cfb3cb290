"""CPU: the argument checks of the six fused-attend entry points and the scratch size they share.

Every call here is rejected from its arguments alone, before anything touches a device, so dummy non-null pointers
are enough and no GPU is needed.  The codes are part of the C ABI: an input with several faults gets the code of the
first check it fails, and that order differs between the single-sequence and the batched entry points.
"""
import ctypes

import pytest

from kvquant_b200 import _lib

E_BITS, E_SHAPE, E_NULL, E_ALIGN, E_UNSUPPORTED = -1, -2, -3, -4, -5
P = ctypes.c_void_p(256)            # never dereferenced
ODD = ctypes.c_void_p(264)          # 8-byte aligned only
SINGLE = ["kvq_attend", "kvq_attend_dyn", "kvq_attend_gqa", "kvq_attend_gqa_dyn"]
BATCHED = ["kvq_attend_batch", "kvq_attend_paged"]
ALL = SINGLE + BATCHED
WITH_KV_HEADS = ["kvq_attend_gqa", "kvq_attend_gqa_dyn"] + BATCHED

DEFAULTS = dict(bits=4, B=2, q=P, kcache=P, klut=P, ko=None, koi=None, vcache=P, vlut=P, vcent=P, vaff=P, vo=None,
                voi=None, n_out=42, Hq=32, Hkv=None, Lmax=640, L=640, len_dev=P, len_add=0, rope=P, npos=4096,
                pos=0, sink_k=None, sink_v=None, n_sink=0, out=P, lse=None, scratch=P, rope_half=None,
                n_pool=8, table=P, max_pages=4, npages=P, page=160)


def call(fn, **kw):
    """Return code of entry point `fn` for DEFAULTS overridden by kw.  Hkv defaults to Hq / 4 where the entry point has
    KV heads of its own (kvq_attend and kvq_attend_dyn take one head count)."""
    a = dict(DEFAULTS, **kw)
    if a["Hkv"] is None:
        a["Hkv"] = a["Hq"] // 4 if fn in WITH_KV_HEADS else a["Hq"]
    lib = _lib.load()
    k = (a["kcache"], a["klut"], a["ko"], a["koi"], a["vcache"])
    v = (a["vcent"], a["vaff"], a["vo"], a["voi"], a["n_out"])
    heads = (a["Hq"], a["Hkv"]) if fn in WITH_KV_HEADS else (a["Hq"],)
    tail = (a["rope"], a["npos"], 10000.0, a["pos"], a["sink_k"], a["sink_v"], a["n_sink"], a["out"], a["lse"],
            a["scratch"], a["rope_half"], None)
    dyn = (a["len_dev"], a["len_add"])
    if fn in ("kvq_attend", "kvq_attend_gqa"):
        return getattr(lib, fn)(a["bits"], a["q"], *k, a["vlut"], *v, *heads, a["Lmax"], a["L"], *tail)
    if fn in ("kvq_attend_dyn", "kvq_attend_gqa_dyn"):
        return getattr(lib, fn)(a["bits"], a["q"], *k, *v, *heads, a["Lmax"], a["L"], *dyn, *tail)
    if fn == "kvq_attend_batch":
        return lib.kvq_attend_batch(a["bits"], a["B"], a["q"], *k, *v, *heads, a["Lmax"], a["L"], *dyn, *tail)
    assert fn == "kvq_attend_paged"
    return lib.kvq_attend_paged(a["bits"], a["B"], a["q"], *k, *v, *heads, a["n_pool"], a["L"], *dyn, *tail,
                                a["table"], a["max_pages"], a["npages"], a["page"])


@pytest.mark.parametrize("fn", ALL)
def test_negative_position_misalignment_and_bits_are_rejected(fn):
    """A negative pos_offset would index the rope table below its start; kcache and scratch are read with 16-byte
    accesses; bits outside 2..4 has no kernel.  Every entry point says so before it launches anything."""
    assert call(fn, pos=-1) == E_SHAPE
    assert call(fn, pos=-1, L=100, npos=99) == E_SHAPE       # rope_npos >= L + pos_offset holds, the offset is still bad
    assert call(fn, kcache=ODD) == E_ALIGN
    assert call(fn, scratch=ODD) == E_ALIGN
    assert call(fn, bits=5) == E_BITS and call(fn, bits=1) == E_BITS
    assert call(fn, kcache=ODD, bits=5) == (E_BITS if fn in BATCHED else E_ALIGN)


@pytest.mark.parametrize("fn", SINGLE)
def test_multi_head_attention_through_the_gqa_entry_points_gets_the_same_checks(fn):
    assert call(fn, Hkv=32, pos=-1) == E_SHAPE
    assert call(fn, Hkv=32, kcache=ODD) == E_ALIGN
    assert call(fn, Hkv=32, bits=5) == E_BITS


@pytest.mark.parametrize("fn", ALL)
def test_rejections_every_entry_point_shares(fn):
    assert call(fn, q=None) == E_NULL
    assert call(fn, out=None) == E_NULL and call(fn, rope=None) == E_NULL
    assert call(fn, Hq=30, Hkv=30) == E_SHAPE                # heads not a multiple of 4
    assert call(fn, Hq=68, Hkv=68) == E_SHAPE                # more than 64 heads
    assert call(fn, L=644) == E_SHAPE                        # L > Lmax (a paged batch: > max_pages * P)
    assert call(fn, n_sink=65, sink_k=P, sink_v=P) == E_SHAPE
    assert call(fn, n_sink=2) == E_SHAPE                     # sinks counted but not given
    assert call(fn, ko=P) == E_NULL and call(fn, voi=P) == E_NULL     # outlier values and indices come in pairs
    assert call(fn, ko=P, koi=P, n_out=0) == E_SHAPE
    assert call(fn, npos=639) == E_SHAPE                     # rope table shorter than L + pos_offset
    assert call(fn, vcache=ODD) == E_ALIGN


@pytest.mark.parametrize("fn", WITH_KV_HEADS)
def test_grouped_query_rejections(fn):
    assert call(fn, Hq=32, Hkv=12) == E_SHAPE                # Hq % Hkv
    assert call(fn, Hq=32, Hkv=6) == E_SHAPE                 # Hkv % 4
    assert call(fn, Hq=32, Hkv=0) == E_SHAPE
    assert call(fn, vcent=None) == E_UNSUPPORTED             # grouped queries read the native V form ...
    assert call(fn, rope_half=P) == E_UNSUPPORTED            # ... and the exact K tables


def test_entry_point_preconditions():
    assert call("kvq_attend", Lmax=642, L=640) == E_ALIGN    # Lmax % 4
    assert call("kvq_attend", vcent=None, vlut=None) == E_NULL
    assert call("kvq_attend", L=0) == E_SHAPE                # nothing to attend: no slot and no sink
    for fn in ("kvq_attend_dyn", "kvq_attend_gqa_dyn"):
        assert call(fn, len_dev=None) == E_NULL
        assert call(fn, L=0) == E_SHAPE
        assert call(fn, Hkv=32, vcent=None) == E_NULL        # the device-length forms need the native V form
    for fn in BATCHED:
        assert call(fn, B=0) == E_SHAPE and call(fn, B=257) == E_SHAPE
        assert call(fn, len_dev=None) == E_NULL and call(fn, L=0) == E_SHAPE
        assert call(fn, Hkv=32, vcent=None) == E_UNSUPPORTED
    assert call("kvq_attend_paged", table=None) == E_NULL and call("kvq_attend_paged", npages=None) == E_NULL
    assert call("kvq_attend_paged", page=100) == E_SHAPE and call("kvq_attend_paged", n_pool=0) == E_SHAPE


def test_first_failed_check_decides_the_code():
    """Inputs with two faults: the single-sequence entry points report pointers and shapes ahead of bits and the
    kcache / scratch alignment, the batched ones report bits first and the alignment ahead of the outlier pairs."""
    for fn in SINGLE:
        assert call(fn, bits=5, q=None) == E_NULL
        assert call(fn, bits=5, L=644) == E_SHAPE
        assert call(fn, kcache=ODD, ko=P) == E_NULL
        assert call(fn, kcache=ODD, n_sink=65, sink_k=P, sink_v=P) == E_SHAPE
    assert call("kvq_attend", q=None, Hq=30) == E_NULL
    assert call("kvq_attend_gqa", q=None, Hq=30, Hkv=30) == E_SHAPE
    assert call("kvq_attend_dyn", len_dev=None, Hq=30) == E_NULL
    assert call("kvq_attend_gqa_dyn", len_dev=None, vcent=None) == E_UNSUPPORTED
    for fn in BATCHED:
        assert call(fn, bits=5, q=None) == E_BITS
        assert call(fn, bits=5, vcent=None) == E_BITS
        assert call(fn, bits=5, Hq=30) == E_SHAPE
        assert call(fn, vcent=None, q=None) == E_UNSUPPORTED
        assert call(fn, kcache=ODD, ko=P) == E_ALIGN
        assert call(fn, kcache=ODD, q=None) == E_NULL
        assert call(fn, kcache=ODD, L=644) == E_SHAPE


def _scratch_bytes(H, L):
    """The layout of one sequence's scratch, in floats: score rows, per-head max, sink scores, 256 partial (o, l)
    rows, the 4-bit K table with its ratios; 256 bytes of slack."""
    r32 = lambda x: (x + 31) // 32 * 32     # noqa: E731
    floats = H * r32(L) + H + H * 64 + 256 * H * 128 + 256 * H + H * 128 * 17
    return 4 * floats + 256


def test_scratch_bytes_closed_form():
    lib = _lib.load()
    for H in range(4, 65, 4):
        for L in (1, 31, 32, 33, 200, 1000, 4096, 32768, 131072, 1 << 20):
            want = _scratch_bytes(H, L)
            assert lib.kvq_attend_scratch_bytes(H, L) == want, (H, L)
            assert want % 16 == 0
            for B in (1, 3, 256):
                assert lib.kvq_attend_batch_scratch_bytes(B, H, L) == B * want, (B, H, L)
    assert lib.kvq_attend_batch_scratch_bytes(0, 32, 4096) == 0 and lib.kvq_attend_batch_scratch_bytes(257, 32, 4096) == 0
    assert lib.kvq_attend_batch_scratch_bytes(2, 0, 4096) == 0 and lib.kvq_attend_batch_scratch_bytes(2, 32, 0) == 0
