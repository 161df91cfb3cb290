"""CPU: the argument checks of the ragged chunk append and attend (kvq_append_kv_fused_chunk_ragged[_paged],
kvq_attend_chunk_ragged[_paged]) and the scratch size of the ragged attend.

Every call here is decided on the host before anything touches a device: the segment table and the paged forms'
mapped counts are host arrays the entry points read, and the data pointers are dummies that are never dereferenced.
An input with several faults gets the code of the first check it fails.
"""
import ctypes

import numpy as np

from kvquant_b200 import _lib

E_BITS, E_SHAPE, E_NULL, E_ALIGN = -1, -2, -3, -4
P = ctypes.c_void_p(256)            # never dereferenced
ODD = ctypes.c_void_p(264)          # 8-byte aligned only


def _segs(*rows):
    """(b, s0, T) per segment -> int64 [n, 4] with rows packed in order."""
    out, row = [], 0
    for b, s0, t in rows:
        out.append((b, s0, t, row))
        row += t
    return np.ascontiguousarray(np.asarray(out, dtype=np.int64).reshape(-1, 4))


def _ptr(a):
    return a.ctypes.data if a is not None else None


def append(segs, N=None, bits=4, B=4, H=8, Lmax=640, n_each=21, k_new=P, klut=P, paged=False, n_mapped=None,
           n_pool=16, max_pages=4, page=160, table=P):
    lib = _lib.load()
    N = int(segs[:, 2].sum()) if N is None and segs is not None else (N or 0)
    n_seg = len(segs) if segs is not None else 1
    data = (n_each, k_new, P, klut) + (P,) * 13 + (None,)
    if not paged:
        return lib.kvq_append_kv_fused_chunk_ragged(bits, B, H, Lmax, n_seg, _ptr(segs), N, *data)
    return lib.kvq_append_kv_fused_chunk_ragged_paged(bits, B, H, n_pool, n_seg, _ptr(segs), N, *data, table,
                                                      max_pages, _ptr(n_mapped), page)


def attend(segs, N=None, bits=4, B=4, Hq=32, Hkv=8, Lmax=640, q=P, scratch=P, npos=4096, pos=0, paged=False,
           n_mapped=None, n_pool=16, max_pages=4, page=160):
    lib = _lib.load()
    N = int(segs[:, 2].sum()) if N is None and segs is not None else (N or 0)
    n_seg = len(segs) if segs is not None else 1
    data = (q, P, P, P, P, None, None, P, P, P, None, None, 42, P, npos, pos, None, None, 0, P, scratch, None)
    if not paged:
        return lib.kvq_attend_chunk_ragged(bits, B, Hq, Hkv, Lmax, n_seg, _ptr(segs), N, *data)
    return lib.kvq_attend_chunk_ragged_paged(bits, B, Hq, Hkv, n_pool, n_seg, _ptr(segs), N, *data, P, max_pages,
                                             _ptr(n_mapped), page)


def test_append_table_checks_and_their_order():
    good = _segs((2, 5, 9), (0, 0, 300), (3, 17, 0))
    assert append(good, k_new=None) == E_NULL                     # a valid table reaches the pointer checks
    assert append(good, klut=ODD) == E_ALIGN
    assert append(good, N=0) == E_SHAPE                           # rows do not add up to N
    assert append(None) == E_NULL                                 # no table
    assert append(_segs((1, 0, 4), (1, 8, 4))) == E_SHAPE         # a slot named twice
    assert append(_segs((4, 0, 4))) == E_SHAPE                    # a slot outside [0, B)
    assert append(_segs((0, 600, 41))) == E_SHAPE                 # past Lmax
    assert append(_segs((0, -1, 4))) == E_SHAPE
    bad_rows = _segs((0, 0, 4), (1, 0, 4))
    bad_rows[1, 3] = 3
    assert append(bad_rows) == E_SHAPE                            # rows not packed in segment order
    assert append(_segs((0, 0, 4), (1, 0, 4), (2, 0, 4), (3, 0, 4)), B=3) == E_SHAPE   # more segments than slots
    assert append(_segs((0, 600, 41)), bits=5) == E_SHAPE         # the table before bits
    assert append(good, bits=5) == E_BITS
    assert append(None, H=0) == E_SHAPE                           # sizes before the table
    assert append(_segs((0, 0, 4)), Lmax=642) == E_SHAPE          # batch strides keep Lmax % 4 == 0
    assert append(_segs((0, 0, 0), (1, 3, 0)), k_new=None, klut=ODD) == 0   # N == 0: nothing to do


def test_append_paged_checks():
    segs = _segs((1, 100, 100), (0, 0, 160))
    mapped = np.asarray([2, 1], dtype=np.int32)
    assert append(segs, paged=True, n_mapped=mapped, k_new=None) == E_NULL
    assert append(segs, paged=True, n_mapped=None) == E_NULL
    assert append(segs, paged=True, n_mapped=np.asarray([1, 1], dtype=np.int32)) == E_SHAPE   # 200 > 1 page
    assert append(segs, paged=True, n_mapped=np.asarray([2, 5], dtype=np.int32)) == E_SHAPE   # > max_pages
    assert append(None, paged=True, page=100) == E_SHAPE          # page geometry first
    assert append(segs, paged=True, n_mapped=mapped, table=None) == E_NULL


def test_attend_checks_and_their_order():
    good = _segs((2, 5, 9), (0, 0, 300), (3, 2000 - 640, 0))
    assert attend(good, Lmax=2000, q=None) == E_NULL
    assert attend(good, Lmax=2000, q=ODD) == E_ALIGN
    assert attend(good, Lmax=2000, npos=1360 - 1) == E_SHAPE      # the table does not cover the largest s0
    assert attend(good, Lmax=2000, npos=1360, q=None) == E_NULL
    assert attend(None, bits=5) == E_BITS                         # bits first, as kvq_attend_chunk
    assert attend(None) == E_NULL
    assert attend(_segs((1, 0, 4), (1, 8, 4))) == E_SHAPE
    assert attend(_segs((0, 0, 4)), Hkv=3) == E_SHAPE
    assert attend(_segs((0, 0, 4)), pos=-1) == E_SHAPE
    assert attend(_segs((0, 0, 0)), q=None, scratch=ODD) == 0     # N == 0


def test_attend_paged_reads_only_the_first_s0_slots():
    segs = _segs((0, 100, 300))                                   # 100 cached tokens in one mapped page
    one = np.asarray([1], dtype=np.int32)
    assert attend(segs, paged=True, n_mapped=one, q=None) == E_NULL   # s0 mapped: valid, the chunk is not written
    assert attend(_segs((0, 161, 3)), paged=True, n_mapped=one) == E_SHAPE
    assert attend(segs, paged=True, n_mapped=None) == E_NULL
    assert attend(_segs((0, 600, 100)), paged=True, n_mapped=np.asarray([4], dtype=np.int32)) == E_SHAPE   # cap 640


def test_ragged_scratch_is_the_sum_of_the_lone_calls():
    lib = _lib.load()
    segs = _segs((2, 2000, 50), (0, 0, 131), (3, 7, 0), (1, 317, 260))
    want = sum(lib.kvq_attend_chunk_scratch_bytes(32, int(t), int(s0)) for _, s0, t, _ in segs if t > 0)
    assert lib.kvq_attend_chunk_ragged_scratch_bytes(32, len(segs), segs.ctypes.data) == want > 0
    assert lib.kvq_attend_chunk_ragged_scratch_bytes(32, 1, None) == 0
