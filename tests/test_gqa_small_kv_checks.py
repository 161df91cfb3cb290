"""The shape rule of two-KV-head and multi-query caches, without a GPU: H_kv in {1, 2} or H_kv % 4 == 0, with
H_q % 4 == 0, H_q <= 64 and H_q % H_kv == 0; everything else is KVQ_E_SHAPE at the C ABI and ValueError in the cache
constructors.  The paths grouped-query attention does not cover stay refused at one KV head.
"""
import ctypes

import numpy as np
import pytest

import test_gpu_gqa as G

E_SHAPE = -2
E_UNSUPPORTED = -5
REJECTED = [(24, 3), (12, 6), (30, 2), (68, 1)]
ACCEPTED = [(8, 1), (32, 1), (64, 1), (12, 2), (16, 2), (32, 2), (64, 2)]


def _lib():
    from kvquant_b200 import _lib
    return _lib.load()


def _dequant_rc(H):
    p = ctypes.c_void_p(16)
    # stop < start: a shape error once H passes, so an accepted H reaches the range check and nothing is launched
    return _lib().kvq_dequant_kv(4, H, 1024, 5, 4, p, p, None, None, p, p, p, None, None, 0, None, 0, 0, p, p, 1024,
                                 None)


def _append_batch_rc(H):
    p = ctypes.c_void_p(16)
    # B = 0: past the shape checks, an accepted H still fails on the batch size
    return _lib().kvq_append_kv_fused_batch(4, 0, H, 64, p, 0, None, 1, p, p, p, p, p, p, p, p, p, p, p, p, p, p, p,
                                            p, None)


@pytest.mark.parametrize("fn_name", ["kvq_attend_gqa", "kvq_attend_gqa_dyn", "kvq_attend_chunk_gqa"])
@pytest.mark.parametrize("Hq,Hkv", REJECTED)
def test_abi_rejects_head_counts_outside_the_rule(fn_name, Hq, Hkv):
    assert G._abi_rc(fn_name, Hq, Hkv) == E_SHAPE


@pytest.mark.parametrize("Hq,Hkv", REJECTED)
def test_layer_cache_rejects_head_counts_outside_the_rule(Hq, Hkv):
    from kvquant_b200.cache import LayerCache
    n = Hkv * 128
    klut = dict(lut=np.zeros((n, 16), np.float32), thr_lower=np.zeros(n, np.float32), thr_upper=np.ones(n, np.float32))
    with pytest.raises(ValueError):
        LayerCache.from_luts(4, Hkv, 64, klut, np.arange(16, dtype=np.float32), device="cpu", q_heads=Hq)


@pytest.mark.parametrize("Hq,Hkv", ACCEPTED)
def test_layer_cache_accepts_one_and_two_kv_heads(Hq, Hkv):
    from kvquant_b200.cache import LayerCache
    n = Hkv * 128
    klut = dict(lut=np.zeros((n, 16), np.float32), thr_lower=np.zeros(n, np.float32), thr_upper=np.ones(n, np.float32))
    lc = LayerCache.from_luts(4, Hkv, 64, klut, np.arange(16, dtype=np.float32), device="cpu", q_heads=Hq)
    assert (lc.H, lc.Hq, lc.group, lc.n_out) == (Hkv, Hq, Hq // Hkv, 2 * Hkv)


def test_dequant_and_batched_append_take_one_and_two_kv_heads_only():
    for H in (1, 2, 4, 8):
        assert _dequant_rc(H) == E_SHAPE        # (the slot range)
        assert _append_batch_rc(H) == E_SHAPE   # (B = 0)
    for H in (3, 6, 30):
        assert _dequant_rc(H) == E_SHAPE
        assert _append_batch_rc(H) == E_SHAPE


def test_unsupported_forms_stay_refused_at_one_kv_head():
    """fp16 tables and the per-token-LUT V form at the C ABI; the sequence-sharded stage in the decode harness."""
    p = ctypes.c_void_p(16)
    lib = _lib()
    # rope_half given (fp16 tables)
    rc = lib.kvq_attend_gqa(4, p, p, p, p, p, p, None, p, p, p, p, 2, 32, 1, 1024, 10, p, 2048, 10000.0, 0, None,
                            None, 0, p, None, p, p, None)
    assert rc == E_UNSUPPORTED
    # the per-token-LUT V form (vlut_tok, no v_cent / v_aff)
    rc = lib.kvq_attend_gqa(4, p, p, p, p, p, p, p, None, None, p, p, 2, 32, 1, 1024, 10, p, 2048, 10000.0, 0, None,
                            None, 0, p, None, p, None, None)
    assert rc == E_UNSUPPORTED
    from kvquant_b200 import decode as kd
    cfg = kd.DecodeConfig(n_layers=1, hidden=2048, n_heads=16, n_kv_heads=1, intermediate=5632, max_len=64)
    with pytest.raises(NotImplementedError):
        kd.DecoderStage(cfg, 0, 1, "cpu", None, sp=(0, 2))
