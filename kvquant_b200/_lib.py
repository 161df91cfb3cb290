"""ctypes binding of libkvquant_b200.so (the C ABI declared in include/kvquant_b200.h).

The product path has NO CPU fallback: if the shared object is missing or an entry point fails, this raises.
"""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libkvquant_b200.so")

_c_int = ctypes.c_int
_c_i64 = ctypes.c_int64
_c_f = ctypes.c_float
_p = ctypes.c_void_p

# name -> (restype, argtypes); mirrors include/kvquant_b200.h one to one
SIGNATURES = {
    "kvq_abi_version": (_c_int, []),
    "kvq_error_string": (ctypes.c_char_p, [_c_int]),
    "kvq_launch_count": (ctypes.c_uint64, []),
    "kvq_append_k": (_c_int, [_c_int, _p, _p, _p, _c_int, _c_i64, _c_i64, _p]),
    "kvq_append_v": (_c_int, [_c_int, _p, _p, _p, _c_int, _c_i64, _c_i64, _p]),
    "kvq_append_k_sparse": (_c_int, [_c_int, _p, _p, _p, _p, _p, _p, _c_int, _c_i64, _c_i64, _p]),
    "kvq_append_v_sparse": (_c_int, [_c_int, _p, _p, _p, _c_f, _c_f, _c_f, _c_int, _c_i64, _c_i64, _p]),
    "kvq_append_k_sparse_parallel": (_c_int, [_c_int, _p, _p, _p, _p, _p, _p, _c_int, _c_i64, _c_i64, _p]),
    "kvq_append_v_sparse_parallel": (_c_int, [_c_int, _p, _p, _p, _p, _p, _c_int, _c_i64, _c_i64, _p]),
    "kvq_rope_table_build": (_c_int, [_p, _c_f, _c_i64, _p]),
    "kvq_rope_table_build_half": (_c_int, [_p, _c_f, _c_i64, _p]),
    "kvq_k_matvec": (_c_int, [_c_int, _p, _p, _p, _p, _c_int, _c_int, _c_i64, _c_i64, _p, _p, _c_int, _p, _c_i64,
                              _c_f, _c_int, _p]),
    "kvq_v_matvec": (_c_int, [_c_int, _p, _p, _p, _p, _c_int, _c_int, _c_i64, _c_i64, _p, _p, _c_int, _p]),
    "kvq_attend_scratch_bytes": (_c_i64, [_c_int, _c_i64]),
    "kvq_attend": (_c_int, [_c_int, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _c_int, _c_int, _c_i64, _c_i64, _p,
                            _c_i64, _c_f, _c_int, _p, _p, _c_int, _p, _p, _p, _p, _p]),
    "kvq_attend_merge": (_c_int, [_p, _c_int, _c_int, _p, _p]),
    "kvq_append_kv_fused": (_c_int, [_c_int, _c_int, _c_i64, _c_i64, _c_int, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p,
                                     _p, _p, _p, _p, _p, _p, _p]),
    "kvq_append_kv_fused_dyn": (_c_int, [_c_int, _c_int, _c_i64, _p, _c_i64, _c_int, _p, _p, _p, _p, _p, _p, _p, _p, _p,
                                         _p, _p, _p, _p, _p, _p, _p, _p]),
    "kvq_attend_dyn": (_c_int, [_c_int, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _c_int, _c_int, _c_i64, _c_i64, _p,
                                _c_i64, _p, _c_i64, _c_f, _c_int, _p, _p, _c_int, _p, _p, _p, _p, _p]),
    "kvq_dequant_kv": (_c_int, [_c_int, _c_int, _c_i64, _c_i64, _c_i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _c_int,
                                _p, _c_i64, _c_int, _p, _p, _c_i64, _p]),
    "kvq_p2p_buffer_bytes": (_c_i64, [_c_int, _c_int]),
    "kvq_p2p_alloc": (_c_int, [_p, _c_i64, _p]),
    "kvq_p2p_open": (_c_int, [_p, _p]),
    "kvq_p2p_close": (_c_int, [_p]),
    "kvq_p2p_free": (_c_int, [_p]),
    "kvq_attend_exchange_merge": (_c_int, [_p, _p, _c_int, _c_int, _c_int, _p, _p, _p, _p]),
    "kvq_k_spmv_csr": (_c_int, [_p, _p, _p, _p, _p, _p, _c_int, _c_i64, _c_int, _c_int, _c_int, _p, _c_i64, _c_int, _p]),
    "kvq_v_spmv_csc": (_c_int, [_p, _p, _p, _p, _p, _p, _c_int, _c_i64, _c_int, _c_int, _c_int, _p]),
    "kvq_append_k_orig": (_c_int, [_p, _p, _p, _p, _p, _p, _p, _p, _p, _c_int, _c_i64, _c_i64, _p]),
    "kvq_append_v_orig": (_c_int, [_p, _p, _p, _c_f, _c_f, _c_f, _p, _p, _p, _c_int, _c_i64, _c_i64, _p]),
    "kvq_dec_rmsnorm": (_c_int, [_p, _p, _p, _c_int, _c_f, _p]),
    "kvq_dec_rope_split": (_c_int, [_p, _p, _c_f, _p, _p, _p, _c_int, _p]),
    "kvq_dec_rope_split_dyn": (_c_int, [_p, _p, _p, _c_i64, _p, _p, _p, _c_int, _p]),
    "kvq_dec_counter_add": (_c_int, [_p, _c_i64, _p]),
    "kvq_dec_silu_mul": (_c_int, [_p, _p, _c_int, _p]),
    "kvq_dec_f32_to_f16": (_c_int, [_p, _p, _c_int, _p]),
    "kvq_dec_gemv": (_c_int, [_p, _c_int, _c_int, _p, _c_int, _p, _c_f, _p, _p, _c_int, _p]),
}

_lib = None


class KVQuantError(RuntimeError):
    pass


def load():
    """Load the shared object (once).  Raises ImportError if it was not built -- there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "kvquant_b200: %s not found -- build it with `python -m kvquant_b200.build` "
            "(the product path has no CPU/PyTorch fallback)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if an export is missing: loud by design
        fn.restype = res
        fn.argtypes = args
    if lib.kvq_abi_version() != 2:
        raise ImportError("kvquant_b200: ABI version mismatch")
    _lib = lib
    return lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().kvq_error_string(rc).decode()
        raise KVQuantError("%s failed: %s (code %d)" % (what or "kvquant_b200 call", msg, rc))


def launch_count() -> int:
    return int(load().kvq_launch_count())
