"""CPU: the C-ABI shared library builds (nvcc cross-compiles sm_90a without a GPU), loads, and exports every
symbol include/kvquant_b200.h declares; the Python surface has exactly the reference's 34 operator names."""
import ctypes
import os
import re
import pytest

from _util import ROOT

REFERENCE_OPS = """
vecquant4matmul_nuq_perchannel_transposed_mha_batched_fused_opt vecquant4matmul_nuq_perchannel_transposed_mha_batched_fused_opt2
vecquant4matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt vecquant4matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2
vecquant4appendvecK vecquant4appendvecKsparse vecquant4appendvecKsparseParallel
vecquant4appendvecV vecquant4appendvecVsparse vecquant4appendvecVsparseParallel
vecquant3matmul_nuq_perchannel_transposed_mha_batched_fused_opt vecquant3matmul_nuq_perchannel_transposed_mha_batched_fused_opt2
vecquant3matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt vecquant3matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2
vecquant3appendvecK vecquant3appendvecKsparse vecquant3appendvecKsparseParallel
vecquant3appendvecV vecquant3appendvecVsparse vecquant3appendvecVsparseParallel
vecquant2matmul_nuq_perchannel_transposed_mha_batched_fused_opt vecquant2matmul_nuq_perchannel_transposed_mha_batched_fused_opt2
vecquant2matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt vecquant2matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2
vecquant2appendvecK vecquant2appendvecKsparse vecquant2appendvecKsparseParallel
vecquant2appendvecV vecquant2appendvecVsparse vecquant2appendvecVsparseParallel
vecquant4matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2_orig vecquant4appendvecKsparseorig
vecquant4matmul_nuq_perchannel_transposed_mha_batched_fused_opt2_orig vecquant4appendvecVsparseorig
""".split()  # the m.def list of reference deployment/kvquant/quant_cuda.cpp:401-436


def _declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "kvquant_b200.h")).read()
    return sorted(set(re.findall(r"KVQ_API\s+[\w\s\*]+?\b(kvq_\w+)\s*\(", hdr)))


def test_library_builds_loads_and_exports_every_declared_symbol():
    from kvquant_b200 import build, _lib
    path = build.build(verbose=False)
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    declared = _declared_symbols()
    assert len(declared) >= 19
    for name in declared:
        assert hasattr(lib, name), "missing export " + name
    assert sorted(_lib.SIGNATURES) == declared          # the ctypes table covers the header one to one
    assert _lib.load().kvq_abi_version() == 2
    assert b"bits" in _lib.load().kvq_error_string(-1)


def test_python_surface_has_exactly_the_reference_ops():
    import quant_cuda  # top-level drop-in shim
    assert len(REFERENCE_OPS) == 34
    assert sorted(quant_cuda.OP_NAMES) == sorted(REFERENCE_OPS)
    for n in REFERENCE_OPS:
        assert callable(getattr(quant_cuda, n))


def test_argument_validation_is_loud_not_a_fallback():
    import pytest
    import torch
    import quant_cuda
    mat = torch.zeros((32, 16, 64), dtype=torch.int32)
    lut = torch.zeros((32, 128, 16))
    with pytest.raises(ValueError):  # CPU tensors are rejected, never computed on the host
        quant_cuda.vecquant4appendvecK(mat, lut, torch.zeros(4096), 0)
    with pytest.raises(ValueError):  # wrong packed height for the bit width
        quant_cuda.vecquant3appendvecK(mat, lut, torch.zeros(4096), 0)


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "kvquant_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("oracle/_ref", ""), os.path.join(dirpath, f)


def test_header_is_plain_c_and_links_against_the_library(tmp_path):
    """include/kvquant_b200.h is a C header (no C++ or torch types): it compiles as C99 and as C++11, and a C program
    that only includes it links against libkvquant_b200.so and runs without a GPU (the cgo / JNI / ctypes view)."""
    import shutil
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "abi_c.c"
    src.write_text('#include "kvquant_b200.h"\n#include <stdio.h>\n'
                   'int main(void) { printf("%d %s\\n", kvq_abi_version(), kvq_error_string(KVQ_E_SHAPE)); return 0; }\n')
    inc = os.path.join(root, "include")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I", inc, str(src)])
    subprocess.check_call(["g++", "-std=c++11", "-fsyntax-only", "-x", "c++", "-I", inc, str(src)])
    lib = os.path.join(root, "kvquant_b200", "libkvquant_b200.so")
    if not os.path.exists(lib) or shutil.which("gcc") is None:
        pytest.skip("library not built")
    exe = tmp_path / "abi_c"
    subprocess.check_call(["gcc", "-std=c99", "-I", inc, str(src), lib, "-o", str(exe),
                           "-Wl,-rpath," + os.path.dirname(lib), "-Wl,-rpath,/usr/local/cuda/lib64"])
    out = subprocess.check_output([str(exe)], text=True).split(None, 1)
    assert out[0] == "2" and out[1].strip()


def test_csr_growth_glue_matches_the_oracle():
    """quant_cuda._grow_csr (host glue of the uncapped 'orig' appends, quant_cuda_kernel.cu:765-823) on CPU tensors
    against the oracle's restatement, token by token, including empty tokens and the 10-nonzeros-per-thread
    start array."""
    import numpy as np
    import torch
    from _util import O
    from kvquant_b200 import quant_cuda as qc
    g = np.random.default_rng(5)
    e = torch.empty(0, dtype=torch.int32)
    ptr, idx, val, start = e, e, torch.empty(0), e
    optr, oidx, oval, ostart = [], [], [], []
    for t in range(60):
        count = int(g.choice([0, 0, 1, 3, 9, 10, 11, 25]))
        ni = torch.tensor(np.sort(g.choice(4096, count, replace=False)), dtype=torch.int32)
        nv = torch.tensor(g.normal(size=count), dtype=torch.float32)
        ptr, idx, val, start, nthr = qc._grow_csr(ptr, idx, val, start, ni, nv, count, t, "cpu")
        optr, oidx, oval, ostart, onthr = O.csr_grow(optr, oidx, oval, ostart, ni.tolist(), nv.tolist(), t)
        assert nthr == onthr == (len(oidx) + 9) // 10
        assert ptr.tolist() == optr and idx.tolist() == oidx and start.tolist() == ostart
        assert np.array_equal(val.numpy(), np.asarray(oval, dtype=np.float32))
    assert ptr.tolist()[-1] == len(oidx) and len(ptr) == 61


def test_algorithmic_bytes_match_the_survey_figures():
    """roofline.achieved is computed from SURVEY.md 8(d)'s per-token figures: 7B 4-bit+1% = 4832 B/token/layer,
    3-bit+1% = 3776, 4-bit dense-only = 4160; outlier width 42 (7B) / 52 (13B)."""
    from kvquant_b200 import decode as kd
    from kvquant_b200.cache import n_outliers_each
    assert kd.layer_step_bytes(kd.DecodeConfig.llama7b(bits=4), 1) == 4832
    assert kd.layer_step_bytes(kd.DecodeConfig.llama7b(bits=3), 1) == 3776
    cfg = kd.DecodeConfig.llama7b(bits=4)
    cfg.include_sparse = False
    assert kd.layer_step_bytes(cfg, 1) == 4160
    assert 2 * n_outliers_each(4096, 0.99) == 42 and 2 * n_outliers_each(5120, 0.99) == 52


def test_ctypes_table_matches_the_header_argument_by_argument():
    """Every prototype of include/kvquant_b200.h against kvquant_b200._lib.SIGNATURES: same number of parameters and the
    same class (pointer / int / int64_t / float) in each position -- a binding that drifts from the header would pass
    garbage in registers without any error."""
    from kvquant_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "kvquant_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    hdr = re.sub(r"//[^\n]*", " ", hdr)
    protos = re.findall(r"KVQ_API\s+([\w\s\*]+?)\b(kvq_\w+)\s*\(([^)]*)\)\s*;", hdr)
    assert len(protos) == len(_lib.SIGNATURES)

    def klass_c(decl):
        decl = decl.strip()
        if "*" in decl:
            return "ptr"
        base = " ".join(decl.split()[:-1]) if len(decl.split()) > 1 else decl     # drop the parameter name
        base = base.replace("const", "").strip()
        return {"int": "int", "int64_t": "i64", "float": "f32", "uint64_t": "u64", "unsigned long long": "u64"}[base]

    def klass_py(t):
        return {ctypes.c_void_p: "ptr", ctypes.c_char_p: "ptr", ctypes.c_int: "int", ctypes.c_int64: "i64",
                ctypes.c_float: "f32", ctypes.c_uint64: "u64"}[t]

    for ret, name, params in protos:
        restype, argtypes = _lib.SIGNATURES[name]
        plist = [p for p in params.split(",") if p.strip() and p.strip() != "void"]
        got = [klass_c(p) for p in plist]
        want = [klass_py(t) for t in argtypes]
        assert got == want, (name, got, want)
        assert klass_c(ret.strip() + " x") == klass_py(restype), (name, ret)
