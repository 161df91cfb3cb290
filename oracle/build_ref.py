#!/usr/bin/env python
"""Build the UNMODIFIED reference CUDA extension into oracle/_ref/ (test infrastructure only).

TEST INFRASTRUCTURE -- never imported by the product path (kvquant_b200/).  Only tests/,
__graft_entry__.smoke() and bench.py's cpu/reference legs may touch anything under oracle/.

What this does
--------------
Compiles the two reference source files *where they lie* in a checkout of the reference (REF_ROOT: $KVQUANT_REFERENCE,
default ../reference next to this repository; deployment/kvquant/quant_cuda.cpp + quant_cuda_kernel.cu, the `quant_cuda` torch extension whose
34 ops are the drop-in boundary, SURVEY.md section 8b) with plain g++/nvcc command lines -- the
reference's own setup_cuda.py is NOT run -- for sm_90a, and links them into

    oracle/_ref/quant_cuda_ref.so      (python module name: quant_cuda_ref)

No reference source is copied into this repository; oracle/_ref/ is git-ignored.  The `-m gpu` parity tests
compare against results of this extension stored under tests/golden/ (tests/_refgold.py), and re-record them from it
when asked to; the bench's `reference_cuda` record times it when it is present.

Without a reference checkout this script is a no-op: a prebuilt .so, if any, is used as is.
"""
import os
import shlex
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(HERE, "_ref")
REF_ROOT = os.environ.get("KVQUANT_REFERENCE") or os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference")
REF_DIR = os.path.join(REF_ROOT, "deployment", "kvquant")
SRC_CPP = os.path.join(REF_DIR, "quant_cuda.cpp")
SRC_CU = os.path.join(REF_DIR, "quant_cuda_kernel.cu")
OUT_SO = os.path.join(OUT_DIR, "quant_cuda_ref.so")
MODNAME = "quant_cuda_ref"


def _run(cmd):
    print("+", " ".join(shlex.quote(c) for c in cmd), flush=True)
    subprocess.check_call(cmd)


def build(force=False):
    if not (os.path.exists(SRC_CPP) and os.path.exists(SRC_CU)):
        print("[oracle/build_ref] no reference checkout at %s -> nothing to build " % REF_ROOT +
              "(prebuilt %s %s)" % (OUT_SO, "exists" if os.path.exists(OUT_SO) else "MISSING"))
        return os.path.exists(OUT_SO)
    if os.path.exists(OUT_SO) and not force:
        newest_src = max(os.path.getmtime(SRC_CPP), os.path.getmtime(SRC_CU))
        if os.path.getmtime(OUT_SO) >= newest_src:
            print("[oracle/build_ref] up to date:", OUT_SO)
            return True
    os.makedirs(OUT_DIR, exist_ok=True)
    import torch  # noqa: F401  (only for include/lib paths)
    from torch.utils import cpp_extension as ce

    cuda_home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    nvcc = os.path.join(cuda_home, "bin", "nvcc")
    incs = []
    for p in ce.include_paths() + [sysconfig.get_paths()["include"], os.path.join(cuda_home, "include")]:
        incs += ["-I", p]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    common_defs = [
        "-DTORCH_EXTENSION_NAME=%s" % MODNAME,
        "-DTORCH_API_INCLUDE_EXTENSION_H",
        "-D_GLIBCXX_USE_CXX11_ABI=%d" % abi,
    ]
    obj_cpp = os.path.join(OUT_DIR, "quant_cuda.o")
    obj_cu = os.path.join(OUT_DIR, "quant_cuda_kernel.o")
    # host binding file: same flags torch's BuildExtension would pass (-DNDEBUG comes from CPython's CFLAGS there)
    _run(["g++", "-O2", "-fPIC", "-std=c++17", "-DNDEBUG", "-w"] + common_defs + incs + ["-c", SRC_CPP, "-o", obj_cpp])
    # device file: no fast-math, no -DNDEBUG (the reference build has neither: asserts stay active,
    # cosf/sinf/powf are the accurate libdevice versions -- parity depends on that)
    _run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
          "--expt-relaxed-constexpr", "-w", "-Xcompiler", "-fPIC",
          "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__",
          "-D__CUDA_NO_BFLOAT16_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__"]
         + common_defs + incs + ["-c", SRC_CU, "-o", obj_cu])
    libdirs = ce.library_paths(device_type="cuda") if hasattr(ce, "library_paths") else []
    ld = []
    for p in libdirs:
        ld += ["-L", p, "-Wl,-rpath," + p]
    _run(["g++", "-shared", obj_cpp, obj_cu, "-o", OUT_SO] + ld +
         ["-lc10", "-ltorch_cpu", "-ltorch", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart"])
    for o in (obj_cpp, obj_cu):
        os.remove(o)
    print("[oracle/build_ref] built", OUT_SO)
    return True


def load():
    """Import the prebuilt reference extension. Returns module or None."""
    if not os.path.exists(OUT_SO):
        return None
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded first)
    spec = importlib.util.spec_from_file_location(MODNAME, OUT_SO)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    ok = build(force="--force" in sys.argv)
    sys.exit(0 if ok else 1)
