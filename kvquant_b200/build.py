"""Build libkvquant_b200.so (hand-written sm_90a CUDA behind a C ABI) in-tree with nvcc.

    python -m kvquant_b200.build [--force]

The shared object lands next to this file (git-ignored).
nvcc cross-compiles without a GPU; the library also loads without one (ctypes export check in tests).
"""
import os
import shlex
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libkvquant_b200.so")
SOURCES = ["kvq_capi.cu", "kvq_append.cu", "kvq_append_ragged.cu", "kvq_kscore.cu", "kvq_k3.cu", "kvq_kfast.cu", "kvq_kratio.cu", "kvq_vaccum.cu", "kvq_vnative.cu", "kvq_attend.cu", "kvq_orig.cu", "kvq_decode_ops.cu", "kvq_decode_gemv.cu", "kvq_p2p.cu", "kvq_dequant.cu", "kvq_chunk.cu", "kvq_page.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",  # H100 only; no fallback archs, no fast-math
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "-cudart", "shared",
]


def _nvcc():
    home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    return os.path.join(home, "bin", "nvcc")


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [
        os.path.join(os.path.dirname(HERE), "include", "kvquant_b200.h"), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=True):
    if not force and not needs_build():
        return OUT
    objs = []
    procs = []
    tmpdir = os.path.join(HERE, "build")
    os.makedirs(tmpdir, exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(tmpdir, src.replace(".cu", ".o"))
        cmd = [_nvcc()] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print("+", " ".join(shlex.quote(c) for c in cmd), flush=True)
        procs.append((subprocess.Popen(cmd), cmd))
        objs.append(obj)
    for p, cmd in procs:
        if p.wait() != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    link = [_nvcc(), "-shared", "-cudart", "shared", "-o", OUT] + objs + [
        "-Xlinker", "-rpath", "-Xlinker", "/usr/local/cuda/lib64", "-ldl"]
    if verbose:
        print("+", " ".join(shlex.quote(c) for c in link), flush=True)
    subprocess.check_call(link)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
