#!/usr/bin/env python
"""Compile oracle/kvq_oracle_port.c -> oracle/_ref/libkvq_oracle_port.so (gcc -O3 -fopenmp).
TEST / BASELINE INFRASTRUCTURE: used by tests/ and bench.py's cpu_baseline / --impl reference legs only."""
import ctypes
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "kvq_oracle_port.c")
OUT = os.path.join(HERE, "_ref", "libkvq_oracle_port.so")


def build(force=False):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= os.path.getmtime(SRC):
        return OUT
    # -march=x86-64-v3 (AVX2/FMA): the .so may be built on one x86-64 host and run on another (the GPU host's cores)
    cmd = ["gcc", "-O3", "-fopenmp", "-march=x86-64-v3", "-fPIC", "-shared", "-std=c11", SRC, "-o", OUT, "-lm"]
    subprocess.check_call(cmd)
    return OUT


def load():
    lib = ctypes.CDLL(build())
    P, I, L64, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
    lib.kvq_port_threads.restype = I
    lib.kvq_port_set_threads.argtypes = [I]
    lib.kvq_port_set_threads.restype = None
    lib.kvq_port_k_scores.argtypes = [I, P, P, P, P, P, I, I, L64, L64, F, I, P]
    lib.kvq_port_v_out.argtypes = [I, P, P, P, P, P, I, I, L64, L64, P]
    lib.kvq_port_attend.argtypes = [I, P, P, P, P, P, P, P, P, P, I, I, L64, L64, F, I, P, P]
    return lib


if __name__ == "__main__":
    print(build(force=True))
