"""Generates tests/golden/rescue_k1024_l512.json: the trace of examples/rescue at BASELINE config 5's shape (K = 2^10
chains of L = 2^9 permutations, 2^22 rows) as the CPU build of ms_rescue_chains (tests/cpp/rescue_cpu_abi.c) writes it
— TEST INFRASTRUCTURE, run offline (about a minute on one core, 400 MB of memory):

    python tests/golden/make_rescue_golden.py

The file holds the seed, K, L, the K digests (canonical words) and the SHA-256 of the (12, 2^22) column-major matrix of
Montgomery words, little-endian.  tests/test_gpu_rescue.py checks the device trace against it."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SEED = [3141592653589793238, 2718281828459045235, 1618033988749894848, 1414213562373095048]
K, L = 1 << 10, 1 << 9
P = 2**64 - 2**32 + 1


def cpu_trace(lib_path, seed, K, L):
    """(12, 8 K L) Montgomery words from the CPU build at lib_path"""
    lib = C.CDLL(lib_path)
    lib.ms_ctx_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
    lib.ms_rescue_chains.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]
    lib.ms_ctx_destroy.argtypes = [C.c_void_p]
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    out = np.empty((12, 8 * K * L), dtype=np.uint64)
    s = np.array(seed, dtype=np.uint64)
    assert lib.ms_rescue_chains(h, s.ctypes.data, K, L, out.ctypes.data) == 0
    lib.ms_ctx_destroy(h)
    return out


def build(out_dir):
    path = os.path.join(out_dir, "librescue_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", path, os.path.join(ROOT, "tests", "cpp", "rescue_cpu_abi.c")])
    return path


def record(trace, seed, K, L):
    rinv = pow(2**64, -1, P)
    ends = trace[:4, 8 * L - 1::8 * L]
    return {"seed": seed, "K": K, "L": L, "trace_sha256": hashlib.sha256(trace.tobytes()).hexdigest(),
            "digests": [[int(w) * rinv % P for w in ends[:, k]] for k in range(K)]}


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as d:
        trace = cpu_trace(build(d), SEED, K, L)
    with open(os.path.join(HERE, "rescue_k1024_l512.json"), "w") as f:
        json.dump(record(trace, SEED, K, L), f)
        f.write("\n")
