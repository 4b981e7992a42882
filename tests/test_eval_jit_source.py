"""CPU-only: the run-time specialised evaluator kernel (csrc/eval_jit.cu) checked WITHOUT a GPU.

ms_eval_jit_check generates the CUDA source of the kernel for a program and compiles it with NVRTC for sm_90a; with
MS_EVAL_JIT_DUMP it also writes that source out.  field.cuh — embedded in the source — has host branches for all its
arithmetic, so the very text NVRTC compiles is compiled here by g++ behind a dozen lines of CUDA stand-ins (blockIdx,
__ldg, __brevll ...), run for every point of a small domain and compared with the compiled CPU interpreter of the same
program (oracle/cpu_abi.c, itself checked against the tree-walking oracle in tests/test_cpp_cpu_abi.py).  Programs: the
composition and DEEP programs of the three example AIRs as the provers build them (grouped DEEP, shared powers, batched
inversions, leaf rematerialisation), bound to random verifier values, in the storage orders the provers use; and every
opcode over every operand-field combination on edge operands, against big integers."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from ministark_b200 import _lib
from ministark_b200 import expr as E
from ministark_b200.air import Air, ProofOptions
from ministark_b200.examples import brainfuck as bf
from ministark_b200.examples import fib, perm

import tests_helpers_expr as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = E.P
R = 2**64
GENERATOR = 7 * R % P

PRELUDE = r"""
#include <cstdint>
#define __global__
#define __launch_bounds__(x)
#define __restrict__
struct Dim3 { unsigned long long x; };
static Dim3 blockIdx, threadIdx;
static const Dim3 blockDim = {128};
static inline unsigned long long __brevll(unsigned long long v) {
    unsigned long long r = 0;
    for (int i = 0; i < 64; i++) r |= ((v >> i) & 1ull) << (63 - i);
    return r;
}
template <class T> static inline T __ldg(const T *p) { return *p; }
"""
DRIVER = r"""
extern "C" void run_all(const u64 *const *col_ptr, const u64 *kc, const u64 *tw_lo, const u64 *tw_hi, unsigned hi_len, u64 offset,
                        unsigned lm, int trace_bitrev, int out_bitrev, u64 *out) {
    const u64 M = 1ull << lm;
    for (u64 t = 0; t < ((M + 127) / 128) * 128; t++) {      // whole blocks, as launched: the kernel's own bounds check applies
        blockIdx.x = t / 128;
        threadIdx.x = t % 128;
        ms_eval_jit(col_ptr, kc, tw_lo, tw_hi, hi_len, offset, lm, trace_bitrev, out_bitrev, out);
    }
}
"""


def _kernel_source(tmp, prog, fq):
    lib = _lib.load()
    src_path = os.path.join(tmp, "k.cu")
    os.environ["MS_EVAL_JIT_DUMP"] = src_path
    try:
        log = C.create_string_buffer(16384)
        rc = lib.ms_eval_jit_check(prog.code.ctypes.data, len(prog), prog.consts.ctypes.data, prog.consts.shape[0], fq, log, 16384)
    finally:
        os.environ.pop("MS_EVAL_JIT_DUMP", None)
    if rc == 1:
        pytest.skip("NVRTC is not installed: no specialised kernel is generated")
    assert rc == 0, log.value.decode()[:2000]
    return open(src_path).read()


def _host_kernel(tmp, prog, fq):
    with open(os.path.join(tmp, "k.cpp"), "w") as f:
        f.write(PRELUDE + _kernel_source(tmp, prog, fq) + DRIVER)
    so = os.path.join(tmp, "k.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-o", so, os.path.join(tmp, "k.cpp")])
    return C.CDLL(so)


def _tables(log_m):
    g = pow(pow(7, (P - 1) >> 32, P), 1 << (32 - log_m), P)
    m = 1 << log_m
    lo = np.array([pow(g, e, P) * R % P for e in range(min(m, 4096))], dtype=np.uint64)
    hi = np.array([pow(g, 4096 * j, P) * R % P for j in range(max(1, m // 4096))], dtype=np.uint64)
    return lo, hi


@pytest.fixture(scope="module")
def cpu_abi(orc):
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "libms_cpu_abi.so"])
    lib = C.CDLL(os.path.join(ROOT, "oracle", "libms_cpu_abi.so"))
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    return lib, h


def _air(which):
    if which == "fib":
        return Air(fib.FibAirConfig, 16, 5, fib.OPTIONS), fib.FibAirConfig
    if which == "perm":
        return Air(perm.PermAirConfig, 16, [], ProofOptions(8, 8, 0, 4, 4)), perm.PermAirConfig
    return Air(bf.BrainfuckAirConfig, 64, bf.BrainfuckClaim("+.", b"", b"\x01"), bf.OPTIONS), bf.BrainfuckAirConfig


@pytest.mark.parametrize("which", ["fib", "perm", "brainfuck"])
@pytest.mark.parametrize("kind", ["composition", "deep"])
def test_generated_kernel_source_runs_like_the_interpreter(tmp_path, orc, cpu_abi, which, kind):
    lib, h = cpu_abi
    rng = random.Random(hash((which, kind)) & 0xFFFF)
    air, cfg = _air(which)
    fq = 1 if cfg.FQ_IS_FP else 3
    q3 = lambda: tuple(rng.randrange(P) for _ in range(fq)) + (0,) * (3 - fq)
    nb, ne = cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS
    if kind == "composition":
        sym = air.composition_program()
        log_m = air.log_n + air.ce_blowup_factor.bit_length() - 1
        nfq, out_bitrev = ne, 0
    else:
        sym, keys = air.deep_program()
        log_m = air.log_n + air.options.lde_blowup_factor.bit_length() - 1
        nfq, out_bitrev = ne + air.ce_blowup_factor, 1
    prog = sym.bind(challenges=[q3() for _ in range(32)], hints=[q3() for _ in range(256)], ccoefs=[q3() for _ in range(256)])
    m = 1 << log_m
    base = orc.rand_matrix(nb, m, 1, seed=rng.randrange(1 << 30))
    ext = orc.rand_matrix(nfq, m, fq, seed=rng.randrange(1 << 30)) if nfq else None
    cols = [np.ascontiguousarray(c) for c in base] + ([np.ascontiguousarray(c) for c in ext] if nfq else [])
    ptrs = (C.c_void_p * len(cols))(*[c.ctypes.data for c in cols])
    isq = (C.c_int * len(cols))(*([0] * nb + [1] * nfq))
    code, consts = np.ascontiguousarray(prog.code), np.ascontiguousarray(prog.consts)
    want = np.zeros(m * fq, dtype=np.uint64)
    assert lib.ms_eval_constraints_ptrs(h, C.c_void_p(code.ctypes.data), len(prog), C.c_void_p(consts.ctypes.data), consts.shape[0], ptrs, isq,
                                        len(cols), fq, log_m, C.c_uint64(GENERATOR), 1, out_bitrev, C.c_void_p(want.ctypes.data)) == 0
    kernel = _host_kernel(str(tmp_path), prog, fq)
    lo, hi = _tables(log_m)
    got = np.zeros(m * fq, dtype=np.uint64)
    kernel.run_all(ptrs, C.c_void_p(consts.ctypes.data), C.c_void_p(lo.ctypes.data), C.c_void_p(hi.ctypes.data), C.c_uint(len(hi)),
                   C.c_uint64(GENERATOR), C.c_uint(log_m), 1, out_bitrev, C.c_void_p(got.ctypes.data))
    assert want.any() and np.array_equal(got, want)


def test_generated_kernel_source_of_the_config3_program(tmp_path, orc, cpu_abi):
    """the synthetic AIR of BASELINE config 3 (ministark_b200/synth_air.py): the specialised kernel's source run on the host
    reproduces oracle/synth_oracle.py's constraint column, read in place from the bit-reversed LDE prefix"""
    from ministark_b200 import synth_air
    from oracle import synth_oracle
    log_n, log_b, ncols = 8, 3, 32
    trace = orc.rand_matrix(ncols, 1 << log_n, 1, seed=9)
    lde = orc.lde(orc.ntt(trace, 1, log_n, inverse=True), 1, log_n, log_b, orc.generator(), True)
    prog = E.compile_program(synth_air.composition(ncols, log_n, 1), ncols, lde_step=1, log_ce=log_n)
    kernel = _host_kernel(str(tmp_path), prog, 1)
    cols = [np.ascontiguousarray(c[:1 << log_n]) for c in lde]       # the ce-domain prefix of every LDE column
    ptrs = (C.c_void_p * ncols)(*[c.ctypes.data for c in cols])
    lo, hi = _tables(log_n)
    consts = np.ascontiguousarray(prog.consts)
    got = np.zeros(1 << log_n, dtype=np.uint64)
    kernel.run_all(ptrs, C.c_void_p(consts.ctypes.data), C.c_void_p(lo.ctypes.data), C.c_void_p(hi.ctypes.data), C.c_uint(len(hi)),
                   C.c_uint64(GENERATOR), C.c_uint(log_n), 1, 0, C.c_void_p(got.ctypes.data))
    assert np.array_equal(got, synth_oracle.constraint_eval(orc, lde, log_n, log_b, ncols))


@pytest.mark.parametrize("fq", [3, 1])
def test_generated_kernel_source_on_edge_operands(tmp_path, fq):
    """every opcode over every operand-field combination on edge operands (tests_helpers_expr.edge_programs, the programs
    tests/test_gpu_eval_edges.py runs on the device): the host branches of the generated source against pyspec's big
    integers.  All kernels go into one host library, the field code once and each kernel under its own name."""
    programs = H.edge_programs()
    kernel_start = 'extern "C" __global__'
    field_src, kernels, drivers = None, [], []
    for k, (_, prog, _, _) in enumerate(programs):
        src = _kernel_source(str(tmp_path), prog, fq)
        head, sep, body = src.partition(kernel_start)
        assert sep and (field_src is None or head == field_src)
        field_src = head
        kernels.append(sep + body.replace("ms_eval_jit(", f"ms_eval_jit_{k}(", 1))
        drivers.append(DRIVER.replace("run_all(", f"run_all_{k}(").replace("ms_eval_jit(", f"ms_eval_jit_{k}("))
    with open(tmp_path / "edges.cpp", "w") as f:
        f.write(PRELUDE + field_src + "".join(kernels) + "".join(drivers))
    so = str(tmp_path / "edges.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-w", "-o", so, str(tmp_path / "edges.cpp")])
    lib = C.CDLL(so)
    log_m = H.EDGE_LOG_M
    m = 1 << log_m
    cols, isq = H.edge_columns(fq)
    words = [np.ascontiguousarray(H.column_words(c, q, fq)) for c, q in zip(cols, isq)]
    ptrs = (C.c_void_p * len(words))(*[w.ctypes.data for w in words])
    lo, hi = _tables(log_m)
    for k, (name, prog, used, ref) in enumerate(programs):
        want, operands = H.edge_reference(cols, used, ref, fq)
        got = np.zeros(m * fq, dtype=np.uint64)
        consts = np.ascontiguousarray(prog.consts)
        getattr(lib, f"run_all_{k}")(ptrs, C.c_void_p(consts.ctypes.data), C.c_void_p(lo.ctypes.data), C.c_void_p(hi.ctypes.data),
                                     C.c_uint(len(hi)), C.c_uint64(GENERATOR), C.c_uint(log_m), 0, 0, C.c_void_p(got.ctypes.data))
        bad = np.nonzero((got.reshape(m, fq) != want.reshape(m, fq)).any(axis=1))[0]
        assert not len(bad), (f"{name} fq_field={fq}: {len(bad)} points differ, first at {bad[0]} operands {operands(bad[0])}: "
                              f"got {[hex(w) for w in got.reshape(m, fq)[bad[0]]]}, want {[hex(w) for w in want.reshape(m, fq)[bad[0]]]}")
