"""CPU-only: the streamed residency of `GpuProver` (ministark_b200/prover.py) and the two entry points it is built on.

  * ms_merkle_commit_block_sha256: a tree committed coset block by coset block, then its top levels from the block
    roots, equals the oracle's whole tree (nodes[1..N) and the root).  The CPU build of these two entry points is
    tests/cpp/stream_cpu_abi.c: the CPU build of the ABI (oracle/cpu_abi.c) plus include/ministark_stream.h;
  * ms_lde_rows: rows of the bit-reversed coset LDE evaluated from the coefficients equal the rows of the oracle's LDE;
  * the streamed prover on the CPU harness (tests/cpu_device.py), its budget forced between the two estimates, emits the
    bytes of oracle/stark_oracle.cpu_prove and the restated verifier accepts them;
  * the residency is chosen from the estimates: resident when it fits, streamed when only that fits, and a ProvingError
    naming both estimates and the budget before any work when neither does.
Prover cases run in spawned workers that install the harness themselves; the pytest process never does."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2**64 - 2**32 + 1
GENERATOR = 7 * 2**64 % P


@pytest.fixture(scope="module")
def stream_abi(tmp_path_factory, orc):
    """tests/cpp/stream_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary directory"""
    out = str(tmp_path_factory.mktemp("stream_abi") / "libms_stream_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out, os.path.join(ROOT, "tests", "cpp", "stream_cpu_abi.c")])
    return out


def _install(path):
    """the CPU harness (tests/cpu_device.py) with the library that also has the streamed-residency entry points"""
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    _lib.bind(lib, _lib._STREAM_SIGS)
    _lib._lib = lib


@pytest.fixture(scope="module")
def abi(stream_abi):
    lib = C.CDLL(stream_abi)
    lib.ms_last_error.restype = C.c_char_p
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    return lib, h


def _ck(abi, rc):
    lib, h = abi
    assert rc == 0, lib.ms_last_error(h).decode()


@pytest.mark.parametrize("field", [1, 3])
@pytest.mark.parametrize("log_block_rows", [0, 1, 3, 7])
@pytest.mark.parametrize("log_blocks", [0, 1, 2, 4])
def test_block_commit_equals_whole_tree(abi, orc, field, log_block_rows, log_blocks):
    if log_block_rows + log_blocks == 0:
        pytest.skip("a Merkle tree needs two leaves")
    lib, h = abi
    nb, beta = 1 << log_block_rows, 1 << log_blocks
    N, ncols = nb * beta, 3
    mat = orc.rand_matrix(ncols, N, field, seed=10 * log_block_rows + log_blocks + field)
    want = orc.merkle_nodes(orc.hash_rows(mat, field))
    nodes = np.zeros((N, 32), dtype=np.uint8)
    roots = np.zeros((beta, 32), dtype=np.uint8)
    for q in range(beta):
        first_row = mat.ctypes.data + q * nb * field * 8
        _ck(abi, lib.ms_merkle_commit_block_sha256(h, field, C.c_void_p(first_row), C.c_size_t(N), ncols, log_block_rows,
                                                   log_blocks, C.c_size_t(q), C.c_void_p(nodes.ctypes.data),
                                                   C.c_void_p(roots[q].ctypes.data)))
    if beta > 1:
        _ck(abi, lib.ms_merkle_nodes_sha256(h, C.c_void_p(roots.ctypes.data), C.c_size_t(beta), C.c_void_p(nodes.ctypes.data)))
    assert np.array_equal(nodes[1:], want[1:])
    assert roots[0].tobytes() == (want[beta] if log_block_rows else orc.hash_rows(mat, field)[0]).tobytes()


def test_block_commit_rejects_a_block_out_of_range(abi, orc):
    lib, h = abi
    mat = orc.rand_matrix(1, 8, 1, seed=1)
    nodes, root = np.zeros((8, 32), dtype=np.uint8), np.zeros(32, dtype=np.uint8)
    assert lib.ms_merkle_commit_block_sha256(h, 1, C.c_void_p(mat.ctypes.data), C.c_size_t(8), 1, 2, 1, C.c_size_t(2),
                                             C.c_void_p(nodes.ctypes.data), C.c_void_p(root.ctypes.data)) != 0
    assert b"block 2 of 2" in lib.ms_last_error(h)


def _lde_rows(abi, coeffs, field, log_n, log_b, positions, offset=GENERATOR):
    lib, h = abi
    ncols = coeffs.shape[0]
    ids = np.ascontiguousarray(positions, dtype=np.uint64)
    out = np.zeros((ids.size, ncols * field), dtype=np.uint64)
    _ck(abi, lib.ms_lde_rows(h, field, C.c_void_p(coeffs.ctypes.data), C.c_size_t(1 << log_n), ncols, log_n, log_b,
                             C.c_uint64(offset), C.c_void_p(ids.ctypes.data), ids.size, C.c_void_p(out.ctypes.data)))
    return out


@pytest.mark.parametrize("field", [1, 3])
@pytest.mark.parametrize("log_n,log_b", [(0, 0), (0, 2), (1, 1), (5, 3), (8, 4), (10, 0)])
def test_lde_rows_equal_the_oracle_lde(abi, orc, field, log_n, log_b):
    n, N = 1 << log_n, 1 << (log_n + log_b)
    coeffs = orc.rand_matrix(5, n, field, seed=log_n * 7 + log_b)
    coeffs[1] = 0                                               # zero column
    coeffs[2] = 0
    coeffs[2][:field] = orc.rand_matrix(1, 1, field, seed=99)[0]   # constant column
    coeffs[3] = np.uint64(P - 1)                                 # every word p - 1
    lde = orc.lde(coeffs, field, log_n, log_b, orc.generator(), True)
    rng = np.random.default_rng(N)
    positions = [0, N - 1, N // 2, 0, N - 1] + [int(v) for v in rng.integers(0, N, size=9)]
    got = _lde_rows(abi, coeffs, field, log_n, log_b, positions)
    for q, pos in enumerate(positions):
        want = np.concatenate([lde[c][pos * field:(pos + 1) * field] for c in range(coeffs.shape[0])])
        assert np.array_equal(got[q], want), (q, pos)


def test_lde_rows_at_another_offset(abi, orc):
    coeffs = orc.rand_matrix(2, 16, 3, seed=4)
    off = 11 * 2**64 % P
    lde = orc.lde(coeffs, 3, 4, 2, off, True)
    got = _lde_rows(abi, coeffs, 3, 4, 2, [63, 5, 17], offset=off)
    for q, pos in enumerate([63, 5, 17]):
        assert np.array_equal(got[q], np.concatenate([lde[c][3 * pos:3 * pos + 3] for c in range(2)]))


# ---------------------------------------------------------------------------------------------- the streamed prover
def _make_case(which):
    from ministark_b200.examples import brainfuck as bf
    from ministark_b200.examples import fib, perm
    if which.startswith("fib"):
        _, log_rows, opts = which.split(":")
        trace, last = fib.gen_trace(8 << int(log_rows))
        return fib.FibClaim(last), tuple(int(v) for v in opts.split(",")), trace
    if which == "perm":
        return perm.PermClaim(), (16, 8, 4, 4, 8), perm.gen_trace(1 << 8, seed=3)
    src = bf.HELLO_WORLD
    trace, output = bf.simulate(src)
    return bf.BrainfuckClaim(src, b"", output), (19, 16, 20, 16, 16), trace


def _estimates(claim, opts, n):
    from ministark_b200 import FP, FQ3
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.prover import peak_bytes
    cfg = claim.AirConfig
    o = ProofOptions(*opts)
    air = Air(cfg, n, None, o)
    return peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, FP if cfg.FQ_IS_FP else FQ3,
                      air.ce_blowup_factor, o.fri_folding_factor)


def _stream_worker(which, lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    from ministark_b200.air import ProofOptions
    from ministark_b200.prover import GpuProver
    claim, opts, trace = _make_case(which)
    est = _estimates(claim, opts, len(trace))
    assert est["streamed"] < est["resident"]
    p = GpuProver(0)
    p.memory_budget = (est["streamed"] + est["resident"]) // 2
    first = p.prove(claim, ProofOptions(*opts), trace).to_bytes()
    q.put((p.last_residency, first))


def _cpu_restatement(which):
    from ministark_b200.air import Air, ProofOptions
    from oracle import stark_oracle as SO
    claim, opts, trace = _make_case(which)
    pub = claim if which == "brainfuck" else claim.get_public_inputs()
    mk = lambda n, o: Air(claim.AirConfig, n, pub, ProofOptions(*o))
    ext = getattr(trace, "build_extension_columns", None)
    want = SO.cpu_prove(claim, opts, trace.base_columns(), mk, ext_builder=ext if claim.AirConfig.NUM_EXTENSION_COLUMNS else None)
    return want, claim, mk


def _spawn(target, *args):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=target, args=args + (q,))
    p.start()
    got = q.get(timeout=900)
    p.join(timeout=60)
    assert p.exitcode == 0
    return got


@pytest.mark.parametrize("which", ["fib:7:16,4,4,8,16", "fib:13:16,4,4,8,16", "perm", "brainfuck"])
def test_streamed_prover_bytes_equal_cpu_restatement(orc, stream_abi, which):
    from oracle import stark_oracle as SO
    residency, got = _spawn(_stream_worker, which, stream_abi)
    assert residency == "streamed"
    want, claim, mk = _cpu_restatement(which)
    assert got == want
    SO.verify(claim, got, 10, mk)


def _selection_worker(lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    from ministark_b200.air import ProofOptions
    from ministark_b200.prover import GpuProver, ProvingError
    claim, opts, trace = _make_case("fib:7:16,4,4,8,16")
    est = _estimates(claim, opts, len(trace))
    p = GpuProver(0)
    out = {"unset": GpuProver.memory_budget, "available": p.memory_available()}
    p.prove(claim, ProofOptions(*opts), trace)
    out["default"] = p.last_residency
    res = {}
    for name, budget in [("at_resident", est["resident"]), ("above", 10 * est["resident"]),
                         ("between", est["resident"] - 1), ("at_streamed", est["streamed"])]:
        p.memory_budget = budget
        proof = p.prove(claim, ProofOptions(*opts), trace).to_bytes()
        res[name] = (p.last_residency, proof)

    class Untouchable:
        """a witness whose columns must not be read: the refusal comes before any work"""
        def __len__(self):
            return len(trace)

        def base_columns(self):
            raise AssertionError("base columns read although the proof cannot fit")

    p.memory_budget = est["streamed"] - 1
    p.last_residency = None
    try:
        p.prove(claim, ProofOptions(*opts), Untouchable())
        err = None
    except ProvingError as e:
        err = str(e)
    out.update(res=res, err=err, est=est, after_refusal=p.last_residency)
    q.put(out)


def test_residency_selection(orc, stream_abi):
    out = _spawn(_selection_worker, stream_abi)
    assert out["unset"] is None and out["available"] == float("inf")     # off a CUDA device an unset budget is unlimited
    assert out["default"] == "resident"
    res = out["res"]
    assert res["at_resident"][0] == res["above"][0] == "resident"
    assert res["between"][0] == res["at_streamed"][0] == "streamed"
    assert len({r[1] for r in res.values()}) == 1                         # one proof, whichever residency made it
    err, est = out["err"], out["est"]
    assert err and "resident" in err and "streamed" in err and "available" in err
    gib = lambda b: f"{b / 2**30:.2f} GiB"
    assert gib(est["resident"]) in err and gib(est["streamed"]) in err and gib(est["streamed"] - 1) in err
    assert out["after_refusal"] is None


def test_stream_header_is_bound_exported_and_covered(stream_abi):
    """include/ministark_stream.h: every entry point is bound by the loader, exported by the CUDA library and by the CPU
    build the harness runs on, and none of them is also declared in include/ministark_b200.h"""
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.STREAM_HEADER_PATH)
    assert declared == sorted(_lib._STREAM_SIGS) == ["ms_lde_rows", "ms_merkle_commit_block_sha256"]
    assert not set(declared) & set(_lib.header_symbols())
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(stream_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)
