"""CPU-only: the "streamed_host" residency, whose Merkle node heaps live in pinned host memory, and the entry point it is
built on (include/ministark_host_nodes.h), on the CPU build of the ABI: tests/cpp/host_nodes_cpu_abi.c, the top of the CPU
ABI chain (oracle, streamed residency, constraint check, brainfuck trace, ms_device_memory) plus the new entry point,
compiled into a temporary directory.

  * every block's local heap is its slice of the whole tree's heap, and the top heap from the block roots gives the root;
  * cosets.heap_location finds every node merkle_walk names in the split heap;
  * GpuProver on the CPU harness (tests/cpu_device.py), with a device budget only streamed_host fits and a host budget,
    picks streamed_host and emits the bytes of oracle/stark_oracle.cpu_prove, with and without validation; without a
    host budget, or with one byte too little, it refuses;
  * the C++ prover does the same, and its four peak_bytes estimates are Python's.
Prover cases run in spawned workers that install the harness themselves; the pytest process never does."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from ministark_b200 import FP, FQ3
from ministark_b200.cosets import heap_location, merkle_walk
from ministark_b200.prover import peak_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")


@pytest.fixture(scope="module")
def cpu_lib(tmp_path_factory, orc):
    d = tmp_path_factory.mktemp("host_nodes_abi")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", str(d / "libms_host_nodes_cpu_abi.so"),
                           os.path.join(ROOT, "tests", "cpp", "host_nodes_cpu_abi.c")])
    return d


@pytest.fixture(scope="module")
def abi(cpu_lib):
    lib = C.CDLL(str(cpu_lib / "libms_host_nodes_cpu_abi.so"))
    lib.ms_last_error.restype = C.c_char_p
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    yield lib, h
    lib.ms_ctx_destroy(h)


def _ck(abi, rc):
    lib, h = abi
    assert rc == 0, lib.ms_last_error(h).decode()


# ---------------------------------------------------------------------------------------------- the split heap
@pytest.mark.parametrize("field", [FP, FQ3])
@pytest.mark.parametrize("log_block_rows", [0, 1, 4, 10])
@pytest.mark.parametrize("log_b", [0, 1, 2, 3, 4])
def test_local_heaps_are_slices_of_the_global_heap(abi, orc, field, log_block_rows, log_b):
    if log_block_rows + log_b == 0:
        pytest.skip("a Merkle tree needs two leaves")
    lib, h = abi
    nb, beta = 1 << log_block_rows, 1 << log_b
    N, ncols = nb * beta, 3
    mat = orc.rand_matrix(ncols, N, field, seed=100 * log_block_rows + 10 * log_b + field)
    want = orc.merkle_nodes(orc.hash_rows(mat, field))
    local = np.full((beta, nb, 32), 0xAB, dtype=np.uint8)
    top = np.zeros((2 * beta, 32), dtype=np.uint8)
    for q in range(beta):
        _ck(abi, lib.ms_merkle_commit_block_sha256_host(h, field, C.c_void_p(mat.ctypes.data + q * nb * field * 8), C.c_size_t(N),
                                                         ncols, log_block_rows, C.c_void_p(local[q].ctypes.data),
                                                         C.c_void_p(top[beta + q].ctypes.data)))
    assert not local[:, 0].any()                                    # slot 0 of every local heap: the unused zero digest
    if beta > 1:
        _ck(abi, lib.ms_merkle_nodes_sha256(h, C.c_void_p(top[beta:].ctypes.data), C.c_size_t(beta), C.c_void_p(top.ctypes.data)))
    for i in range(1, N):
        b, j = heap_location(i, log_b)
        got = top[j] if b is None else local[b, j]
        assert np.array_equal(got, want[i]), (i, b, j)
    if log_block_rows:
        assert np.array_equal(top[beta:], want[beta:2 * beta])      # the block roots are the heap's level log_b
        assert all(np.array_equal(local[q, 1], top[beta + q]) for q in range(beta))
    else:
        assert np.array_equal(top[beta:], orc.hash_rows(mat, field))   # one row per block: its leaf digest
    assert np.array_equal(top[1], want[1])                          # the root


def _split(heap, log_n, log_b):
    """the split layout built level by level, as the block commitment writes it: on level L > log_b, block q owns the
    2^d (d = L - log_b) nodes from 2^L + q * 2^d, and its local heap holds them from 2^d"""
    beta, n = 1 << log_b, 1 << log_n
    top = heap[:2 * beta].copy()
    local = np.full((beta, n), -1, dtype=np.int64)
    for d in range(1, log_n):
        for q in range(beta):
            local[q, 1 << d:2 << d] = heap[(1 << (d + log_b)) + q * (1 << d):(1 << (d + log_b)) + (q + 1) * (1 << d)]
    return top, local


def test_heap_location_finds_every_node_merkle_walk_names():
    rng = random.Random(5)
    cases = [(1, 0, [0]), (1, 0, [1, 1, 0]), (1, 1, [0, 1]), (0, 1, [1])]    # 2-leaf trees, split either way
    for _ in range(300):
        log_N = rng.randint(1, 14)
        log_b = rng.randint(0, min(log_N, 5))
        N = 1 << log_N
        k = rng.randint(1, 40)
        pos = [rng.randrange(N) for _ in range(k)]
        pos += rng.sample(pos, min(len(pos), 5))                     # duplicates
        cases.append((log_N - log_b, log_b, pos))
    for log_n, log_b, pos in cases:
        N = 1 << (log_n + log_b)
        heap = np.arange(N, dtype=np.int64)
        top, local = _split(heap, log_n, log_b)
        _, _, path = merkle_walk(N, pos)
        for i in path:
            b, j = heap_location(i, log_b)
            assert (top[j] if b is None else local[b, j]) == i, (log_n, log_b, i, b, j)


def test_heap_location_at_the_largest_heaps():
    """heap indices up to 2^30 (a 2^26-row trace at blow-up 16): Python ints, no narrowing"""
    log_b, log_N = 4, 30
    i = (1 << log_N) - 1                                            # the last leaf pair's parent level, last node
    assert heap_location(i, log_b) == ((1 << log_b) - 1, (1 << (log_N - log_b)) - 1)
    assert heap_location(1 << (log_b + 1), log_b) == (0, 2)
    assert heap_location((1 << (log_b + 1)) - 1, log_b) == (None, (1 << (log_b + 1)) - 1)


def test_host_nodes_header_is_bound_exported_and_separate(cpu_lib):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.HOST_NODES_HEADER_PATH)
    assert declared == sorted(_lib._HOST_NODES_SIGS) == ["ms_merkle_commit_block_sha256_host"]
    others = set(_lib.header_symbols()) | set(_lib.header_symbols(_lib.STREAM_HEADER_PATH)) | \
        set(_lib.header_symbols(_lib.BF_HEADER_PATH)) | set(_lib.header_symbols(_lib.CHECK_HEADER_PATH)) | \
        set(_lib.header_symbols(_lib.DEVICE_HEADER_PATH))
    assert not set(declared) & others
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(str(cpu_lib / "libms_host_nodes_cpu_abi.so"))
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)


# ---------------------------------------------------------------------------------------------- the Python prover
def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._BF_SIGS, _lib._DEVICE_SIGS, _lib._HOST_NODES_SIGS):
        _lib.bind(lib, sigs)
    _lib._lib = lib


def _make_case(which):
    from ministark_b200.examples import brainfuck as bf
    from ministark_b200.examples import fib, perm
    if which == "fib":
        trace, last = fib.gen_trace(8 << 7)
        return fib.FibClaim(last), (16, 4, 4, 8, 16), trace
    if which == "perm":
        return perm.PermClaim(), (16, 8, 4, 4, 8), perm.gen_trace(1 << 8, seed=3)
    trace, output = bf.simulate(bf.HELLO_WORLD)
    return bf.BrainfuckClaim(bf.HELLO_WORLD, b"", output), (19, 16, 20, 16, 16), trace


def _estimates(claim, opts, n):
    from ministark_b200.air import Air, ProofOptions
    cfg = claim.AirConfig
    o = ProofOptions(*opts)
    return peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, FP if cfg.FQ_IS_FP else FQ3,
                      Air(cfg, n, None, o).ce_blowup_factor, o.fri_folding_factor)


def _between(est):
    return (est["streamed_host"] + est["streamed"]) // 2


def _prove_worker(which, lib_path, q):
    try:
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        _install(lib_path)
        from ministark_b200.air import ProofOptions
        from ministark_b200.prover import GpuProver, ProvingError
        claim, opts, trace = _make_case(which)
        est = _estimates(claim, opts, len(trace))
        p = GpuProver(0)
        p.memory_budget = _between(est)
        p.host_memory_budget = est["host"]
        out = {"est": est}
        for validate in (False, True):
            proof = p.prove(claim, ProofOptions(*opts), trace, validate=validate)
            out[validate] = (p.last_residency, proof.to_bytes(), p.pinned_bytes, "pin_host_memory" in proof.timings)
        for name, host in [("no_host", None), ("host_short", est["host"] - 1)]:
            p.host_memory_budget = host
            p.last_residency = None
            try:
                p.prove(claim, ProofOptions(*opts), trace)
                out[name] = ("proved", p.last_residency)
            except ProvingError as e:
                out[name] = ("refused", str(e))
            out[name + "_pinned"] = p.pinned_bytes
        p.host_memory_budget = est["host"]
        p.prove(claim, ProofOptions(*opts), trace)
        out["pinned_again"] = p.pinned_bytes
        p.release_host_memory()
        out["released"] = p.pinned_bytes
        q.put(out)
    except Exception:                       # reported, not left for the queue's timeout
        import traceback
        q.put(traceback.format_exc())


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


def _cpu_restatement(which):
    from ministark_b200.air import Air, ProofOptions
    from oracle import stark_oracle as SO
    claim, opts, trace = _make_case(which)
    pub = claim if which == "brainfuck" else claim.get_public_inputs()
    mk = lambda n, o: Air(claim.AirConfig, n, pub, ProofOptions(*o))
    ext = getattr(trace, "build_extension_columns", None)
    want = SO.cpu_prove(claim, opts, trace.base_columns(), mk, ext_builder=ext if claim.AirConfig.NUM_EXTENSION_COLUMNS else None)
    return want, claim, mk


@pytest.mark.parametrize("which", ["fib", "perm", "brainfuck"])
def test_streamed_host_prover_bytes_equal_cpu_restatement(orc, cpu_lib, which):
    from oracle import stark_oracle as SO
    out = _spawn(_prove_worker, which, str(cpu_lib / "libms_host_nodes_cpu_abi.so"))
    assert isinstance(out, dict), out
    est = out["est"]
    assert est["streamed_host"] < est["streamed"] < est["resident"]
    want, claim, mk = _cpu_restatement(which)
    for validate in (False, True):
        residency, got, pinned, timed = out[validate]
        assert residency == "streamed_host" and got == want and pinned == est["host"] and timed
    SO.verify(claim, want, 10, mk)
    gib = lambda b: f"{b / 2**30:.2f} GiB"
    status, err = out["no_host"]
    assert status == "refused" and "host memory" not in err          # no host budget: the streamed refusal, word for word
    assert err == (f"the proof does not fit on the device: it needs about {gib(est['resident'])} resident or "
                   f"{gib(est['streamed'])} streamed, and {gib(_between(est))} is available")
    status, err = out["host_short"]
    assert status == "refused" and err.startswith(out["no_host"][1] + "; ")
    assert gib(est["streamed_host"]) in err and gib(est["host"]) in err and gib(est["host"] - 1) in err
    # heaps pinned under a larger budget are freed when a proof starts under a lower one (here: none), and pinned again
    assert out["no_host_pinned"] == out["host_short_pinned"] == 0
    assert out["pinned_again"] == est["host"] and out["released"] == 0


def _drop_worker(lib_path, q):
    """pinned allocations and frees of the context, across a dropped prover"""
    try:
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        _install(lib_path)
        import gc
        from ministark_b200 import Context
        from ministark_b200.air import ProofOptions
        from ministark_b200.prover import GpuProver
        pinned, freed = [], []
        alloc, free = Context.alloc_host_pinned, Context.free
        Context.alloc_host_pinned = lambda self, nbytes: pinned.append(alloc(self, nbytes)) or pinned[-1]
        Context.free = lambda self, ptr: freed.append(ptr) or free(self, ptr)
        claim, opts, trace = _make_case("fib")
        est = _estimates(claim, opts, len(trace))
        out = {}
        for how in ("dropped", "released"):
            p = GpuProver(0)
            p.memory_budget, p.host_memory_budget = _between(est), est["host"]
            p.prove(claim, ProofOptions(*opts), trace)
            out[how + "_held"] = (list(pinned), list(freed))
            if how == "released":
                p.release_host_memory()
            del p
            gc.collect()
            out[how] = (list(pinned), list(freed))
        q.put(out)
    except Exception:
        import traceback
        q.put(traceback.format_exc())


def test_a_dropped_prover_frees_its_pinned_heaps(orc, cpu_lib):
    out = _spawn(_drop_worker, str(cpu_lib / "libms_host_nodes_cpu_abi.so"))
    assert isinstance(out, dict), out
    pinned, freed = out["dropped_held"]
    assert len(pinned) == 1 and freed == []                           # held between proofs
    pinned, freed = out["dropped"]
    assert freed == pinned                                            # freed with the prover, once
    pinned, freed = out["released"]
    assert len(pinned) == 2 and freed == pinned                       # an explicit release is not freed twice


# ---------------------------------------------------------------------------------------------- the C++ prover
@pytest.fixture(scope="module")
def driver(cpu_lib):
    exe = cpu_lib / "host_nodes_test"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I", INCLUDE,
                           os.path.join(ROOT, "tests", "cpp", "host_nodes_test.cpp"), "-o", str(exe), "-L", str(cpu_lib),
                           "-lms_host_nodes_cpu_abi", f"-Wl,-rpath,{cpu_lib}"])

    def run(*args):
        return subprocess.run([str(exe)] + [str(a) for a in args], capture_output=True, text=True, timeout=900)
    return run


@pytest.mark.parametrize("log_n", [3, 10, 20, 25])
@pytest.mark.parametrize("beta", [1, 2, 16])
@pytest.mark.parametrize("nbase,next_,fq", [(8, 0, FP), (17, 9, FQ3), (3, 2, FQ3)])
@pytest.mark.parametrize("ce,ff", [(1, 2), (4, 8), (16, 16)])
def test_cpp_peak_bytes_equal_python(driver, log_n, beta, nbase, next_, fq, ce, ff):
    if ce > beta:
        pytest.skip("ce blow-up above the LDE blow-up")
    r = driver("peak", 1 << log_n, beta, nbase, next_, fq, ce, ff)
    assert r.returncode == 0, r.stderr
    want = peak_bytes(1 << log_n, beta, nbase, next_, fq, ce, ff)
    assert [int(v) for v in r.stdout.split()] == [want["resident"], want["streamed"], want["streamed_host"], want["host"]]


def test_cpp_streamed_host_fib_bytes_equal_cpu_restatement(driver, orc):
    from oracle import stark_oracle as SO
    want, claim, mk = _cpu_restatement("fib")
    est = _estimates(*_make_case("fib")[:2], 1 << 7)
    r = driver("fib", 7, 16, 4, 4, 8, 16, _between(est), est["host"])
    assert r.returncode == 0, r.stderr
    residency, pinned, proof = r.stdout.split()
    assert residency == "streamed_host" and int(pinned) == est["host"] and bytes.fromhex(proof) == want
    SO.verify(claim, want, 10, mk)


@pytest.mark.parametrize("second", ["none", "short", "same"])
def test_cpp_heaps_over_a_lowered_budget_are_freed(driver, second):
    est = _estimates(*_make_case("fib")[:2], 1 << 7)
    host2 = {"none": 0, "short": est["host"] - 1, "same": est["host"]}[second]
    r = driver("fib", 7, 16, 4, 4, 8, 16, _between(est), est["host"], host2)
    assert r.returncode == 0, r.stderr
    residency, pinned, _, pinned_after = r.stdout.split()
    assert residency == "streamed_host" and int(pinned) == est["host"]
    assert int(pinned_after) == (est["host"] if second == "same" else 0)


def test_cpp_streamed_host_brainfuck_bytes_equal_cpu_restatement(driver, orc):
    want, claim, mk = _cpu_restatement("brainfuck")
    _, opts, trace = _make_case("brainfuck")
    est = _estimates(claim, opts, len(trace))
    r = driver("bf", "hello", *opts, _between(est), est["host"])
    assert r.returncode == 0, r.stderr
    residency, pinned, out, proof = r.stdout.split()
    assert residency == "streamed_host" and int(pinned) == est["host"] and bytes.fromhex(proof) == want


def test_cpp_refusals_match_python(driver):
    _, opts, trace = _make_case("brainfuck")
    from ministark_b200.examples import brainfuck as bf
    claim = bf.BrainfuckClaim(bf.HELLO_WORLD, b"", bf.simulate(bf.HELLO_WORLD)[1])
    est = _estimates(claim, opts, len(trace))
    gib = lambda b: f"{b / 2**30:.2f} GiB"
    base = (f"the proof does not fit on the device: it needs about {gib(est['resident'])} resident or "
            f"{gib(est['streamed'])} streamed, and {gib(_between(est))} is available")
    r = driver("bf", "hello", *opts, _between(est), 0)
    assert r.returncode == 1 and r.stderr.strip() == "host_nodes_test: " + base
    r = driver("bf", "hello", *opts, _between(est), est["host"] - 1)
    assert r.returncode == 1
    assert r.stderr.strip() == ("host_nodes_test: " + base + f"; with the Merkle node heaps in pinned host memory it needs about "
                                f"{gib(est['streamed_host'])} on the device and {gib(est['host'])} of host memory, and "
                                f"{gib(est['host'] - 1)} of host memory is allowed")
