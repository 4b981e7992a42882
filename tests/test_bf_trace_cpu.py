"""CPU-only: the brainfuck execution trace built natively (include/ministark_bf.h).

  * ms_bf_run of the product library: the records and the output of `simulate` (the host path) on a program corpus and
    on seeded random programs, and its three errors (tape left, input exhausted, cycle cap);
  * the table entry points of the CPU build (tests/cpp/bf_trace_cpu_abi.c, the CPU build of the constraint check plus
    include/ministark_bf.h): `simulate(..., device=...)` on the CPU harness (tests/cpu_device.py) gives the host trace's
    17 base columns and eight helper columns word for word, and proofs from that trace equal the host trace's, in both
    residencies;
  * the header is bound, exported, and disjoint from include/ministark_b200.h.
Harness cases run in spawned workers that install it themselves; the pytest process never does."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ECHO = ",>,<.>."
TAPE_WALK = ">+" * 1000 + "[<]>."                           # marks 1000 cells, then walks back over them
CORPUS = [
    ("hello_world", None, b""),
    ("echo", ECHO, b"hi"),
    ("burner", "burner:3,4,5", b""),
    ("tape_walk", TAPE_WALK, b""),
    ("reads_in_loop", ",[.-]", b"\x05"),
    ("wrap", "-.+.", b""),
]


def _source(src):
    from ministark_b200.examples import brainfuck as bf
    if src is None:
        return bf.HELLO_WORLD
    head, _, burner = src.partition("burner:")
    return head + (bf.cycle_burner(*(int(v) for v in burner.split(","))) if burner else "")


def random_program(rng, size):
    """balanced brackets over the eight opcodes; loops are short so that many runs end"""
    out, depth = [], 0
    for _ in range(size):
        r = rng.random()
        if r < 0.1:
            out.append("[")
            depth += 1
        elif r < 0.2 and depth:
            out.append("-]")
            depth -= 1
        else:
            out.append(rng.choice("+-<>.,>+"))
    return "".join(out) + "-]" * depth


def random_cases(count, seed, cap=5000):
    """(source, input) of seeded random programs that end within `cap` cycles on the tape and the input they are given"""
    import ministark_b200 as ms
    from ministark_b200.examples import brainfuck as bf
    rng = random.Random(seed)
    cases = []
    while len(cases) < count:
        src = random_program(rng, rng.randint(1, 60))
        inp = bytes(rng.randrange(256) for _ in range(rng.randint(0, 40)))
        try:
            ms.bf_run(np.array(bf.compile_program(src), dtype=np.uint32), inp, cap)
        except ms.MsError:
            continue
        cases.append((src, inp))
    return cases


def _host_records(trace):
    """the processor rows of a host trace up to the final state, packed like ms_bf_run's records"""
    from ministark_b200.examples import brainfuck as bf
    recs = []
    for row in trace.rows:
        recs.append(row[bf.IP] | row[bf.MP] << 32 | row[bf.MEM_VAL] << 48)
        if row[bf.CURR_INSTR] == 0:
            break
    return np.array(recs, dtype=np.uint64)


# ------------------------------------------------------------------------------------------------- 1. the VM
@pytest.mark.parametrize("name,src,inp", CORPUS)
def test_bf_run_matches_simulate(name, src, inp):
    import ministark_b200 as ms
    from ministark_b200.examples import brainfuck as bf
    source = _source(src)
    trace, output = bf.simulate(source, inp)
    log, out = ms.bf_run(np.array(bf.compile_program(source), dtype=np.uint32), inp)
    assert out == output
    assert np.array_equal(log, _host_records(trace))


def test_bf_run_matches_simulate_random():
    import ministark_b200 as ms
    from ministark_b200.examples import brainfuck as bf
    for src, inp in random_cases(100, seed=11):
        trace, output = bf.simulate(src, inp)
        log, out = ms.bf_run(np.array(bf.compile_program(src), dtype=np.uint32), inp)
        assert out == output, src
        assert np.array_equal(log, _host_records(trace)), src


@pytest.mark.parametrize("src,inp,msg", [
    ("<+", b"", "memory pointer leaves"),
    (">" * 1024, b"", "memory pointer leaves"),
    (",,", b"a", "input exhausted"),
    ("+[]", b"", "cycle cap"),
])
def test_bf_run_errors(src, inp, msg):
    import ministark_b200 as ms
    from ministark_b200.examples import brainfuck as bf
    with pytest.raises(ms.MsError, match=msg):
        ms.bf_run(np.array(bf.compile_program(src), dtype=np.uint32), inp, max_cycles=10_000)


def test_bf_run_error_message_lasts_until_the_next_run():
    import ministark_b200 as ms
    from ministark_b200 import _lib
    from ministark_b200.examples import brainfuck as bf
    lib = _lib.load()
    with pytest.raises(ms.MsError, match="input exhausted"):
        ms.bf_run(np.array(bf.compile_program(","), dtype=np.uint32), b"")
    assert b"input exhausted" in lib.ms_last_error(None)
    ms.bf_run(np.array(bf.compile_program("+."), dtype=np.uint32), b"")
    assert lib.ms_last_error(None) == b"null context"


# --------------------------------------------------------------------------------------- 2. tables and proofs
@pytest.fixture(scope="module")
def bf_abi(tmp_path_factory, orc):
    """tests/cpp/bf_trace_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary directory"""
    out = str(tmp_path_factory.mktemp("bf_abi") / "libms_bf_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out, os.path.join(ROOT, "tests", "cpp", "bf_trace_cpu_abi.c")])
    return out


def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._BF_SIGS):
        _lib.bind(lib, sigs)
    _lib._lib = lib


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


def _tables_worker(lib_path, cases, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    from ministark_b200 import Context
    from ministark_b200.examples import brainfuck as bf
    bad = []
    for src, inp in cases:
        host, out_h = bf.simulate(src, inp)
        dev, out_d = bf.simulate(src, inp, device="cpu")
        base = dev.base_columns().numpy().view(np.uint64)
        aux = dev.helper_columns_device(Context(0)).numpy().view(np.uint64)
        ok = (out_h == out_d and len(dev) == len(host) and np.array_equal(base, host.base_columns())
              and np.array_equal(aux, host.helper_columns()))
        if not ok:
            bad.append(src)
    q.put(bad)


def test_cpu_tables_equal_host_trace(bf_abi):
    cases = [(_source(src), inp) for _, src, inp in CORPUS] + random_cases(40, seed=5)
    assert _spawn(_tables_worker, bf_abi, cases) == []


OPTS = (8, 16, 4, 16, 16)


def _prove_worker(lib_path, src, inp, valid, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    try:
        q.put(_prove_both(src, inp, valid))
    except Exception:                       # reported, not left for the queue's timeout
        import traceback
        q.put(traceback.format_exc())


def _prove_both(src, inp, validate):
    from ministark_b200 import FQ3
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.examples import brainfuck as bf
    from ministark_b200.prover import GpuProver, peak_bytes
    host, out = bf.simulate(src, inp)
    claim = bf.BrainfuckClaim(src, inp, out)
    o = ProofOptions(*OPTS)
    n = len(host)
    est = peak_bytes(n, o.lde_blowup_factor, 17, 9, FQ3, Air(claim.AirConfig, n, None, o).ce_blowup_factor, o.fri_folding_factor)
    got = {}
    for residency, budget in [("resident", None), ("streamed", (est["streamed"] + est["resident"]) // 2)]:
        for kind in ("host", "device"):
            trace = host if kind == "host" else bf.simulate(src, inp, device="cpu")[0]
            p = GpuProver(0)
            p.memory_budget = budget
            got[residency, kind] = (p.prove(claim, o, trace, validate=validate).to_bytes(), p.last_residency)
    return got


# The echo program alone pads to 16 rows, too few for any blowup of this AIR, so it runs ahead of a small burner.  Its
# trace does not satisfy the AIR (a cell's first memory row must hold 0, and ',' writes into a fresh cell), so its proofs
# are compared without validation and not verified.
@pytest.mark.parametrize("src,inp,valid", [(None, b"", True), (ECHO + ">" + "burner:3,4,5", b"hi", False),
                                           ("burner:3,4,5", b"", True)])
def test_device_trace_proofs_equal_host_trace_proofs(bf_abi, src, inp, valid):
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.examples import brainfuck as bf
    from oracle import stark_oracle as SO
    source = _source(src)
    got = _spawn(_prove_worker, bf_abi, source, inp, valid)
    assert isinstance(got, dict), got
    for residency in ("resident", "streamed"):
        assert got[residency, "device"] == got[residency, "host"]
        assert got[residency, "device"][1] == residency
    assert got["resident", "device"][0] == got["streamed", "device"][0]
    if not valid:
        return
    _, out = bf.simulate(source, inp)
    claim = bf.BrainfuckClaim(source, inp, out)
    SO.verify(claim, got["resident", "device"][0], 10, lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o)))


# ------------------------------------------------------------------------------------------------ 3. the header
def test_bf_header_bound_and_exported(bf_abi):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.BF_HEADER_PATH)
    assert declared == sorted(_lib._BF_SIGS) == ["ms_bf_helper_columns", "ms_bf_run", "ms_bf_trace_fill", "ms_bf_trace_sizes"]
    assert not set(declared) & set(_lib.header_symbols())
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(bf_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)
