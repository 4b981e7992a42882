"""CPU-only: extension columns declared by the AIR (air.RunningColumn, AirConfig.extension_columns) and built on the device.

  * Air rejects a malformed declaration with a ValueError naming the column and the problem;
  * expr.compile_extension_program stores mul_k / add_k to slots 2k / 2k + 1, and the single-output programs of the
    example AIRs are word for word what they were before multi-slot stores existed;
  * ms_extension_columns of the CPU build (tests/cpp/extension_cpu_abi.c) equals oracle/extension_oracle.py word for word
    over Fp and Fq3, exclusive and inclusive columns, row offsets with wrap-around, X / Periodic / Hint leaves, division
    with zero denominators, one to 2^16 rows and one to four columns, and rejects malformed arguments and programs;
  * GpuProver on the CPU harness (tests/cpu_device.py), resident and streamed: the declared perm AIR proves to the bytes of
    the callback perm AIR and of oracle/stark_oracle.cpu_prove, the LogUp example to cpu_prove's bytes, Stark.verify
    accepts both, validate=True passes, and a wrong declaration or multiplicity raises ConstraintViolation;
  * ShardedProver over gloo with two ranks gives the same bytes.
Prover cases run in spawned workers that install the harness themselves; the pytest process never does."""
import ctypes as C
import hashlib
import os
import random
import socket
import subprocess
import sys

import numpy as np
import pytest

from ministark_b200 import expr as E
from ministark_b200.air import Air, AirConfig, ProofOptions, RunningColumn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = E.P
_R = 2**64
OPTS = ProofOptions(16, 8, 4, 4, 8)


def _mont(v):
    return int(v) % P * _R % P


# ------------------------------------------------------------------------------------------- 1. declarations
def _config(decl, nbase=2, next_=None, fq_is_fp=False):
    class Cfg(AirConfig):
        NUM_BASE_COLUMNS = nbase
        NUM_EXTENSION_COLUMNS = len(decl) if next_ is None else next_
        FQ_IS_FP = fq_is_fp

        @staticmethod
        def constraints(trace_len):
            return [(E.Trace(0) - E.Challenge(0) * E.Challenge(1)) / (E.X() - 1)]

        @staticmethod
        def extension_columns(trace_len):
            return decl
    return Cfg


@pytest.mark.parametrize("decl,next_,msg", [
    ([RunningColumn(1, E.Challenge(0) - E.Trace(0))], 2, "declares 1 columns but NUM_EXTENSION_COLUMNS is 2"),
    ([RunningColumn(1, E.Trace(2, 1))], None, "extension column 2: mul reads Trace(2, 1), which is not a base column"),
    ([RunningColumn(1), RunningColumn(0, add=E.Trace(3, 0))], None, "extension column 3: add reads Trace(3, 0)"),
    ([RunningColumn(E.Trace(0) + 1)], None, "extension column 2: init reads the trace"),
    ([RunningColumn(E.X())], None, "extension column 2: init reads X"),
    ([RunningColumn(1, add=E.Challenge(2))], None, "extension column 2: add reads Challenge(2), but the constraints make the "
                                                   "channel draw 2 challenges"),
    ([RunningColumn(E.Challenge(5))], None, "init reads Challenge(5)"),
    (["not a column"], None, "extension column 2: expected a RunningColumn"),
])
def test_invalid_declarations_raise(decl, next_, msg):
    with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(")", r"\)")):
        Air(_config(decl, next_=next_), 8, None, OPTS)


def test_valid_declaration_and_default():
    air = Air(_config([RunningColumn((1, 2, 3), E.Challenge(1) - E.Trace(1, -1), E.Hint(0) / E.Trace(0, 1), True)]), 8, None, OPTS)
    (col,) = air.extension_declaration
    assert isinstance(col.init, E.Expr) and col.inclusive
    assert air.extension_program() is air.extension_program()          # compiled once per Air
    from ministark_b200.examples import perm
    assert Air(perm.PermAirConfig, 8, None, OPTS).extension_declaration is None
    assert AirConfig.extension_columns(8) is None


# ---------------------------------------------------------------------------------------------- 2. compiler
# SHA-256 of the composition, DEEP and check programs (code and constants) of the fib, perm and brainfuck AIRs as the
# compiler emitted them before OP_STORE carried a slot
_PROGRAMS_DIGEST = "442e746ec1b0148807705db0df85afef3a8ab4344846ead32a6ed271f49e4e90"


def test_single_output_programs_are_unchanged():
    from ministark_b200.examples import brainfuck as bf
    from ministark_b200.examples import fib, perm
    h = hashlib.sha256()
    for cfg, n, o in ((fib.FibAirConfig, 1 << 8, (16, 4, 6, 8, 16)), (perm.PermAirConfig, 1 << 8, (16, 8, 4, 4, 8)),
                      (bf.BrainfuckAirConfig, 1 << 10, (19, 16, 20, 16, 16))):
        a = Air(cfg, n, None, ProofOptions(*o))
        for p in (a.composition_program(), a.deep_program()[0], a.check_program()):
            h.update(p.code.tobytes())
            h.update(p.consts.tobytes())
            stores = [w for w in p.code if int(w[0]) & 0xff == E.OP_STORE]
            assert all(int(w[1]) == 0 for w in stores)
    assert h.hexdigest() == _PROGRAMS_DIGEST


def test_extension_program_slots_and_sharing():
    a, b, al = E.Trace(0), E.Trace(1, 1), E.Challenge(0)
    shared = al - a
    prog = E.compile_extension_program([shared, E.Constant(1), shared * b], [E.Constant(0), E.Constant(1) / shared, b],
                                       2, 4, 2)
    stores = [(int(w[1]), int(w[2])) for w in prog.code if int(w[0]) & 0xff == E.OP_STORE]
    assert sorted(s for s, _ in stores) == list(range(6))
    ops = [int(w[0]) & 0xff for w in prog.code]
    assert ops.count(E.OP_TRACE) == 2                       # every cell loaded once
    assert ops.count(E.OP_NEG) == 1                         # alpha - a computed once for three roots
    assert E.OP_INV in ops and E.OP_DIV not in ops
    assert prog.bindings == [(prog.bindings[0][0], "chal", 0)]


# ------------------------------------------------------------------------------------------------ 3. CPU ABI
@pytest.fixture(scope="module")
def ext_abi(tmp_path_factory, orc):
    """tests/cpp/extension_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary directory"""
    out = str(tmp_path_factory.mktemp("ext_abi") / "libms_extension_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out, os.path.join(ROOT, "tests", "cpp", "extension_cpu_abi.c")])
    return out


@pytest.fixture(scope="module")
def abi(ext_abi):
    from ministark_b200 import _lib
    lib = C.CDLL(ext_abi)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    _lib.bind(lib, _lib._EXTENSION_SIGS)
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    return lib, h


def _periodic_tables(prog, log_n, lanes):
    """the program's periodic tables over <g_n> by their definition (natural order), Montgomery words"""
    if not prog.periodic:
        return []
    g = pow(pow(7, (P - 1) >> 32, P), 1 << (32 - log_n), P)
    n = 1 << log_n
    out = []
    for _, coeffs, interval, is_q, log_len in prog.periodic:
        words = []
        for i in range(1 << log_len):
            y = pow(g, i * (n // interval), P)
            v = (0, 0, 0)
            for c in reversed(coeffs):
                v = E.q_add(E.q_mul(v, (y, 0, 0)), E._q(c))
            words += [_mont(w) for w in (v if is_q and lanes == 3 else v[:1])]
        out.append(np.array(words, dtype=np.uint64))
    return out


def run_abi(abi, prog, base, lanes, log_n, init_words, inclusive, code=None, isq=None, ncolumns=None):
    lib, h = abi
    code = prog.code if code is None else np.ascontiguousarray(code, dtype=np.uint32)
    tables = _periodic_tables(prog, log_n, lanes)
    cols = [np.ascontiguousarray(c) for c in base] + tables
    isq = [0] * len(base) + [int(p[3]) for p in prog.periodic] if isq is None else isq
    ptrs = (C.c_void_p * max(len(cols), 1))(*[c.ctypes.data for c in cols])
    q = (C.c_int * max(len(cols), 1))(*isq)
    K = len(inclusive) if ncolumns is None else ncolumns
    inc = (C.c_int * max(len(inclusive), 1))(*[int(v) for v in inclusive])
    ini = np.ascontiguousarray(init_words, dtype=np.uint64).reshape(-1)
    out = np.zeros((max(K, 1), (1 << min(log_n, 16)) * lanes), dtype=np.uint64)    # refused calls write nothing
    rc = lib.ms_extension_columns(h, code.ctypes.data, code.shape[0], prog.consts.ctypes.data, prog.consts.shape[0], ptrs, q,
                                  len(cols), lanes, log_n, K, ini.ctypes.data, inc, out.ctypes.data)
    return rc, lib.ms_last_error(h).decode() if rc else "", out


def random_declaration(seed, log_n, nbase, K, fq3, nchal=2, nhint=2):
    """K RunningColumns over nbase base columns: offsets -1..1, X, Periodic, Challenge, Hint leaves, divisions (zero
    denominators planted where the trace is zero), random inclusive flags"""
    rng = random.Random(seed)
    X = E.X()

    def leaf():
        r = rng.random()
        if r < 0.4:
            return E.Trace(rng.randrange(nbase), rng.choice([-1, 0, 1]))
        if r < 0.5:
            return X
        if r < 0.6:
            return E.Challenge(rng.randrange(nchal))
        if r < 0.7:
            return E.Hint(rng.randrange(nhint))
        if r < 0.8:
            iv = 1 << rng.randint(0, log_n)
            return E.Periodic([rng.randrange(P) for _ in range(rng.choice([c for c in (1, 2, 4) if c <= iv]))], iv)
        if r < 0.9 and fq3:
            return E.Constant((rng.randrange(P), rng.randrange(P), rng.randrange(P)))
        return E.Constant(rng.randrange(P))

    def expr(depth):
        if depth == 0 or rng.random() < 0.25:
            return leaf()
        op = rng.choice(["add", "sub", "mul", "mul", "div", "pow", "neg"])
        a = expr(depth - 1)
        if op == "neg":
            return -a
        if op == "pow":
            return a ** rng.randint(0, 5)
        if op == "div":
            return a / rng.choice([E.Trace(rng.randrange(nbase), rng.choice([-1, 0, 1])), expr(depth - 1), E.Constant(0)])
        b = expr(depth - 1)
        return {"add": a + b, "sub": a - b, "mul": a * b}[op]

    sym = [E.Challenge(0), E.Hint(1), E.Constant(rng.randrange(P)), E.Constant(0)]
    return [RunningColumn(rng.choice(sym) + rng.choice(sym), expr(3), expr(3), rng.random() < 0.5) for _ in range(K)]


def _case_inputs(seed, log_n, nbase, fq3):
    rng = random.Random(seed * 7 + 1)
    n = 1 << log_n
    base = [[0 if rng.random() < 0.2 else rng.randrange(P) for _ in range(n)] for _ in range(nbase)]
    chal = [(rng.randrange(P), rng.randrange(P), rng.randrange(P)) if fq3 else rng.randrange(P) for _ in range(2)]
    hints = [(rng.randrange(P), 0, rng.randrange(P)) if fq3 else rng.randrange(P) for _ in range(2)]
    return np.array([[_mont(v) for v in c] for c in base], dtype=np.uint64).reshape(nbase, n), chal, hints


def _check_against_oracle(abi, decl, base, lanes, log_n, chal, hints):
    from oracle import extension_oracle as XO
    nbase = base.shape[0]
    prog = E.compile_extension_program([c.mul for c in decl], [c.add for c in decl], nbase, log_n, nbase)
    prog = prog.bind(challenges=chal, hints=hints)
    init = [[_mont(w) for w in E.evaluate_at(E.Expr._lift(c.init), 0, challenges=chal, hints=hints)[:lanes]] for c in decl]
    rc, err, got = run_abi(abi, prog, list(base), lanes, log_n, init, [c.inclusive for c in decl])
    assert rc == 0, err
    want = XO.columns([(c.init, c.mul, c.add, c.inclusive) for c in decl], base, lanes, chal, hints)
    assert np.array_equal(got, want)


CASES = [(s, log_n, K, fq3) for s, (log_n, K, fq3) in enumerate(
    [(0, 1, True), (0, 4, False), (1, 1, False), (1, 4, True), (11, 1, True), (11, 4, False), (12, 1, False), (12, 4, True),
     (4, 4, True), (5, 1, False), (16, 1, True), (16, 4, False)])]


@pytest.mark.parametrize("seed,log_n,K,fq3", CASES)
def test_cpu_abi_equals_oracle(abi, seed, log_n, K, fq3):
    lanes = 3 if fq3 else 1
    decl = random_declaration(seed, log_n, 3, K, fq3)
    base, chal, hints = _case_inputs(seed, log_n, 3, fq3)
    _check_against_oracle(abi, decl, base, lanes, log_n, chal, hints)


@pytest.mark.parametrize("fq3", [False, True])
@pytest.mark.parametrize("inclusive", [False, True])
def test_cpu_abi_named_shapes(abi, fq3, inclusive):
    """the shapes the examples use, and a division whose denominator vanishes on chosen rows (0 there, not an error)"""
    lanes = 3 if fq3 else 1
    log_n = 6
    base, chal, hints = _case_inputs(99, log_n, 3, fq3)
    base[1, ::5] = 0
    al, T = E.Challenge(0), E.Trace
    decl = [RunningColumn(1, al - T(0), inclusive=inclusive),                           # running product
            RunningColumn(0, al, T(2, -1), inclusive=inclusive),                        # running evaluation, wrap-around
            RunningColumn(E.Hint(0), add=T(2, 1) / T(1) - E.Constant(1) / (al - T(0)), inclusive=inclusive),   # LogUp sum
            RunningColumn(E.Challenge(1), E.X() * E.Periodic([3, 5], 4), E.Constant(7) / E.Constant(0), inclusive=inclusive)]
    _check_against_oracle(abi, decl, base, lanes, log_n, chal, hints)


def test_cpu_abi_rejects_malformed_arguments_and_programs(abi):
    lib, h = abi
    base, chal, hints = _case_inputs(5, 3, 2, True)
    decl = [RunningColumn(1, E.Challenge(0) - E.Trace(0)), RunningColumn(0, add=E.Trace(1, 1))]
    prog = E.compile_extension_program([c.mul for c in decl], [c.add for c in decl], 2, 3, 2).bind(challenges=chal)
    init = [[_mont(1), 0, 0], [0, 0, 0]]
    ok = lambda **kw: run_abi(abi, prog, list(base), kw.pop("lanes", 3), kw.pop("log_n", 3), kw.pop("init", init),
                              kw.pop("inclusive", [0, 0]), **kw)
    assert ok()[0] == 0
    assert "bad Fq field id" in ok(lanes=2)[1]
    assert "domain too large" in ok(log_n=33)[1]
    assert "0 columns" in ok(ncolumns=0)[1]
    assert "9 columns (1 to 8)" in ok(ncolumns=9)[1]
    assert "non-canonical init of column 1" in ok(init=[[_mont(1), 0, 0], [0, P, 0]])[1]
    assert "never stores slot 4 of 6" in ok(inclusive=[0, 0, 0], init=init + [[0, 0, 0]])[1]
    assert "wrong field" in ok(isq=[1, 0])[1]
    bad = prog.code.copy()
    bad[0, 0] = E.OP_DIV
    assert "bad instruction 0" in ok(code=bad)[1]
    bad = prog.code.copy()
    st = [i for i, w in enumerate(bad) if int(w[0]) & 0xff == E.OP_STORE][-1]
    bad[st, 1] = 4
    assert "stores to slot 4 of 4" in ok(code=bad)[1]
    bad = prog.code.copy()
    bad[st, 2] = 40
    assert "before it is written" in ok(code=bad)[1]
    bad = prog.code.copy()
    tr = [i for i, w in enumerate(bad) if int(w[0]) & 0xff == E.OP_TRACE][0]
    bad[tr, 2] = 7
    assert "column 7 out of range" in ok(code=bad)[1]


# ------------------------------------------------------------------------------------------------- 4. the prover
def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS):
        _lib.bind(lib, sigs)
    _lib._lib = lib


def _make_case(which):
    """(claim, options, trace) of a named case; 'perm' keeps its host callback, the others declare"""
    from ministark_b200.examples import lookup, perm
    kind, _, variant = which.partition(":")
    if kind == "perm":
        return perm.PermClaim(), (16, 8, 4, 4, 8), perm.gen_trace(1 << 8, seed=3)
    if kind == "declared":
        claim = perm.PermDeclaredClaim()
        if variant == "init2":
            class Wrong(perm.PermDeclaredAirConfig):
                @staticmethod
                def extension_columns(trace_len):
                    ok = perm.PermDeclaredAirConfig.extension_columns(trace_len)
                    return [RunningColumn(2, ok[0].mul), ok[1]]

            claim = type("WrongClaim", (perm.PermDeclaredClaim,), {"AirConfig": Wrong})()
        return claim, (16, 8, 4, 4, 8), perm.gen_trace(1 << 8, seed=3, extension=False)
    trace = lookup.gen_trace(1 << 8, seed=4)
    if variant == "bad_m":
        from ministark_b200.prover import Trace
        base = np.array(trace.base_columns(), copy=True)
        base[2, 0] += np.uint64(_R % P)                         # multiplicity of t_0 one too high
        trace = Trace(base)
    return lookup.LookupClaim(), (16, 8, 4, 4, 8), trace


def _prove_worker(which, lib_path, residency, validate, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    from ministark_b200 import FP, FQ3
    from ministark_b200.prover import GpuProver, peak_bytes
    from ministark_b200.validate import ConstraintViolation
    claim, opts, trace = _make_case(which)
    p = GpuProver(0)
    if residency == "streamed":
        cfg, o, n = claim.AirConfig, ProofOptions(*opts), len(trace)
        est = peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, FP if cfg.FQ_IS_FP else FQ3,
                         Air(cfg, n, None, o).ce_blowup_factor, o.fri_folding_factor)
        p.memory_budget = (est["streamed"] + est["resident"]) // 2
    out = {}
    try:
        proof = p.prove(claim, ProofOptions(*opts), trace, validate=validate)
        out["bytes"] = proof.to_bytes()
        claim.verify(out["bytes"], 10)
        out["verified"] = True
    except ConstraintViolation as e:
        out["violations"] = [(v.constraint, v.first_row, v.count) for v in e.violations]
    out["residency"] = p.last_residency
    q.put(out)


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
    from oracle import extension_oracle as XO
    from oracle import stark_oracle as SO
    claim, opts, trace = _make_case(which)
    mk = lambda n, o: Air(claim.AirConfig, n, claim.get_public_inputs(), ProofOptions(*o))
    if trace._ext is not None:                                  # the trace's own host callback
        ext = trace.build_extension_columns
    else:
        ext = XO.builder(claim.AirConfig, trace.base_columns(), claim.get_public_inputs())
    want = SO.cpu_prove(claim, opts, trace.base_columns(), mk, ext_builder=ext)
    SO.verify(claim, want, 10, mk)
    return want


@pytest.mark.parametrize("residency", ["resident", "streamed"])
@pytest.mark.parametrize("which", ["declared", "lookup"])
def test_declared_airs_prove_to_the_restatement(orc, ext_abi, which, residency):
    out = _spawn(_prove_worker, which, ext_abi, residency, True)
    assert "violations" not in out, out["violations"]
    assert out["residency"] == residency and out["verified"]
    want = _cpu_restatement(which)
    assert out["bytes"] == want
    if which == "declared":                                     # the host callback's AIR gives the same proof
        assert _spawn(_prove_worker, "perm", ext_abi, residency, False)["bytes"] == want


@pytest.mark.parametrize("which,constraints", [("declared:init2", [0, 4]), ("lookup:bad_m", [4])])
def test_wrong_declaration_or_multiplicity_fails_validation(ext_abi, which, constraints):
    """init = 2 breaks the boundary op_0 = 1 (and with it the final product check); a multiplicity one too high breaks the
    zero sum at the last row"""
    out = _spawn(_prove_worker, which, ext_abi, "resident", True)
    assert "violations" in out, "the wrong trace passed validation"
    assert [v[0] for v in out["violations"]] == constraints


def _hint_worker(lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    from ministark_b200.examples import perm
    from ministark_b200.prover import GpuProver, ProvingError

    class HintCfg(perm.PermDeclaredAirConfig):
        @staticmethod
        def extension_columns(trace_len):
            ok = perm.PermDeclaredAirConfig.extension_columns(trace_len)
            return [RunningColumn(E.Hint(3), ok[0].mul), ok[1]]

    claim = type("HintClaim", (perm.PermDeclaredClaim,), {"AirConfig": HintCfg})()
    try:
        GpuProver(0).prove(claim, OPTS, perm.gen_trace(1 << 6, extension=False))
        q.put(None)
    except ProvingError as e:
        q.put(str(e))


def test_hint_beyond_gen_hints_raises_proving_error(ext_abi):
    assert _spawn(_hint_worker, ext_abi) == "extension column 3 reads Hint(3), but gen_hints returned 0 hints"


def _sharded_worker(rank, world, port, which, lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.setdefault("OMP_NUM_THREADS", "2")
    _install(lib_path)
    import torch.distributed as dist
    from ministark_b200.prover_mgpu import ShardedProver
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        claim, opts, trace = _make_case(which)
        q.put((rank, ShardedProver(dist, rank).prove(claim, ProofOptions(*opts), trace).to_bytes()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("which", ["declared", "lookup"])
def test_sharded_prover_over_gloo(orc, ext_abi, which):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, which, ext_abi, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=900) for _ in range(2)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    want = _cpu_restatement(which)
    for rank, b in got:
        assert b == want, f"rank {rank}"


# ---------------------------------------------------------------------------------------------------- 5. header
def test_extension_header_is_bound_exported_and_separate(ext_abi):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.EXTENSION_HEADER_PATH)
    assert declared == sorted(_lib._EXTENSION_SIGS) == ["ms_extension_columns"]
    others = set(_lib.header_symbols()) | set(_lib.header_symbols(_lib.STREAM_HEADER_PATH)) | \
        set(_lib.header_symbols(_lib.CHECK_HEADER_PATH)) | set(_lib.header_symbols(_lib.BF_HEADER_PATH))
    assert not set(declared) & others
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(ext_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)
