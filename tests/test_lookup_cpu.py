"""CPU-only: LogUp lookups declared by the AIR (air.Lookup, AirConfig.lookups), their generated constraints and running sums,
and their multiplicity columns filled by ms_lookup_multiplicities.

  * Air rejects a malformed lookup with a ValueError naming the lookup and the problem, merges the generated running sums
    into extension_columns by the None / RunningColumn rules, and assigns the challenges after the AIR's own;
  * ms_lookup_multiplicities of the CPU build (tests/cpp/lookup_cpu_abi.c) equals oracle/lookup_oracle.py word for word:
    widths and tuple counts 1 to 4, selectors, wrapping offsets, X and Periodic leaves, runs of duplicate table tuples,
    words 0 and p - 1, misses and bad selectors, one to 2^16 rows; malformed arguments are refused;
  * GpuProver on the CPU harness (tests/cpu_device.py), resident and streamed: DeclaredLookupClaim proves to the bytes of
    the hand-written LookupClaim and of oracle/stark_oracle.cpu_prove, SquareLookupClaim to cpu_prove's bytes; a wrong value
    raises LookupViolation, and a corrupted fill is refused by validate=True and by Stark.verify;
  * ShardedProver over gloo with two ranks gives the same bytes.
Prover cases run in spawned workers that install the harness themselves; the pytest process never does."""
import ctypes as C
import os
import random
import re
import socket
import subprocess
import sys

import numpy as np
import pytest

from ministark_b200 import expr as E
from ministark_b200.air import Air, AirConfig, Lookup, ProofOptions, RunningColumn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = E.P
_R = 2**64
OPTS = ProofOptions(16, 8, 4, 4, 8)
T = E.Trace


def _mont(v):
    return int(v) % P * _R % P


# ------------------------------------------------------------------------------------------- 1. declarations
def _config(lookups, nbase=4, next_=1, ext=None, fq_is_fp=False):
    class Cfg(AirConfig):
        NUM_BASE_COLUMNS = nbase
        NUM_EXTENSION_COLUMNS = next_
        FQ_IS_FP = fq_is_fp

        @staticmethod
        def constraints(trace_len):
            return [(T(0) - E.Challenge(0) * E.Challenge(1)) / (E.X() - 1)]

        @staticmethod
        def extension_columns(trace_len):
            return ext

        @staticmethod
        def lookups(trace_len):
            return lookups
    return Cfg


def _lk(table=(T(0),), values=((T(1),),), m=2, s=4, sel=None):
    return Lookup(table, values, m, s, sel)


@pytest.mark.parametrize("lookups,next_,msg", [
    ([_lk(m=4)], 1, "lookup 0: multiplicity column 4 is not a base column (0..3)"),
    ([_lk(), _lk(s=5)], 2, "lookup 1: multiplicity column 2 is also lookup 0's"),
    ([_lk(s=3)], 1, "lookup 0: running-sum column 3 is not an extension column (4..4)"),
    ([_lk(), _lk(m=3)], 2, "lookup 1: running-sum column 4 is also lookup 0's"),
    ([_lk(values=((T(1), T(0)),))], 1, "lookup 0: value tuple 0 has width 2, the table 1"),
    ([_lk(table=(T(0),) * 5, values=((T(1),) * 5,))], 1, "lookup 0: table tuples of width 5; 1 to 4 are supported"),
    ([_lk(values=((T(1),),) * 5)], 1, "lookup 0: 5 value tuples; 1 to 4 are supported"),
    ([_lk(table=())], 1, "lookup 0: table tuples of width 0"),
    ([_lk(sel=(T(3), T(3)))], 1, "lookup 0: 2 selectors for 1 value tuples"),
    ([_lk(values=((T(2, 1),),))], 1, "lookup 0: values[0][0] reads Trace(2, 1), the multiplicity column of lookup 0"),
    ([_lk(table=(T(0) + E.Challenge(0),))], 1, "lookup 0: table[0] reads a challenge"),
    ([_lk(sel=(E.Hint(0),))], 1, "lookup 0: selectors[0] reads a hint"),
    ([_lk(values=((T(4),),))], 1, "lookup 0: values[0][0] reads Trace(4, 0), which is not a base column"),
    ([_lk(table=(E.Expr("ccoef", 0),))], 1, "lookup 0: table[0] reads a composition coefficient"),
    ([_lk(table=(E.Constant((1, 2, 3)),))], 1, "lookup 0: table[0] reads an extension-field constant"),
    (["not a lookup"], 1, "lookup 0: expected a Lookup"),
])
def test_invalid_lookups_raise(lookups, next_, msg):
    with pytest.raises(ValueError, match=re.escape(msg)):
        Air(_config(lookups, next_=next_), 8, None, OPTS)


def test_extension_columns_merge_rules():
    rc = RunningColumn(1, E.Challenge(0) - T(0))
    # None at every lookup position, RunningColumns elsewhere
    air = Air(_config([_lk(s=5)], next_=2, ext=[rc, None]), 8, None, OPTS)
    user, gen = air.extension_declaration
    assert user.mul is rc.mul and user.init is E.Constant(1) and gen.init is E.Constant(0) and gen.mul is E.Constant(1)
    bad = [([rc, rc], "extension column 5: lookup 0's running sum is declared by the package"),
           ([None, None], "extension column 4: expected a RunningColumn, got NoneType"),
           (None, "extension_columns returned None, but only 1 of the 2 extension columns are lookup running sums"),
           ([None], "extension_columns declares 1 columns but NUM_EXTENSION_COLUMNS is 2")]
    for ext, msg in bad:
        with pytest.raises(ValueError, match=re.escape(msg)):
            Air(_config([_lk(s=5)], next_=2, ext=ext), 8, None, OPTS)
    # None as a whole when every extension column is a lookup sum
    air = Air(_config([_lk(), _lk(m=3, s=5)], next_=2), 8, None, OPTS)
    assert [c.init for c in air.extension_declaration] == [E.Constant(0)] * 2


def test_challenge_indices_and_default():
    # the AIR's own constraints draw 2; W = 1 takes alpha only, W = 2 takes alpha and beta
    air = Air(_config([_lk(), _lk(table=(T(0), T(1)), values=((T(1), T(0)),), m=3, s=5)], next_=2), 8, None, OPTS)
    assert air.lookup_challenges == [(2, None), (3, 4)]
    assert air.num_challenges() == 5
    assert len(air.constraints) == 1 + 3 * 2
    assert AirConfig.lookups(8) == []
    from ministark_b200.examples import lookup, perm
    assert Air(perm.PermAirConfig, 8, None, OPTS).lookups == []
    assert Air(lookup.LookupAirConfig, 8, None, OPTS).lookups == []
    a = Air(lookup.DeclaredLookupAirConfig, 8, None, OPTS)
    assert a.lookup_programs() is a.lookup_programs()


def test_generated_constraints_are_the_hand_written_ones():
    """Q = W = 1 without selectors: node for node LookupAirConfig's constraints, and the same running sum"""
    from ministark_b200.examples import lookup
    for n in (8, 1 << 10):
        a, b = Air(lookup.DeclaredLookupAirConfig, n, None, OPTS), Air(lookup.LookupAirConfig, n, None, OPTS)
        assert len(a.constraints) == len(b.constraints) and all(x is y for x, y in zip(a.constraints, b.constraints))
        assert a.ce_blowup_factor == b.ce_blowup_factor and a.num_challenges() == b.num_challenges() == 1
        (sa,), (sb,) = a.extension_declaration, b.extension_declaration
        assert sa.add is sb.add and sa.mul is sb.mul and sa.init is sb.init


def test_lookup_program_slots():
    prog = E.compile_lookup_program((T(0), T(1, 1)), ((T(2), T(0, -1)), (E.X(), T(1))), (E.Constant(1), T(3)), 4, 3)
    stores = sorted(int(w[1]) for w in prog.code if int(w[0]) & 0xff == E.OP_STORE)
    assert stores == list(range(E.lookup_slots(2, 2))) == list(range(8))
    assert all(not (int(w[0]) >> 8) & 1 for w in prog.code if int(w[0]) & 0xff == E.OP_STORE)


# ------------------------------------------------------------------------------------------------ 2. CPU ABI
@pytest.fixture(scope="module")
def lookup_abi(tmp_path_factory, orc):
    """tests/cpp/lookup_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary directory"""
    out = str(tmp_path_factory.mktemp("lookup_abi") / "libms_lookup_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out, os.path.join(ROOT, "tests", "cpp", "lookup_cpu_abi.c")])
    return out


@pytest.fixture(scope="module")
def abi(lookup_abi):
    from ministark_b200 import _lib
    lib = C.CDLL(lookup_abi)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    _lib.bind(lib, _lib._LOOKUP_SIGS)
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    return lib, h


def periodic_tables(prog, log_n):
    """the program's periodic tables over <g_n> by their definition (natural order), Montgomery words"""
    g = pow(pow(7, (P - 1) >> 32, P), 1 << (32 - log_n), P)
    n, out = 1 << log_n, []
    for _, coeffs, interval, _, log_len in prog.periodic:
        words = []
        for i in range(1 << log_len):
            y, v = pow(g, i * (n // interval), P), 0
            for c in reversed(coeffs):
                v = (v * y + c) % P
            words.append(_mont(v))
        out.append(np.array(words, dtype=np.uint64))
    return out


def run_abi(abi, lk, base, log_n, code=None, width=None, ntuples=None, ws_bytes=None, isq=None, prog=None):
    lib, h = abi
    W, Q = len(lk.table), len(lk.values)
    prog = prog or E.compile_lookup_program(lk.table, lk.values, lk.selectors, base.shape[0], log_n)
    code = prog.code if code is None else np.ascontiguousarray(code, dtype=np.uint32)
    cols = [np.ascontiguousarray(c) for c in base] + periodic_tables(prog, log_n)
    ptrs = (C.c_void_p * max(len(cols), 1))(*[c.ctypes.data for c in cols])
    q = (C.c_int * max(len(cols), 1))(*([0] * len(cols) if isq is None else isq))
    W, Q = width or W, ntuples or Q
    need = C.c_size_t()
    assert lib.ms_lookup_workspace_bytes(min(log_n, 16), min(max(W, 1), 4), min(max(Q, 1), 4), C.byref(need)) == 0
    work = np.zeros(need.value if ws_bytes is None else ws_bytes, dtype=np.uint8)
    out = np.zeros(1 << min(log_n, 16), dtype=np.uint64)
    status = np.zeros(2 * 4 + 2, dtype=np.uint64)
    rc = lib.ms_lookup_multiplicities(h, code.ctypes.data, code.shape[0], prog.consts.ctypes.data, prog.consts.shape[0], ptrs,
                                      q, len(cols), log_n, W, Q, work.ctypes.data, work.size, out.ctypes.data,
                                      status.ctypes.data)
    if rc:
        return rc, lib.ms_last_error(h).decode(), out, None
    none = lambda r: None if int(r) == 2**64 - 1 else int(r)
    st = ([(int(status[2 * k]), none(status[2 * k + 1])) for k in range(Q)], (int(status[2 * Q]), none(status[2 * Q + 1])))
    return rc, lib.ms_last_error(h).decode() if rc else "", out, st


def _check(abi, lk, base):
    from oracle import lookup_oracle as LO
    log_n = base.shape[1].bit_length() - 1
    rc, err, got, (missing, bad) = run_abi(abi, lk, base, log_n)
    assert rc == 0, err
    want, wmiss, wbad = LO.multiplicities(lk.table, lk.values, lk.selectors, base)
    assert np.array_equal(got, want)
    assert missing == wmiss and bad == wbad
    return missing, bad


def random_lookup(seed, W, Q, selectors, log_n, nbase=4):
    """tuples over base columns 0..2 (small values, so runs of duplicate table tuples), selectors from column 3: value
    tuple q is the table tuple shifted by a row offset (a hit, wrapping) or with one word replaced (mostly misses)"""
    rng = random.Random(seed)
    iv = 1 << rng.randint(0, log_n)

    def word(k, sh):
        kind = rng.choice(["trace", "trace", "sum", "periodic", "x0"])
        c, o = rng.randrange(3), rng.choice([-1, 0, 1])
        if kind == "trace":
            return lambda s: T(c, o + s)
        if kind == "sum":
            return lambda s: T(c, o + s) * T((c + 1) % 3, s) + E.Constant(P - 1)
        if kind == "periodic":
            coeffs = [rng.randrange(3) for _ in range(rng.choice([x for x in (1, 2) if x <= iv]))]
            return lambda s: T(c, o + s) + E.Periodic(coeffs, iv) * 0
        return lambda s: T(c, o + s) + E.X() * 0
    fs = [word(k, 0) for k in range(W)]
    table = tuple(f(0) for f in fs)
    values = []
    for q in range(Q):
        sh = rng.randrange(-3, 4)
        v = [f(sh) for f in fs]
        if rng.random() < 0.4:
            v[rng.randrange(W)] = T(rng.randrange(3), rng.choice([-2, 2])) + E.Constant(rng.choice([1, 2]))
        values.append(tuple(v))
    sel = tuple(T(3, rng.choice([0, 1])) if rng.random() < 0.7 else E.Constant(1) for _ in range(Q)) if selectors else None
    return Lookup(table, tuple(values), 4, 5, sel)


def _base(seed, log_n, nbase=5, lo=4, sel_vals=(0, 1)):
    rng = np.random.default_rng(seed)
    n = 1 << log_n
    cols = rng.integers(0, lo, size=(nbase, n))
    cols[3] = rng.choice(sel_vals, size=n)
    out = np.array([[_mont(v) for v in c] for c in cols.tolist()], dtype=np.uint64)
    return out


CASES = [(s, W, Q, sel, log_n) for s, (W, Q, sel, log_n) in enumerate(
    [(1, 1, False, 0), (1, 1, False, 1), (1, 2, True, 4), (2, 1, True, 5), (2, 2, False, 8), (3, 3, True, 9), (4, 4, True, 10),
     (4, 1, False, 7), (1, 4, True, 11), (3, 2, False, 12), (2, 4, True, 6), (4, 3, False, 16)])]


@pytest.mark.parametrize("seed,W,Q,sel,log_n", CASES)
def test_cpu_abi_equals_oracle(abi, seed, W, Q, sel, log_n):
    _check(abi, random_lookup(seed, W, Q, sel, log_n), _base(seed, log_n))


def test_cpu_abi_duplicate_runs_and_extreme_words(abi):
    log_n = 9
    n = 1 << log_n
    base = _base(3, log_n)
    base[0] = _mont(P - 1)                              # the table is one tuple repeated n times
    base[1] = np.array([_mont(v) for v in np.random.default_rng(1).choice([0, P - 1], size=n)], dtype=np.uint64)
    lk = Lookup((T(0), T(1)), ((T(0, 3), T(1, -1)), (T(1), T(0))), 4, 5, (E.Constant(1), T(3)))
    _check(abi, lk, base)
    missing, _ = _check(abi, Lookup((T(0),), ((T(0, 1),), (T(1),)), 4, 5), base)
    assert missing[0] == (0, None)
    # every row counts at row 0, the lowest of the run
    from oracle import lookup_oracle as LO
    m, _, _ = LO.multiplicities((T(0),), ((T(0, 1),),), None, base)
    assert int(m[0]) == _mont(n) and not m[1:].any()


def test_cpu_abi_misses_and_bad_selectors(abi):
    log_n = 6
    n = 1 << log_n
    base = _base(4, log_n)
    base[0] = np.array([_mont(i) for i in range(n)], dtype=np.uint64)            # table 0..n-1
    base[1] = base[0].copy()
    base[1][0] = _mont(n + 5)                                                    # misses at the first row,
    base[1][n - 1] = _mont(P - 1)                                                # the last row
    base[2] = np.full(n, _mont(n), dtype=np.uint64)                              # and every row
    base[3] = np.array([_mont(v) for v in [1] * (n - 3) + [2, P - 1, 0]], dtype=np.uint64)
    lk = Lookup((T(0),), ((T(1),), (T(2),), (T(1, 1),)), 4, 5, (E.Constant(1), E.Constant(1), T(3)))
    missing, bad = _check(abi, lk, base)
    assert missing[0] == (2, 0) and missing[1] == (n, 0) and bad == (2, n - 3)


def test_cpu_abi_rejects_malformed_arguments(abi):
    base = _base(5, 3)
    lk = Lookup((T(0), T(1)), ((T(1), T(0)),), 4, 5)
    prog = E.compile_lookup_program(lk.table, lk.values, None, 5, 3)
    assert run_abi(abi, lk, base, 3)[0] == 0
    assert "domain too large" in run_abi(abi, lk, base, 31)[1]
    assert "tuples of 5 words (1 to 4)" in run_abi(abi, lk, base, 3, width=5)[1]
    assert "5 value tuples (1 to 4)" in run_abi(abi, lk, base, 3, ntuples=5)[1]
    assert "workspace of 100 bytes" in run_abi(abi, lk, base, 3, ws_bytes=100)[1]
    assert "never stores slot 5 of 8" in run_abi(abi, lk, base, 3, ntuples=2)[1]
    assert "is not a base-field column" in run_abi(abi, lk, base, 3, isq=[1, 0, 0, 0, 0])[1]
    bad = prog.code.copy()
    st = [i for i, w in enumerate(bad) if int(w[0]) & 0xff == E.OP_STORE][-1]
    bad[st, 1] = 7
    assert "stores to slot 7 of 5" in run_abi(abi, lk, base, 3, code=bad)[1]
    bad = prog.code.copy()
    bad[st, 0] |= 1 << 8
    assert "stores an extension-field value" in run_abi(abi, lk, base, 3, code=bad)[1]
    bad = prog.code.copy()
    tr = [i for i, w in enumerate(bad) if int(w[0]) & 0xff == E.OP_TRACE][0]
    bad[tr, 2] = 9
    assert "column 9 out of range" in run_abi(abi, lk, base, 3, code=bad)[1]
    lib, _ = abi
    out = C.c_size_t()
    assert lib.ms_lookup_workspace_bytes(31, 1, 1, C.byref(out)) != 0
    assert lib.ms_lookup_workspace_bytes(10, 0, 1, C.byref(out)) != 0
    assert lib.ms_lookup_workspace_bytes(10, 1, 5, C.byref(out)) != 0


# ------------------------------------------------------------------------------------------------- 3. the prover
def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS, _lib._LOOKUP_SIGS):
        _lib.bind(lib, sigs)
    _lib._lib = lib


SQ_OPTS = (16, 8, 4, 4, 8)


def _make_case(which):
    """(claim, options, trace) of a named case"""
    from ministark_b200.examples import lookup as L
    from ministark_b200.prover import Trace
    kind, _, variant = which.partition(":")
    if kind == "hand":
        return L.LookupClaim(), SQ_OPTS, L.gen_trace(1 << 8, seed=4)
    if kind == "declared":
        return L.DeclaredLookupClaim(), SQ_OPTS, L.DeclaredLookupClaim.gen_trace(1 << 8, seed=4)
    trace = L.SquareLookupClaim.gen_trace(1 << 8, seed=6)
    if variant == "wrong_c":
        base = np.array(trace.base_columns(), copy=True)
        base[L.CS, 37] = np.uint64(_mont(12345))
        trace = Trace(base)
    return L.SquareLookupClaim(), SQ_OPTS, trace


def _prove_worker(which, lib_path, residency, validate, corrupt, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    from ministark_b200 import FP, FQ3
    from ministark_b200.examples import lookup as L
    from ministark_b200.prover import GpuProver, LookupViolation, peak_bytes
    from ministark_b200.validate import ConstraintViolation
    from ministark_b200.verifier import VerificationError
    claim, opts, trace = _make_case(which)
    before = np.array(trace.base_columns(), copy=True)

    class Corrupting(GpuProver):
        """a wrong fill injected after the kernel"""
        def _lookup_base(self, r, host_base):
            base = super()._lookup_base(r, host_base)
            import torch
            if corrupt == "zero":
                base[L.MS] = 0
            else:                       # every count one row late
                base[L.MS] = torch.roll(base[L.MS], 1)
            return base

    p = Corrupting(0) if corrupt else GpuProver(0)
    if residency == "streamed":
        cfg, o, n = claim.AirConfig, ProofOptions(*opts), len(trace)
        est = peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, FP if cfg.FQ_IS_FP else FQ3,
                         Air(cfg, n, None, o).ce_blowup_factor, o.fri_folding_factor)
        p.memory_budget = (est["streamed"] + est["resident"]) // 2
    out = {}
    try:
        proof = p.prove(claim, ProofOptions(*opts), trace, validate=validate)
        out["bytes"] = proof.to_bytes()
        out["lookup_timed"] = "lookup_multiplicities" in proof.timings
        claim.verify(out["bytes"], 10)
        out["verified"] = True
    except ConstraintViolation as e:
        out["violations"] = [v.constraint for v in e.violations]
    except LookupViolation as e:
        out["misses"] = [(m.lookup, m.tuple, m.kind, m.first_row, m.count, m.values) for m in e.misses]
        out["message"] = str(e)
    except VerificationError as e:
        out["rejected"] = str(e)
    out["unchanged"] = bool(np.array_equal(np.asarray(trace.base_columns()), before))
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
    """cpu_prove with the oracle's multiplicities in the oracle's trace, and the running sums evaluated by the oracle"""
    from oracle import extension_oracle as XO
    from oracle import lookup_oracle as LO
    from oracle import stark_oracle as SO
    claim, opts, trace = _make_case(which)
    cfg = claim.AirConfig
    mk = lambda n, o: Air(cfg, n, claim.get_public_inputs(), ProofOptions(*o))
    base = LO.fill(cfg, trace.base_columns())
    n = base.shape[1]
    decl = [(c.init, c.mul, c.add, c.inclusive) for c in mk(n, opts).extension_declaration]
    ext = lambda ch: XO.columns(decl, base, 1 if cfg.FQ_IS_FP else 3, ch, cfg.gen_hints(n, None, ch))
    want = SO.cpu_prove(claim, opts, base, mk, ext_builder=ext)
    SO.verify(claim, want, 10, mk)
    return want


@pytest.mark.parametrize("residency", ["resident", "streamed"])
@pytest.mark.parametrize("which", ["declared", "square"])
def test_lookup_airs_prove_to_the_restatement(orc, lookup_abi, which, residency):
    out = _spawn(_prove_worker, which, lookup_abi, residency, True, None)
    assert "violations" not in out and "misses" not in out, out
    assert out["residency"] == residency and out["verified"] and out["lookup_timed"] and out["unchanged"]
    want = _cpu_restatement(which)
    assert out["bytes"] == want
    if which == "declared":             # the hand-written AIR with host multiplicities: the same proof
        assert _spawn(_prove_worker, "hand", lookup_abi, residency, False, None)["bytes"] == want


def test_wrong_value_raises_lookup_violation(lookup_abi):
    from ministark_b200.examples import lookup as L
    out = _spawn(_prove_worker, "square:wrong_c", lookup_abi, "resident", False, None)
    assert "misses" in out, out
    (miss,) = out["misses"]
    claim, _, trace = _make_case("square:wrong_c")
    a = int(np.asarray(trace.base_columns())[L.AS, 37]) * pow(_R, -1, P) % P
    assert miss == (0, 0, "missing", 37, 1, (a, 12345))
    assert "lookup 0, value tuple 0" in out["message"] and "row 37" in out["message"]
    assert out["unchanged"]


@pytest.mark.parametrize("corrupt", ["zero", "shift"])
def test_corrupted_fill_is_refused(lookup_abi, corrupt):
    out = _spawn(_prove_worker, "square", lookup_abi, "resident", True, corrupt)
    n_user = len(__import__("ministark_b200.examples.lookup", fromlist=["x"]).SquareLookupAirConfig.constraints(1 << 8))
    assert out.get("violations") and all(k >= n_user for k in out["violations"]), out
    out = _spawn(_prove_worker, "square", lookup_abi, "resident", False, corrupt)
    assert "rejected" in out, out


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


@pytest.mark.parametrize("which", ["declared", "square"])
def test_sharded_prover_over_gloo(orc, lookup_abi, which):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, which, lookup_abi, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=900) for _ in range(2)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    want = _cpu_restatement(which)
    for rank, b in got:
        assert b == want, f"rank {rank}"


def _own_builder_worker(lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    from ministark_b200.examples import lookup as L
    from ministark_b200.prover import GpuProver, ProvingError, Trace
    trace = L.DeclaredLookupClaim.gen_trace(1 << 6)
    try:
        GpuProver(0).prove(L.DeclaredLookupClaim(), OPTS, Trace(trace.base_columns(), lambda ch: None))
        q.put(None)
    except ProvingError as e:
        q.put(str(e))


def test_trace_with_its_own_extension_builder_is_refused(lookup_abi):
    assert "the trace must not bring its own extension columns" in _spawn(_own_builder_worker, lookup_abi)


# ---------------------------------------------------------------------------------------------------- 4. header
def test_lookup_header_is_bound_exported_and_separate(lookup_abi):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.LOOKUP_HEADER_PATH)
    assert declared == sorted(_lib._LOOKUP_SIGS) == ["ms_lookup_multiplicities", "ms_lookup_workspace_bytes"]
    others = set(_lib.header_symbols()) | set(_lib.header_symbols(_lib.STREAM_HEADER_PATH)) | \
        set(_lib.header_symbols(_lib.CHECK_HEADER_PATH)) | set(_lib.header_symbols(_lib.EXTENSION_HEADER_PATH)) | \
        set(_lib.header_symbols(_lib.BF_HEADER_PATH))
    assert not set(declared) & others
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(lookup_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)
