"""CPU-only: the constraint check behind `GpuProver.prove(..., validate=True)` (ministark_b200/validate.py).

  * oracle/check_oracle.py restates Constraint::check (src/constraints.rs:168-249): every Option branch on hand-built
    expressions;
  * expr.compile_check_program: a big-integer interpreter of the checked instruction set (written here) runs the compiled
    program row by row and equals the oracle on random DAGs (vanishing denominators, zerofiers, row offsets with
    wrap-around, periodic columns, challenges, hints, register eviction, 100 constraints);
  * ms_check_constraints of the CPU build (tests/cpp/check_cpu_abi.c) equals the oracle and rejects malformed programs;
  * both residencies of the prover on the CPU harness (tests/cpu_device.py) with validate=True: valid traces give the
    bytes of validate=False and of oracle/stark_oracle.cpu_prove, corrupted traces raise ConstraintViolation with the
    oracle's report before the composition commitment;
  * the three warnings of the reference, and the header include/ministark_check.h.
Prover cases run in spawned workers that install the harness themselves; the pytest process never does."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from ministark_b200 import expr as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = E.P
_R = 2**64
_RINV = pow(_R, -1, P)


def _mont(v):
    return int(v) % P * _R % P


def _cols(rows, lanes=1):
    """canonical values (ints, or 3-tuples for lanes = 3) -> one column of Montgomery words"""
    if lanes == 1:
        return np.array([_mont(v) for v in rows], dtype=np.uint64)
    return np.array([_mont(c) for v in rows for c in E._q(v)], dtype=np.uint64)


# --------------------------------------------------------------------------------------------- 1. oracle semantics
@pytest.fixture(scope="module")
def CO(orc):
    from oracle import check_oracle
    return check_oracle


def _none_rows(CO, expr, base, ext=None, lanes=1, log_n=2):
    """rows where the single constraint `expr` is None, by the oracle"""
    b = np.stack([_cols(c) for c in base]) if base else None
    e = np.stack([_cols(c, lanes) for c in ext]) if ext else None
    first, count = CO.check([expr.to_tuple()], log_n, b, e, lanes)[0]
    return first, count


def test_oracle_option_semantics(CO):
    T, X, K = E.Trace, E.X, E.Constant
    base = [[0, 0, 5, 5], [0, 3, 0, 3]]             # a = col 0, b = col 1: rows (0,0) (0,3) (5,0) (5,3)
    a, b = T(0), T(1)
    none_ = K(1) / K(0)                              # a / 0 with a != 0: None everywhere
    cases = [
        (a + b, []),
        (a / b, [2]),                                # 0/0 Some(0) at row 0, 0/3 at row 1, 5/0 None at row 2
        (a * none_, [2, 3]),                         # Some(x) * None: Some(0) iff x = 0
        (none_ * a, [2, 3]),
        (none_ * none_, [0, 1, 2, 3]),
        (a + none_, [0, 1, 2, 3]),
        (none_ + a, [0, 1, 2, 3]),
        (a / none_, [2, 3]),                         # 0 / None = Some(0)
        (none_ / b, [1, 3]),                         # None / 0 = Some(0)
        (none_ / none_, [0, 1, 2, 3]),
        (-none_, [0, 1, 2, 3]),
        (none_ ** 3, [0, 1, 2, 3]),
        (none_ ** 0, [0, 1, 2, 3]),
        ((a / b) * 0, []),                           # None * Some(0) = Some(0): the None of row 2 is absorbed
        (K(0) * (a / b), []),
        (K(0) / K(0), []),
        ((X() - 1) / (X() - 1), []),                 # 0/0 at row 0
        (a / (X() - 1), []),                         # a = 0 at row 0
        (b / (X() - 1), []),
        (K(7) / (X() - 1), [0]),
        (K(7) / (X() ** 4 - 1), [0, 1, 2, 3]),       # the zerofier of the whole domain
    ]
    for expr, want in cases:
        first, count = _none_rows(CO, expr, base)
        assert count == len(want) and (first == (want[0] if want else None)), (expr.to_tuple(), first, count, want)


def test_oracle_fq3_zero_needs_all_coordinates(CO):
    T = E.Trace
    ext = [[(0, 0, 0), (0, 1, 0), (0, 0, 1), (2, 0, 0)]]
    base = [[1, 1, 1, 1]]
    first, count = _none_rows(CO, T(0) / T(1), base, ext, lanes=3)
    assert (first, count) == (0, 1)
    first, count = _none_rows(CO, (E.Constant(1) / E.Constant(0)) * T(1), base, ext, lanes=3)
    assert (first, count) == (1, 3)                  # None * Some(x): Some(0) only where all of x is 0
    first, count = _none_rows(CO, T(0) / (T(0) - 1), base, ext, lanes=3)
    assert (first, count) == (0, 4)                  # Fp zero test on the base column


# ------------------------------------------------------------------------------------ 2. compiler vs interpreter
def _q(v):
    return E._q(v)


def interpret(prog, nconstraints, log_n, cols, col_is_q, fq_lanes, periodic_tables):
    """the checked instruction set over canonical big integers, one row at a time; returns [(first_row | None, count)].
    cols: per column a list of canonical values (ints or 3-tuples), periodic_tables likewise (natural order)."""
    n = 1 << log_n
    g = pow(7, (P - 1) >> 32, P)
    g = pow(g, 1 << (32 - log_n), P)
    consts = [tuple(int(w) * _RINV % P for w in c) for c in prog.consts]
    table = list(cols) + list(periodic_tables)
    res = [[None, 0] for _ in range(nconstraints)]
    zero = lambda v: not any(v)
    for i in range(n):
        reg, none = {}, {}
        for w in prog.code:
            op, d, a, b = int(w[0]) & 0xff, int(w[1]), int(w[2]), int(w[3])
            qa, qb = (int(w[0]) >> 8) & 1 and fq_lanes == 3, (int(w[0]) >> 9) & 1 and fq_lanes == 3
            vn = False
            if op == E.OP_X:
                v = (pow(g, i, P), 0, 0)
            elif op == E.OP_CONST:
                v = consts[a] if qa else (consts[a][0], 0, 0)
            elif op in (E.OP_TRACE, E.OP_PERIODIC):
                pos = (i + b) % n if op == E.OP_TRACE else i % (1 << b)
                v = _q(table[a][pos])
            elif op == E.OP_NEG:
                v, vn = E.q_neg(reg[a]), none[a]
            elif op == E.OP_ADD:
                v, vn = E.q_add(reg[a], reg[b]), none[a] or none[b]
            elif op == E.OP_POW:
                v, vn = E.q_pow(reg[a], b), none[a]
            elif op in (E.OP_MUL, E.OP_DIV):
                x, y, nx, ny = reg[a], reg[b], none[a], none[b]
                v = (0, 0, 0)
                if nx and ny:
                    vn = True
                elif nx or ny:
                    vn = not zero(y if nx else x)
                elif op == E.OP_MUL:
                    v = E.q_mul(x, y)
                elif zero(y):
                    vn = not zero(x)
                else:
                    v = E.q_mul(x, E.q_inv(y))
            elif op == E.OP_CHECK:
                if none[a]:
                    if res[b][1] == 0:
                        res[b][0] = i
                    res[b][1] += 1
                continue
            else:
                raise AssertionError(f"opcode {op} in a checked program")
            reg[d], none[d] = v, vn
    return [tuple(r) for r in res]


def random_constraints(seed, log_n, nbase, next_, k, nchal=3, nhint=2, fq3=True):
    """k random constraint DAGs over nbase + next_ columns (extension columns only when fq3).  Denominators: zerofier
    shapes, trace-dependent values that vanish on chosen rows, Fq3 ones, constant zeros; numerators sometimes zero where
    the denominator is."""
    rng = random.Random(seed)
    n = 1 << log_n
    g = pow(pow(7, (P - 1) >> 32, P), 1 << (32 - log_n), P)
    ncols = nbase + next_
    X = E.X()

    def leaf():
        r = rng.random()
        if r < 0.45:
            return E.Trace(rng.randrange(ncols), rng.randint(-3, 3))
        if r < 0.55:
            return X
        if r < 0.65:
            return E.Challenge(rng.randrange(nchal))
        if r < 0.72:
            return E.Hint(rng.randrange(nhint))
        if r < 0.8:
            iv = 1 << rng.randint(0, log_n)
            return E.Periodic([rng.randrange(P) for _ in range(rng.choice([c for c in (1, 2, 4) if c <= iv]))], iv)
        if r < 0.9:
            return E.Constant(rng.choice([0, 1, 2, rng.randrange(P)]))
        return E.Constant((rng.randrange(P), rng.randrange(P), 0), ext=True) if fq3 else E.Constant(rng.randrange(P))

    def denom():
        r = rng.random()
        if r < 0.2:
            return X - 1
        if r < 0.35:
            return X ** n - 1
        if r < 0.5:
            return X - pow(g, n - 1, P)                  # x - g^-1
        if r < 0.6:
            return E.Constant(0)
        if r < 0.8:
            return E.Trace(rng.randrange(ncols), rng.randint(-3, 3))   # zero where the trace is (the tests plant zeros)
        return E.Trace(rng.randrange(nbase), 0) - rng.randrange(3)

    def tree(depth):
        if depth == 0 or rng.random() < 0.2:
            return leaf()
        r = rng.random()
        if r < 0.3:
            return tree(depth - 1) + tree(depth - 1)
        if r < 0.55:
            return tree(depth - 1) * tree(depth - 1)
        if r < 0.65:
            return tree(depth - 1) - tree(depth - 1)
        if r < 0.72:
            return -tree(depth - 1)
        if r < 0.78:
            return tree(depth - 1) ** rng.randint(0, 5)
        num = tree(depth - 1)
        if rng.random() < 0.4:
            num = num * E.Trace(rng.randrange(nbase), 0)                # zero on the rows the trace is zero
        return num / denom()

    return [tree(rng.randint(1, 5)) for _ in range(k)]


def random_trace(seed, log_n, nbase, next_, lanes):
    """columns with zeros planted on a chosen subset of rows (canonical values)"""
    rng = random.Random(seed ^ 0x5EED)
    n = 1 << log_n
    zrows = set(rng.sample(range(n), max(1, n // 4)))
    base = [[0 if (i in zrows and rng.random() < 0.7) else rng.choice([1, 2, rng.randrange(P)]) for i in range(n)]
            for _ in range(nbase)]
    zero = (0, 0, 0) if lanes == 3 else 0
    ext = [[zero if (i in zrows and rng.random() < 0.7) else (rng.randrange(P), rng.randrange(P), rng.randrange(P))
            if lanes == 3 else rng.randrange(P) for i in range(n)] for _ in range(next_)]
    return base, ext


def _periodic_canon(prog, log_n):
    """the periodic tables of `prog` (what periodic_tables(.., offset_canonical=1) computes on the device), canonical"""
    n = 1 << log_n
    out = []
    for _, coeffs, interval, is_q, log_len in prog.periodic:
        gi = pow(pow(7, (P - 1) >> 32, P), 1 << (32 - log_len), P) if log_len else 1
        tab = []
        for j in range(1 << log_len):
            y = pow(gi, j, P)
            acc = (0, 0, 0)
            for c in reversed(coeffs):
                acc = E.q_add(E.q_mul(acc, (y, 0, 0)), _q(c))
            tab.append(acc if is_q else acc[0])
        out.append(tab)
        assert n % interval == 0
    return out


def _case(seed, log_n, k, fq3, with_ext=True):
    nbase, next_ = 3, (2 if with_ext else 0)
    lanes = 3 if fq3 else 1
    cons = random_constraints(seed, log_n, nbase, next_, k, fq3=fq3)
    base, ext = random_trace(seed, log_n, nbase, next_, lanes)
    rng = random.Random(seed + 1)
    chal = [(rng.randrange(P), rng.randrange(P), rng.randrange(P)) if fq3 else rng.randrange(P) for _ in range(3)]
    hints = [0, (rng.randrange(P), 0, 0) if fq3 else rng.randrange(P)]
    return cons, nbase, next_, lanes, base, ext, chal, hints


CASES = [(s, log_n, k, fq3, wx) for s, (log_n, k, fq3, wx) in enumerate(
    [(0, 8, True, True), (1, 16, True, True), (3, 48, True, False), (6, 100, True, True), (3, 100, False, True),
     (1, 20, False, False), (6, 30, False, True)])]


def _oracle(CO, cons, log_n, base, ext, lanes, chal, hints):
    b = np.stack([_cols(c) for c in base])
    e = np.stack([_cols(c, lanes) for c in ext]) if ext else None
    return [(f, c) for f, c in CO.check([x.to_tuple() for x in cons], log_n, b, e, lanes, chal, hints)]


@pytest.mark.parametrize("seed,log_n,k,fq3,with_ext", CASES)
def test_compiled_program_equals_oracle(CO, seed, log_n, k, fq3, with_ext):
    cons, nbase, next_, lanes, base, ext, chal, hints = _case(seed, log_n, k, fq3, with_ext)
    prog = E.compile_check_program(cons, nbase, log_n, nbase + next_).bind(challenges=chal, hints=hints)
    got = interpret(prog, k, log_n, base + ext, [0] * nbase + [1] * next_, lanes, _periodic_canon(prog, log_n))
    want = _oracle(CO, cons, log_n, base, ext, lanes, chal, hints)
    assert got == want
    assert any(c for _, c in want) and not all(c for _, c in want) or k < 20


def test_compiler_evicts_and_shares():
    cons, nbase, next_, *_ = _case(6, 6, 100, True)
    prog = E.compile_check_program(cons, nbase, 6, nbase + next_)
    assert prog.nregs == E.MAX_REGS                          # more live values than registers: leaves were evicted
    ops = [int(w[0]) & 0xff for w in prog.code]
    assert ops.count(E.OP_CHECK) == 100 and E.OP_INV not in ops and E.OP_STORE not in ops
    z = E.X() ** 64 - 1
    shared = E.compile_check_program([E.Trace(0) / z, E.Trace(1) / z], 2, 6, 2)
    assert [int(w[0]) & 0xff for w in shared.code].count(E.OP_POW) == 1     # x^n - 1 computed once
    folded = E.compile_check_program([E.Constant(3) / E.Constant(0)], 1, 2, 1)
    assert E.OP_DIV in [int(w[0]) & 0xff for w in folded.code]               # a zero denominator is left to the kernel


# ------------------------------------------------------------------------------------------------- 3. CPU ABI
@pytest.fixture(scope="module")
def check_abi(tmp_path_factory, orc):
    """tests/cpp/check_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary directory"""
    out = str(tmp_path_factory.mktemp("check_abi") / "libms_check_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out, os.path.join(ROOT, "tests", "cpp", "check_cpu_abi.c")])
    return out


@pytest.fixture(scope="module")
def abi(check_abi):
    from ministark_b200 import _lib
    lib = C.CDLL(check_abi)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    _lib.bind(lib, _lib._CHECK_SIGS)
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    return lib, h


def _run_abi(abi, prog, cols, isq, fq_field, log_n, k, code=None):
    lib, h = abi
    code = prog.code if code is None else np.ascontiguousarray(code, dtype=np.uint32)
    ptrs = (C.c_void_p * max(len(cols), 1))(*[c.ctypes.data for c in cols])
    q = (C.c_int * max(len(cols), 1))(*isq)
    first, count = np.zeros(k, dtype=np.uint64), np.zeros(k, dtype=np.uint64)
    rc = lib.ms_check_constraints(h, code.ctypes.data, code.shape[0], prog.consts.ctypes.data, prog.consts.shape[0], ptrs, q,
                                  len(cols), fq_field, log_n, k, first.ctypes.data, count.ctypes.data)
    return rc, lib.ms_last_error(h).decode() if rc else "", first, count


def _device_tables(prog, log_n, lanes):
    return [_cols(t, 3 if is_q and lanes == 3 else 1) for t, (_, _, _, is_q, _) in zip(_periodic_canon(prog, log_n), prog.periodic)]


@pytest.mark.parametrize("seed,log_n,k,fq3,with_ext", CASES)
def test_cpu_abi_equals_oracle(CO, abi, seed, log_n, k, fq3, with_ext):
    cons, nbase, next_, lanes, base, ext, chal, hints = _case(seed, log_n, k, fq3, with_ext)
    prog = E.compile_check_program(cons, nbase, log_n, nbase + next_).bind(challenges=chal, hints=hints)
    cols = [_cols(c) for c in base] + [_cols(c, lanes) for c in ext] + _device_tables(prog, log_n, lanes)
    isq = [0] * nbase + [1] * next_ + [int(p[3]) for p in prog.periodic]
    rc, err, first, count = _run_abi(abi, prog, cols, isq, lanes, log_n, k)
    assert rc == 0, err
    want = _oracle(CO, cons, log_n, base, ext, lanes, chal, hints)
    assert [(None if int(f) == 2**64 - 1 else int(f), int(c)) for f, c in zip(first, count)] == want


def test_cpu_abi_rejects_malformed_programs(abi):
    prog = E.compile_check_program([E.Trace(0) / (E.X() - 1), E.Trace(1, 1) * E.Trace(0)], 1, 3, 2)
    cols = [_cols(range(8)), _cols([(i, 0, 0) for i in range(8)], 3)]
    assert _run_abi(abi, prog, cols, [0, 1], 3, 3, 2)[0] == 0
    bad = prog.code.copy()
    bad[0, 0] = 13
    assert "bad instruction 0" in _run_abi(abi, prog, cols, [0, 1], 3, 3, 2, bad)[1]
    for op, name in ((E.OP_STORE, "STORE"), (E.OP_INV, "INV")):
        bad = prog.code.copy()
        last = [i for i, w in enumerate(bad) if int(w[0]) & 0xff == E.OP_CHECK][0]
        bad[last] = [op, 0, bad[last][2], 0]
        assert f"{name} has no place" in _run_abi(abi, prog, cols, [0, 1], 3, 3, 2, bad)[1]
    bad = prog.code.copy()
    bad[-1][2] = 40                                          # OP_CHECK of a register never written
    assert "before it is written" in _run_abi(abi, prog, cols, [0, 1], 3, 3, 2, bad)[1]
    assert "wrong field" in _run_abi(abi, prog, cols, [0, 0], 3, 3, 2)[1]
    assert "checks constraint 1 of 1" in _run_abi(abi, prog, cols, [0, 1], 3, 3, 1)[1]


# ------------------------------------------------------------------------------------ 4. the prover, both residencies
def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    _lib.bind(lib, _lib._STREAM_SIGS)
    _lib.bind(lib, _lib._CHECK_SIGS)
    _lib._lib = lib


class _Tampered:
    """a trace whose base cell or (host-built) extension cell is changed; canonical value += 1"""

    def __init__(self, inner, base_cell=None, ext_cell=None, lanes=1):
        self.inner, self.base_cell, self.ext_cell, self.lanes = inner, base_cell, ext_cell, lanes
        self.base = np.array(inner.base_columns(), copy=True)
        if base_cell is not None:
            c, r = base_cell
            self.base[c, r] = np.uint64(_mont(int(self.base[c, r]) * _RINV % P + 1))

    def __len__(self):
        return len(self.inner)

    def base_columns(self):
        return self.base

    def build_extension_columns(self, challenges):
        ext = self.inner.build_extension_columns(challenges)
        if ext is not None and self.ext_cell is not None:
            ext = np.array(ext, copy=True)
            c, r = self.ext_cell
            ext[c, r * self.lanes] = np.uint64(_mont(int(ext[c, r * self.lanes]) * _RINV % P + 1))
        return ext


def _make_case(which):
    from ministark_b200.examples import brainfuck as bf
    from ministark_b200.examples import fib, perm
    kind, _, rest = which.partition(":")
    if kind == "fib":
        log_rows, _, tamper = rest.partition(":")
        n = 8 << int(log_rows)
        trace, last = fib.gen_trace(n)
        rows = n // 8
        cells = {"": None, "cell": (3, 17), "boundary": (0, 0), "terminal": (7, rows - 1), "wrap": (0, rows - 1)}
        t = _Tampered(trace, base_cell=cells[tamper]) if tamper else trace
        return fib.FibClaim(last), (16, 4, 4, 8, 16), t
    if kind == "perm":
        return perm.PermClaim(), (16, 8, 4, 4, 8), perm.gen_trace(1 << 8, seed=3)
    trace, output = bf.simulate(bf.HELLO_WORLD)
    claim = bf.BrainfuckClaim(bf.HELLO_WORLD, b"", output)
    if rest == "base":
        trace = _Tampered(trace, base_cell=(1, 5))
    elif rest == "ext":
        trace = _Tampered(trace, ext_cell=(2, 9), lanes=3)
    return claim, (19, 16, 20, 16, 16), trace


def _prove_worker(which, lib_path, residency, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    import warnings
    from ministark_b200 import prover as PR
    from ministark_b200.air import ProofOptions
    from ministark_b200.prover import GpuProver, peak_bytes
    from ministark_b200.validate import ConstraintViolation
    claim, opts, trace = _make_case(which)
    p = GpuProver(0)
    if residency == "streamed":
        from ministark_b200 import FP, FQ3
        from ministark_b200.air import Air
        cfg, o, n = claim.AirConfig, ProofOptions(*opts), len(trace)
        est = peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, FP if cfg.FQ_IS_FP else FQ3,
                         Air(cfg, n, None, o).ce_blowup_factor, o.fri_folding_factor)
        p.memory_budget = (est["streamed"] + est["resident"]) // 2
    commits = []
    orig = PR.ProverChannel.commit_composition_trace
    PR.ProverChannel.commit_composition_trace = lambda self, root: (commits.append(root), orig(self, root))[1]
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("error")                  # the example AIRs use every column, challenge and hint
        try:
            proof = p.prove(claim, ProofOptions(*opts), trace, validate=True)
            out["bytes"] = proof.to_bytes()
            out["keys"] = sorted(proof.timings) if hasattr(proof, "timings") else None
            out["plain"] = p.prove(claim, ProofOptions(*opts), trace).to_bytes()
        except ConstraintViolation as e:
            out["violations"] = [(v.constraint, v.first_row, v.count, v.values) for v in e.violations]
            out["message"] = str(e)
            out["commits"] = len(commits)
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
    from ministark_b200.air import Air, ProofOptions
    from oracle import stark_oracle as SO
    claim, opts, trace = _make_case(which)
    pub = claim if which.startswith("brainfuck") else claim.get_public_inputs()
    mk = lambda n, o: Air(claim.AirConfig, n, pub, ProofOptions(*o))
    ext = getattr(trace, "build_extension_columns", None)
    return SO.cpu_prove(claim, opts, trace.base_columns(), mk, ext_builder=ext if claim.AirConfig.NUM_EXTENSION_COLUMNS else None)


@pytest.mark.parametrize("residency", ["resident", "streamed"])
@pytest.mark.parametrize("which", ["fib:4", "fib:10", "perm", "brainfuck"])
def test_valid_traces_prove_identically_with_validation(orc, check_abi, which, residency):
    out = _spawn(_prove_worker, which, check_abi, residency)
    assert "violations" not in out, out.get("message")
    assert out["residency"] == residency
    assert out["bytes"] == out["plain"] == _cpu_restatement(which)


@pytest.mark.parametrize("residency", ["resident", "streamed"])
@pytest.mark.parametrize("which", ["fib:6:cell", "fib:6:boundary", "fib:6:terminal", "fib:6:wrap", "brainfuck:base",
                                   "brainfuck:ext"])
def test_corrupted_traces_raise_the_oracle_report(CO, check_abi, which, residency):
    out = _spawn(_prove_worker, which, check_abi, residency)
    assert "violations" in out, "the corrupted trace proved"
    assert out["commits"] == 0                          # raised before the composition commitment
    got = out["violations"]
    want = _expected(CO, which, out)
    assert [(k, f, c) for k, f, c, _ in got] == want["counts"]
    k0, f0, _, vals = got[0]
    assert out["message"].startswith(f"Constraint {k0} does not evaluate to a low degree polynomial. Divide by zero occurs "
                                     f"at row {f0} ")
    assert list(vals) == want["values"]


def _expected(CO, which, out):
    """the oracle's report for the corrupted trace: every constraint checked over the trace the prover saw, with the
    challenges the prover drew (replayed: the oracle's base commitment into the prover's channel)"""
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.channel import ProverChannel
    from oracle import oracle as orc
    claim, opts, trace = _make_case(which)
    cfg = claim.AirConfig
    n = len(trace)
    o = ProofOptions(*opts)
    air = Air(cfg, n, claim.get_public_inputs(), o)
    lanes = 1 if cfg.FQ_IS_FP else 3
    base = np.asarray(trace.base_columns())
    log_n = n.bit_length() - 1
    polys = orc.ntt(base, 1, log_n, inverse=True)
    lde = orc.lde(polys, 1, log_n, o.lde_blowup_factor.bit_length() - 1, orc.generator(), True)
    root = orc.merkle_nodes(orc.hash_rows(lde, 1))[1].tobytes()
    ch = ProverChannel(air, claim.gen_public_coin(air), None)
    ch.commit_base_trace(root)
    chal = [ch.public_coin.draw() for _ in range(air.num_challenges())]
    hints = air.gen_hints(chal)
    ext = trace.build_extension_columns(chal) if cfg.NUM_EXTENSION_COLUMNS else None
    ext = None if ext is None else np.asarray(ext)
    res = CO.check([c.to_tuple() for c in air.constraints], log_n, base, ext, lanes, chal, hints)
    counts = [(k, f, c) for k, (f, c) in enumerate(res) if c]
    k0, f0, _ = counts[0]
    vals = CO.leaf_values(air.constraints[k0].to_tuple(), f0, log_n, base, ext, lanes, chal, hints)
    return {"counts": counts, "values": vals}


# ------------------------------------------------------------------------------------------------- 5. warnings
def _warn_worker(lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    import warnings
    import torch
    from ministark_b200 import Context
    from ministark_b200.air import Air, AirConfig, ProofOptions
    from ministark_b200.validate import validate_constraints

    class Toy(AirConfig):
        NUM_BASE_COLUMNS = 3
        FQ_IS_FP = True

        @staticmethod
        def constraints(trace_len):
            return [(E.Trace(0) - E.Trace(1) * E.Challenge(1)) / (E.X() - 1)]

        @staticmethod
        def gen_hints(trace_len, public_inputs, challenges):
            return [5]

    air = Air(Toy, 8, None, ProofOptions(4, 4, 0, 2, 4))
    base = torch.from_numpy(np.stack([_cols([3] * 8), _cols([1] * 8), _cols([0] * 8)]).view(np.int64))
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        v = validate_constraints(Context(0), air, [7, 3], [5], base, None)
    q.put(([str(x.message) for x in w], [(x.constraint, x.first_row, x.count, x.values) for x in v]))


def test_unused_column_challenge_and_hint_warn(check_abi):
    msgs, v = _spawn(_warn_worker, check_abi)
    assert msgs == ["no constraints for execution trace column 2", "challenge at index 0 never used",
                    "hint at index 0 never used"]
    # (3 - 1 * 3) / (x - 1) = 0/0 at row 0: Some(0); the constraint holds everywhere
    assert v == []


# ---------------------------------------------------------------------------------------------------- 6. header
def test_check_header_is_bound_exported_and_covered(check_abi):
    """include/ministark_check.h: bound by the loader, exported by the CUDA library and by the CPU build, declares
    nothing that include/ministark_b200.h declares, and the product's modules import no oracle"""
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.CHECK_HEADER_PATH)
    assert declared == sorted(_lib._CHECK_SIGS) == ["ms_check_constraints"]
    assert not set(declared) & set(_lib.header_symbols())
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(check_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)
    for mod in ("validate.py", "prover.py", "expr.py", "air.py"):
        src = open(os.path.join(ROOT, "ministark_b200", mod)).read()
        assert "from oracle" not in src and "import oracle" not in src
