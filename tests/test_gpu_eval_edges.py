"""GPU: both device implementations of the fused constraint evaluator — the run-time specialised kernel (csrc/eval_jit.cu,
the default) and the interpreter (eval_point in csrc/eval.cuh, the fallback and the evaluator of extension.cu and
lookup.cu) — against big-integer references, word for word:

  1. every opcode over every operand-field combination on edge operands (0, 1, p - 1, 2^32, 2^63, Fq3 elements with zero
     components ...), where the carry chains of field.cuh's device branches turn over, with Fq = Fq3 and with Fq = Fp;
  2. domain and layout edges: domain sizes from 2 to 2^20 (partial and exact blocks, the two-level twiddle table),
     row offsets that wrap the domain, the four storage-order combinations, domain offsets, strided columns, periodic
     columns of interval 1 and of the trace length;
  3. program-shape edges: the 48-register file, and one cached specialised kernel rebound to new constants.

Every case runs on the specialised kernel (after asserting that it is built for the program: eval_launch_jit falls back to
the interpreter silently) and on the interpreter (MS_EVAL_NO_JIT=1).  References: big integers per point (pyspec for the
opcode grid, expr.evaluate_at for expressions) for domains up to 2^12 points, oracle.eval_oracle (C, u128) above."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import ministark_b200 as ms
from ministark_b200 import _lib
from ministark_b200 import deep
from ministark_b200 import expr as E
from oracle import pyspec as S

import tests_helpers_expr as H

pytestmark = pytest.mark.gpu
P = E.P
R = 2**64
LEGS = ("specialised kernel", "interpreter")


@pytest.fixture(scope="module")
def ctx():
    return ms.Context(0)


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


_jit_built = set()


def _assert_specialised(prog, fq, name):
    """the default leg is the specialised kernel only if NVRTC builds it for this program"""
    key = (prog.code.tobytes(), fq)
    if key in _jit_built:
        return
    log = C.create_string_buffer(4096)
    rc = _lib.load().ms_eval_jit_check(prog.code.ctypes.data, len(prog), prog.consts.ctypes.data, prog.consts.shape[0], fq, log, 4096)
    assert rc == 0, f"{name}: no specialised kernel (ms_eval_jit_check = {rc}): {log.value.decode()[:800]}"
    _jit_built.add(key)


def _first_difference(got, want, fq, what, operands=None):
    got, want = got.reshape(-1, fq), want.reshape(-1, fq)
    bad = np.nonzero((got != want).any(axis=1))[0]
    if len(bad):
        k = int(bad[0])
        fmt = lambda r: "(" + ", ".join(f"{int(w):#x}" for w in r) + ")"
        at = f" operands {operands(k)}" if operands else ""
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} points differ; first at output position {k}{at}: "
                             f"got {fmt(got[k])}, want {fmt(want[k])}")


def _both_legs(name, prog, fq, run, want, operands=None):
    """run() evaluates `prog` and returns the output words; compared with `want` on each leg"""
    for leg in LEGS:
        if leg == LEGS[0]:
            _assert_specialised(prog, fq, name)
        else:
            os.environ["MS_EVAL_NO_JIT"] = "1"
        try:
            got = run()
        finally:
            os.environ.pop("MS_EVAL_NO_JIT", None)
        _first_difference(got, want, fq, f"{name} [{leg}]", operands)


def _device(torch, words):
    return torch.from_numpy(np.ascontiguousarray(words, dtype=np.uint64).view(np.int64).copy()).cuda()


def _launcher(ctx, torch, prog, log_m, dcols, isq, fq, **kw):
    out = torch.empty((1 << log_m) * fq, dtype=torch.int64, device="cuda")

    def run():
        out.fill_(-1)                # not a canonical word: a point the kernel never stores shows up
        torch.cuda.synchronize()
        ctx.eval_constraints_ptrs(prog, out, log_m, dcols, isq, fq_field=fq, **kw)
        ctx.sync()
        return out.cpu().numpy().view(np.uint64).copy()
    return run


# ---- 1. opcode x operand-field grid on edge operands -------------------------------------------------------------------
@pytest.fixture(scope="module", params=[3, 1], ids=["fq3", "fq_is_fp"])
def edge(request, torch):
    fq = request.param
    cols, isq = H.edge_columns(fq)
    dcols = [_device(torch, H.column_words(c, q, fq)) for c, q in zip(cols, isq)]
    return fq, cols, isq, dcols


@pytest.mark.parametrize("op", ["ADD", "SUB", "MUL", "NEG", "POW", "INV", "STORE"])
def test_opcode_grid_on_edge_operands(ctx, torch, edge, op):
    fq, cols, isq, dcols = edge
    progs = [p for p in H.edge_programs() if p[0].startswith(op)]
    assert progs
    for name, prog, used, ref in progs:
        name = f"{name} fq_field={fq}"
        want, operands = H.edge_reference(cols, used, ref, fq)
        _both_legs(name, prog, fq, _launcher(ctx, torch, prog, H.EDGE_LOG_M, dcols, isq, fq), want, operands)


# ---- 2. domain and layout edges ----------------------------------------------------------------------------------------
class _Row:
    """the trace cells of point i for expr.evaluate_at: Trace(col, off) is row (i + lde_step * off) mod M"""

    def __init__(self, canon, i, lde_step):
        self.canon, self.i, self.lde_step = canon, i, lde_step

    def __getitem__(self, cell):
        col = self.canon[cell[0]]
        return col[(self.i + self.lde_step * cell[1]) % len(col)]


def _ref_eval(expr, log_m, offset, cols, nbase, fq, chal=(), hints=(), lde_step=1):
    """expr.evaluate_at, big integers, at every point of the domain offset * <g_M> (natural order, Montgomery words); cols
    are numpy columns as the evaluator reads them (Fq columns with fq words per point)"""
    m = 1 << log_m
    g = S.root_of_unity(log_m)
    canon = []
    for c, col in enumerate(cols):
        v = [int(w) * S.R_INV % P for w in col]
        canon.append(v if c < nbase else [tuple(v[i * fq:(i + 1) * fq]) for i in range(m)])
    out = np.empty(m * fq, dtype=np.uint64)
    x = S.from_mont(int(offset))
    for i in range(m):
        v = E.evaluate_at(expr, x, _Row(canon, i, lde_step), chal, hints, trace_len=m // lde_step)
        out[i * fq:(i + 1) * fq] = [w * R % P for w in v[:fq]]
        x = x * g % P
    return out


def _reference(expr, log_m, offset, cols, nbase, fq, chal=(), hints=(), lde_step=1):
    """big integers per point up to 2^12 points, the C oracle (u128) above"""
    if log_m <= 12:
        return _ref_eval(expr, log_m, offset, cols, nbase, fq, chal, hints, lde_step)
    from oracle import eval_oracle
    base = np.stack(cols[:nbase]) if nbase else None
    ext = np.stack(cols[nbase:]) if len(cols) > nbase else None
    return eval_oracle.evaluate(expr.to_tuple(), log_m, int(offset), base, ext, fq_lanes=fq, challenges=chal, hints=hints,
                                lde_step=lde_step)


def _bitrev(words, lanes, log_m):
    idx = np.array([S.bit_reverse_index(1 << log_m, i) for i in range(1 << log_m)]) if log_m else np.zeros(1, dtype=np.int64)
    return np.ascontiguousarray(words.reshape(-1, lanes)[idx].reshape(-1))


def _random_cols(seed, log_m, nbase=3, next_=2, fq=3):
    rng = np.random.default_rng(seed)
    m = 1 << log_m
    draw = lambda n: (rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)) % np.uint64(P)
    return [draw(m) for _ in range(nbase)] + [draw(m * fq) for _ in range(next_)]


CHAL = [(11, 2**63 + 5, P - 1), (P - 2, 0, 2**32)]
HINT = [(7, P - 2**32, 3)]
PA = E.Periodic([3, 5], 2)
PB = E.Periodic([(1, 2, 3), (4, 5, 6)], 2)


def _expression_set():
    x = E.X()
    return [
        ("X", x),
        ("X^2+5", x * x + 5),
        ("(X^3-1)/(X-3)", (x ** 3 - 1) / (x - 3)),
        ("Fp offsets", E.Trace(0, 0) * E.Trace(1, 1) - E.Trace(2, -1)),
        ("mixed Fp/Fq3", E.Trace(3, 0) * E.Trace(0, 1) + E.Trace(4, 2) * E.Trace(3, -2)),
        ("Fq3 inverse", (E.Trace(3, 1) + E.Challenge(0)) / (E.Trace(4, 0) - E.Hint(0))),
        ("Fq3 constant", E.Constant((1, 2, 3)) * x ** 5 - E.Challenge(1) ** 3),
        ("-(t^7)+9", -(E.Trace(1, 0) ** 7) + E.Constant(9)),
        ("folded constant", E.Constant(4) * E.Constant(5) + E.Challenge(0) / E.Challenge(1)),
        ("periodic", (E.Trace(0, 1) - PA * E.Trace(1, 0)) * PB + E.Trace(3, 0) * PA * PA - x * PB),
    ]


def _run_set(ctx, torch, log_m, lde_step, cases, cols, nbase=3, fq=3, offset=ms.GENERATOR, trace_bitrev=False,
             out_bitrev=False, log_ce="domain", tag=""):
    """each (name, expr) of `cases` over natural-order columns `cols`, on both legs"""
    ncols = len(cols)
    isq = [c >= nbase for c in range(ncols)]
    stored = [_bitrev(c, fq if q else 1, log_m) if trace_bitrev else c for c, q in zip(cols, isq)]
    dcols = [_device(torch, c) for c in stored]
    for name, ex in cases:
        prog = E.compile_program(ex, nbase, CHAL, HINT, lde_step=lde_step, log_ce=log_m if log_ce == "domain" else log_ce,
                                 num_cols=ncols)
        tabs = E.periodic_tables(ctx, prog, log_m - (lde_step.bit_length() - 1), lde_step, S.from_mont(int(offset))) if prog.periodic else []
        want = _reference(ex, log_m, offset, cols, nbase, fq, CHAL, HINT, lde_step)
        if trace_bitrev and out_bitrev:
            want = _bitrev(want, fq, log_m)
        try:
            run = _launcher(ctx, torch, prog, log_m, dcols + [p for p, _ in tabs], isq + [q for _, q in tabs], fq, offset=offset,
                            trace_bitrev=trace_bitrev, out_bitrev=out_bitrev)
            _both_legs(f"{name} log_m={log_m} lde_step={lde_step}{tag}", prog, fq, run, want)
        finally:
            for p, _ in tabs:
                ctx.free(p)


@pytest.mark.parametrize("log_m", [1, 2, 5, 7, 8, 12, 13, 16, 20])
def test_domain_sizes(ctx, torch, log_m):
    """partial and whole 128-thread blocks, and the two-level twiddle table X reads (tw_hi from 2^13 points on)"""
    lde_step = 1 if log_m < 5 else 4
    _run_set(ctx, torch, log_m, lde_step, _expression_set(), _random_cols(log_m, log_m))


@pytest.mark.parametrize("lde_step", [1, 2, 8])
@pytest.mark.parametrize("off", [-3, -1, 0, 1, 5])
def test_row_offsets_wrap_the_domain(ctx, torch, off, lde_step):
    """Trace(col, off) reads row (i + lde_step * off) mod M; compiled without the domain size, the kernels see the raw shift
    (40 for 5 x 8 at M = 32, 2^32 - 24 for -3 x 8) and must wrap it themselves"""
    log_m = 5
    ex = E.Trace(0, off) * E.Trace(3, off) - E.Trace(1, -off) + E.Trace(4, off) * E.X() + E.Trace(2, 2 * off)
    prog = E.compile_program(ex, 3, lde_step=lde_step)
    shifts = [int(w[3]) for w in prog.code if w[0] & 0xFF == E.OP_TRACE]
    assert off == 0 or any(s >= 1 << log_m for s in shifts)
    _run_set(ctx, torch, log_m, lde_step, [(f"offset {off}", ex)], _random_cols(100 + off, log_m), log_ce=None)


@pytest.mark.parametrize("out_bitrev", [False, True])
@pytest.mark.parametrize("trace_bitrev", [False, True])
def test_storage_orders(ctx, torch, trace_bitrev, out_bitrev):
    """bit-reversed columns are read in place; the output is bit-reversed only together with them (out_bitrev alone is
    ignored: natural order)"""
    log_m = 8
    cases = [c for c in _expression_set() if c[0] in ("X", "Fp offsets", "mixed Fp/Fq3", "Fq3 inverse", "periodic")]
    _run_set(ctx, torch, log_m, 4, cases, _random_cols(200, log_m), trace_bitrev=trace_bitrev, out_bitrev=out_bitrev,
             tag=f" trace_bitrev={trace_bitrev} out_bitrev={out_bitrev}")


@pytest.mark.parametrize("offset", [ms.ONE, ms.GENERATOR, 0x9E3779B97F4A7C15 % P], ids=["one", "generator", "random"])
def test_domain_offsets(ctx, torch, offset):
    log_m = 7
    cases = [c for c in _expression_set() if c[0] in ("X", "(X^3-1)/(X-3)", "Fq3 constant", "periodic")]
    _run_set(ctx, torch, log_m, 2, cases, _random_cols(300, log_m), offset=offset, tag=f" offset={offset:#x}")


def test_strided_columns(ctx, torch):
    """ms_eval_constraints over base and extension matrices whose column strides exceed the domain, against
    ms_eval_constraints_ptrs on the same columns and against the reference"""
    log_m, fq, lde_step = 9, 3, 2
    m = 1 << log_m
    cols = _random_cols(400, log_m)
    bs, es = m + 37, m + 5
    base = np.zeros((3, bs), dtype=np.uint64)
    ext = np.zeros((2, es * fq), dtype=np.uint64)
    for c in range(3):
        base[c, :m] = cols[c]
        base[c, m:] = np.arange(bs - m, dtype=np.uint64) + np.uint64(P)      # padding: not canonical, never read
    for c in range(2):
        ext[c, :m * fq] = cols[3 + c]
        ext[c, m * fq:] = np.uint64(2**64 - 1)
    dcols = [_device(torch, c) for c in cols]
    for name, ex in [c for c in _expression_set() if c[0] in ("Fp offsets", "mixed Fp/Fq3", "Fq3 inverse", "-(t^7)+9")]:
        prog = E.compile_program(ex, 3, CHAL, HINT, lde_step=lde_step, log_ce=log_m)
        want = _reference(ex, log_m, ms.GENERATOR, cols, 3, fq, CHAL, HINT, lde_step)

        def strided():
            out = np.full(m * fq, 2**64 - 1, dtype=np.uint64)
            ctx.eval_constraints(prog, out, log_m, base_cols=base, nbase=3, base_stride=bs, ext_cols=ext, next_=2,
                                 ext_stride=es, fq_field=fq)
            return out
        _both_legs(f"{name} strided", prog, fq, strided, want)
        _both_legs(f"{name} pointers", prog, fq, _launcher(ctx, torch, prog, log_m, dcols, [False] * 3 + [True] * 2, fq), want)


def test_periodic_interval_one_and_trace_length(ctx, torch):
    """a periodic column of interval 1 is a constant; one of interval trace_len is its polynomial in x itself"""
    log_m, lde_step = 8, 4
    n = (1 << log_m) // lde_step
    rng = random.Random(17)
    full = [rng.randrange(P) for _ in range(n)]
    fullq = [tuple(rng.randrange(P) for _ in range(3)) for _ in range(n // 2)]
    cases = [
        ("interval 1", E.Periodic([P - 1], 1) * E.Trace(0, 0) + E.Periodic([(2**63, 0, 5)], 1)),
        ("interval trace_len", E.Periodic(full, n) - E.Trace(3, 1) * E.Periodic(fullq, n)),
        ("interval trace_len, Fp only", E.Periodic(full, n) * E.X() + E.Periodic([1], n)),
    ]
    _run_set(ctx, torch, log_m, lde_step, cases, _random_cols(500, log_m))


# ---- 3. program-shape edges --------------------------------------------------------------------------------------------
def test_full_register_file_rematerialises_leaves(ctx, torch):
    """60 trace cells used early and again late: the allocation reaches all 48 registers and has to drop and reload leaves"""
    log_m, nbase, next_ = 6, 40, 20
    leaves = [E.Trace(j, 0) for j in range(nbase + next_)]
    early = leaves[0] * E.Constant(2)
    for j, t in enumerate(leaves[1:], 1):
        early = early + t * E.Constant(j + 2)
    late = leaves[-1]
    for t in reversed(leaves[:-1]):
        late = late + t
    ex = early * late
    prog = E.compile_program(ex, nbase, log_ce=log_m)
    assert prog.nregs == E.MAX_REGS
    loads = [tuple(w[2:]) for w in prog.code.tolist() if w[0] & 0xFF == E.OP_TRACE]
    assert len(loads) > len(set(loads)), "no leaf was rematerialised"
    cols = _random_cols(600, log_m, nbase, next_)
    want = _reference(ex, log_m, ms.GENERATOR, cols, nbase, 3)
    isq = [c >= nbase for c in range(nbase + next_)]
    _both_legs("48-register program", prog, 3, _launcher(ctx, torch, prog, log_m, [_device(torch, c) for c in cols], isq, 3), want)


def test_48_live_temporaries_are_refused():
    """48 products that are all still needed when the last is formed, plus the accumulator: more than the register file"""
    temps = [E.Trace(j, 0) * E.Trace(j, 1) for j in range(E.MAX_REGS)]
    total, prod = temps[0], temps[0] + 1
    for t in temps[1:]:
        total = total + t
        prod = prod * (t + 1)
    with pytest.raises(ValueError, match="live temporaries"):
        E.compile_program(total + prod, E.MAX_REGS)


@pytest.mark.parametrize("where", ["write", "read"])
def test_register_48_is_refused(ctx, torch, where):
    r = E.MAX_REGS
    code = [[E.OP_X, r, 0, 0], [E.OP_STORE, 0, r, 0]] if where == "write" else \
        [[E.OP_X, 0, 0, 0], [E.OP_ADD, 1, 0, r], [E.OP_STORE, 0, 1, 0]]
    prog = E.Program(np.array(code, dtype=np.uint32), np.zeros((1, 3), dtype=np.uint64), r + 1, False)
    out = torch.empty(64, dtype=torch.int64, device="cuda")
    for leg in LEGS:
        if leg == LEGS[1]:
            os.environ["MS_EVAL_NO_JIT"] = "1"
        try:
            with pytest.raises(ms.MsError):
                ctx.eval_constraints_ptrs(prog, out, 6, [], [], fq_field=1)
        finally:
            os.environ.pop("MS_EVAL_NO_JIT", None)


def test_cached_kernel_reads_new_constants(ctx, torch):
    """a DEEP-shaped program compiled as Air.deep_program does, bound to two different hint / challenge sets and evaluated
    with each back to back: the specialised kernel is cached by instruction stream only, so the second run must read the
    second constant table"""
    log_m, nbase, next_, ncomp = 7, 3, 2, 2
    targs = [(0, 0), (1, 0), (0, 1), (2, 0), (3, 0), (4, 1), (3, -1)]
    ex, keys = deep.deep_expression_symbolic(targs, nbase, next_, ncomp)
    sym = E.compile_program(ex, nbase, log_ce=log_m, symbolic=True, max_live_leaves=8, batch_inverses=True)
    cols = _random_cols(700, log_m, nbase, next_ + ncomp)
    isq = [c >= nbase for c in range(len(cols))]
    dcols = [_device(torch, _bitrev(c, 3 if q else 1, log_m)) for c, q in zip(cols, isq)]
    rng = random.Random(23)
    bound = []
    for k in range(2):
        hints = [tuple(rng.randrange(P) for _ in range(3)) for _ in keys]
        chal = [tuple(rng.randrange(P) for _ in range(3)) for _ in range(2)]
        prog = sym.bind(challenges=chal, hints=hints)
        want = _bitrev(_ref_eval(ex, log_m, ms.GENERATOR, cols, nbase, 3, chal, hints), 3, log_m)
        bound.append((prog, want))
    assert not np.array_equal(bound[0][0].consts, bound[1][0].consts) and np.array_equal(bound[0][0].code, bound[1][0].code)
    for leg in LEGS:
        for k, (prog, want) in enumerate(bound):
            if leg == LEGS[0]:
                _assert_specialised(prog, 3, "DEEP program")
            else:
                os.environ["MS_EVAL_NO_JIT"] = "1"
            try:
                got = _launcher(ctx, torch, prog, log_m, dcols, isq, 3, trace_bitrev=True, out_bitrev=True)()
            finally:
                os.environ.pop("MS_EVAL_NO_JIT", None)
            _first_difference(got, want, 3, f"DEEP program, constant set {k} [{leg}]")
