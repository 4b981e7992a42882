"""GPU: the constraint check (csrc/check.cu, ms_check_constraints) and `GpuProver.prove(..., validate=True)`.

  * the kernel against oracle/check_oracle.py, per constraint (first_row, count) bit for bit: log_n in {0, 1, 5, 10, 16},
    Fp and Fq3, with and without extension columns, failures nowhere / only at row 0 / only at row n - 1 / on every row /
    several in one warp, with 1, 48 and 100 constraints;
  * at 2^20 rows, violations planted at known rows are all found, with exact counts;
  * proofs with validate=True, resident and streamed, equal validate=False; corrupted traces raise the oracle's report;
  * the streamed 2^16-row cycle_burner needs at most 1 MiB more torch peak memory with validation.
The random constraint DAGs, traces and corrupted cases are those of tests/test_validate_cpu.py."""
import numpy as np
import pytest
import torch

import ministark_b200 as ms
from ministark_b200 import expr as E
from ministark_b200.air import ProofOptions
from ministark_b200.prover import GpuProver, peak_bytes
from ministark_b200.validate import ConstraintViolation

import test_validate_cpu as V

pytestmark = pytest.mark.gpu
P = E.P
NONE = 2**64 - 1


@pytest.fixture(scope="module")
def ctx():
    return ms.Context(0)


def _patterned(log_n, nbase):
    """constraints whose failing rows are known: nowhere, row 0, row n - 1, every row, the rows where column 1 is zero"""
    n = 1 << log_n
    g = pow(pow(7, (P - 1) >> 32, P), 1 << (32 - log_n), P)
    X, T = E.X(), E.Trace
    return [T(0) * 0 + 1, E.Constant(5) / (X - 1), E.Constant(5) / (X - pow(g, n - 1, P)), E.Constant(3) / (X ** n - 1),
            (T(0) + 1) / T(nbase - 1)]


def _run(ctx, cons, nbase, next_, lanes, base, ext, chal, hints, log_n):
    prog = E.compile_check_program(cons, nbase, log_n, nbase + next_).bind(challenges=chal, hints=hints)
    dev = [torch.from_numpy(V._cols(c).view(np.int64)).cuda() for c in base]
    dev += [torch.from_numpy(V._cols(c, lanes).view(np.int64)).cuda() for c in ext]
    tables = E.periodic_tables(ctx, prog, log_n, 1, offset_canonical=1)
    try:
        first, count = ctx.check_constraints(prog, dev + [p for p, _ in tables], [False] * nbase + [True] * next_ +
                                             [q for _, q in tables], lanes, log_n, len(cons))
    finally:
        for p, _ in tables:
            ctx.free(p)
    return [(None if int(f) == NONE else int(f), int(c)) for f, c in zip(first, count)]


@pytest.mark.parametrize("log_n", [0, 1, 5, 10, 16])
@pytest.mark.parametrize("fq3", [False, True])
@pytest.mark.parametrize("with_ext", [False, True])
@pytest.mark.parametrize("k", [1, 48, 100])
def test_kernel_equals_oracle(orc, ctx, log_n, fq3, with_ext, k):
    from oracle import check_oracle as CO
    seed = 1000 * log_n + 10 * k + 2 * fq3 + with_ext
    nbase, next_, lanes = 3, (2 if with_ext else 0), (3 if fq3 else 1)
    pattern = _patterned(log_n, nbase)
    cons = (pattern + V.random_constraints(seed, min(log_n, 6), nbase, next_, max(k - len(pattern), 0), fq3=fq3))[:k]
    base, ext = V.random_trace(seed, log_n, nbase, next_, lanes)
    n = 1 << log_n
    base[nbase - 1] = [0 if i in (0, 3, 4, 9, n - 1) else v for i, v in enumerate(base[nbase - 1])]   # several in one warp
    chal = [(5, 6, 7) if fq3 else 5, 11, (0, 0, 1) if fq3 else 2]
    hints = [0, 3]
    got = _run(ctx, cons, nbase, next_, lanes, base, ext, chal, hints, log_n)
    b = np.stack([V._cols(c) for c in base])
    e = np.stack([V._cols(c, lanes) for c in ext]) if ext else None
    want = CO.check([c.to_tuple() for c in cons], log_n, b, e, lanes, chal, hints)
    assert got == want
    if k >= len(pattern):
        assert got[0] == (None, 0) and got[1] == (0, 1) and got[2] == (n - 1, 1) and got[3] == (0, n)


def test_planted_violations_at_2_20_rows(ctx):
    log_n, n = 20, 1 << 20
    rng = np.random.default_rng(7)
    a = rng.integers(1, 2**63, size=n, dtype=np.uint64)                     # canonical, non-zero
    b = rng.integers(1, 2**63, size=n, dtype=np.uint64)
    planted = np.array(sorted(set(rng.integers(0, n, size=300).tolist()) | {0, 1, 2, 31, 32, n - 1}), dtype=np.int64)
    b[planted] = 0
    cq = np.zeros(3 * n, dtype=np.uint64)
    cq[0::3], cq[2::3] = a, b                                              # Fq3 column (a, 0, b): zero nowhere
    mont = lambda v: torch.from_numpy(np.array([x * 2**64 % P for x in v.tolist()], dtype=np.uint64).view(np.int64)).cuda()
    cols = [mont(a), mont(b), mont(cq)]
    g = pow(pow(7, (P - 1) >> 32, P), 1 << (32 - log_n), P)
    T, X = E.Trace, E.X()
    cons = [T(0) / T(1),                                 # fails exactly at the planted rows
            T(0) / T(1, -1),                             # ... shifted by one row, across the wrap
            T(1) / T(1),                                 # 0/0 = Some(0): never fails
            T(2) / T(1),                                 # Fq3 numerator, never zero: the planted rows
            E.Constant(1) / (X - pow(g, 12345, P)),      # row 12345 only
            T(2) * (E.Constant(1) / T(1))]               # None * Some(non-zero Fq3): the planted rows
    prog = E.compile_check_program(cons, 2, log_n, 3)
    first, count = ctx.check_constraints(prog, cols, [False, False, True], ms.FQ3, log_n, len(cons))
    shifted = np.sort((planted + 1) % n)
    assert [(int(f), int(c)) for f, c in zip(first, count)] == [
        (int(planted[0]), len(planted)), (int(shifted[0]), len(planted)), (NONE, 0), (int(planted[0]), len(planted)),
        (12345, 1), (int(planted[0]), len(planted))]


def _streamed(claim, opts, n):
    from ministark_b200.air import Air
    cfg, o = claim.AirConfig, ProofOptions(*opts)
    est = peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS,
                     ms.FP if cfg.FQ_IS_FP else ms.FQ3, Air(cfg, n, None, o).ce_blowup_factor, o.fri_folding_factor)
    return GpuProver(0, memory_budget=(est["streamed"] + est["resident"]) // 2)


def _case(which):
    from ministark_b200.examples import brainfuck as bf
    if which == "burner":
        trace, output = bf.simulate(bf.cycle_burner(14, 14, 30))                          # 2^16 rows
        return bf.BrainfuckClaim(bf.cycle_burner(14, 14, 30), b"", output), (19, 16, 20, 16, 16), trace
    if which == "fib:18":
        from ministark_b200.examples import fib
        trace, last = fib.gen_trace(8 << 18)
        return fib.FibClaim(last), (16, 4, 4, 8, 16), trace
    return V._make_case(which)


@pytest.mark.parametrize("residency", ["resident", "streamed"])
@pytest.mark.parametrize("which", ["fib:7", "fib:13", "fib:18", "perm", "brainfuck", "burner"])
def test_validated_proof_equals_plain_proof(which, residency):
    claim, opts, trace = _case(which)
    p = GpuProver(0) if residency == "resident" else _streamed(claim, opts, len(trace))
    plain = p.prove(claim, ProofOptions(*opts), trace)
    checked = p.prove(claim, ProofOptions(*opts), trace, validate=True)
    assert p.last_residency == residency
    assert checked.to_bytes() == plain.to_bytes()
    assert "validate_constraints" in checked.timings and "validate_constraints" not in plain.timings


@pytest.mark.parametrize("residency", ["resident", "streamed"])
@pytest.mark.parametrize("which", ["fib:6:cell", "fib:6:boundary", "fib:6:terminal", "fib:6:wrap", "brainfuck:base",
                                   "brainfuck:ext"])
def test_corrupted_traces_raise_the_oracle_report(orc, which, residency):
    from oracle import check_oracle as CO
    claim, opts, trace = V._make_case(which)
    p = GpuProver(0) if residency == "resident" else _streamed(claim, opts, len(trace))
    with pytest.raises(ConstraintViolation) as ei:
        p.prove(claim, ProofOptions(*opts), trace, validate=True)
    assert p.last_residency == residency
    want = V._expected(CO, which, None)
    got = ei.value.violations
    assert [(v.constraint, v.first_row, v.count) for v in got] == want["counts"]
    assert list(got[0].values) == want["values"]
    assert str(ei.value).startswith(f"Constraint {got[0].constraint} does not evaluate to a low degree polynomial. "
                                    f"Divide by zero occurs at row {got[0].first_row} ")


def test_validation_adds_no_peak_memory_streamed():
    claim, opts, trace = _case("burner")
    p = _streamed(claim, opts, len(trace))
    peaks = {}
    for validate in (False, True, False, True):           # the second pair: plans and scratch are warm for both
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        p.prove(claim, ProofOptions(*opts), trace, validate=validate)
        torch.cuda.synchronize()
        peaks[validate] = torch.cuda.max_memory_allocated() - base
    assert p.last_residency == "streamed"
    assert peaks[True] <= peaks[False] + (1 << 20), peaks
