"""GPU: the lookup multiplicity fill (csrc/lookup.cu, ms_lookup_multiplicities) and proofs of AIRs that declare lookups.

  * the kernel equals oracle/lookup_oracle.py word for word on random declarations up to 2^14 rows, the duplicate-run table
    and the miss and bad-selector rows, and a numpy lexicographic reference on the two examples' shapes at 2^16 to 2^22 rows
    and a W = 1, Q = 2 lookup at 2^24 rows;
  * DeclaredLookupClaim proves to the bytes of the hand-written LookupClaim at 2^10, 2^14 and 2^20 rows;
  * SquareLookupClaim proves from a device trace at 2^20 rows, resident and streamed under a forced budget, and verifies;
    the caller's tensor is unchanged and the torch peak stays within peak_bytes; a device trace with a miss raises
    LookupViolation."""
import numpy as np
import pytest
import torch

from ministark_b200 import FQ3, Context
from ministark_b200 import expr as E
from ministark_b200.air import Air, Lookup, ProofOptions

pytestmark = pytest.mark.gpu

P = E.P
_R = 2**64
_RINV = pow(_R, -1, P)
T = E.Trace
OPTS = ProofOptions(16, 8, 4, 4, 8)


@pytest.fixture(scope="module")
def ctx():
    return Context(0)


def run_kernel(ctx, lk, base):
    """base: (nbase, n) Montgomery words, numpy or a cuda tensor.  Returns (out words, missing, bad)"""
    nbase, n = base.shape
    log_n = n.bit_length() - 1
    dev = base if isinstance(base, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(base).view(np.int64)).cuda()
    prog = E.compile_lookup_program(lk.table, lk.values, lk.selectors, nbase, log_n)
    W, Q = len(lk.table), len(lk.values)
    work = torch.empty(ctx.lookup_workspace_bytes(log_n, W, Q), dtype=torch.uint8, device="cuda")
    out = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    tables = E.periodic_tables(ctx, prog, log_n, 1, offset_canonical=1)
    torch.cuda.synchronize()
    try:
        missing, bad = ctx.lookup_multiplicities(prog, out, log_n, [dev[c] for c in range(nbase)] + [p for p, _ in tables],
                                                 W, Q, work)
    finally:
        for p, _ in tables:
            ctx.free(p)
    return out.cpu().numpy().view(np.uint64), missing, bad


def numpy_multiplicities(table, values, selectors=None):
    """the lexicographic reference: table (W, n) and values (Q, W, n) canonical uint64, selectors (Q, n) or None.
    Returns the n multiplicities (ints) and the per-tuple miss counts"""
    W, n = table.shape
    allv = np.concatenate([table.T] + [v.T for v in values])
    if W == 1:
        uniq, inv = np.unique(allv[:, 0], return_inverse=True)
    else:
        uniq, inv = np.unique(allv, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    first = np.full(len(uniq), -1, dtype=np.int64)
    first[inv[:n][::-1]] = np.arange(n, dtype=np.int64)[::-1]       # the lowest row of every table tuple
    counts, misses = np.zeros(n, dtype=np.int64), []
    for q in range(len(values)):
        hit = first[inv[n * (q + 1):n * (q + 2)]]
        on = np.ones(n, dtype=bool) if selectors is None else selectors[q] == 1
        counts += np.bincount(hit[on & (hit >= 0)], minlength=n)
        misses.append(int((on & (hit < 0)).sum()))
    return counts, misses


def _mont_np(x):
    x = np.asarray(x, dtype=np.uint64)
    h, l = x >> np.uint64(32), x & np.uint64(0xFFFFFFFF)
    v, s = l << np.uint64(32), h + l
    return np.where(v >= s, v - s, v + (np.uint64(P) - s))


@pytest.mark.parametrize("seed,W,Q,sel,log_n", [(0, 1, 1, False, 0), (1, 2, 2, True, 5), (2, 4, 4, True, 10), (3, 3, 2, False, 12),
                                                (4, 1, 4, True, 14), (5, 4, 1, False, 14), (6, 2, 3, True, 13)])
def test_kernel_equals_oracle(ctx, seed, W, Q, sel, log_n):
    from oracle import lookup_oracle as LO
    from test_lookup_cpu import _base, random_lookup
    lk, base = random_lookup(seed, W, Q, sel, log_n), _base(seed, log_n)
    got, missing, bad = run_kernel(ctx, lk, base)
    want, wmiss, wbad = LO.multiplicities(lk.table, lk.values, lk.selectors, base)
    assert np.array_equal(got, want) and missing == wmiss and bad == wbad


def test_kernel_duplicate_runs_misses_and_bad_selectors(ctx):
    from oracle import lookup_oracle as LO
    from test_lookup_cpu import _base
    log_n = 12
    n = 1 << log_n
    base = _base(7, log_n)
    base[0] = np.uint64((P - 1) * _R % P)                                          # one tuple repeated n times
    base[1] = np.array([(v * _R) % P for v in np.random.default_rng(2).choice([0, P - 1, 5], size=n).tolist()], dtype=np.uint64)
    base[3] = np.array([(v * _R) % P for v in [1] * (n - 3) + [2, P - 1, 0]], dtype=np.uint64)
    for lk in (Lookup((T(0), T(1)), ((T(0, 3), T(1, -1)), (T(1), T(0))), 4, 5, (E.Constant(1), T(3))),
               Lookup((T(1),), ((T(0, 1),), (T(2),)), 4, 5, (T(3), E.Constant(1)))):
        got, missing, bad = run_kernel(ctx, lk, base)
        want, wmiss, wbad = LO.multiplicities(lk.table, lk.values, lk.selectors, base)
        assert np.array_equal(got, want) and missing == wmiss and bad == wbad
    assert bad == (2, n - 3)


def _shape_case(kind, log_n, seed):
    """the two examples' lookups over random columns, with canonical columns for the numpy reference"""
    n = 1 << log_n
    rng = np.random.default_rng(seed)
    if kind == "range":                     # DeclaredLookupAirConfig: v in t = 0..n-1
        v = rng.integers(0, n, size=n, dtype=np.uint64)
        canon = np.stack([v, np.arange(n, dtype=np.uint64), np.zeros(n, dtype=np.uint64)])
        lk = Lookup((T(1),), ((T(0),),), 2, 3)
        return lk, canon, canon[[1]], [canon[[0]]], None
    if kind == "two_values":                # W = 1, Q = 2 over a table with duplicates
        t = rng.integers(0, n // 4, size=n, dtype=np.uint64)
        a, b = t[rng.permutation(n)], t[rng.permutation(n)]
        b[::97] = np.uint64(n)              # some misses
        canon = np.stack([t, a, b, np.zeros(n, dtype=np.uint64)])
        lk = Lookup((T(0),), ((T(1),), (T(2),)), 3, 4)
        return lk, canon, canon[[0]], [canon[[1]], canon[[2]]], None
    from ministark_b200.examples import lookup as L   # SquareLookupAirConfig
    canon = L._square_columns(n, seed).astype(np.uint64)
    lk = L.SquareLookupAirConfig.lookups(n)[0]
    return lk, canon, canon[[0, 1]], [canon[[2, 4]], canon[[3, 5]]], np.stack([np.ones(n, dtype=np.uint64), canon[6]])


@pytest.mark.parametrize("kind,log_n", [("range", 16), ("square", 16), ("range", 20), ("square", 20), ("range", 22),
                                        ("square", 22), ("two_values", 24)])
def test_kernel_equals_numpy_on_example_shapes(ctx, kind, log_n):
    lk, canon, table, values, sel = _shape_case(kind, log_n, 11)
    got, missing, bad = run_kernel(ctx, lk, _mont_np(canon))
    counts, misses = numpy_multiplicities(table, values, sel)
    assert np.array_equal(got, _mont_np(counts.astype(np.uint64)))
    assert [m for m, _ in missing] == misses and bad == (0, None)


# ------------------------------------------------------------------------------------------------- proofs
@pytest.mark.parametrize("log_n", [10, 14, 20])
def test_declared_lookup_proves_to_the_hand_written_bytes(log_n):
    from ministark_b200.examples import lookup as L
    n = 1 << log_n
    declared = L.DeclaredLookupClaim().prove(OPTS, L.DeclaredLookupClaim.gen_trace(n, seed=log_n))
    hand = L.LookupClaim().prove(OPTS, L.gen_trace(n, seed=log_n))
    assert declared.to_bytes() == hand.to_bytes()
    assert "lookup_multiplicities" in declared.timings
    L.DeclaredLookupClaim().verify(declared.to_bytes(), 10)


@pytest.mark.parametrize("residency", ["resident", "streamed"])
def test_square_lookup_from_a_device_trace(residency):
    from ministark_b200.examples import lookup as L
    from ministark_b200.prover import GpuProver, peak_bytes
    n = 1 << 20
    trace = L.SquareLookupClaim.gen_trace(n, seed=3, device=0)
    before = trace.base_columns().clone()
    cfg = L.SquareLookupAirConfig
    est = peak_bytes(n, OPTS.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, FQ3,
                     Air(cfg, n, None, OPTS).ce_blowup_factor, OPTS.fri_folding_factor)
    p = GpuProver(0)
    if residency == "streamed":
        p.memory_budget = (est["streamed"] + est["resident"]) // 2
    claim = L.SquareLookupClaim()
    p.prove(claim, OPTS, trace)                         # warm: programs, plans
    torch.cuda.synchronize()
    base_alloc = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    proof = p.prove(claim, OPTS, trace, validate=True)
    peak = torch.cuda.max_memory_allocated() - base_alloc
    assert p.last_residency == residency
    assert peak <= est[residency], (peak, est[residency])
    assert torch.equal(trace.base_columns(), before)
    claim.verify(proof.to_bytes(), 10)


def test_device_trace_with_a_miss_raises():
    from ministark_b200.examples import lookup as L
    from ministark_b200.prover import LookupViolation, Trace
    n = 1 << 12
    trace = L.SquareLookupClaim.gen_trace(n, seed=5, device=0)
    cols = trace.base_columns().clone()
    cols[L.CS, 100] = int(np.uint64(12345 * _R % P).view(np.int64))
    torch.cuda.synchronize()
    with pytest.raises(LookupViolation) as e:
        L.SquareLookupClaim().prove(OPTS, Trace(cols))
    (m,) = e.value.misses
    a = int(cols[L.AS, 100]) % 2**64 * _RINV % P
    assert (m.lookup, m.tuple, m.kind, m.first_row, m.count, m.values) == (0, 0, "missing", 100, 1, (a, 12345))
