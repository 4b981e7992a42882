"""GPU: extension columns declared by the AIR (air.RunningColumn) and built by ms_extension_columns (csrc/extension.cu).

  * the kernel equals oracle/extension_oracle.py word for word from 1 to 2^22 rows (random declarations with offsets,
    X, Periodic, Hint leaves and zero denominators up to 2^14 rows, the examples' shapes beyond), and at 2^24 rows for two
    Fq3 columns;
  * declaring brainfuck's input and output evaluations reproduces columns 7 and 8 of its device builder;
  * the declared perm AIR proves to the bytes of the callback perm AIR at 2^10 and 2^14 rows;
  * the declared perm and LogUp AIRs prove and verify at 2^20 rows, resident and streamed under a forced budget, with the
    torch peak within peak_bytes."""
import os
import sys

import numpy as np
import pytest
import torch

import ministark_b200 as ms
from ministark_b200 import expr as E
from ministark_b200.air import Air, ProofOptions, RunningColumn

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_extension_cpu import _case_inputs, _mont, _periodic_tables, random_declaration  # noqa: E402

P = E.P


@pytest.fixture(scope="module")
def ctx():
    return ms.Context(0)


def _device(words):
    return torch.from_numpy(np.ascontiguousarray(words, dtype=np.uint64).view(np.int64)).cuda()


def _build(ctx, decl, base, lanes, log_n, chal, hints):
    """ms_extension_columns over device copies of `base`; returns (K, n * lanes) host words"""
    nbase = base.shape[0]
    prog = E.compile_extension_program([c.mul for c in decl], [c.add for c in decl], nbase, log_n, nbase)
    prog = prog.bind(challenges=chal, hints=hints)
    init = np.array([[_mont(w) for w in E.evaluate_at(E.Expr._lift(c.init), 0, challenges=chal, hints=hints)[:lanes]]
                     for c in decl], dtype=np.uint64)
    d_base = _device(base)
    tables = [_device(t) for t in _periodic_tables(prog, log_n, lanes)]
    out = torch.empty((len(decl), (1 << log_n) * lanes), dtype=torch.int64, device="cuda")
    ctx.extension_columns(prog, out, log_n, [d_base[c] for c in range(nbase)] + tables,
                          [False] * nbase + [p[3] for p in prog.periodic], lanes, init, [c.inclusive for c in decl])
    ctx.sync()
    return out.cpu().numpy().view(np.uint64)


def _examples_declaration():
    al, T = E.Challenge(0), E.Trace
    return [RunningColumn(1, al - T(0)),                                                   # running product
            RunningColumn(0, al, T(2, -1), inclusive=True),                                 # running evaluation
            RunningColumn(E.Hint(0), add=T(2, 1) / (al - T(1)) - E.Constant(1) / (al - T(0)))]   # LogUp sum


@pytest.mark.parametrize("log_n", list(range(0, 23)))
@pytest.mark.parametrize("fq3", [False, True])
def test_kernel_equals_oracle(ctx, log_n, fq3):
    from oracle import extension_oracle as XO
    lanes = 3 if fq3 else 1
    if log_n <= 14:
        decl = random_declaration(log_n * 2 + fq3, log_n, 3, 1 + (log_n % 4), fq3)
        base, chal, hints = _case_inputs(log_n, log_n, 3, fq3)
    else:
        from oracle import oracle as orc
        decl = _examples_declaration()
        base = orc.rand_matrix(3, 1 << log_n, 1, seed=log_n)
        base[1, ::7] = base[0, ::7]                              # alpha - t = alpha - v there: shared denominators
        _, chal, hints = _case_inputs(log_n, 0, 3, fq3)
    got = _build(ctx, decl, base, lanes, log_n, chal, hints)
    want = XO.columns([(c.init, c.mul, c.add, c.inclusive) for c in decl], base, lanes, chal, hints)
    assert np.array_equal(got, want)


def test_kernel_equals_oracle_at_2p24_for_two_fq3_columns(ctx):
    from oracle import extension_oracle as XO
    from oracle import oracle as orc
    log_n = 24
    decl = _examples_declaration()[:2]
    base = orc.rand_matrix(3, 1 << log_n, 1, seed=24)
    _, chal, hints = _case_inputs(24, 0, 3, True)
    got = _build(ctx, decl, base, 3, log_n, chal, hints)
    want = XO.columns([(c.init, c.mul, c.add, c.inclusive) for c in decl], base, 3, chal, hints)
    assert np.array_equal(got, want)


def test_declared_brainfuck_evaluations_reproduce_its_builder(ctx):
    from ministark_b200.examples import brainfuck as bf
    trace, _ = bf.simulate(",[.,]", b"extension columns\x00")       # cat: both columns carry data
    n = len(trace)
    log_n = n.bit_length() - 1
    nchal = Air(bf.BrainfuckAirConfig, n, None, ProofOptions(19, 16, 20, 16, 16)).num_challenges()
    rng = np.random.default_rng(7)
    chal = [tuple(int(v) for v in rng.integers(0, P, size=3, dtype=np.uint64)) for _ in range(nchal)]
    base = _device(trace.base_columns())
    want = trace.build_extension_columns_device(chal, ctx, base)
    ctx.sync()                                                  # built on the context's stream
    want = want.cpu().numpy().view(np.uint64)
    decl = [RunningColumn(0, E.Challenge(bf.CH_GAMMA), E.Trace(bf.IN_VALUE), inclusive=True),
            RunningColumn(0, E.Challenge(bf.CH_DELTA), E.Trace(bf.OUT_VALUE), inclusive=True)]
    got = _build(ctx, decl, np.asarray(trace.base_columns()), 3, log_n, chal, [])
    assert np.any(got != 0)
    assert np.array_equal(got[0], want[7]) and np.array_equal(got[1], want[8])


@pytest.mark.parametrize("log_n", [10, 14])
def test_declared_perm_proves_to_the_callback_bytes(log_n):
    from ministark_b200.examples import perm
    from ministark_b200.prover import GpuProver
    opts = ProofOptions(16, 8, 4, 4, 8)
    p = GpuProver(0)
    want = p.prove(perm.PermClaim(), opts, perm.gen_trace(1 << log_n, seed=5)).to_bytes()
    got = p.prove(perm.PermDeclaredClaim(), opts, perm.gen_trace(1 << log_n, seed=5, extension=False)).to_bytes()
    assert got == want


def _case(which, n):
    from ministark_b200.examples import lookup, perm
    if which == "perm":
        return perm.PermDeclaredClaim(), perm.gen_trace(n, seed=9, extension=False)
    return lookup.LookupClaim(), lookup.gen_trace(n, seed=9)


@pytest.mark.parametrize("residency", ["resident", "streamed"])
@pytest.mark.parametrize("which", ["perm", "lookup"])
def test_declared_airs_prove_and_verify_at_2p20(which, residency):
    from ministark_b200 import FQ3
    from ministark_b200.prover import GpuProver, peak_bytes
    n = 1 << 20
    opts = ProofOptions(16, 8, 4, 4, 8)
    claim, trace = _case(which, n)
    cfg = claim.AirConfig
    est = peak_bytes(n, 8, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, FQ3, Air(cfg, n, None, opts).ce_blowup_factor, 4)
    p = GpuProver(0)
    if residency == "streamed":
        p.memory_budget = (est["streamed"] + est["resident"]) // 2
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    proof = p.prove(claim, opts, trace)
    peak = torch.cuda.max_memory_allocated() - base
    assert p.last_residency == residency
    assert peak <= est[residency], (peak, est)
    claim.verify(proof.to_bytes(), 10)
