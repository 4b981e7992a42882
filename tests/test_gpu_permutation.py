"""GPU: the permutation target fill (csrc/permutation.cu, ms_permutation_fill) and proofs of AIRs that declare permutations.

  * the kernel equals oracle/permutation_oracle.py word for word for W = 1 to 4 up to 2^14 rows (duplicate tuples, words
    0 and p - 1, row offsets), and a numpy lexsort up to 2^24 rows;
  * MemoryDeclaredClaim proves to the bytes of the hand-written MemoryClaim at 2^10, 2^14 and 2^20 rows, and to the CPU
    restatement's bytes (oracle/stark_oracle.cpu_prove) at 2^8 rows;
  * MemoryDeclaredClaim proves from a device trace at 2^20 rows, resident and streamed under a forced budget, validated,
    and verifies; the caller's tensor is unchanged and the torch peak stays within peak_bytes."""
import numpy as np
import pytest
import torch

from ministark_b200 import FQ3, Context
from ministark_b200 import expr as E
from ministark_b200.air import Air, ProofOptions

pytestmark = pytest.mark.gpu

P = E.P
_R = 2**64
T = E.Trace
OPTS = ProofOptions(16, 8, 4, 4, 8)


@pytest.fixture(scope="module")
def ctx():
    return Context(0)


def run_kernel(ctx, source, base):
    """base: (nbase, n) Montgomery words, numpy or a cuda tensor.  Returns the (W, n) target words"""
    nbase, n = base.shape
    log_n = n.bit_length() - 1
    dev = base if isinstance(base, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(base).view(np.int64)).cuda()
    prog = E.compile_lookup_program(source, (), None, nbase, log_n)
    W = len(source)
    work = torch.empty(ctx.permutation_workspace_bytes(log_n, W), dtype=torch.uint8, device="cuda")
    out = torch.full((W, n), -1, dtype=torch.int64, device="cuda")
    tables = E.periodic_tables(ctx, prog, log_n, 1, offset_canonical=1)
    torch.cuda.synchronize()
    try:
        ctx.permutation_fill(prog, [out[k] for k in range(W)], log_n, [dev[c] for c in range(nbase)] + [p for p, _ in tables],
                             W, work)
        ctx.sync()
    finally:
        for p, _ in tables:
            ctx.free(p)
    return out.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("W,log_n,hi", [(1, 0, 4), (1, 12, 2**40), (2, 5, 3), (2, 14, 4), (3, 10, 3), (3, 13, 2**20),
                                        (4, 11, 3), (4, 14, 5)])
def test_kernel_equals_oracle(ctx, W, log_n, hi):
    from oracle import permutation_oracle as PO
    from test_permutation_cpu import SOURCES, _base
    base = _base(W * 100 + log_n, log_n, hi=hi)
    assert np.array_equal(run_kernel(ctx, SOURCES[W], base), PO.targets(SOURCES[W], base))


def _mont_np(x):
    """Montgomery words of canonical uint64 values below 2^62"""
    x = np.asarray(x, dtype=np.uint64)
    h, l = x >> np.uint64(32), x & np.uint64(0xFFFFFFFF)
    v, s = l << np.uint64(32), h + l
    return np.where(v >= s, v - s, v + (np.uint64(P) - s))


@pytest.mark.parametrize("W,log_n", [(1, 20), (2, 20), (4, 20), (1, 24), (2, 24), (3, 24), (4, 24)])
def test_kernel_equals_numpy_lexsort(ctx, W, log_n):
    """word k of the source is column k shifted by one row for odd k; columns of few distinct values make long runs of
    equal tuples, whose rows the stable sort keeps in order"""
    n = 1 << log_n
    rng = np.random.default_rng(W + log_n)
    canon = np.stack([rng.integers(0, hi, size=n, dtype=np.uint64) for hi in (1 << 62, 7, 1 << 20, 3)[:W]])
    source = tuple(T(k, k & 1) for k in range(W))
    words = np.stack([np.roll(canon[k], -(k & 1)) for k in range(W)])
    order = np.lexsort(words[::-1])
    got = run_kernel(ctx, source, _mont_np(canon))
    assert np.array_equal(got, _mont_np(words[:, order]))


# ------------------------------------------------------------------------------------------------- proofs
@pytest.mark.parametrize("log_n", [10, 14, 20])
def test_declared_memory_proves_to_the_hand_written_bytes(log_n):
    from ministark_b200.examples import memory as MM
    n = 1 << log_n
    trace, reads = MM.MemoryDeclaredClaim.gen_trace(n, n // 16, seed=log_n)
    declared = MM.MemoryDeclaredClaim(reads).prove(OPTS, trace)
    hand_trace, hand_reads = MM.MemoryClaim.gen_trace(n, n // 16, seed=log_n)
    assert hand_reads == reads
    hand = MM.MemoryClaim(reads).prove(OPTS, hand_trace)
    assert declared.to_bytes() == hand.to_bytes()
    assert "permutation_fill" in declared.timings and "lookup_multiplicities" in declared.timings
    MM.MemoryDeclaredClaim(reads).verify(declared.to_bytes(), 10)


def test_memory_proves_to_the_cpu_restatement(orc):
    from ministark_b200.prover import GpuProver
    from test_permutation_cpu import _cpu_restatement, _make_case
    claim, opts, trace = _make_case("memory")
    assert GpuProver(0).prove(claim, ProofOptions(*opts), trace, validate=True).to_bytes() == _cpu_restatement("memory")


@pytest.mark.parametrize("residency", ["resident", "streamed"])
def test_memory_from_a_device_trace(residency):
    from ministark_b200.examples import memory as MM
    from ministark_b200.prover import GpuProver, peak_bytes
    n = 1 << 20
    trace, reads = MM.MemoryDeclaredClaim.gen_trace(n, 1 << 12, seed=3, device=0)
    before = trace.base_columns().clone()
    cfg = MM.MemoryDeclaredAirConfig
    est = peak_bytes(n, OPTS.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, FQ3,
                     Air(cfg, n, None, OPTS).ce_blowup_factor, OPTS.fri_folding_factor)
    p = GpuProver(0)
    if residency == "streamed":
        p.memory_budget = (est["streamed"] + est["resident"]) // 2
    claim = MM.MemoryDeclaredClaim(reads)
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
