"""GPU: the streamed residency of `GpuProver` and its two kernels against their resident counterparts.

  * ms_merkle_commit_block_sha256 over every coset block, then ms_merkle_nodes_sha256 over the block roots, gives the
    node heap and root of ms_merkle_commit_sha256 over the whole matrix, bit for bit, and both equal the CPU oracle's
    up to 2^16 rows; a single row, which ms_merkle_commit_sha256 refuses, gives its leaf digest as the block root;
  * ms_lde_rows gives the rows ms_gather_rows reads from ms_lde_batch(..., bitrev_out = 1);
  * a proof made with the budget forced between the two estimates (streamed) has the bytes of the resident prover's;
  * for brainfuck the streamed torch peak stays within its own estimate and far below the resident peak."""
import numpy as np
import pytest
import torch

import ministark_b200 as ms
from ministark_b200.air import ProofOptions
from ministark_b200.examples import brainfuck as bf
from ministark_b200.examples import fib, perm
from ministark_b200.prover import GpuProver, peak_bytes

pytestmark = pytest.mark.gpu
P = ms.P


@pytest.fixture(scope="module")
def ctx():
    return ms.Context(0)


def _rand(ctx, ncols, words, seed):
    t = torch.empty((ncols, words), dtype=torch.int64, device="cuda")
    ctx.fill_random(t, t.numel(), seed)
    return t


# (field, ncols): three columns at every block size; the other counts, without the 2^20-row blocks, put the one-block
# (Fp 1, 7; Fq3 1), constant-padding (Fp 8; Fq3 8 = 24 words) and multi-block (Fp 17) leaf shapes through the block
# commit.  The three-column cases keep the ids they had before the column count was a parameter.
_BLOCK_CASES = [(field, ncols, log_n, log_b)
                for field, ncols in [(ms.FP, 3), (ms.FQ3, 3), (ms.FP, 1), (ms.FP, 7), (ms.FP, 8), (ms.FP, 17), (ms.FQ3, 1),
                                     (ms.FQ3, 8)]
                for log_n in ([0, 1, 5, 12, 20] if ncols == 3 else [0, 1, 5, 12]) for log_b in [0, 1, 3, 4]]


@pytest.mark.parametrize("field,ncols,log_n,log_b", _BLOCK_CASES,
                         ids=[f"{b}-{n}-{f}" + ("" if c == 3 else f"-{c}cols") for f, c, n, b in _BLOCK_CASES])
def test_block_commit_equals_resident_commit(ctx, orc, field, ncols, log_n, log_b):
    n, beta = 1 << log_n, 1 << log_b
    N = n * beta
    mat = _rand(ctx, ncols, N * field, seed=log_n * 16 + log_b + field)
    ctx.sync()
    cols = np.ascontiguousarray(mat.cpu().numpy().view(np.uint64)) if N <= 1 << 16 else None
    if N == 1:                                      # no tree: the resident commit refuses one leaf, the block root is it
        with pytest.raises(ms.MsError):
            ctx.merkle_commit(mat, field, N, ncols)
        root = torch.empty(4, dtype=torch.int64, device="cuda")
        ctx.merkle_commit_block(mat, field, 0, 0, 0, ncols, torch.empty(4, dtype=torch.int64, device="cuda"), root)
        assert root.cpu().numpy().tobytes() == orc.hash_rows(cols, field)[0].tobytes()
        return
    want = torch.empty((N, 4), dtype=torch.int64, device="cuda")
    root = ctx.merkle_commit(mat, field, N, ncols, nodes=want)
    if cols is not None:                            # the resident commit itself against the serial CPU oracle
        assert root == orc.merkle_nodes(orc.hash_rows(cols, field))[1].tobytes()
    nodes = torch.full((N, 4), -1, dtype=torch.int64, device="cuda")
    roots = torch.empty((beta, 4), dtype=torch.int64, device="cuda")
    for q in range(beta):
        ctx.merkle_commit_block(mat.data_ptr() + q * n * field * 8, field, log_n, log_b, q, ncols, nodes, roots[q], col_stride=N)
    if beta > 1:
        ctx.merkle_nodes(roots, nodes, beta)
    torch.cuda.synchronize()
    assert torch.equal(nodes[1:], want[1:])
    assert nodes[1].cpu().numpy().tobytes() == root


@pytest.mark.parametrize("field", [ms.FP, ms.FQ3])
@pytest.mark.parametrize("log_n", [0, 1, 5, 12, 20])
@pytest.mark.parametrize("log_b", [0, 1, 3, 4])
def test_lde_rows_equal_gathered_lde_rows(ctx, field, log_n, log_b):
    n, N = 1 << log_n, 1 << (log_n + log_b)
    ncols = 5
    coeffs = _rand(ctx, ncols, n * field, seed=log_n * 16 + log_b + 7 * field)
    coeffs[1].zero_()                                         # zero column
    coeffs[2].zero_()
    coeffs[2][:field] = _rand(ctx, 1, field, seed=99)[0]     # constant column
    coeffs[3].fill_(P - 1 - 2**64)                           # every word p - 1 (as int64)
    lde = torch.empty((ncols, N * field), dtype=torch.int64, device="cuda")
    ctx.lde_batch(coeffs, lde, field, log_n, log_b, ncols, offset=ms.GENERATOR, bitrev=True)
    rng = np.random.default_rng(N + field)
    positions = [0, N - 1, N // 2, 0, N - 1] + [int(v) for v in rng.integers(0, N, size=75)]
    want = ctx.gather_rows(lde, field, N, ncols, positions)
    got = ctx.lde_rows(coeffs, field, log_n, log_b, ncols, positions)
    assert np.array_equal(got, want)


def _case(which):
    if which.startswith("fib"):
        log_rows = int(which.split(":")[1])
        trace, last = fib.gen_trace(8 << log_rows)
        return fib.FibClaim(last), (16, 4, 4, 8, 16), trace
    if which == "perm":
        return perm.PermClaim(), (16, 8, 4, 4, 8), perm.gen_trace(1 << 10, seed=5)
    src = bf.HELLO_WORLD if which == "brainfuck" else bf.cycle_burner(14, 14, 30)     # (14, 14, 30): 2^16 rows
    trace, output = bf.simulate(src)
    return bf.BrainfuckClaim(src, b"", output), (19, 16, 20, 16, 16), trace


def _estimates(claim, opts, n):
    from ministark_b200.air import Air
    cfg = claim.AirConfig
    o = ProofOptions(*opts)
    return peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS,
                      ms.FP if cfg.FQ_IS_FP else ms.FQ3, Air(cfg, n, None, o).ce_blowup_factor, o.fri_folding_factor)


def _peak_prove(prover, claim, opts, trace):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    proof = prover.prove(claim, ProofOptions(*opts), trace).to_bytes()
    torch.cuda.synchronize()
    return proof, torch.cuda.max_memory_allocated() - base


@pytest.fixture(scope="module")
def resident():
    return GpuProver(0)


@pytest.mark.parametrize("which", ["fib:7", "fib:13", "fib:18", "perm", "brainfuck", "burner"])
def test_streamed_proof_equals_resident_proof(resident, which):
    claim, opts, trace = _case(which)
    est = _estimates(claim, opts, len(trace))
    want, res_peak = _peak_prove(resident, claim, opts, trace)
    assert resident.last_residency == "resident"
    streamed = GpuProver(0, memory_budget=(est["streamed"] + est["resident"]) // 2)
    got, str_peak = _peak_prove(streamed, claim, opts, trace)
    assert streamed.last_residency == "streamed"
    assert got == want
    if which == "burner":
        assert str_peak <= est["streamed"], (str_peak, est)
        assert str_peak <= 0.35 * res_peak, (str_peak, res_peak)


def test_streamed_proof_verifies(orc):
    from ministark_b200.air import Air
    from oracle import stark_oracle as SO
    claim, opts, trace = _case("brainfuck")
    est = _estimates(claim, opts, len(trace))
    p = GpuProver(0, memory_budget=est["resident"] - 1)
    proof = p.prove(claim, ProofOptions(*opts), trace).to_bytes()
    assert p.last_residency == "streamed"
    SO.verify(claim, proof, 10, lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o)))
