"""GPU: the full prover (ministark_b200/prover.py = default_prove, src/prover.rs:25-174) against the CPU restatement.

For every case the proof produced on the GPU must be BYTE-IDENTICAL to the one the reference-formulation CPU prover
(oracle/stark_oracle.cpu_prove: coefficient-form DEEP, apply_drp through two transforms, CPU Merkle) emits for the
same trace, and the restated `default_verify` must accept it.  Covers examples/fib (Fq = Fp, ce_blowup 1) and the
permutation AIR (Fq = Fq3 extension columns, challenge, ce_blowup 4)."""
import numpy as np
import pytest

import ministark_b200 as ms
from ministark_b200.air import Air, ProofOptions
from ministark_b200.examples import fib, perm
from ministark_b200.prover import GpuProver

pytestmark = pytest.mark.gpu


def air_factory(stark):
    return lambda n, o: Air(stark.AirConfig, n, stark.get_public_inputs(), ProofOptions(*o))


@pytest.fixture(scope="module")
def prover():
    return GpuProver(0)


@pytest.mark.parametrize("log_rows,opts", [(7, (32, 4, 8, 8, 64)), (10, (20, 8, 5, 4, 16)), (6, (10, 2, 0, 2, 8)),
                                           (13, (32, 4, 10, 8, 64)), (11, (24, 16, 6, 16, 8))])
def test_fib_proof_bytes_match_cpu_prover(prover, orc, log_rows, opts):
    from oracle import stark_oracle as SO
    trace, last = fib.gen_trace(8 << log_rows)
    claim = fib.FibClaim(last)
    proof = prover.prove(claim, ProofOptions(*opts), trace)
    got = proof.to_bytes()
    want = SO.cpu_prove(claim, opts, trace.base_columns(), air_factory(claim))
    assert got == want
    SO.verify(claim, got, 10, air_factory(claim))
    assert proof.pow_nonce >= (1 if opts[2] else 0)
    assert set(proof.timings) >= {"base_trace_commitment", "constraint_eval", "fri", "total"}


@pytest.mark.parametrize("log_n,opts", [(6, (12, 8, 4, 4, 8)), (9, (20, 16, 6, 16, 4)), (10, (16, 8, 0, 8, 16))])
def test_perm_fq3_proof_bytes_match_cpu_prover(prover, orc, log_n, opts):
    from oracle import stark_oracle as SO
    claim = perm.PermClaim()
    tr = perm.gen_trace(1 << log_n, seed=log_n)
    proof = prover.prove(claim, ProofOptions(*opts), tr)
    got = proof.to_bytes()
    want = SO.cpu_prove(claim, opts, tr.base_columns(), air_factory(claim), ext_builder=tr.build_extension_columns)
    assert got == want
    SO.verify(claim, got, 10, air_factory(claim))


def test_fib_native_size_verifies_and_trace_on_device(prover, orc):
    """examples/fib at 2^18 rows with the reference's OPTIONS, trace handed over as a resident device tensor;
    too large for the CPU prover in a unit test, so soundness is checked by the restated verifier."""
    torch = pytest.importorskip("torch")
    from oracle import stark_oracle as SO
    from ministark_b200.prover import Trace
    trace, last = fib.gen_trace(8 << 18)
    dev = torch.from_numpy(trace.base_columns().view(np.int64)).cuda()
    claim = fib.FibClaim(last)
    proof = prover.prove(claim, fib.OPTIONS, Trace(dev))
    art = SO.verify(claim, proof.to_bytes(), fib.SECURITY_LEVEL, air_factory(claim))
    assert len(proof.fri_proof.layers) == fib.OPTIONS.fri_num_layers(4 << 18) == len(art["fri_alphas"])
    assert len(proof.fri_proof.remainder_coeffs) == fib.OPTIONS.fri_remainder_size(4 << 18) // 4
    bad = fib.FibClaim((last + 1) % fib.P)
    with pytest.raises(SO.VerificationError):
        SO.verify(bad, proof.to_bytes(), fib.SECURITY_LEVEL, air_factory(bad))


EVERY_SMALL_SET = "every index set of 1, 2 or 3 leaves"


@pytest.mark.parametrize("n,ids", [(8, [3]), (4, [0, 1, 2, 3]), (1 << 10, [378]), (64, [5, 4, 63, 17, 16, 5]), (2, [1]),
                                   (1 << 16, list(range(0, 1 << 16, 2049))),
                                   pytest.param(16, EVERY_SMALL_SET, id="16-every-set-of-1-2-3"),       # 696 sets, one tree
                                   (16, [11, 4, 15, 0, 7, 4, 2, 13, 9, 1, 14, 6, 0, 10, 3, 12, 8, 5, 15, 11]),
                                   (1 << 20, [int(i) for i in np.random.default_rng(64).integers(0, 1 << 20, size=64)]),
                                   (1 << 20, [0, (1 << 20) - 1, (1 << 19) - 1, 1 << 19])])
def test_merkle_prove_resident_tree(orc, n, ids):
    # MerkleTreeImpl::prove (src/merkle.rs:149-207; tests :528-581) from the device-resident leaf / node arrays
    import itertools
    torch = pytest.importorskip("torch")
    from oracle import stark_oracle as SO
    ctx = ms.Context(0)
    rng = np.random.default_rng(n)
    leaves = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    nodes = orc.merkle_nodes(leaves)
    if n == 2:
        nodes[0] = 0          # nodes[0] is the unused default digest (src/merkle.rs:441)
    d_leaves, d_nodes = torch.from_numpy(leaves).cuda(), torch.from_numpy(nodes).cuda()
    sets = [ids] if ids is not EVERY_SMALL_SET else [list(s) for k in (1, 2, 3) for s in itertools.combinations(range(n), k)]
    for ids in sets:
        path, init, sib, height = ctx.merkle_prove(d_leaves, d_nodes, n, ids)
        want = SO._merkle_prove(leaves, nodes, ids)
        assert (path, init, sib, height) == (want["nodes"], want["initial_leaves"], want["sibling_leaves"], want["height"]), ids
        SO.merkle_verify(nodes[1].tobytes(), dict(nodes=path, initial_leaves=init, sibling_leaves=sib, height=height), ids)
        # host-resident arrays go through the same kernel (staged)
        assert ctx.merkle_prove(leaves, nodes, n, ids)[0] == path
    with pytest.raises(ms.MsError):
        ctx.merkle_prove(d_leaves, d_nodes, n, [n])      # LeafIndexOutOfBounds


def test_gather_rows_rowmajor():
    torch = pytest.importorskip("torch")
    ctx = ms.Context(0)
    rng = np.random.default_rng(9)
    rows = rng.integers(0, 2**63, size=(4096, 24), dtype=np.uint64)
    ids = [0, 4095, 17, 17, 1000]
    assert np.array_equal(ctx.gather_rows_rowmajor(torch.from_numpy(rows.view(np.int64)).cuda(), 24, 4096, ids), rows[ids])
    assert np.array_equal(ctx.gather_rows_rowmajor(rows, 24, 4096, ids), rows[ids])
    with pytest.raises(ms.MsError):
        ctx.gather_rows_rowmajor(rows, 24, 4096, [4096])


def test_brainfuck_hello_world_proof_bytes_match_cpu_prover(prover, orc):
    """BASELINE config 2: brainfuck hello_world.bf, full prove -> verify, proof bytes identical to the CPU path"""
    from oracle import stark_oracle as SO
    from ministark_b200.examples import brainfuck as bf
    trace, out = bf.simulate(bf.HELLO_WORLD)
    claim = bf.BrainfuckClaim(bf.HELLO_WORLD, b"", out)
    mk = lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o))
    proof = prover.prove(claim, bf.OPTIONS, trace)
    got = proof.to_bytes()
    want = SO.cpu_prove(claim, (19, 16, 20, 16, 16), trace.base_columns(), mk, ext_builder=trace.build_extension_columns)
    assert got == want
    SO.verify(claim, got, bf.SECURITY_LEVEL, mk)
    assert proof.pow_nonce > 0 and len(proof.fri_proof.layers) == 2


def test_brainfuck_extension_columns_on_device_match_host_loops(orc):
    """§8(f) rank 3: the nine Fq3 running-product / running-evaluation columns from ms_eval_constraints + ms_scan_affine
    equal the sequential host construction (examples/brainfuck/trace.rs:108-279) word for word"""
    torch = pytest.importorskip("torch")
    from ministark_b200.examples import brainfuck as bf
    ctx = ms.Context(0)
    for src, inp in ((bf.HELLO_WORLD, b""), (",>,<.>.+[-].", b"hi")):
        trace, out = bf.simulate(src, inp)
        ch = [tuple(int(x) for x in np.random.default_rng(k).integers(1, ms.P, size=3, dtype=np.uint64)) for k in range(11)]
        want = trace.build_extension_columns(ch)
        base = torch.from_numpy(trace.base_columns().view(np.int64)).cuda()
        got = trace.build_extension_columns_device(ch, ctx, base)
        ctx.sync()
        assert np.array_equal(got.cpu().numpy().view(np.uint64), want)


def test_brainfuck_cycle_burner_proof_bytes_match_cpu_prover(prover, orc):
    """a loop-heavy program (1024 rows): exercises LoopBegin / LoopEnd jumps, dummy memory rows and the device-built
    extension columns inside the full prover"""
    from oracle import stark_oracle as SO
    from ministark_b200.examples import brainfuck as bf
    src = bf.cycle_burner(4, 4, 4)
    trace, out = bf.simulate(src)
    assert len(trace) == 1024
    claim = bf.BrainfuckClaim(src, b"", out)
    mk = lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o))
    opts = (16, 16, 6, 8, 8)
    got = prover.prove(claim, ProofOptions(*opts), trace).to_bytes()
    want = SO.cpu_prove(claim, opts, trace.base_columns(), mk, ext_builder=trace.build_extension_columns)
    assert got == want
    SO.verify(claim, got, 60, mk)


def test_stark_prove_entry_point(orc):
    """`claim.prove(OPTIONS, trace)` as in examples/fib/main.rs:234-240, through the shared per-device prover"""
    from oracle import stark_oracle as SO
    trace, last = fib.gen_trace(8 << 9)
    claim = fib.FibClaim(last)
    opts = ProofOptions(12, 4, 4, 8, 16)
    p1 = claim.prove(opts, trace)
    p2 = claim.prove(opts, trace)
    assert p1.to_bytes() == p2.to_bytes()                      # deterministic: smallest-nonce PoW
    assert GpuProver.shared(0) is GpuProver.shared(0)
    SO.verify(claim, p1.to_bytes(), 20, air_factory(claim))
