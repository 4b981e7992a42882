"""GPU: proofs made on the device, in every residency, are accepted by the product's verifier (`Stark.verify`).

  * fib, the Fq3 permutation AIR and brainfuck hello_world (its trace built on the device), resident: the bytes equal
    oracle/stark_oracle.cpu_prove's and verify;
  * brainfuck cycle_burner(40, 40, 60) (2^20 rows, trace built on the device) resident, streamed (device budget between
    the two estimates) and streamed_host (node heaps in pinned host memory): the recorded proof, accepted;
  * one changed composition row of a device proof is CompositionTraceQueryDoesNotMatchCommitment."""
import hashlib

import pytest
import torch

from ministark_b200 import FQ3
from ministark_b200.air import Air, ProofOptions
from ministark_b200.examples import brainfuck as bf
from ministark_b200.examples import fib, perm
from ministark_b200.proof import Proof
from ministark_b200.prover import GpuProver, peak_bytes
from ministark_b200.verifier import VerificationError

pytestmark = pytest.mark.gpu
BF_OPTS = (19, 16, 20, 16, 16)
PROOF_SHA256_2P20 = "cbf317503bf28883d7a008838857a4b905063d8eb2e0bf03a5cd499aab87c4a1"    # cycle_burner(40, 40, 60)


def _small(which):
    """(claim, options, trace for the prover, base columns on the host, extension builder on the host)"""
    if which == "fib":
        trace, last = fib.gen_trace(8 << 13)
        return fib.FibClaim(last), (32, 4, 8, 8, 64), trace, trace.base_columns(), None
    if which == "perm":
        trace = perm.gen_trace(1 << 10, seed=5)
        return perm.PermClaim(), (16, 8, 4, 4, 8), trace, trace.base_columns(), trace.build_extension_columns
    host, out = bf.simulate(bf.HELLO_WORLD)
    dev, _ = bf.simulate(bf.HELLO_WORLD, device=0)
    return bf.BrainfuckClaim(bf.HELLO_WORLD, b"", out), BF_OPTS, dev, host.base_columns(), host.build_extension_columns


@pytest.mark.parametrize("which", ["fib", "perm", "brainfuck"])
def test_resident_proofs_equal_cpu_prove_and_verify(orc, which):
    from oracle import stark_oracle as SO
    claim, opts, trace, base, ext = _small(which)
    proof = GpuProver.shared(0).prove(claim, ProofOptions(*opts), trace)
    assert GpuProver.shared(0).last_residency == "resident"
    mk = lambda n, o: Air(claim.AirConfig, n, claim.get_public_inputs(), ProofOptions(*o))
    data = proof.to_bytes()
    assert data == SO.cpu_prove(claim, opts, base, mk, ext_builder=ext)
    bits = proof.security_level_bits()
    art = claim.verify(data, bits)
    assert art.query_positions == SO.verify(claim, data, bits, mk)["query_positions"]
    assert claim.verify(proof, bits).query_positions == art.query_positions


@pytest.fixture(scope="module")
def burner():
    src = bf.cycle_burner(40, 40, 60)
    _, output = bf.simulate(src, device=0)
    claim = bf.BrainfuckClaim(src, b"", output)
    n = 1 << 20
    est = peak_bytes(n, 16, 17, 9, FQ3, Air(claim.AirConfig, n, None, ProofOptions(*BF_OPTS)).ce_blowup_factor, 16)
    return src, claim, est


@pytest.mark.parametrize("residency", ["resident", "streamed", "streamed_host"])
def test_2p20_brainfuck_proofs_verify_in_every_residency(burner, residency):
    src, claim, est = burner
    if residency == "resident":
        p = GpuProver(0)
    elif residency == "streamed":
        p = GpuProver(0, memory_budget=(est["streamed"] + est["resident"]) // 2)
    else:
        p = GpuProver(0, memory_budget=(est["streamed_host"] + est["streamed"]) // 2, host_memory_budget=est["host"])
    trace, _ = bf.simulate(src, device=0)
    proof = p.prove(claim, ProofOptions(*BF_OPTS), trace)
    p.release_host_memory()
    assert p.last_residency == residency
    data = proof.to_bytes()
    assert hashlib.sha256(data).hexdigest() == PROOF_SHA256_2P20
    art = claim.verify(data, bf.SECURITY_LEVEL)
    assert 0 < len(art.query_positions) <= BF_OPTS[0] and len(art.fri_alphas) == len(proof.fri_proof.layers)
    if residency == "resident":
        bad = Proof.from_bytes(data, False)
        values = bad.trace_queries.composition_trace_values
        values[5] = ((values[5][0] + 1) % fib.P,) + values[5][1:]
        with pytest.raises(VerificationError) as e:
            claim.verify(bad, bf.SECURITY_LEVEL)
        assert e.value.kind == "CompositionTraceQueryDoesNotMatchCommitment"
    del p, proof, trace
    torch.cuda.empty_cache()
