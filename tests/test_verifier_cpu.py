"""CPU-only: the product's verifier (ministark_b200/verifier.py, `Stark.verify`) and proof reader (`Proof.from_bytes`).

  * acceptance: proofs of oracle/stark_oracle.cpu_prove (fib 2^7 and 2^13 rows, the Fq3 permutation AIR, brainfuck
    hello_world) and of the product's `GpuProver` on the CPU harness (tests/cpu_device.py), resident and streamed, are
    accepted with the artifacts (challenges, hints, FRI alphas, query positions) of the restated verifier;
  * round trip: from_bytes(b).to_bytes() == b, and malformed bytes raise ProofFormatError naming the field;
  * rejection parity: a fixed list of single-field mutations per proof, refused (or accepted) by both verifiers, with the
    reference's variant as `kind`; for brainfuck the C++ verifier (include/ministark_verifier.hpp) gives the same verdicts;
  * the FRI layer and remainder checks, which every proof mutation stops short of, on the verifier's own inputs with
    one evaluation, alpha or remainder coefficient changed;
  * security bits: the reference's formula, and one bit too many is InvalidProofSecurity."""
import copy
import os
import subprocess
import sys

import pytest

from ministark_b200.air import Air, ProofOptions
from ministark_b200.examples import brainfuck as bf
from ministark_b200.examples import fib, perm
from ministark_b200.proof import Proof, ProofFormatError
from ministark_b200.verifier import VerificationError
from oracle import stark_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = fib.P
BITS = 10                      # below every case's security level, so mutated options still reach the later checks


def _case(which):
    """(claim, options, trace)"""
    if which.startswith("fib"):
        log_rows = int(which.split(":")[1])
        trace, last = fib.gen_trace(8 << log_rows)
        return fib.FibClaim(last), ((32, 4, 8, 8, 64) if log_rows == 7 else (16, 4, 0, 8, 16)), trace
    if which == "perm":
        return perm.PermClaim(), (16, 8, 4, 4, 8), perm.gen_trace(1 << 8, seed=3)
    trace, output = bf.simulate(bf.HELLO_WORLD)
    return bf.BrainfuckClaim(bf.HELLO_WORLD, b"", output), (19, 16, 20, 16, 16), trace


def _make_air(claim):
    return lambda n, o: Air(claim.AirConfig, n, claim.get_public_inputs(), ProofOptions(*o))


def _oracle_verify(claim, data, bits=BITS):
    """the restated verifier's verdict: its artifacts, or None for any refusal"""
    try:
        return SO.verify(claim, data, bits, _make_air(claim))
    except Exception:
        return None


CASES = ["fib:7", "fib:13", "perm", "brainfuck"]


@pytest.fixture(scope="module")
def cpu_proofs(orc):
    out = {}
    for which in CASES:
        claim, opts, trace = _case(which)
        ext = trace.build_extension_columns if claim.AirConfig.NUM_EXTENSION_COLUMNS else None
        out[which] = SO.cpu_prove(claim, opts, trace.base_columns(), _make_air(claim), ext_builder=ext)
    return out


def _prover_worker(lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ctypes as C
    import cpu_device
    cpu_device.install()
    from ministark_b200 import FP, FQ3, _lib
    from ministark_b200.prover import GpuProver, peak_bytes
    lib = C.CDLL(lib_path)                  # the CPU ABI with the streamed-residency entry points
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    _lib.bind(lib, _lib._STREAM_SIGS)
    _lib._lib = lib
    out = {}
    for which in ("fib:7", "perm", "brainfuck"):
        claim, opts, trace = _case(which)
        cfg, o = claim.AirConfig, ProofOptions(*opts)
        n = len(trace)
        est = peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, FP if cfg.FQ_IS_FP else FQ3,
                         Air(cfg, n, None, o).ce_blowup_factor, o.fri_folding_factor)
        for residency, budget in (("resident", None), ("streamed", (est["streamed"] + est["resident"]) // 2)):
            p = GpuProver(0)
            p.memory_budget = budget
            proof = p.prove(claim, o, trace)
            out[which, residency] = (p.last_residency, proof.to_bytes())
    q.put(out)


@pytest.fixture(scope="module")
def harness_proofs(orc, tmp_path_factory):
    import torch.multiprocessing as mp
    lib = str(tmp_path_factory.mktemp("verifier_abi") / "libms_stream_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", lib, os.path.join(ROOT, "tests", "cpp", "stream_cpu_abi.c")])
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_prover_worker, args=(lib, q))
    p.start()
    got = q.get(timeout=900)
    p.join(timeout=60)
    assert p.exitcode == 0
    return got


def _same_artifacts(art, want):
    assert [SO.q(c) for c in art.air_challenges] == want["air_challenges"]
    assert art.air_hints == want["air_hints"]
    assert [SO.q(a) for a in art.fri_alphas] == want["fri_alphas"]
    assert art.query_positions == want["query_positions"]


@pytest.mark.parametrize("which", CASES)
def test_cpu_prover_proofs_are_accepted_with_the_oracle_artifacts(cpu_proofs, which):
    claim, _, _ = _case(which)
    data = cpu_proofs[which]
    art = claim.verify(data, BITS)
    _same_artifacts(art, SO.verify(claim, data, BITS, _make_air(claim)))
    _same_artifacts(claim.verify(Proof.from_bytes(data, claim.AirConfig.FQ_IS_FP), BITS), SO.verify(claim, data, BITS,
                                                                                                       _make_air(claim)))


@pytest.mark.parametrize("which", ["fib:7", "perm", "brainfuck"])
def test_gpu_prover_proofs_on_the_cpu_harness_are_accepted(cpu_proofs, harness_proofs, which):
    claim, _, _ = _case(which)
    want = SO.verify(claim, cpu_proofs[which], BITS, _make_air(claim))
    for residency in ("resident", "streamed"):
        ran, data = harness_proofs[which, residency]
        assert ran == residency and data == cpu_proofs[which]
        _same_artifacts(claim.verify(data, BITS), want)


@pytest.mark.parametrize("which", CASES)
def test_round_trip_and_malformed_bytes(cpu_proofs, which):
    claim, _, _ = _case(which)
    fq_is_fp = claim.AirConfig.FQ_IS_FP
    data = cpu_proofs[which]
    proof = Proof.from_bytes(data, fq_is_fp)
    assert proof.to_bytes() == data
    assert isinstance(proof.trace_queries.base_trace_values[0], int)
    assert isinstance(proof.composition_trace_ood_evals[0], int if fq_is_fp else tuple)
    # every prefix is truncated: a ProofFormatError, never an IndexError
    for k in list(range(0, 200)) + list(range(200, len(data), 61)) + [len(data) - 1]:
        with pytest.raises(ProofFormatError, match="truncated"):
            Proof.from_bytes(data[:k], fq_is_fp)
    with pytest.raises(ProofFormatError, match="trailing bytes"):
        Proof.from_bytes(data + b"\x00", fq_is_fp)
    bad = bytearray(data)
    bad[13] = 31                                                  # the length of the base trace commitment
    with pytest.raises(ProofFormatError, match="base_trace_commitment: digest length 31"):
        Proof.from_bytes(bytes(bad), fq_is_fp)
    bad = bytearray(data)
    bad[5 + 8 + 40] = 2                                           # the Option tag of the extension trace commitment
    with pytest.raises(ProofFormatError, match="extension_trace_commitment: Option tag 2"):
        Proof.from_bytes(bytes(bad), fq_is_fp)
    bad = bytearray(data)
    bad[3] = 3                                                    # fri_folding_factor
    with pytest.raises(ProofFormatError, match="options.fri_folding_factor"):
        Proof.from_bytes(bytes(bad), fq_is_fp)
    for field, set_p in [("base_trace_values", lambda p: p.trace_queries.base_trace_values.__setitem__(0, P)),
                         ("composition_trace_ood_evals", lambda p: p.composition_trace_ood_evals.__setitem__(
                             0, P if fq_is_fp else (1, P, 0))),
                         ("remainder_coeffs", lambda p: p.fri_proof.remainder_coeffs.__setitem__(
                             0, P + 5 if fq_is_fp else (0, 0, P)))]:
        p = copy.deepcopy(proof)
        set_p(p)
        with pytest.raises(ProofFormatError, match=f"{field}.*not a canonical field element"):
            Proof.from_bytes(p.to_bytes(), fq_is_fp)


def _mutations(which, proof):
    """(name, claim, mutated Proof, the kind the product must raise — or a tuple of kinds that depend on a hash — or None
    for acceptance)"""
    claim, _, _ = _case(which)
    grind = proof.options.grinding_factor
    # a changed FRI commitment or remainder reseeds the coin: the proof of work fails (the old nonce still passes with
    # probability 2^-grinding), or the query positions move and the base trace rows no longer open
    reseeded = ("FriProofOfWork", "BaseTraceQueryDoesNotMatchCommitment") if grind else "BaseTraceQueryDoesNotMatchCommitment"
    flip = lambda d: bytes([d[0] ^ 1]) + d[1:]
    bump = lambda v: (v + 1) % P if isinstance(v, int) else ((v[0] + 1) % P,) + tuple(v[1:])
    out = []

    def mutate(name, kind, f, who=claim):
        p = copy.deepcopy(proof)
        f(p)
        out.append((name, who, p, kind))

    q = lambda p: p.trace_queries
    mutate("base_trace_commitment", "InconsistentOodConstraintEvaluations",
           lambda p: setattr(p, "base_trace_commitment", flip(p.base_trace_commitment)))
    if proof.extension_trace_commitment is not None:
        mutate("extension_trace_commitment", "InconsistentOodConstraintEvaluations",
               lambda p: setattr(p, "extension_trace_commitment", flip(p.extension_trace_commitment)))
    mutate("composition_trace_commitment", "InconsistentOodConstraintEvaluations",
           lambda p: setattr(p, "composition_trace_commitment", flip(p.composition_trace_commitment)))
    mutate("execution_trace_ood_eval", "InconsistentOodConstraintEvaluations",
           lambda p: p.execution_trace_ood_evals.__setitem__(3, bump(p.execution_trace_ood_evals[3])))
    mutate("composition_trace_ood_eval", "InconsistentOodConstraintEvaluations",
           lambda p: p.composition_trace_ood_evals.__setitem__(0, bump(p.composition_trace_ood_evals[0])))
    mutate("base_trace_value", "BaseTraceQueryDoesNotMatchCommitment",
           lambda p: q(p).base_trace_values.__setitem__(1, bump(q(p).base_trace_values[1])))
    if q(proof).extension_trace_values:
        mutate("extension_trace_value", "ExtensionTraceQueryDoesNotMatchCommitment",
               lambda p: q(p).extension_trace_values.__setitem__(-1, bump(q(p).extension_trace_values[-1])))
    mutate("composition_trace_value", "CompositionTraceQueryDoesNotMatchCommitment",
           lambda p: q(p).composition_trace_values.__setitem__(2, bump(q(p).composition_trace_values[2])))
    for tree, kind in (("base_trace_proof", "BaseTraceQueryDoesNotMatchCommitment"),
                       ("extension_trace_proof", "ExtensionTraceQueryDoesNotMatchCommitment"),
                       ("composition_trace_proof", "CompositionTraceQueryDoesNotMatchCommitment")):
        if getattr(q(proof), tree) is not None:
            def sib(p, tree=tree):
                view = getattr(q(p), tree)
                digests = view.nodes if view.nodes else view.sibling_leaves
                digests[0] = flip(digests[0])
            mutate(tree + ".sibling", kind, sib)
    mutate("fri_layer_value", "LayerCommitmentInvalid",
           lambda p: p.fri_proof.layers[0].flattenend_rows.__setitem__(0, bump(p.fri_proof.layers[0].flattenend_rows[0])))
    mutate("fri_layer_commitment", reseeded,
           lambda p: setattr(p.fri_proof.layers[-1], "commitment", flip(p.fri_proof.layers[-1].commitment)))
    mutate("remainder_coeff", reseeded,
           lambda p: p.fri_proof.remainder_coeffs.__setitem__(0, bump(p.fri_proof.remainder_coeffs[0])))
    # the nonce is only read when the options ask for grinding; another nonce changes the query positions if it passes
    mutate("pow_nonce", reseeded if grind else None, lambda p: setattr(p, "pow_nonce", p.pow_nonce + 1))
    mutate("trace_len", "InconsistentOodConstraintEvaluations", lambda p: setattr(p, "trace_len", 2 * p.trace_len))
    mutate("trace_len_not_power_of_two", "InvalidTraceLength", lambda p: setattr(p, "trace_len", p.trace_len + 1))
    o = proof.options
    for name, new in (("num_queries", dict(num_queries=o.num_queries - 1)),
                      ("lde_blowup_factor", dict(lde_blowup_factor=2 * o.lde_blowup_factor)),
                      ("grinding_factor", dict(grinding_factor=o.grinding_factor + 1)),
                      ("fri_folding_factor", dict(fri_folding_factor=o.fri_folding_factor // 2)),
                      ("fri_max_remainder_coeffs", dict(fri_max_remainder_coeffs=o.fri_max_remainder_coeffs + 1))):
        mutate("options." + name, "InconsistentOodConstraintEvaluations",
               lambda p, new=new: setattr(p, "options", ProofOptions(**{**p.options.__dict__, **new})))
    # copies of the last FRI layer until a layer that is not the last one has a codeword shorter than the folding factor
    surplus, cw = 0, proof.trace_len * o.lde_blowup_factor
    while cw % o.fri_folding_factor == 0:
        cw //= o.fri_folding_factor
        surplus += 1
    mutate("fri_layers_surplus", "CodewordTruncation",
           lambda p: p.fri_proof.layers.extend(copy.deepcopy(p.fri_proof.layers[-1]) for _ in range(surplus + 2 - len(p.fri_proof.layers))))
    if which == "brainfuck":
        # 128 bits of security, but a trace shorter than the output: the AIR's hints refuse it instead of raising the
        # challenge to a negative power
        mutate("trace_len_shorter_than_output", "InvalidAir",
               lambda p: (setattr(p, "trace_len", 8), setattr(p, "options", ProofOptions(**{**p.options.__dict__,
                                                                                            "lde_blowup_factor": 128}))))
    if which.startswith("fib"):
        out.append(("public_inputs", fib.FibClaim((claim.claimed_value + 1) % P), proof, "InconsistentOodConstraintEvaluations"))
    elif which == "brainfuck":
        out.append(("public_inputs", bf.BrainfuckClaim(bf.HELLO_WORLD, b"", b"Hello World?"), proof,
                    "InconsistentOodConstraintEvaluations"))
    return out


def _product_kind(claim, data):
    try:
        claim.verify(data, BITS)
        return None
    except VerificationError as e:
        return e.kind
    except ProofFormatError:
        return "ProofFormatError"


@pytest.mark.parametrize("which", CASES)
def test_rejection_parity_with_the_oracle(cpu_proofs, which):
    claim, _, _ = _case(which)
    proof = Proof.from_bytes(cpu_proofs[which], claim.AirConfig.FQ_IS_FP)
    muts = _mutations(which, proof)
    assert len(muts) >= 17
    for name, who, p, kind in muts:
        data = p.to_bytes()
        got = _product_kind(who, data)
        assert got in kind if isinstance(kind, tuple) else got == kind, (name, got, kind)
        assert (got is None) == (_oracle_verify(who, data) is not None), name


def test_security_bits(cpu_proofs):
    for which in CASES:
        claim, opts, _ = _case(which)
        lanes = 1 if claim.AirConfig.FQ_IS_FP else 3
        proof = Proof.from_bytes(cpu_proofs[which], claim.AirConfig.FQ_IS_FP)
        bits = proof.security_level_bits()
        assert bits == proof.security_level_bits(claim.AirConfig.FQ_IS_FP) == SO.security_level_bits(opts, proof.trace_len, lanes)
        claim.verify(proof, bits)
        with pytest.raises(VerificationError) as e:
            claim.verify(proof, bits + 1)
        assert e.value.kind == "InvalidProofSecurity"
    assert Proof.from_bytes(cpu_proofs["brainfuck"], False).security_level_bits() == bf.SECURITY_LEVEL


def test_brainfuck_verdicts_equal_the_cpp_verifier(cpu_proofs, tmp_path):
    exe = str(tmp_path / "host_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "host_test.cpp"), "-o", exe])
    claim, _, _ = _case("brainfuck")
    proof = Proof.from_bytes(cpu_proofs["brainfuck"], False)
    cases = [("unchanged", claim, proof, None)] + _mutations("brainfuck", proof)
    for name, who, p, _ in cases:
        data = p.to_bytes()
        cpp = subprocess.run([exe, "verify", "bf", who.source_code,
                              who.output.hex(), str(BITS)], input=data.hex(), capture_output=True, text=True, check=True)
        assert cpp.stdout.startswith(("ok", "error:")), (name, cpp.stdout)
        assert cpp.stdout.startswith("ok") == (_product_kind(who, data) is None), (name, cpp.stdout)


def _fri_inputs(claim, data, monkeypatch):
    """the arguments verify() hands to the FRI check of an accepted proof"""
    from ministark_b200 import verifier
    seen = []
    real = verifier._verify_fri
    monkeypatch.setattr(verifier, "_verify_fri", lambda *a: (seen.append(a), real(*a))[1])
    claim.verify(data, BITS)
    monkeypatch.undo()
    return real, seen[0]


@pytest.mark.parametrize("which", CASES)
def test_fri_checks_after_the_commitments(cpu_proofs, which, monkeypatch):
    """the FRI checks that no proof mutation reaches (each one reseeds the coin or breaks a Merkle opening first), run
    on the verifier's own inputs with one value changed: the DEEP evaluations against the first layer, each folding
    step against the next layer or the remainder, and the remainder's degree and values"""
    claim, _, _ = _case(which)
    fri_check, (fri_proof, options, alphas, positions, evals, size, gen) = _fri_inputs(claim, cpu_proofs[which], monkeypatch)
    bump = lambda v: ((v[0] + 1) % P,) + tuple(v[1:])

    def kind(fp=fri_proof, al=alphas, ev=evals):
        try:
            fri_check(fp, options, al, positions, ev, size, gen)
            return None
        except VerificationError as e:
            return e.kind, e.layer, e.degree

    assert kind() is None
    assert kind(ev=[bump(evals[0])] + evals[1:]) == ("InvalidDegreeRespectingProjection", 0, None)
    assert kind(ev=evals[:-1]) == ("NumPositionEvaluationMismatch", None, None)
    layers = len(fri_proof.layers)
    for i in range(layers):
        al = list(alphas)
        al[i] = bump(al[i])
        want = ("InvalidDegreeRespectingProjection", i + 1, None) if i + 1 < layers else ("RemainderCommitmentInvalid", None, None)
        assert kind(al=al) == want, i
    rem = fri_proof.remainder_coeffs
    zero, one = (0, 1) if isinstance(rem[0], int) else ((0, 0, 0), (1, 0, 0))
    with_rem = lambda coeffs: type(fri_proof)(fri_proof.layers, coeffs)
    rem0 = (rem[0] + 1) % P if isinstance(rem[0], int) else bump(rem[0])
    assert kind(fp=with_rem([rem0] + rem[1:])) == ("RemainderCommitmentInvalid", None, None)
    assert kind(fp=with_rem(rem + [zero])) is None                 # a trailing zero coefficient leaves the degree
    deg = len(rem) - 1
    assert kind(fp=with_rem(rem + [one])) == ("RemainderDegreeMismatch", None, deg)
    assert kind(fp=with_rem([])) == ("RemainderCommitmentInvalid", None, None)
