"""CPU-only: examples/rescue, K chains of Rescue-Prime permutations over Goldilocks.

  * the parameters: alpha alpha^-1 = 1 mod p - 1, 168 round constants, an invertible MDS matrix whose 1x1 and 2x2 minors
    are all non-zero, the product's parameters equal oracle/rescue_oracle.py's and csrc/rescue_params.cuh is current;
  * the CPU build of ms_rescue_chains (tests/cpp/rescue_cpu_abi.c) through `gen_trace(..., device="cpu")` on the CPU
    harness (tests/cpu_device.py), and the host path, equal the oracle's trace word for word;
  * the oracle's trace satisfies every constraint (oracle/check_oracle.py, with R from oracle/extension_oracle.py), and
    the AIR's ce blow-up by oracle/air_oracle.py's degree rule is 8;
  * a 2^12-row proof from the stand-in's trace verifies with Stark.verify and oracle/stark_oracle.verify; a wrong digest,
    a wrong seed word and a swapped pair of digests are refused.
Harness cases run in spawned workers that install it themselves; the pytest process never does."""
import ctypes as C
import os
import subprocess
import sys
from itertools import combinations

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

P = 2**64 - 2**32 + 1
SEED = [11, 22, 33, 44]
SHAPES = [(1, 1), (4, 2), (64, 4), (1, 64)]


# --------------------------------------------------------------------------------------------------- parameters
def test_alphas():
    from oracle import rescue_oracle as RO
    assert RO.ALPHA == 7 and RO.ALPHA_INV == 10540996611094048183
    assert RO.ALPHA * RO.ALPHA_INV % (P - 1) == 1
    x = 0x1234567890abcdef
    assert pow(pow(x, RO.ALPHA, P), RO.ALPHA_INV, P) == x


def test_round_constants_and_mds():
    from oracle import rescue_oracle as RO
    assert len(RO.RC) == 2 * 12 * 7 == 168 and all(0 <= c < P for c in RO.RC)
    m = RO.MDS
    assert len(m) == 12 and all(len(r) == 12 for r in m)
    assert all(v for r in m for v in r)                                           # every 1x1 minor
    for r0, r1 in combinations(range(12), 2):                                     # every 2x2 minor
        for c0, c1 in combinations(range(12), 2):
            assert (m[r0][c0] * m[r1][c1] - m[r0][c1] * m[r1][c0]) % P, (r0, r1, c0, c1)
    inv = RO.rref([list(r) + [int(i == j) for j in range(12)] for i, r in enumerate(m)])
    assert [r[:12] for r in inv] == [[int(i == j) for j in range(12)] for i in range(12)]     # invertible


def test_product_parameters_equal_oracle():
    from ministark_b200.examples import rescue as R
    from oracle import rescue_oracle as RO
    assert (R.ALPHA, R.ALPHA_INV, R.RC, R.MDS) == (RO.ALPHA, RO.ALPHA_INV, RO.RC, RO.MDS)
    ident = [[sum(a * b for a, b in zip(row, col)) % P for col in zip(*R.MDS_INV)] for row in R.MDS]
    assert ident == [[int(i == j) for j in range(12)] for i in range(12)]
    state = list(range(12))
    assert R.permute(state) == RO.permute(state)


def test_params_header_is_current():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_rescue_params
    with open(os.path.join(ROOT, "ministark_b200", "csrc", "rescue_params.cuh")) as f:
        assert f.read() == gen_rescue_params.render(), "run tools/gen_rescue_params.py"


def test_chain_tag_is_x_at_the_chain_start():
    from ministark_b200.air import domain_generator
    for log_k, log_n in [(0, 3), (2, 6), (10, 22), (6, 12)]:
        n, K = 1 << log_n, 1 << log_k
        assert pow(domain_generator(log_n), n // K, P) == domain_generator(log_k)


def test_bad_shapes_refused():
    from ministark_b200.examples import rescue as R
    for seed, K, L in [(SEED, 3, 1), (SEED, 1, 6), (SEED, 0, 1), (SEED[:3], 1, 1), ([P] + SEED[1:], 1, 1), (SEED, 1 << 20, 1 << 10)]:
        with pytest.raises(ValueError):
            R.gen_trace(seed, K, L)


# ------------------------------------------------------------------------------------------------------ traces
def _mont_cols(rows):
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T.copy()


def test_host_trace_equals_oracle():
    from ministark_b200.examples import rescue as R
    from oracle import rescue_oracle as RO
    for K, L in [(1, 1), (4, 2)]:
        trace, digests = R.gen_trace(SEED, K, L)
        rows, want = RO.chain_trace(SEED, K, L)
        assert np.array_equal(trace.base_columns(), _mont_cols(rows))
        assert [list(d) for d in digests] == want


@pytest.fixture(scope="module")
def rescue_abi(tmp_path_factory, orc):
    """tests/cpp/rescue_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary directory"""
    out = str(tmp_path_factory.mktemp("rescue_abi") / "libms_rescue_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out, os.path.join(ROOT, "tests", "cpp", "rescue_cpu_abi.c")])
    return out


def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS, _lib._RESCUE_SIGS):
        _lib.bind(lib, sigs)
    _lib._lib = lib


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


def _worker(lib_path, fn, args, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    try:
        q.put(fn(*args))
    except Exception:                       # reported, not left for the queue's timeout
        import traceback
        q.put(traceback.format_exc())


def _stand_in_traces(shapes):
    from ministark_b200.examples import rescue as R
    out = []
    for K, L in shapes:
        trace, digests = R.gen_trace(SEED, K, L, device="cpu")
        out.append((trace.base_columns().numpy().view(np.uint64).copy(), digests))
    return out


def test_stand_in_trace_equals_oracle(rescue_abi):
    from oracle import rescue_oracle as RO
    got = _spawn(_worker, rescue_abi, _stand_in_traces, (SHAPES,))
    assert isinstance(got, list), got
    for (K, L), (cols, digests) in zip(SHAPES, got):
        rows, want = RO.chain_trace(SEED, K, L)
        assert np.array_equal(cols, _mont_cols(rows)), (K, L)
        assert [list(d) for d in digests] == want, (K, L)


def _stand_in_errors():
    from ministark_b200 import Context, MsError
    import torch
    ctx, out, msgs = Context(0), torch.empty((12, 64), dtype=torch.int64), []
    for seed, K, L in [(SEED, 3, 1), (SEED, 1, 0), ([1, 2, 3, P], 1, 1), (SEED, 1 << 20, 1 << 10)]:
        try:
            ctx.rescue_chains(seed, K, L, out)
            msgs.append(None)
        except MsError as e:
            msgs.append(str(e))
    return msgs


def test_stand_in_refuses_bad_arguments(rescue_abi):
    msgs = _spawn(_worker, rescue_abi, _stand_in_errors, ())
    assert isinstance(msgs, list), msgs
    assert "powers of two" in msgs[0] and "powers of two" in msgs[1]
    assert "not canonical" in msgs[2] and "exceed 2^32" in msgs[3]


# ------------------------------------------------------------------------------------------------------- the AIR
def test_oracle_trace_satisfies_every_constraint():
    from ministark_b200.examples import rescue as R
    from oracle import air_oracle, check_oracle, extension_oracle
    from oracle import rescue_oracle as RO
    K, L = 4, 4
    n = 8 * K * L
    rows, digests = RO.chain_trace(SEED, K, L)
    base = _mont_cols(rows)
    claim = R.RescueChainsClaim(SEED, K, L, digests)
    cfg = claim.AirConfig
    gamma = (123456789, 987654321, 55555)
    hints = cfg.gen_hints(n, claim, [gamma])
    ext = extension_oracle.builder(cfg, base, claim)([gamma])
    cons = [c.to_tuple() for c in cfg.constraints(n)]
    assert len(cons) == 40
    got = check_oracle.check(cons, n.bit_length() - 1, base, ext, 3, [gamma], hints)
    assert all(first is None for first, _ in got), [k for k, (first, _) in enumerate(got) if first is not None]
    # R's last row is the Horner evaluation gen_hints makes from the digests
    last = tuple(int(w) * pow(2**64, -1, P) % P for w in ext[0, 3 * (n - 1):])
    assert last == tuple(hints[0])
    # the reference's degree rule: ce blow-up 8 at the config 5 shape and at the test shapes
    for K, L in [(4, 4), (64, 8), (1 << 10, 1 << 9)]:
        n = 8 * K * L
        assert air_oracle.composition_constraint([c.to_tuple() for c in R.air_config(K).constraints(n)], n)[1] == 8
    # one wrong word: a round constraint and a link constraint name it
    bad = base.copy()
    bad[5, 8 * 2 + 7] ^= np.uint64(1)
    got = check_oracle.check(cons, 7, bad, ext, 3, [gamma], hints)
    failing = [k for k, (first, _) in enumerate(got) if first is not None]
    assert any(k in R.ROUND for k in failing) and any(k in R.LINK for k in failing)


OPTS = (40, 8, 8, 8, 64)


def _prove(K, L):
    from ministark_b200.air import ProofOptions
    from ministark_b200.examples import rescue as R
    from ministark_b200.prover import GpuProver
    trace, digests = R.gen_trace(SEED, K, L, device="cpu")
    claim = R.RescueChainsClaim(SEED, K, L, digests)
    got = {}
    for residency, budget in [("resident", None), ("streamed", 1)]:
        p = GpuProver(0)
        if budget:
            from ministark_b200.prover import peak_bytes
            from ministark_b200 import FQ3
            est = peak_bytes(len(trace), 8, 12, 1, FQ3, 8, 8)
            p.memory_budget = (est["streamed"] + est["resident"]) // 2
        got[residency] = (p.prove(claim, ProofOptions(*OPTS), trace).to_bytes(), p.last_residency)
    return got, digests


def test_cpu_harness_proof_verifies(rescue_abi):
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.examples import rescue as R
    from ministark_b200.verifier import VerificationError
    from oracle import stark_oracle as SO
    K, L = 64, 8                                   # 2^12 rows
    got = _spawn(_worker, rescue_abi, _prove, (K, L))
    assert isinstance(got, tuple), got
    proofs, digests = got
    assert proofs["resident"][1] == "resident" and proofs["streamed"][1] == "streamed"
    assert proofs["resident"][0] == proofs["streamed"][0]
    proof = proofs["resident"][0]
    claim = R.RescueChainsClaim(SEED, K, L, digests)
    claim.verify(proof, R.SECURITY_LEVEL)
    SO.verify(claim, proof, R.SECURITY_LEVEL, lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o)))
    wrong_digest = [list(d) for d in digests]
    wrong_digest[17][2] = (wrong_digest[17][2] + 1) % P
    swapped = list(digests)
    swapped[3], swapped[40] = swapped[40], swapped[3]
    wrong_seed = list(SEED)
    wrong_seed[1] += 1
    for bad in (R.RescueChainsClaim(SEED, K, L, wrong_digest), R.RescueChainsClaim(SEED, K, L, swapped),
                R.RescueChainsClaim(wrong_seed, K, L, digests)):
        with pytest.raises(VerificationError):
            bad.verify(proof, R.SECURITY_LEVEL)
    # the same proof claimed for another split of its 2^12 rows into chains is refused too
    with pytest.raises(VerificationError):
        R.RescueChainsClaim(SEED, K // 2, 2 * L, digests[:K // 2]).verify(proof, R.SECURITY_LEVEL)


def test_header_bound_and_exported(rescue_abi):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.RESCUE_HEADER_PATH)
    assert declared == sorted(_lib._RESCUE_SIGS) == ["ms_rescue_chains"]
    assert not set(declared) & set(_lib.header_symbols())
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(rescue_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)
