"""CPU-only: examples/rescue's hash claim, K messages absorbed by the Rescue-Prime sponge over Goldilocks.

  * rescue.hash equals the restated sponge (tests/rescue_hash_oracle.py) over message lengths around the rate;
  * the host trace and the CPU build of ms_rescue_hash (tests/cpp/rescue_hash_cpu_abi.c, through
    `gen_hash_trace(..., device="cpu")` on the CPU harness, tests/cpu_device.py) equal the restated trace word for word,
    and bad arguments are refused before anything is written;
  * the restated trace satisfies every constraint (oracle/check_oracle.py, with R from oracle/extension_oracle.py), at
    L = 1 too; the constraint count is 48 - t (36 - t at L = 1) and the ce blow-up is 8; a flipped message word breaks
    a LINK or START constraint, a flipped padding word the PAD constraint of its position;
  * 2^12-row proofs verify with Stark.verify and oracle/stark_oracle.verify, resident and streamed give the same bytes,
    and a changed digest, swapped digests and other message lengths are refused.
Harness cases run in spawned workers that install it themselves; the pytest process never does."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rescue_hash_oracle as HO  # noqa: E402

P = 2**64 - 2**32 + 1
# (K, length): one message of zero words; L = 1 (B = 1); B = L = 2; B = 3 < L = 4; B = L = 8
SHAPES = [(1, 0), (4, 7), (2, 8), (4, 20), (2, 63)]


def messages(K, length, salt=0):
    """K messages of `length` canonical words, some near p"""
    return [[(0x9E3779B97F4A7C15 * (1 + salt + k * length + i) + (P - 1 if i % 5 == 3 else 0)) % P
             for i in range(length)] for k in range(K)]


def _mont_cols(rows):
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T.copy()


# ------------------------------------------------------------------------------------------------------- the hash
def test_hash_equals_sponge():
    from ministark_b200.examples import rescue as R
    for length in (0, 1, 7, 8, 9, 20, 60, 63):
        words = messages(1, length, salt=length)[0]
        assert list(R.hash(words)) == HO.sponge_hash(words), length
    assert R.hash([]) == tuple(R.permute([1] + [0] * 11)[:4])
    a = 123456789
    assert R.hash([a]) != R.hash([a, 0])
    for bad in ([P], [1, -1], [2**64]):
        with pytest.raises(ValueError):
            R.hash(bad)


def test_bad_shapes_refused():
    from ministark_b200.examples import rescue as R
    for msgs in ([[1]] * 3, [[1, 2], [3]], [[P]], [[-1]], [], np.zeros((2, 3), dtype=np.int64),
                 np.array([[P]], dtype=np.uint64), np.zeros((1 << 30, 0), dtype=np.uint64)):
        with pytest.raises(ValueError):
            R.gen_hash_trace(msgs)
    with pytest.raises(ValueError):
        R.RescueHashClaim(4, [(1, 2, 3, 4)] * 3)                       # K = 3
    with pytest.raises(ValueError):
        R.RescueHashClaim(4, [(1, 2, 3, P)])                            # not canonical
    with pytest.raises(ValueError):
        R.hash_air_config(4, 20).constraints(8 * 4 * 2)                 # 20 words take L = 4, not 2
    assert R.hash_air_config(4, 20) is R.hash_air_config(4, 20)


def test_host_trace_equals_oracle():
    from ministark_b200.examples import rescue as R
    for K, length in SHAPES:
        msgs = messages(K, length)
        trace, digests = R.gen_hash_trace(msgs)
        rows, want = HO.hash_trace(msgs)
        assert np.array_equal(trace.base_columns(), _mont_cols(rows)), (K, length)
        assert [list(d) for d in digests] == want == [list(R.hash(m)) for m in msgs], (K, length)
    # a uint64 array gives the same trace
    msgs = messages(4, 20)
    assert np.array_equal(R.gen_hash_trace(np.array(msgs, dtype=np.uint64))[0].base_columns(),
                          R.gen_hash_trace(msgs)[0].base_columns())


# ------------------------------------------------------------------------------------------- the CPU stand-in
@pytest.fixture(scope="module")
def rescue_hash_abi(tmp_path_factory, orc):
    """tests/cpp/rescue_hash_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary directory"""
    out = str(tmp_path_factory.mktemp("rescue_hash_abi") / "libms_rescue_hash_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "cpp", "rescue_hash_cpu_abi.c")])
    return out


def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS, _lib._RESCUE_SIGS, _lib._RESCUE_HASH_SIGS):
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
    for K, length in shapes:
        trace, digests = R.gen_hash_trace(messages(K, length), device="cpu")
        out.append((trace.base_columns().numpy().view(np.uint64).copy(), digests))
    return out


def test_stand_in_trace_equals_oracle(rescue_hash_abi):
    got = _spawn(_worker, rescue_hash_abi, _stand_in_traces, (SHAPES,))
    assert isinstance(got, list), got
    for (K, length), (cols, digests) in zip(SHAPES, got):
        rows, want = HO.hash_trace(messages(K, length))
        assert np.array_equal(cols, _mont_cols(rows)), (K, length)
        assert [list(d) for d in digests] == want, (K, length)


def _stand_in_errors():
    from ministark_b200 import Context, MsError
    import torch
    ctx, out, msgs = Context(0), torch.zeros((13, 64), dtype=torch.int64), []
    words = np.arange(3 * 4, dtype=np.uint64)
    for m, K, length in [(words, 3, 4), (None, 1, 4), (None, 1 << 30, 0), (words, 1 << 27, 64)]:
        try:
            ctx.rescue_hash(m, K, length, out)
            msgs.append(None)
        except MsError as e:
            msgs.append(str(e))
    return msgs, bool(out.any())


def test_stand_in_refuses_bad_arguments(rescue_hash_abi):
    got = _spawn(_worker, rescue_hash_abi, _stand_in_errors, ())
    assert isinstance(got, tuple), got
    msgs, written = got
    assert "not a power of two" in msgs[0] and "null argument" in msgs[1]
    assert "exceed 2^32" in msgs[2] and "exceed 2^32" in msgs[3]
    assert not written


# ------------------------------------------------------------------------------------------------------- the AIR
def _check(length, rows, digests):
    from ministark_b200.examples import rescue as R
    from oracle import check_oracle, extension_oracle
    base = _mont_cols(rows)
    n = base.shape[1]
    claim = R.RescueHashClaim(length, digests)
    cfg = claim.AirConfig
    gamma = (123456789, 987654321, 55555)
    hints = cfg.gen_hints(n, claim, [gamma])
    ext = extension_oracle.builder(cfg, base, claim)([gamma])
    cons = [c.to_tuple() for c in cfg.constraints(n)]
    got = check_oracle.check(cons, n.bit_length() - 1, base, ext, 3, [gamma], hints)
    return [k for k, (first, _) in enumerate(got) if first is not None], ext, hints


@pytest.mark.parametrize("K,length", [(4, 20), (4, 4), (8, 7), (2, 8), (2, 0), (1, 63)])
def test_oracle_trace_satisfies_every_constraint(K, length):
    from ministark_b200.examples import rescue as R
    rows, digests = HO.hash_trace(messages(K, length))
    failing, ext, hints = _check(length, rows, digests)
    assert failing == []
    n = len(rows)
    B = length // 8 + 1
    t = length - 8 * (B - 1)
    L = n // (8 * K)
    groups = R.hash_air_config(K, length).groups(n)
    # ROUND 12, LINK 12 (none at L = 1), START 12, PAD 8 - t, R 4
    assert len(R.hash_air_config(K, length).constraints(n)) == (36 - t if L == 1 else 48 - t)
    assert [len(groups[g]) for g in ("ROUND", "LINK", "START", "PAD", "R")] == [12, 0 if L == 1 else 12, 12, 8 - t, 4]
    # R's last row is the Horner evaluation gen_hints makes from the digests
    last = tuple(int(w) * pow(2**64, -1, P) % P for w in ext[0, 3 * (n - 1):])
    assert last == tuple(hints[0])


def test_digests_leave_montgomery_form_exactly():
    import random
    from ministark_b200.examples import rescue as R
    rng = random.Random(5)
    words = [0, 1, 2, P - 1, P, P + 1, 2**64 - 1, 2**63, 2**32 - 1, 2**32, 2**32 + 1, 2**64 - 2**32, (2**32 - 1) << 32]
    words += [rng.randrange(2**64) for _ in range(10000)]
    got = R._from_mont(np.array(words, dtype=np.uint64)).tolist()
    assert got == [w * pow(2**64, -1, P) % P for w in words]


def test_digest_evaluation_is_horner():
    """the blocked evaluation of R's last row equals acc <- acc gamma^4 + d_0 + gamma d_1 + gamma^2 d_2 + gamma^3 d_3"""
    import random
    from ministark_b200 import expr as E
    from ministark_b200.examples import rescue as R
    rng = random.Random(7)
    for K in (0, 1, 2, 255, 256, 257, 1024, 3000):
        digests = [tuple(rng.randrange(P) for _ in range(4)) for _ in range(K)]
        gamma = tuple(rng.randrange(P) for _ in range(3))
        gp = [(1, 0, 0), gamma]
        for _ in range(3):
            gp.append(E.q_mul(gp[-1], gamma))
        acc = (0, 0, 0)
        for dg in digests:
            acc = E.q_mul(acc, gp[4])
            for w in range(4):
                acc = E.q_add(acc, E.q_mul(gp[w], (dg[w], 0, 0)))
        assert R.digest_evaluation(digests, gamma) == acc, K


def test_ce_blowup_is_8():
    from ministark_b200.examples import rescue as R
    from oracle import air_oracle
    # from 16 rows up: at 8 rows y = x^(n / 8) is x itself and the degree rule gives 18, for the chains AIR as well
    for K, length in SHAPES[1:] + [(2, 0), (128, 20), (512, 4), (1 << 16, 60), (1 << 19, 4)]:
        n = 8 * K * (1 << (length // 8).bit_length())
        cons = [c.to_tuple() for c in R.hash_air_config(K, length).constraints(n)]
        assert air_oracle.composition_constraint(cons, n)[1] == 8, (K, length)


def test_flipped_words_break_their_constraints():
    from ministark_b200.examples import rescue as R
    K, length = 4, 20                                   # B = 3, L = 4: 32 rows per message
    rows, digests = HO.hash_trace(messages(K, length))
    groups = R.hash_air_config(K, length).groups(len(rows))
    for p, group in [(3, "START"), (8 + 5, "LINK"), (16 + 2, "LINK")]:      # message 2's word p
        bad = [list(r) for r in rows]
        bad[32 * 2 + p][12] = (bad[32 * 2 + p][12] + 1) % P
        failing, _, _ = _check(length, bad, digests)
        assert any(k in groups[group] for k in failing), (p, failing)
    for p in range(length, 24):                          # message 1's padding: its 1 at 20, then zeros
        bad = [list(r) for r in rows]
        bad[32 + p][12] = (bad[32 + p][12] + 1) % P
        failing, _, _ = _check(length, bad, digests)
        assert groups["PAD"][p - length] in failing, (p, failing)


# ------------------------------------------------------------------------------------------------------ proofs
OPTS = (40, 8, 8, 8, 64)


def _prove(shapes):
    from ministark_b200.air import ProofOptions
    from ministark_b200.examples import rescue as R
    from ministark_b200.prover import GpuProver, peak_bytes
    from ministark_b200 import FQ3
    out = []
    for K, length, streamed in shapes:
        trace, digests = R.gen_hash_trace(messages(K, length), device="cpu")
        claim = R.RescueHashClaim(length, digests)
        got = {}
        for residency in ("resident", "streamed")[:1 + streamed]:
            p = GpuProver(0)
            if residency == "streamed":
                est = peak_bytes(len(trace), 8, 13, 1, FQ3, 8, 8)
                p.memory_budget = (est["streamed"] + est["resident"]) // 2
            got[residency] = (p.prove(claim, ProofOptions(*OPTS), trace).to_bytes(), p.last_residency)
        out.append((got, digests))
    return out


def test_cpu_harness_proofs_verify(rescue_hash_abi):
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.examples import rescue as R
    from ministark_b200.verifier import VerificationError
    from oracle import stark_oracle as SO
    shapes = [(128, 20, True), (512, 4, False)]         # 2^12 rows each: B = 3 < L = 4, and L = 1
    got = _spawn(_worker, rescue_hash_abi, _prove, (shapes,))
    assert isinstance(got, list), got
    (proofs, digests), (proofs1, digests1) = got
    assert proofs["resident"][1] == "resident" and proofs["streamed"][1] == "streamed"
    assert proofs["resident"][0] == proofs["streamed"][0]
    assert digests == [R.hash(m) for m in messages(128, 20)] and digests1 == [R.hash(m) for m in messages(512, 4)]
    for length, dg, proof in [(20, digests, proofs["resident"][0]), (4, digests1, proofs1["resident"][0])]:
        claim = R.RescueHashClaim(length, dg)
        claim.verify(proof, R.SECURITY_LEVEL)
        SO.verify(claim, proof, R.SECURITY_LEVEL, lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o)))
    proof = proofs["resident"][0]
    wrong_digest = [list(d) for d in digests]
    wrong_digest[17][2] = (wrong_digest[17][2] + 1) % P
    swapped = list(digests)
    swapped[3], swapped[40] = swapped[40], swapped[3]
    # 19 words: the same B and L, a different padding; 27 words: B = 4, the same L
    for bad in (R.RescueHashClaim(20, wrong_digest), R.RescueHashClaim(20, swapped), R.RescueHashClaim(19, digests),
                R.RescueHashClaim(27, digests)):
        with pytest.raises(VerificationError):
            bad.verify(proof, R.SECURITY_LEVEL)


def test_header_bound_and_exported(rescue_hash_abi):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.RESCUE_HASH_HEADER_PATH)
    assert declared == sorted(_lib._RESCUE_HASH_SIGS) == ["ms_rescue_hash"]
    others = set(_lib.header_symbols())
    for path in (_lib.STREAM_HEADER_PATH, _lib.CHECK_HEADER_PATH, _lib.EXTENSION_HEADER_PATH, _lib.LOOKUP_HEADER_PATH,
                 _lib.BF_HEADER_PATH, _lib.DEVICE_HEADER_PATH, _lib.HOST_NODES_HEADER_PATH, _lib.RESCUE_HEADER_PATH):
        others |= set(_lib.header_symbols(path))
    assert not set(declared) & others
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(rescue_hash_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)
