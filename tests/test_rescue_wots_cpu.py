"""CPU-only: examples/wots's signature claim, K Winternitz one-time signatures over Rescue-Prime proved valid in one proof.

  * the host scheme (digits, public_key, sign, sign_batch) equals the restatement (tests/rescue_wots_oracle.py), and
    verify refuses a flipped word, a wrong message and a wrong key;
  * the host trace and the CPU build of ms_rescue_wots_sign / ms_rescue_wots_trace (tests/cpp/rescue_wots_cpu_abi.c,
    through `device="cpu"` on the CPU harness, tests/cpu_device.py) equal the restatement; a signature that does not
    verify is refused with its k named and nothing written, and so are bad arguments;
  * the restated trace satisfies every constraint (oracle/check_oracle.py), and each of these breaks its own group and
    no other: an ACT pattern with the right count in the wrong slots (ACT), CNT off by one (CNT), a wrong tweak word
    (CAP), a seed changed from one slot on (CAP), a seed changed in a whole block (R), a broken fold carry (ACC), LAST
    moved to another chain (R) and a padding block that carries its fold into the next (R).  Each changed trace is
    otherwise recomputed, down to the root its claim states;
  * every padding block is the same independent block, ending in pad_root(), and R binds it as such;
  * the constraint counts, the ce blow-up of 8 and a composition program that fits the evaluator; the specialised
    evaluator's generated source (csrc/eval_jit.cu, compiled here by g++) and the CPU interpreter agree on it;
  * 2^14-row (K = 1) and padded 2^15-row (K = 3) proofs verify with Stark.verify and oracle/stark_oracle.verify, and a
    wrong key, a wrong message, two swapped signatures and a claim with K - 1 entries are refused.
Harness cases run in spawned workers that install it themselves; the pytest process never does."""
import ctypes as C
import functools
import os
import random
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rescue_wots_oracle as WO  # noqa: E402

P = 2**64 - 2**32 + 1


def keys_of(K, salt=0):
    """(secrets, seeds, messages) of K keys: key 0 signs the all-zero message, key 1 (when K > 1) shares key 0's seed
    and signs words p - 1"""
    rng = random.Random(77 + salt)
    secrets = [[rng.randrange(P) for _ in range(4)] for _ in range(K)]
    seeds = [[rng.randrange(P) for _ in range(2)] for _ in range(K)]
    msgs = [[rng.randrange(P) for _ in range(4)] for _ in range(K)]
    msgs[0] = [0] * 4
    if K > 1:
        seeds[1] = list(seeds[0])
        msgs[1] = [P - 1] * 4
    return secrets, seeds, msgs


@functools.lru_cache(maxsize=None)
def material(K, salt=0):
    """(public keys, messages, signatures) by the restatement"""
    secrets, seeds, msgs = keys_of(K, salt)
    pks = [WO.keygen(s, r)[0] for s, r in zip(secrets, seeds)]
    sigs = [WO.sign(s, r, m) for s, r, m in zip(secrets, seeds, msgs)]
    return pks, msgs, sigs


@functools.lru_cache(maxsize=None)
def oracle_rows(K, salt=0):
    pks, msgs, sigs = material(K, salt)
    rows, roots = WO.wots_trace(pks, msgs, sigs)
    assert roots == [pk[2:] for pk in pks]
    return rows


def _mont_cols(rows):
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T.copy()


# ------------------------------------------------------------------------------------------------------ the scheme
def test_host_scheme_equals_oracle_and_verify_refuses_tampering():
    from ministark_b200.examples import wots as W
    secrets, seeds, msgs = keys_of(2)
    pks, _, sigs = material(2)
    assert W.digits([0] * 4)[64:] == [0, 12, 3] and W.digits([P - 1] * 4)[:16] == [0] * 8 + [15] * 8
    for m in msgs + [[1, 2, 3, 4], [2**63, 5, P - 2, 17]]:
        assert W.digits(m) == WO.digits(m)
    got_sigs, got_pks = W.sign_batch(secrets, seeds, msgs)
    assert [list(pk) for pk in got_pks] == pks and [[list(x) for x in s] for s in got_sigs] == sigs
    assert list(W.public_key(secrets[0], seeds[0])) == pks[0]
    assert [list(x) for x in W.sign(secrets[1], seeds[1], msgs[1])] == sigs[1]
    for k in range(2):
        assert W.verify(pks[k], msgs[k], sigs[k])
    flipped = [list(x) for x in sigs[0]]
    flipped[40][2] = (flipped[40][2] + 1) % P
    assert not W.verify(pks[0], msgs[0], flipped)
    assert not W.verify(pks[0], [1, 0, 0, 0], sigs[0])
    assert not W.verify(pks[1], msgs[0], sigs[0])                 # the same seed, another secret
    for bad in [lambda: W.verify(pks[0], msgs[0], sigs[0][:-1]), lambda: W.digits([P, 0, 0, 0]),
                lambda: W.public_key([1, 2, 3], [4, 5]), lambda: W.sign([1, 2, 3, 4], [P, 0], [0] * 4),
                lambda: W.verify(pks[0][:5], msgs[0], sigs[0])]:
        with pytest.raises(ValueError):
            bad()


def test_host_trace_equals_oracle_and_names_invalid_signatures():
    from ministark_b200.examples import wots as W
    pks, msgs, sigs = material(1)
    trace = W.gen_trace(pks, msgs, sigs)
    assert trace.base_columns().shape == (15, 1 << 14)
    assert np.array_equal(trace.base_columns(), _mont_cols(oracle_rows(1)))
    pks2, msgs2, sigs2 = material(2)
    bad = [list(s) for s in sigs2]
    bad[1] = [list(x) for x in bad[1]]
    bad[1][66][0] = (bad[1][66][0] + 1) % P
    with pytest.raises(ValueError, match="signature 1 does not verify"):
        W.gen_trace(pks2, msgs2, bad)
    with pytest.raises(ValueError):
        W.gen_trace(pks2, msgs2, sigs2[:1])
    with pytest.raises(ValueError):
        W.gen_trace([], [], [])


def test_shapes_and_claim_arguments():
    from ministark_b200.examples import wots as W
    assert W.MAX_KEYS == 500812 and W._blocks(1) == 128 and W._blocks(7) == 512 and W._blocks(489) == 1 << 15
    assert 128 * W._blocks(W.MAX_KEYS) == 1 << 32
    for K in (0, W.MAX_KEYS + 1):
        with pytest.raises(ValueError):
            W.air_config(K)
    assert W.air_config(3) is W.air_config(3)
    pks, msgs, _ = material(1)
    with pytest.raises(ValueError):
        W.SignaturesClaim(pks, msgs + msgs)
    with pytest.raises(ValueError):
        W.SignaturesClaim([pks[0][:5]], msgs)
    with pytest.raises(ValueError):
        W.air_config(3).constraints(1 << 14)                 # 3 signatures take 2^15 rows
    claim = W.SignaturesClaim(pks, msgs)
    assert claim.public_inputs_bytes(claim) == np.array([1] + pks[0] + msgs[0], dtype="<u8").tobytes()


# ------------------------------------------------------------------------------------------------ the CPU stand-in
@pytest.fixture(scope="module")
def wots_abi(tmp_path_factory, orc):
    out = str(tmp_path_factory.mktemp("rescue_wots_abi") / "libms_rescue_wots_cpu_abi.so")
    build_stand_in(out)
    return out


def build_stand_in(out):
    """tests/cpp/rescue_wots_cpu_abi.c on top of the rollup stand-in, linked like it with tests/cpp/lookup_cpu_abi.c"""
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "cpp", "rescue_wots_cpu_abi.c"),
                           os.path.join(ROOT, "tests", "cpp", "lookup_cpu_abi.c"), "-Wl,--allow-multiple-definition"])


def _install(path):
    from test_rescue_rollup_cpu import _install as install_rollup
    from ministark_b200 import _lib
    install_rollup(path)
    _lib.bind(_lib._lib, _lib._RESCUE_WOTS_SIGS)


def _spawn(target, *args):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=target, args=args + (q,))
    p.start()
    got = q.get(timeout=1800)
    p.join(timeout=60)
    assert p.exitcode == 0
    return got


def _worker(lib_path, fn, args, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    try:
        _install(lib_path)
        q.put(fn(*args))
    except Exception:                       # reported, not left for the queue's timeout
        import traceback
        q.put(traceback.format_exc())


def _stand_in(K):
    from ministark_b200.examples import wots as W
    secrets, seeds, msgs = keys_of(K)
    sigs, pks = W.sign_batch(secrets, seeds, msgs, device="cpu")
    trace = W.gen_trace(pks, msgs, sigs, device="cpu")
    from_lists = W.gen_trace(pks.numpy().view(np.uint64).tolist(), msgs, sigs.numpy().view(np.uint64).tolist(),
                            device="cpu")
    return (sigs.numpy().view(np.uint64).tolist(), pks.numpy().view(np.uint64).tolist(),
            trace.base_columns().numpy().view(np.uint64).copy(), bool((from_lists.base_columns() == trace.base_columns()).all()))


def test_stand_in_equals_oracle(wots_abi):
    got = _spawn(_worker, wots_abi, _stand_in, (2,))
    assert isinstance(got, tuple), got
    sigs, pks, cols, same = got
    want_pks, _, want_sigs = material(2)
    assert pks == want_pks and sigs == want_sigs and same
    rows, _ = WO.wots_trace(*material(2))
    assert np.array_equal(cols, _mont_cols(rows))


def _stand_in_errors():
    import torch
    from ministark_b200 import Context, MsError
    from ministark_b200.examples import wots as W
    pks, msgs, sigs = (np.array(v, dtype=np.uint64) for v in material(2))
    ctx, msgs_out = Context(0), []
    out = torch.zeros((15, 1 << 15), dtype=torch.int64)
    bad_sig = sigs.copy()
    bad_sig[1, 3, 2] ^= np.uint64(1)
    noncanon = sigs.copy()
    noncanon[1, 5, 3] = np.uint64(P)
    bad_msg = msgs.copy()
    bad_msg[0, 2] = np.uint64(P + 3)
    for args in [(pks, msgs, bad_sig, 2), (pks, msgs, noncanon, 2), (pks, bad_msg, sigs, 2), (pks, msgs, None, 2),
                 (pks, msgs, sigs, 0)]:
        try:
            ctx.rescue_wots_trace(*args, out)
            msgs_out.append(None)
        except MsError as e:
            msgs_out.append(str(e))
    sig_out, pk_out = torch.zeros((1, 67, 4), dtype=torch.int64), torch.zeros((1, 6), dtype=torch.int64)
    try:
        ctx.rescue_wots_sign(np.array([[1, 2, 3, P]], dtype=np.uint64), np.array([[1, 2]], dtype=np.uint64),
                             np.zeros((1, 4), dtype=np.uint64), 1, sig_out, pk_out)
        msgs_out.append(None)
    except MsError as e:
        msgs_out.append(str(e))
    try:
        W.gen_trace(pks, msgs, bad_sig, device="cpu")
        msgs_out.append(None)
    except ValueError as e:
        msgs_out.append(str(e))
    return msgs_out, bool(out.any()), bool(sig_out.any() or pk_out.any())


def test_stand_in_refuses_invalid_signatures_and_bad_arguments(wots_abi):
    got = _spawn(_worker, wots_abi, _stand_in_errors, ())
    assert isinstance(got, tuple), got
    msgs, out_written, sign_written = got
    assert "signature 1 does not verify: its root differs from its public key" in msgs[0]
    assert f"word 3 of element 5 of signature 1 ({P}) is not canonical" in msgs[1]
    assert f"word 2 of message 0 ({P + 3}) is not canonical" in msgs[2]
    assert "null argument" in msgs[3] and "K = 0 is outside 1..500812" in msgs[4]
    assert f"word 3 of secret 0 ({P}) is not canonical" in msgs[5]
    assert msgs[6] == "signature 1 does not verify: its root differs from its public key"
    assert not out_written and not sign_written


def test_header_bound_and_exported(wots_abi):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.RESCUE_WOTS_HEADER_PATH)
    assert declared == sorted(_lib._RESCUE_WOTS_SIGS) == ["ms_rescue_wots_sign", "ms_rescue_wots_trace"]
    others = set(_lib.header_symbols())
    for path in (_lib.STREAM_HEADER_PATH, _lib.CHECK_HEADER_PATH, _lib.EXTENSION_HEADER_PATH, _lib.LOOKUP_HEADER_PATH,
                 _lib.PERMUTATION_HEADER_PATH, _lib.BF_HEADER_PATH, _lib.DEVICE_HEADER_PATH, _lib.HOST_NODES_HEADER_PATH,
                 _lib.RESCUE_HEADER_PATH, _lib.RESCUE_HASH_HEADER_PATH, _lib.RESCUE_MERKLE_HEADER_PATH,
                 _lib.RESCUE_MERKLE_UPDATES_HEADER_PATH, _lib.RESCUE_ROLLUP_HEADER_PATH):
        others |= set(_lib.header_symbols(path))
    assert not set(declared) & others
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(wots_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)


# ------------------------------------------------------------------------------------------------------- the AIR
GAMMA = (123456789, 987654321, 55555)


def _check(rows, pks, msgs):
    """{constraint: first failing row} of the rows against SignaturesClaim(pks, msgs)"""
    from ministark_b200.air import Air
    from ministark_b200.examples import wots as W
    from oracle import check_oracle, extension_oracle
    base = _mont_cols(rows)
    n = base.shape[1]
    claim = W.SignaturesClaim(pks, msgs)
    air = Air(claim.AirConfig, n, claim, W.OPTIONS)
    hints = claim.AirConfig.gen_hints(n, claim, [GAMMA])
    decl = [(c.init, c.mul, c.add, c.inclusive) for c in air.extension_declaration]
    ext = extension_oracle.columns(decl, base, 3, [GAMMA], hints)
    got = check_oracle.check([c.to_tuple() for c in air.constraints], n.bit_length() - 1, base, ext, 3, [GAMMA], hints)
    return {k: first for k, (first, _) in enumerate(got) if first is not None}, ext, hints


def test_oracle_trace_satisfies_every_constraint():
    from ministark_b200.air import Air
    from ministark_b200.examples import wots as W
    for K in (1, 3):
        pks, msgs, _ = material(K)
        rows = oracle_rows(K)
        failing, ext, hints = _check(rows, pks, msgs)
        assert failing == {}, K
        n = len(rows)
        cfg = W.air_config(K)
        groups = cfg.groups(n)
        sizes = {"ROUND": 12, "CAP": 8, "LINK": 4, "ACT": 2, "CNT": 2, "ACC": 9, "R": 4}
        assert {g: len(r) for g, r in groups.items()} == sizes and list(groups) == list(sizes)
        assert len(cfg.constraints(n)) == 41
        assert tuple(int(w) * pow(2**64, -1, P) % P for w in ext[0, 3 * (n - 1):]) == tuple(hints[0])


def test_ce_blowup_is_8_and_the_program_fits_the_evaluator():
    from ministark_b200.air import Air
    from ministark_b200.examples import rescue as R
    from ministark_b200.examples import wots as W
    assert W.OPTIONS is R.OPTIONS and W.SECURITY_LEVEL == R.SECURITY_LEVEL
    for K in (1, 3, 7, 489, 978, W.MAX_KEYS):
        n = 128 * W._blocks(K)
        air = Air(W.air_config(K), n, None, W.OPTIONS)
        assert air.ce_blowup_factor == 8, K
        if K <= 978:
            assert len(air.composition_program()) > 0
            assert max(o for _, o in air.trace_arguments()) == 128


def _mutated(K, changes):
    """(rows, public keys): the restated trace of material(K) with per-block changes {b: {acts, cnts, tweaks, rhos,
    carry, last}}, every block after a change recomputed from it, and each key's root replaced by the root its last
    block (LAST = 1) reaches"""
    from ministark_b200.examples import wots as W
    pks, msgs, sigs = material(K)
    rows, roots, acc = [], [], [0] * 4
    for b in range(W._blocks(K)):
        k, i = divmod(b, WO.CHAINS)
        if k < K:
            d, x, rho, last = WO.digits(msgs[k])[i], sigs[k][i], pks[k][:2], int(i == WO.CHAINS - 1)
        else:
            d, x, i, rho, last = 0, [0] * 4, 0, [0, 0], 1
        ch = changes.get(b, {})
        last = ch.get("last", last)
        acts = ch.get("acts", [int(s >= d) for s in range(15)])
        cnts = ch.get("cnts", [max(d - s, 0) for s in range(15)])
        block, out = WO.block_rows(x, acts, cnts, i, rho, ch.get("carry", acc), last, ch.get("tweaks"), ch.get("rhos"))
        rows += block
        if last and k < K:
            roots.append(out)
        acc = [0] * 4 if last else out
    return rows, [pk[:2] + r for pk, r in zip(pks, roots)]


def test_changes_break_their_own_constraints():
    from ministark_b200.examples import wots as W
    K = 1
    pks, msgs, _ = material(K)
    groups = W.air_config(K).groups(1 << 14)
    dig = WO.digits(msgs[0])
    i = next(i for i, d in enumerate(dig) if 2 <= d <= 12)          # a chain that skips some steps and applies others
    d = dig[i]

    def only(changes, group, rows=None, keys=None):
        if rows is None:
            rows, keys = _mutated(K, changes)
        got = _check(rows, keys, msgs)[0]
        assert got and set(got) <= set(groups[group]), (group, got)
        return got

    acts = [1] + [0] * d + [1] * (14 - d)                              # 15 - d steps, but not the last ones
    cnts, c = [], d
    for a in acts:
        cnts.append(c)
        c += a - 1
    assert c == 0 and sum(acts) == 15 - d
    only({i: {"acts": acts, "cnts": cnts}}, "ACT")
    rows = [list(r) for r in oracle_rows(K)]
    rows[128 * i + 8 * 6][W.CNT] += 1                                 # CNT off by one at slot 6's input
    assert only({}, "CNT", rows, pks) == {groups["CNT"][0]: 128 * i + 40}
    tweaks = [1 + s for s in range(15)]
    tweaks[7] = 9                                                      # step 7 run with step 8's tweak
    only({i: {"tweaks": tweaks}}, "CAP")
    other = [(pks[0][0] + 1) % P, pks[0][1]]
    only({i: {"rhos": [pks[0][:2]] * 5 + [other] * 11}}, "CAP")        # the seed changed from slot 5 on
    only({i: {"rhos": [other] * 16}}, "R")                             # the seed changed in a whole block
    only({i + 1: {"carry": [0] * 4}}, "ACC")                           # block i + 1's fold restarts from 0^4
    only({65: {"last": 1}, 66: {"last": 0}}, "R")                      # LAST on chain 65 instead of 66
    only({100: {"last": 0}}, "R")                                      # padding block 100 carries into block 101


def test_padding_blocks_are_independent():
    """every padding block is the same block: LAST = 1, its fold on 0^4, ending in pad_root(), which the restatement
    gives too; its tuple (0, 1, 0, 0, 0, pad_root()) is what R binds"""
    from ministark_b200.examples import wots as W
    rows = oracle_rows(1)                                              # blocks 67..127 are padding
    pad = [r for r in rows[128 * 67:128 * 68]]
    assert all(rows[128 * b:128 * (b + 1)] == pad for b in range(68, 128))
    assert all(r[W.LAST] == 1 for r in pad) and pad[120][4:8] == [0] * 4
    acc = [0] * 4
    _, x = WO.block_rows([0] * 4, [1] * 15, [0] * 15, 0, [0, 0], acc, 1)
    assert tuple(x) == W.pad_root() == tuple(pad[127][:4])
    pks, msgs, _ = material(1)
    assert W.block_tuples(pks, msgs, 128)[67:] == [(0, 1, 0, 0, 0) + W.pad_root()] * 61


# ------------------------------------------------------------------------------------------ the evaluator's source
def test_generated_kernel_source_equals_the_interpreter(tmp_path, orc):
    """the composition program of the K = 1 AIR (reads at row offsets 0, 1, 7, 8, 120, 121, 127 and 128), the
    generated kernel source against the CPU interpreter on random columns"""
    from test_eval_jit_source import GENERATOR, _host_kernel, _tables
    from ministark_b200.air import Air
    from ministark_b200.examples import wots as W
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "libms_cpu_abi.so"])
    lib = C.CDLL(os.path.join(ROOT, "oracle", "libms_cpu_abi.so"))
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    rng = random.Random(5)
    pks, msgs, _ = material(1)
    claim = W.SignaturesClaim(pks, msgs)
    air = Air(claim.AirConfig, 1 << 14, claim, W.OPTIONS)
    assert {o for _, o in air.trace_arguments()} >= {0, 1, 7, 8, 120, 121, 127, 128}
    q3 = lambda: tuple(rng.randrange(P) for _ in range(3))
    prog = air.composition_program().bind(challenges=[q3() for _ in range(32)], hints=[q3() for _ in range(256)],
                                          ccoefs=[q3() for _ in range(256)])
    log_m = air.log_n + air.ce_blowup_factor.bit_length() - 1
    m = 1 << log_m
    base = orc.rand_matrix(15, m, 1, seed=rng.randrange(1 << 30))
    ext = orc.rand_matrix(1, m, 3, seed=rng.randrange(1 << 30))
    cols = [np.ascontiguousarray(c) for c in base] + [np.ascontiguousarray(e) for e in ext]
    ptrs = (C.c_void_p * len(cols))(*[c.ctypes.data for c in cols])
    isq = (C.c_int * len(cols))(*([0] * 15 + [1]))
    code, consts = np.ascontiguousarray(prog.code), np.ascontiguousarray(prog.consts)
    want = np.zeros(m * 3, dtype=np.uint64)
    assert lib.ms_eval_constraints_ptrs(h, C.c_void_p(code.ctypes.data), len(prog), C.c_void_p(consts.ctypes.data),
                                        consts.shape[0], ptrs, isq, len(cols), 3, log_m, C.c_uint64(GENERATOR), 1, 0,
                                        C.c_void_p(want.ctypes.data)) == 0
    kernel = _host_kernel(str(tmp_path), prog, 3)
    lo, hi = _tables(log_m)
    got = np.zeros(m * 3, dtype=np.uint64)
    kernel.run_all(ptrs, C.c_void_p(consts.ctypes.data), C.c_void_p(lo.ctypes.data), C.c_void_p(hi.ctypes.data),
                   C.c_uint(len(hi)), C.c_uint64(GENERATOR), C.c_uint(log_m), 1, 0, C.c_void_p(got.ctypes.data))
    assert np.array_equal(got, want)


# ------------------------------------------------------------------------------------------------------ proofs
def _prove(K):
    from ministark_b200.examples import wots as W
    from ministark_b200.prover import GpuProver
    pks, msgs, sigs = material(K)
    trace = W.gen_trace(np.array(pks, dtype=np.uint64), msgs, sigs, device="cpu")
    return GpuProver(0).prove(W.SignaturesClaim(pks, msgs), W.OPTIONS, trace).to_bytes()


@pytest.mark.parametrize("K", [1, 3])
def test_cpu_harness_proofs_verify_and_tampered_claims_are_refused(wots_abi, K):
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.examples import wots as W
    from ministark_b200.verifier import VerificationError
    from oracle import stark_oracle as SO
    proof = _spawn(_worker, wots_abi, _prove, (K,))
    assert isinstance(proof, bytes), proof
    pks, msgs, _ = material(K)
    claim = W.SignaturesClaim(pks, msgs)
    claim.verify(proof, W.SECURITY_LEVEL)
    SO.verify(claim, proof, W.SECURITY_LEVEL, lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o)))
    wrong_key = [list(pk) for pk in pks]
    wrong_key[-1][3] = (wrong_key[-1][3] + 1) % P
    wrong_msg = [list(m) for m in msgs]
    wrong_msg[0][1] ^= 1 << 8
    bad = [W.SignaturesClaim(wrong_key, msgs), W.SignaturesClaim(pks, wrong_msg)]
    if K > 1:
        bad += [W.SignaturesClaim([pks[1], pks[0]] + pks[2:], [msgs[1], msgs[0]] + msgs[2:]),
                W.SignaturesClaim(pks[:-1], msgs[:-1])]        # 2 signatures also take 2^15 rows
    for c in bad:
        with pytest.raises(VerificationError):
            c.verify(proof, W.SECURITY_LEVEL)
