"""GPU: examples/wots's signature claim with the signatures (ms_rescue_wots_sign) and the chain trace
(ms_rescue_wots_trace) built on the device (csrc/rescue.cu).

  * device signatures, public keys and traces equal tests/rescue_wots_oracle.py, with inputs in device and host memory;
  * at K = 7 the keys, the signatures and the trace equal tests/golden/rescue_wots_k7.json, which the restatement wrote
    (the all-zero message, a message of words p - 1, a checksum with a zero digit, two keys sharing a seed), and the
    proof verifies;
  * a signature that does not verify is refused with its k named and nothing written; bad arguments are refused;
  * a K = 489 batch (2^22 rows) signs and traces on the device, and a sample of its signatures verifies on the host;
  * at 2^14 rows the proof bytes from the device trace equal the CPU harness's (tests/cpu_device.py with
    tests/cpp/rescue_wots_cpu_abi.c, in a spawned worker), resident and streamed, with validate=True, with the
    specialised evaluator and with the interpreter;
  * a broken chain raises ConstraintViolation naming LINK and its row;
  * ShardedProver with 2 ranks run as threads on one GPU gives the single-GPU bytes."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from make_rescue_wots_golden import keys, messages, sha  # noqa: E402
from ministark_b200 import FQ3  # noqa: E402
from ministark_b200.examples import wots as W  # noqa: E402
from ministark_b200.prover import GpuProver, peak_bytes  # noqa: E402
from test_rescue_wots_cpu import _mont_cols, build_stand_in, keys_of, material, oracle_rows  # noqa: E402

pytestmark = pytest.mark.gpu

P = 2**64 - 2**32 + 1


def _host(t):
    return t.cpu().numpy().view(np.uint64)


def test_device_sign_and_trace_equal_oracle():
    secrets, seeds, msgs = keys_of(2)
    pks, _, sigs = material(2)
    d_sigs, d_pks = W.sign_batch(secrets, seeds, msgs, device=0)
    assert d_sigs.is_cuda and tuple(d_sigs.shape) == (2, 67, 4) and tuple(d_pks.shape) == (2, 6)
    assert _host(d_pks).tolist() == pks and _host(d_sigs).tolist() == sigs
    # inputs already on the device give the same
    dev = lambda a: torch.from_numpy(np.array(a, dtype=np.uint64).view(np.int64)).cuda()
    s2, p2 = W.sign_batch(dev(secrets), dev(seeds), dev(msgs), device=0)
    assert torch.equal(s2, d_sigs) and torch.equal(p2, d_pks)
    pks1, msgs1, sigs1 = material(1)
    trace = W.gen_trace(pks1, msgs1, sigs1, device=0)
    base = trace.base_columns()
    assert base.is_cuda and tuple(base.shape) == (15, 1 << 14)
    assert np.array_equal(_host(base), _mont_cols(oracle_rows(1)))
    t2 = W.gen_trace(dev(pks1), dev(msgs1), dev(sigs1), device=0)
    assert torch.equal(t2.base_columns(), base)


def test_device_refuses_invalid_signatures_and_bad_arguments():
    from ministark_b200 import Context, MsError
    ctx = Context(0)
    pks, msgs, sigs = (np.array(v, dtype=np.uint64) for v in material(2))
    out = torch.zeros((15, 1 << 15), dtype=torch.int64, device="cuda")
    dsig = torch.from_numpy(sigs.view(np.int64)).cuda()
    bad_sig = dsig.clone()
    bad_sig[1, 3, 2] ^= 1
    noncanon = sigs.copy()
    noncanon[1, 5, 3] = np.uint64(P)
    bad_msg = msgs.copy()
    bad_msg[0, 2] = np.uint64(P + 3)
    for args, msg in [((pks, msgs, bad_sig, 2), "signature 1 does not verify: its root differs from its public key"),
                      ((pks, msgs, noncanon, 2), f"word 3 of element 5 of signature 1 \\({P}\\) is not canonical"),
                      ((pks, bad_msg, dsig, 2), f"word 2 of message 0 \\({P + 3}\\) is not canonical"),
                      ((pks, msgs, None, 2), "null argument"), ((pks, msgs, dsig, 0), "K = 0 is outside 1..500812")]:
        with pytest.raises(MsError, match=msg):
            ctx.rescue_wots_trace(*args, out)
    sig_out = torch.zeros((1, 67, 4), dtype=torch.int64, device="cuda")
    pk_out = torch.zeros((1, 6), dtype=torch.int64, device="cuda")
    with pytest.raises(MsError, match=f"word 1 of seed 0 \\({P}\\) is not canonical"):
        ctx.rescue_wots_sign(np.array([[1, 2, 3, 4]], dtype=np.uint64), np.array([[1, P]], dtype=np.uint64),
                             np.zeros((1, 4), dtype=np.uint64), 1, sig_out, pk_out)
    ctx.sync()
    assert not out.any() and not sig_out.any() and not pk_out.any()        # refused before anything was written
    with pytest.raises(ValueError, match="^signature 1 does not verify"):
        W.gen_trace(pks, msgs, bad_sig, device=0)


# ------------------------------------------------------------------------------------------ the golden batch
@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "rescue_wots_k7.json")) as f:
        gold = json.load(f)
    K, seed = gold["K"], gold["seed"]
    secrets, seeds = keys(K, seed)
    msgs = messages(K, seed)
    sigs, pks = W.sign_batch(secrets, seeds, msgs, device=0)
    return gold, msgs, sigs, pks, W.gen_trace(pks, msgs, sigs, device=0)


def test_golden_signatures_and_trace(golden):
    gold, msgs, sigs, pks, trace = golden
    assert W.digits(msgs[0])[64:] == [0, 12, 3] and W.digits(msgs[1]).count(15) == 32
    assert 0 in W.digits(msgs[2])[64:] and gold["public_keys"][3][:2] == gold["public_keys"][4][:2]
    assert _host(pks).tolist() == gold["public_keys"]
    assert sha(_host(sigs)) == gold["signatures_sha256"] and sha(_host(pks)) == gold["public_keys_sha256"]
    assert tuple(trace.base_columns().shape) == (15, 1 << 16)
    assert hashlib.sha256(_host(trace.base_columns()).tobytes()).hexdigest() == gold["trace_sha256"]


def test_golden_proof_verifies(golden):
    gold, msgs, _, _, trace = golden
    claim = W.SignaturesClaim(gold["public_keys"], msgs)
    proof = GpuProver(0).prove(claim, W.OPTIONS, trace)
    claim.verify(proof.to_bytes(), W.SECURITY_LEVEL)


def test_benchmark_batch_verifies_on_the_host():
    K = 489
    secrets, seeds = keys(K, 2)
    msgs = messages(K, 2)
    sigs, pks = W.sign_batch(secrets, seeds, msgs, device=0)
    trace = W.gen_trace(pks, msgs, sigs, device=0)
    assert tuple(trace.base_columns().shape) == (15, 1 << 22)
    hs, hp = _host(sigs), _host(pks)
    for k in (0, 137, K - 1):
        assert W.verify(hp[k], msgs[k], hs[k]), k
        assert hp[k][:2].tolist() == seeds[k].tolist()
    bad = sigs.clone()
    bad[300, 66, 0] ^= 1
    with pytest.raises(ValueError, match="^signature 300 does not verify"):
        W.gen_trace(pks, msgs, bad, device=0)


# ------------------------------------------------------------------ device-trace proofs against the CPU harness's
def _cpu_harness_worker(lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    try:
        from test_rescue_wots_cpu import _install
        _install(lib_path)
        pks, msgs, sigs = material(1)
        trace = W.gen_trace(pks, msgs, sigs, device="cpu")
        q.put(GpuProver(0).prove(W.SignaturesClaim(pks, msgs), W.OPTIONS, trace).to_bytes())
    except Exception:
        import traceback
        q.put(traceback.format_exc())


def _case14():
    pks, msgs, sigs = material(1)
    return W.SignaturesClaim(pks, msgs), W.gen_trace(pks, msgs, sigs, device=0)


def test_device_trace_proofs_equal_cpu_harness(tmp_path, orc):
    import torch.multiprocessing as mp
    lib = str(tmp_path / "libms_rescue_wots_cpu_abi.so")
    build_stand_in(lib)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_cpu_harness_worker, args=(lib, q))
    visible = os.environ.get("CUDA_VISIBLE_DEVICES")
    os.environ["CUDA_VISIBLE_DEVICES"] = ""             # the harness's host tensors and no-op streams want no device
    try:
        p.start()
    finally:
        if visible is None:
            del os.environ["CUDA_VISIBLE_DEVICES"]
        else:
            os.environ["CUDA_VISIBLE_DEVICES"] = visible
    want = q.get(timeout=1800)
    p.join(timeout=60)
    assert isinstance(want, bytes), want
    claim, trace = _case14()
    est = peak_bytes(len(trace), 8, 15, 1, FQ3, 8, 8)
    for no_jit in (False, True):
        if no_jit:
            os.environ["MS_EVAL_NO_JIT"] = "1"              # the interpreter kernel instead of the specialised one
        try:
            for residency, budget in [("resident", None), ("streamed", (est["streamed"] + est["resident"]) // 2)]:
                prover = GpuProver(0, memory_budget=budget)
                got = prover.prove(claim, W.OPTIONS, trace, validate=True).to_bytes()
                assert prover.last_residency == residency
                assert got == want, (residency, no_jit)
        finally:
            os.environ.pop("MS_EVAL_NO_JIT", None)
    claim.verify(want, W.SECURITY_LEVEL)


def test_broken_chain_names_link_and_its_row():
    from ministark_b200.validate import ConstraintViolation
    claim, trace = _case14()
    groups = W.air_config(1).groups(len(trace))
    b, s = 40, 6                                             # block 40: slot 7's input no longer follows slot 6
    base = trace.base_columns()
    row = W.BLOCK * b + 8 * (s + 1)
    base[0, row] = int(np.array([(int(_host(base[0, row:row + 1])[0]) + 1) % P], dtype=np.uint64).view(np.int64)[0])
    with pytest.raises(ConstraintViolation) as e:
        GpuProver(0).prove(claim, W.OPTIONS, trace, validate=True)
    by_constraint = {v.constraint: v.first_row for v in e.value.violations}
    assert by_constraint.get(groups["LINK"][0]) == row - 8, by_constraint
    assert set(by_constraint) <= set(groups["LINK"]) | set(groups["ROUND"]), by_constraint
    first = min(by_constraint)                               # the message names the first violated constraint
    assert f"Constraint {first} " in str(e.value) and f"row {by_constraint[first]} " in str(e.value)


def test_sharded_prover_on_thread_ranks_gives_the_same_bytes():
    from test_gpu_sharded_one_gpu import _prove_on_thread_ranks
    claim, trace = _case14()
    single = GpuProver(0).prove(claim, W.OPTIONS, trace).to_bytes()
    proofs = _prove_on_thread_ranks(2, claim, W.OPTIONS, trace)
    assert all(p == [single, single] for p in proofs)
