"""GPU: examples/rescue's hash claim with the trace built on the device (csrc/rescue.cu, ms_rescue_hash).

  * the device trace equals tests/rescue_hash_oracle.py word for word at one message of zero words, L = 1, B = L and
    B < L, with the messages in host or in device memory; bad arguments are refused before anything is written;
  * at K = 2^16 messages of 60 words (2^22 rows) the SHA-256 of the trace and of the digests, and the first digests,
    equal tests/golden/rescue_hash_k65536_len60.json, which the restated sponge wrote
    (tests/golden/make_rescue_hash_golden.py), and the proof verifies; at K = 2^19 messages of 4 words (2^22 rows, one
    permutation per message) the proof verifies;
  * at 2^14 rows the proof bytes from the device trace equal the CPU harness's (tests/cpu_device.py with
    tests/cpp/rescue_hash_cpu_abi.c, in a spawned worker), resident and streamed, with validate=True;
  * a flipped message word raises ConstraintViolation naming the LINK or START constraint of the row that absorbs it;
  * with two or more GPUs, ShardedProver gives the single-GPU bytes."""
import hashlib
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from make_rescue_hash_golden import digests_sha256, messages  # noqa: E402
from ministark_b200 import FQ3  # noqa: E402
from ministark_b200.examples import rescue as R  # noqa: E402
from ministark_b200.prover import GpuProver, peak_bytes  # noqa: E402

pytestmark = pytest.mark.gpu

P = 2**64 - 2**32 + 1


def _mont_cols(rows):
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T.copy()


@pytest.mark.parametrize("K,length", [(1, 0), (4, 7), (2, 8), (4, 20), (2, 63), (1024, 9)])
def test_device_trace_equals_oracle(K, length):
    import rescue_hash_oracle as HO
    msgs = messages(K, length)
    trace, digests = R.gen_hash_trace(msgs, device=0)
    base = trace.base_columns()
    assert base.is_cuda and tuple(base.shape) == (13, 8 * K * (1 << (length // 8).bit_length()))
    rows, want = HO.hash_trace([[int(w) for w in m] for m in msgs])
    cols = base.cpu().numpy().view(np.uint64)
    assert np.array_equal(cols, _mont_cols(rows))
    assert [list(d) for d in digests] == want
    # the messages in device memory give the same trace
    from ministark_b200 import Context
    ctx, out = Context(0), torch.zeros_like(base)
    ctx.rescue_hash(torch.from_numpy(msgs.view(np.int64)).cuda(), K, length, out)
    ctx.sync()
    assert torch.equal(out, base)


def test_device_trace_refuses_bad_arguments():
    from ministark_b200 import Context, MsError
    ctx, out = Context(0), torch.zeros((13, 64), dtype=torch.int64, device="cuda")
    words = np.arange(12, dtype=np.uint64)
    for m, K, length, msg in [(words, 3, 4, "not a power of two"), (None, 1, 4, "null argument"),
                              (None, 1 << 30, 0, "exceed 2\\^32"), (words, 1 << 27, 64, "exceed 2\\^32")]:
        with pytest.raises(MsError, match=msg):
            ctx.rescue_hash(m, K, length, out)
    ctx.sync()
    assert not out.any()                                      # refused before anything was written


# --------------------------------------------------------------------------------------------------- 2^22 rows
@pytest.fixture(scope="module")
def config5():
    with open(os.path.join(ROOT, "tests", "golden", "rescue_hash_k65536_len60.json")) as f:
        gold = json.load(f)
    trace, digests = R.gen_hash_trace(messages(gold["K"], gold["length"]), device=0)
    return gold, trace, digests


def test_config5_trace_equals_golden(config5):
    gold, trace, digests = config5
    words = trace.base_columns().cpu().numpy().view(np.uint64)
    assert hashlib.sha256(words.tobytes()).hexdigest() == gold["trace_sha256"]
    assert digests_sha256(digests) == gold["digests_sha256"]
    assert [list(d) for d in digests[:8]] == gold["first_digests"]


def test_config5_proof_verifies(config5):
    gold, trace, digests = config5
    claim = R.RescueHashClaim(gold["length"], digests)
    proof = GpuProver(0).prove(claim, R.OPTIONS, trace)
    claim.verify(proof.to_bytes(), R.SECURITY_LEVEL)


def test_one_permutation_per_message_proof_verifies():
    K, length = 1 << 19, 4                                    # L = 1: 2^22 rows
    trace, digests = R.gen_hash_trace(messages(K, length), device=0)
    claim = R.RescueHashClaim(length, digests)
    proof = GpuProver(0).prove(claim, R.OPTIONS, trace)
    claim.verify(proof.to_bytes(), R.SECURITY_LEVEL)


# ------------------------------------------------------------------ device-trace proofs against the CPU harness's
K14, LEN14 = 512, 20                # B = 3, L = 4: 2^14 rows


def _budget(n):
    est = peak_bytes(n, 8, 13, 1, FQ3, 8, 8)
    return (est["streamed"] + est["resident"]) // 2


def _cpu_harness_worker(lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    try:
        import ctypes as C
        import cpu_device
        cpu_device.install()
        from ministark_b200 import _lib
        lib = C.CDLL(lib_path)
        _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
        for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS, _lib._RESCUE_SIGS, _lib._RESCUE_HASH_SIGS):
            _lib.bind(lib, sigs)
        _lib._lib = lib
        trace, digests = R.gen_hash_trace(messages(K14, LEN14), device="cpu")
        claim = R.RescueHashClaim(LEN14, digests)
        q.put(GpuProver(0).prove(claim, R.OPTIONS, trace).to_bytes())
    except Exception:
        import traceback
        q.put(traceback.format_exc())


def test_device_trace_proofs_equal_cpu_harness(tmp_path):
    import torch.multiprocessing as mp
    lib = str(tmp_path / "libms_rescue_hash_cpu_abi.so")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "libms_cpu_abi.so"])
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", lib,
                           os.path.join(ROOT, "tests", "cpp", "rescue_hash_cpu_abi.c")])
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
    trace, digests = R.gen_hash_trace(messages(K14, LEN14), device=0)
    claim = R.RescueHashClaim(LEN14, digests)
    for residency, budget in [("resident", None), ("streamed", _budget(len(trace)))]:
        prover = GpuProver(0, memory_budget=budget)
        got = prover.prove(claim, R.OPTIONS, trace, validate=True).to_bytes()
        assert prover.last_residency == residency
        assert got == want, residency
    claim.verify(want, R.SECURITY_LEVEL)


def test_flipped_message_word_names_its_constraint_and_row():
    from ministark_b200.validate import ConstraintViolation
    K, length = 64, 20                                       # B = 3, L = 4: 32 rows per message
    groups = R.hash_air_config(K, length).groups(8 * K * 4)
    claim = R.RescueHashClaim(length, [R.hash(m) for m in messages(K, length)])
    # message 5, word 8 + 3 (block 1): the link into permutation 1 absorbs it at the r = 7 row of permutation 0;
    # message 9, word 6 (block 0): the start constraint absorbs it at the message's first row
    for k, p, group, absorbing_row in [(5, 11, "LINK", 32 * 5 + 7), (9, 6, "START", 32 * 9)]:
        trace, _ = R.gen_hash_trace(messages(K, length), device=0)
        trace.base_columns()[12, 32 * k + p] ^= 1
        with pytest.raises(ConstraintViolation) as e:
            GpuProver(0).prove(claim, R.OPTIONS, trace, validate=True)
        by_constraint = {v.constraint: v.first_row for v in e.value.violations}
        assert by_constraint == {groups[group][p % 8]: absorbing_row}, by_constraint
        assert f"row {absorbing_row}" in str(e.value)


# ------------------------------------------------------------------------------------------ sharded, two GPUs
def _sharded_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from ministark_b200.prover_mgpu import ShardedProver
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        trace, digests = R.gen_hash_trace(messages(K14, LEN14), device=rank)
        claim = R.RescueHashClaim(LEN14, digests)
        q.put((rank, ShardedProver(dist, rank).prove(claim, R.OPTIONS, trace).to_bytes()))
    finally:
        dist.destroy_process_group()


def test_sharded_prover_gives_the_same_bytes():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=900) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    trace, digests = R.gen_hash_trace(messages(K14, LEN14), device=0)
    single = GpuProver(0).prove(R.RescueHashClaim(LEN14, digests), R.OPTIONS, trace).to_bytes()
    assert got[0] == got[1] == single
