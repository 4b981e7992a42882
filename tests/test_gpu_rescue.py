"""GPU: examples/rescue with the trace built on the device (csrc/rescue.cu, ms_rescue_chains).

  * the device trace equals oracle/rescue_oracle.py word for word at (K, L) = (1, 1), (4, 2), (64, 4), (1, 64), (1024, 1);
  * at BASELINE config 5's shape, K = 2^10 and L = 2^9 (2^22 rows), the digests and the SHA-256 of the trace equal
    tests/golden/rescue_k1024_l512.json, which the CPU build of the entry point wrote (tests/golden/make_rescue_golden.py);
  * at 2^14 rows the proof bytes from the device trace equal the CPU harness's (tests/cpu_device.py with
    tests/cpp/rescue_cpu_abi.c, in a spawned worker), in the resident and the streamed residency;
  * validate=True passes on a good trace, and one flipped word raises ConstraintViolation naming a round or link
    constraint at the row it breaks;
  * the 2^22-row proof verifies with Stark.verify;
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

from ministark_b200 import FQ3  # noqa: E402
from ministark_b200.air import ProofOptions  # noqa: E402
from ministark_b200.examples import rescue as R  # noqa: E402
from ministark_b200.prover import GpuProver, peak_bytes  # noqa: E402

pytestmark = pytest.mark.gpu

P = 2**64 - 2**32 + 1
SEED = [11, 22, 33, 44]


def _mont_cols(rows):
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T.copy()


@pytest.mark.parametrize("K,L", [(1, 1), (4, 2), (64, 4), (1, 64), (1024, 1)])
def test_device_trace_equals_oracle(K, L):
    from oracle import rescue_oracle as RO
    trace, digests = R.gen_trace(SEED, K, L, device=0)
    base = trace.base_columns()
    assert base.is_cuda and tuple(base.shape) == (12, 8 * K * L)
    rows, want = RO.chain_trace(SEED, K, L)
    assert np.array_equal(base.cpu().numpy().view(np.uint64), _mont_cols(rows))
    assert [list(d) for d in digests] == want


def test_device_trace_refuses_bad_arguments():
    from ministark_b200 import Context, MsError
    ctx, out = Context(0), torch.zeros((12, 64), dtype=torch.int64, device="cuda")
    for seed, K, L, msg in [(SEED, 3, 1, "powers of two"), ([1, 2, 3, P], 1, 1, "not canonical"),
                            (SEED, 1 << 20, 1 << 10, "exceed 2\\^32")]:
        with pytest.raises(MsError, match=msg):
            ctx.rescue_chains(seed, K, L, out)
    ctx.sync()
    assert not out.any()                                      # refused before anything was written


@pytest.fixture(scope="module")
def config5():
    with open(os.path.join(ROOT, "tests", "golden", "rescue_k1024_l512.json")) as f:
        gold = json.load(f)
    trace, digests = R.gen_trace(gold["seed"], gold["K"], gold["L"], device=0)
    return gold, trace, digests


def test_config5_trace_equals_golden(config5):
    gold, trace, digests = config5
    words = trace.base_columns().cpu().numpy().view(np.uint64)
    assert hashlib.sha256(words.tobytes()).hexdigest() == gold["trace_sha256"]
    assert [list(d) for d in digests] == gold["digests"]


def test_config5_proof_verifies(config5):
    gold, trace, digests = config5
    claim = R.RescueChainsClaim(gold["seed"], gold["K"], gold["L"], digests)
    proof = GpuProver(0).prove(claim, R.OPTIONS, trace)
    claim.verify(proof.to_bytes(), R.SECURITY_LEVEL)


# ------------------------------------------------------------------ device-trace proofs against the CPU harness's
K14, L14 = 256, 8                   # 2^14 rows


def _budget(n):
    est = peak_bytes(n, 8, 12, 1, FQ3, 8, 8)
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
        for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS, _lib._RESCUE_SIGS):
            _lib.bind(lib, sigs)
        _lib._lib = lib
        trace, digests = R.gen_trace(SEED, K14, L14, device="cpu")
        claim = R.RescueChainsClaim(SEED, K14, L14, digests)
        q.put(GpuProver(0).prove(claim, R.OPTIONS, trace).to_bytes())
    except Exception:
        import traceback
        q.put(traceback.format_exc())


def test_device_trace_proofs_equal_cpu_harness(tmp_path):
    import torch.multiprocessing as mp
    lib = str(tmp_path / "libms_rescue_cpu_abi.so")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "libms_cpu_abi.so"])
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", lib, os.path.join(ROOT, "tests", "cpp", "rescue_cpu_abi.c")])
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
    trace, digests = R.gen_trace(SEED, K14, L14, device=0)
    claim = R.RescueChainsClaim(SEED, K14, L14, digests)
    for residency, budget in [("resident", None), ("streamed", _budget(len(trace)))]:
        prover = GpuProver(0, memory_budget=budget)
        got = prover.prove(claim, R.OPTIONS, trace, validate=True).to_bytes()
        assert prover.last_residency == residency
        assert got == want, residency
    claim.verify(want, R.SECURITY_LEVEL)


def test_flipped_word_names_its_constraint_and_row():
    from ministark_b200.validate import ConstraintViolation
    K, L = 64, 8
    trace, digests = R.gen_trace(SEED, K, L, device=0)
    row = 8 * L * 5 + 8 * 3 + 2                               # chain 5, permutation 3, state before round 2
    trace.base_columns()[7, row] ^= 1
    claim = R.RescueChainsClaim(SEED, K, L, digests)
    with pytest.raises(ConstraintViolation) as e:
        GpuProver(0).prove(claim, R.OPTIONS, trace, validate=True)
    by_constraint = {v.constraint: v.first_row for v in e.value.violations}
    assert set(by_constraint) <= set(R.ROUND), sorted(by_constraint)
    assert sorted(set(by_constraint.values())) == [row - 1]    # round 1's step into it fails first
    assert "Constraint" in str(e.value) and f"row {row - 1}" in str(e.value)
    # a permutation's output changed mid-chain: the round into it and the link out of it fail
    trace2, _ = R.gen_trace(SEED, K, L, device=0)
    row2 = 8 * L * 2 + 8 * 4 + 7                              # chain 2, output of permutation 4
    trace2.base_columns()[0, row2] ^= 1
    with pytest.raises(ConstraintViolation) as e:
        GpuProver(0).prove(claim, R.OPTIONS, trace2, validate=True)
    by_constraint = {v.constraint: v.first_row for v in e.value.violations}
    assert any(k in R.LINK and r in (row2 - 1, row2) for k, r in by_constraint.items()), by_constraint


# ------------------------------------------------------------------------------------------ sharded, two GPUs
def _sharded_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from ministark_b200.prover_mgpu import ShardedProver
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        trace, digests = R.gen_trace(SEED, K14, L14, device=rank)
        claim = R.RescueChainsClaim(SEED, K14, L14, digests)
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
    trace, digests = R.gen_trace(SEED, K14, L14, device=0)
    single = GpuProver(0).prove(R.RescueChainsClaim(SEED, K14, L14, digests), R.OPTIONS, trace).to_bytes()
    assert got[0] == got[1] == single
