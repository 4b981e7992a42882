"""GPU: examples/rollup's transfer claim with the balances resolved and the trace, the roots and the final heap built on
the device (csrc/rescue.cu, ms_rescue_rollup).

  * the device trace, roots and final heap equal tests/rescue_rollup_oracle.py word for word over the CPU test's
    shapes, with the heap in device and in host memory; the caller's heap is left alone;
  * at D = 16, K = 2^9 the roots, the final heap and the trace equal tests/golden/rescue_rollup_d16_k512.json, which
    the restatement wrote (a self-transfer, an account touched 8 times, a sender left at 0, a receiver brought to
    2^32 - 1 and a zero amount), and the proof verifies;
  * at D = 24 the final root equals that of merkle.tree(final leaves, device=0);
  * an invalid batch fails with its first failing transfer named and nothing written; bad arguments are refused;
  * at 2^14 rows the proof bytes from the device trace equal the CPU harness's (tests/cpu_device.py with
    tests/cpp/rescue_rollup_cpu_abi.c, in a spawned worker), resident and streamed, with validate=True, with the
    specialised evaluator and with the interpreter;
  * a broken BAL raises ConstraintViolation naming BAL and its row;
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

from make_rescue_merkle_golden import heap_sha256  # noqa: E402
from make_rescue_rollup_golden import accounts, transfers  # noqa: E402
from ministark_b200 import FQ3  # noqa: E402
from ministark_b200.examples import merkle as M  # noqa: E402
from ministark_b200.examples import rollup as RL  # noqa: E402
from ministark_b200.prover import GpuProver, peak_bytes  # noqa: E402
from test_rescue_rollup_cpu import SHAPES, accounts_of, build_stand_in, transfers_of  # noqa: E402

pytestmark = pytest.mark.gpu

P = 2**64 - 2**32 + 1


def _mont_cols(rows):
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T.copy()


def _host(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("depth,K,case", SHAPES)
def test_device_apply_equals_oracle(depth, K, case):
    import rescue_merkle_oracle as MO
    import rescue_rollup_oracle as RO
    lv = accounts_of(depth)
    txs = transfers_of(depth, K, case)
    nodes = M.tree(lv, device=0)
    before = nodes.clone()
    trace, heap, roots = RL.apply(nodes, depth, txs, device=0)
    assert torch.equal(nodes, before)                       # the caller's heap is left alone
    rows, want_roots, want_heap = RO.rollup_trace(MO.heap([list(a) for a in lv]), depth, txs)
    base = trace.base_columns()
    L = 1 << (depth - 1).bit_length()
    assert base.is_cuda and heap.is_cuda and tuple(base.shape) == (23, 32 * K * L)
    assert np.array_equal(_host(base), _mont_cols(rows))
    assert [list(r) for r in roots] == want_roots
    got = _host(heap)
    assert got[0].tolist() == [0, 0, 0, 0] and got[1:].tolist() == want_heap[1:]
    # the heap in host memory gives the same trace, roots and heap, and so does the context with host arrays
    trace2, heap2, roots2 = RL.apply(_host(nodes).copy(), depth, txs, device=0)
    assert torch.equal(trace2.base_columns(), base) and torch.equal(heap2, heap) and roots2 == roots
    from ministark_b200 import Context
    ctx = Context(0)
    host_heap, out, host_roots = _host(nodes).copy(), torch.zeros_like(base), np.zeros((K + 1, 4), dtype=np.uint64)
    ctx.rescue_rollup(host_heap, depth, np.array(txs, dtype=np.uint64).reshape(K, 3), K, out, host_roots)
    ctx.sync()
    assert torch.equal(out, base) and np.array_equal(host_heap, got) and host_roots.tolist() == want_roots


def test_device_refuses_invalid_batches_and_bad_arguments():
    from ministark_b200 import Context, MsError
    ctx = Context(0)
    lv = torch.tensor([[100, 0, 9, 9], [2**32 - 6, 0, 0, 0], [0, 0, 0, 0], [7, 0, 0, 0]] * 2, dtype=torch.int64,
                      device="cuda")
    nodes = M.tree(lv, device=0)
    heap = nodes.clone()
    out = torch.zeros((23, 256), dtype=torch.int64, device="cuda")
    roots = torch.zeros((3, 4), dtype=torch.int64, device="cuda")
    t = lambda rows: torch.tensor(rows, dtype=torch.int64, device="cuda")
    ok = [3, 2, 7]
    for args, msg in [((heap, 3, t([ok] * 3), 3), "not a power of two"), ((heap, 3, None, 2), "null argument"),
                      ((heap, 0, t([ok] * 2), 2), "outside 1..32"),
                      ((heap, 3, t([ok, [1, 8, 0]]), 2), "receiver 8 of transfer 1 is not below 2\\^3"),
                      ((heap, 3, t([[0, 1, 2**32], ok]), 2), "amount 4294967296 of transfer 0 is not below 2\\^32"),
                      ((heap, 3, t([ok]), 1), "are not in 2\\^8..2\\^32"),
                      ((heap, 3, t([ok, [0, 2, 101]]), 2),
                       f"the sender step of transfer 1 leaves account 0 with balance {P - 1}, not below 2\\^32"),
                      ((heap, 3, t([[0, 1, 6], ok]), 2),
                       f"the receiver step of transfer 0 leaves account 1 with balance {2**32}, not below 2\\^32"),
                      ((heap, 3, t([ok, [0, 1, 50], [0, 1, 1], ok, [0, 2, 101]] + [ok] * 3), 8),
                       "the receiver step of transfer 1 leaves account 1")]:
        with pytest.raises(MsError, match=msg):
            ctx.rescue_rollup(*args, out, roots)
    ctx.sync()
    assert torch.equal(heap, nodes) and not out.any() and not roots.any()     # refused before anything was written
    with pytest.raises(ValueError, match="the sender step of transfer 1 leaves account 0"):
        RL.apply(nodes, 3, [ok, (0, 2, 101)], device=0)
    assert torch.equal(heap, nodes)


# ------------------------------------------------------------------------------------------ the golden shape
@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "rescue_rollup_d16_k512.json")) as f:
        gold = json.load(f)
    depth, K, seed = gold["depth"], gold["K"], gold["seed"]
    lv = accounts(depth, seed)
    txs = transfers(lv, depth, K, seed)
    nodes = M.tree(lv, device=0)
    trace, heap, roots = RL.apply(nodes, depth, txs, device=0)
    return gold, txs, trace, heap, roots


def test_golden_apply(golden):
    gold, txs, trace, heap, roots = golden
    assert any(s == d for s, d, _ in txs) and any(a == 0 for _, _, a in txs)
    assert list(roots[0]) == gold["old_root"] and list(roots[-1]) == gold["new_root"]
    assert [list(r) for r in roots[:4]] == gold["first_roots"]
    assert heap_sha256(_host(heap)) == gold["heap_sha256"]
    assert hashlib.sha256(_host(trace.base_columns()).tobytes()).hexdigest() == gold["trace_sha256"]


def test_golden_proof_verifies(golden):
    gold, txs, trace, _, roots = golden
    claim = RL.TransfersClaim(gold["depth"], roots[0], roots[-1], txs)
    proof = GpuProver(0).prove(claim, RL.OPTIONS, trace)
    claim.verify(proof.to_bytes(), RL.SECURITY_LEVEL)


def test_benchmark_depth_final_root_equals_rebuilt_tree():
    depth, K = 24, 1 << 13
    lv = accounts(depth, 2)
    txs = transfers(lv, depth, K, 2)
    nodes = M.tree(lv, device=0)
    _, heap, roots = RL.apply(nodes, depth, txs, device=0)
    final = lv.copy()
    for s, d, a in txs:                                      # one after another
        final[s, 0] -= np.uint64(a)
        final[s, 1] += np.uint64(1)
        final[d, 0] += np.uint64(a)
    rebuilt = M.tree(final, device=0)
    assert roots[-1] == M.root(rebuilt) and roots[0] == M.root(nodes)
    assert torch.equal(heap, rebuilt)


# ------------------------------------------------------------------ device-trace proofs against the CPU harness's
DEPTH14, K14, SALT14 = 5, 64, 14    # L = 8: 2^14 rows


def _cpu_harness_worker(lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    try:
        from test_rescue_rollup_cpu import _install
        _install(lib_path)
        nodes = M.tree(np.array(accounts_of(DEPTH14, SALT14), dtype=np.uint64), device="cpu")
        txs = transfers_of(DEPTH14, K14, "edges", SALT14)
        trace, _, roots = RL.apply(nodes, DEPTH14, txs, device="cpu")
        claim = RL.TransfersClaim(DEPTH14, roots[0], roots[-1], txs)
        q.put(GpuProver(0).prove(claim, RL.OPTIONS, trace).to_bytes())
    except Exception:
        import traceback
        q.put(traceback.format_exc())


def _case14():
    nodes = M.tree(accounts_of(DEPTH14, SALT14), device=0)
    txs = transfers_of(DEPTH14, K14, "edges", SALT14)
    trace, _, roots = RL.apply(nodes, DEPTH14, txs, device=0)
    return RL.TransfersClaim(DEPTH14, roots[0], roots[-1], txs), trace


def test_device_trace_proofs_equal_cpu_harness(tmp_path, orc):
    import torch.multiprocessing as mp
    lib = str(tmp_path / "libms_rescue_rollup_cpu_abi.so")
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
    est = peak_bytes(len(trace), 8, 23, 2, FQ3, 8, 8)
    for no_jit in (False, True):
        if no_jit:
            os.environ["MS_EVAL_NO_JIT"] = "1"              # the interpreter kernel instead of the specialised one
        try:
            for residency, budget in [("resident", None), ("streamed", (est["streamed"] + est["resident"]) // 2)]:
                prover = GpuProver(0, memory_budget=budget)
                got = prover.prove(claim, RL.OPTIONS, trace, validate=True).to_bytes()
                assert prover.last_residency == residency
                assert got == want, (residency, no_jit)
        finally:
            os.environ.pop("MS_EVAL_NO_JIT", None)
    claim.verify(want, RL.SECURITY_LEVEL)


def test_broken_balance_names_bal_and_its_row():
    from ministark_b200.validate import ConstraintViolation
    claim, trace = _case14()
    L = 8
    groups = RL.rollup_air_config(K14, DEPTH14).groups(len(trace))
    w = 37                                                   # write 37's DELTA, and R's binding of it, changed
    base = trace.base_columns()
    row = 16 * L * w
    delta = int(_host(base[RL.DELTA, row:row + 1])[0]) * pow(2**64, -1, P) % P
    base[RL.DELTA, row] = int(np.array([(delta + 1) % P * 2**64 % P], dtype=np.uint64).view(np.int64)[0])
    with pytest.raises(ConstraintViolation) as e:
        GpuProver(0).prove(claim, RL.OPTIONS, trace, validate=True)
    by_constraint = {v.constraint: v.first_row for v in e.value.violations}
    bal_row = 16 * L * w - 1                                 # write 36's new path end, where write 37 is checked
    assert by_constraint.get(groups["BAL"][0]) == bal_row, by_constraint
    assert set(by_constraint) <= set(groups["BAL"]) | set(groups["R"]), by_constraint
    assert f"row {bal_row}" in str(e.value)


def test_sharded_prover_on_thread_ranks_gives_the_same_bytes():
    from test_gpu_sharded_one_gpu import _prove_on_thread_ranks
    claim, trace = _case14()
    single = GpuProver(0).prove(claim, RL.OPTIONS, trace).to_bytes()
    proofs = _prove_on_thread_ranks(2, claim, RL.OPTIONS, trace)
    assert all(p == [single, single] for p in proofs)
