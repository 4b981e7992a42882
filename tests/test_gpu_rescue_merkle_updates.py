"""GPU: examples/merkle's ordered-write claim with the trace, the roots and the final heap built on the device
(csrc/rescue.cu, ms_rescue_merkle_updates).

  * the device trace, roots and final heap equal tests/rescue_merkle_updates_oracle.py word for word at D = 1, at D
    not a power of two, at K = 1, with repeated indices, consecutive writes to i and i ^ 1 and a write of a leaf's
    current value, and at depths whose tree takes the per-level kernel as well as the one-block top levels, with the
    heap in device and in host memory; the caller's heap is left alone; bad arguments are refused before anything is
    written;
  * at D = 16, K = 2^10 the roots, the final heap and the trace equal tests/golden/rescue_merkle_updates_d16_k1024.json,
    which the restatement wrote (tests/golden/make_rescue_merkle_updates_golden.py), and the proof verifies;
  * at D = 24 (the benchmark's 2^24-leaf tree) the final root equals that of merkle.tree(final leaves, device=0), and
    the heap equals that tree everywhere;
  * at 2^14 rows the proof bytes from the device trace equal the CPU harness's (tests/cpu_device.py with
    tests/cpp/rescue_merkle_updates_cpu_abi.c, in a spawned worker), resident and streamed, with validate=True, with the
    specialised evaluator and with the interpreter (SIB and CHAIN read the trace 8 L rows ahead);
  * a broken root link raises ConstraintViolation naming CHAIN and its row;
  * ShardedProver with 2 ranks run as threads on one GPU gives the single-GPU bytes."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from make_rescue_merkle_golden import heap_sha256, leaves  # noqa: E402
from make_rescue_merkle_updates_golden import writes  # noqa: E402
from ministark_b200 import FQ3  # noqa: E402
from ministark_b200.examples import merkle as M  # noqa: E402
from ministark_b200.examples import rescue as R  # noqa: E402
from ministark_b200.prover import GpuProver, peak_bytes  # noqa: E402

pytestmark = pytest.mark.gpu

P = 2**64 - 2**32 + 1


def _mont_cols(rows):
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T.copy()


def _host(t):
    return t.cpu().numpy().view(np.uint64)


def _writes(depth, K, case, seed):
    idx, new = writes(K, depth, seed)
    idx, new = [int(i) for i in idx], [tuple(int(w) for w in r) for r in new]
    if case == "repeat" and K > 2:
        idx[K - 1] = idx[K - 3] = idx[0]
    elif case == "siblings" and K > 4:
        idx[2], idx[3], idx[4] = idx[1], idx[1] ^ 1, idx[1]
    elif case == "same value" and K > 1:
        idx[1] = idx[0]
        new[1] = new[0]
    return idx, new


# (depth, K, case): L = 1; D = 3 < L = 4; K = 1; D = L = 4; then depths whose tree takes the per-level kernel too
SHAPES = [(1, 4, "repeat"), (3, 8, "siblings"), (3, 1, "single"), (4, 4, "same value"), (5, 16, "repeat"),
          (7, 64, "siblings"), (9, 32, "repeat"), (11, 8, "siblings")]


@pytest.mark.parametrize("depth,K,case", SHAPES)
def test_device_update_equals_oracle(depth, K, case):
    import rescue_merkle_oracle as MO
    import rescue_merkle_updates_oracle as UO
    lv = leaves(depth, 7)
    idx, new = _writes(depth, K, case, 7)
    nodes = M.tree(lv, device=0)
    before = nodes.clone()
    trace, heap, roots = M.update(nodes, depth, idx, new, device=0)
    assert torch.equal(nodes, before)                       # the caller's heap is left alone
    rows, want_roots, want_heap = UO.updates_trace(MO.heap([[int(w) for w in leaf] for leaf in lv]), depth, idx, new)
    base = trace.base_columns()
    L = 1 << (depth - 1).bit_length()
    assert base.is_cuda and heap.is_cuda and tuple(base.shape) == (15, 16 * K * L)
    assert np.array_equal(_host(base), _mont_cols(rows))
    assert [list(r) for r in roots] == want_roots
    got = _host(heap)
    assert got[0].tolist() == [0, 0, 0, 0] and got[1:].tolist() == want_heap[1:]
    # the heap in host memory gives the same trace, roots and heap
    trace2, heap2, roots2 = M.update(_host(nodes).copy(), depth, idx, new, device=0)
    assert torch.equal(trace2.base_columns(), base) and torch.equal(heap2, heap) and roots2 == roots
    from ministark_b200 import Context
    ctx = Context(0)
    host_heap, out, host_roots = _host(nodes).copy(), torch.zeros_like(base), np.zeros((K + 1, 4), dtype=np.uint64)
    ctx.rescue_merkle_updates(host_heap, depth, np.array(idx, dtype=np.uint64), np.array(new, dtype=np.uint64), K, out,
                              host_roots)
    ctx.sync()
    assert torch.equal(out, base) and np.array_equal(host_heap, got) and host_roots.tolist() == want_roots


def test_device_refuses_bad_arguments():
    from ministark_b200 import Context, MsError
    ctx = Context(0)
    nodes = M.tree(torch.arange(32, dtype=torch.int64, device="cuda").reshape(8, 4), device=0)
    heap = nodes.clone()
    out = torch.zeros((15, 256), dtype=torch.int64, device="cuda")
    roots = torch.zeros((5, 4), dtype=torch.int64, device="cuda")
    idx = torch.tensor([1, 7, 8, 2], dtype=torch.int64, device="cuda")
    lv = torch.arange(16, dtype=torch.int64, device="cuda").reshape(4, 4)
    bad_lv = lv.clone()
    bad_lv[2, 1] = 1 - 2**32                                 # the word p = 2^64 - 2^32 + 1 as an int64
    for args, msg in [((heap, 3, idx, lv, 3), "not a power of two"), ((heap, 3, None, lv, 4), "null argument"),
                      ((heap, 0, idx, lv, 4), "outside 1..32"), ((heap, 3, idx, lv, 4), "index 8 of write 2 is not below 2\\^3"),
                      ((heap, 3, idx % 8, bad_lv, 4), f"word 1 of new leaf 2 \\({P}\\) is not canonical"),
                      ((heap, 1, idx, lv, 1 << 30), "exceed 2\\^32")]:
        with pytest.raises(MsError, match=msg):
            ctx.rescue_merkle_updates(*args, out, roots)
    ctx.sync()
    assert torch.equal(heap, nodes) and not out.any() and not roots.any()     # refused before anything was written


# ------------------------------------------------------------------------------------------ the golden shape
@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "rescue_merkle_updates_d16_k1024.json")) as f:
        gold = json.load(f)
    depth, K, seed = gold["depth"], gold["K"], gold["seed"]
    nodes = M.tree(leaves(depth, seed), device=0)
    idx, new = writes(K, depth, seed)
    trace, heap, roots = M.update(nodes, depth, idx, new, device=0)
    return gold, idx, new, trace, heap, roots


def test_golden_update(golden):
    gold, _, _, trace, heap, roots = golden
    assert list(roots[0]) == gold["old_root"] and list(roots[-1]) == gold["new_root"]
    assert [list(r) for r in roots[:4]] == gold["first_roots"]
    assert heap_sha256(_host(heap)) == gold["heap_sha256"]
    assert hashlib.sha256(_host(trace.base_columns()).tobytes()).hexdigest() == gold["trace_sha256"]


def test_golden_proof_verifies(golden):
    gold, idx, new, trace, _, roots = golden
    claim = M.MerkleUpdatesClaim(gold["depth"], roots[0], roots[-1], idx, new)
    proof = GpuProver(0).prove(claim, M.OPTIONS, trace)
    claim.verify(proof.to_bytes(), M.SECURITY_LEVEL)


def test_benchmark_depth_final_root_equals_rebuilt_tree():
    depth, K = 24, 1 << 14
    lv = leaves(depth, 2)
    idx, new = writes(K, depth, 2)
    nodes = M.tree(lv, device=0)
    _, heap, roots = M.update(nodes, depth, idx, new, device=0)
    final = lv.copy()
    for i, leaf in zip(idx.tolist(), new):                   # one after another: the last write to a leaf wins
        final[i] = leaf
    rebuilt = M.tree(final, device=0)
    assert roots[-1] == M.root(rebuilt) and roots[0] == M.root(nodes)
    assert torch.equal(heap, rebuilt)


# ------------------------------------------------------------------ device-trace proofs against the CPU harness's
DEPTH14, K14, SEED14 = 5, 128, 3    # L = 8: 2^14 rows


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
        for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS, _lib._RESCUE_SIGS,
                     _lib._RESCUE_MERKLE_SIGS, _lib._RESCUE_MERKLE_UPDATES_SIGS):
            _lib.bind(lib, sigs)
        _lib._lib = lib
        nodes = M.tree(leaves(DEPTH14, SEED14), device="cpu")
        idx, new = _writes(DEPTH14, K14, "siblings", SEED14)
        trace, _, roots = M.update(nodes, DEPTH14, idx, new, device="cpu")
        claim = M.MerkleUpdatesClaim(DEPTH14, roots[0], roots[-1], idx, new)
        q.put(GpuProver(0).prove(claim, M.OPTIONS, trace).to_bytes())
    except Exception:
        import traceback
        q.put(traceback.format_exc())


def _case14():
    nodes = M.tree(leaves(DEPTH14, SEED14), device=0)
    idx, new = _writes(DEPTH14, K14, "siblings", SEED14)
    trace, _, roots = M.update(nodes, DEPTH14, idx, new, device=0)
    return M.MerkleUpdatesClaim(DEPTH14, roots[0], roots[-1], idx, new), trace


def test_device_trace_proofs_equal_cpu_harness(tmp_path):
    import torch.multiprocessing as mp
    lib = str(tmp_path / "libms_rescue_merkle_updates_cpu_abi.so")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "libms_cpu_abi.so"])
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", lib,
                           os.path.join(ROOT, "tests", "cpp", "rescue_merkle_updates_cpu_abi.c")])
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
                got = prover.prove(claim, M.OPTIONS, trace, validate=True).to_bytes()
                assert prover.last_residency == residency
                assert got == want, (residency, no_jit)
        finally:
            os.environ.pop("MS_EVAL_NO_JIT", None)
    claim.verify(want, M.SECURITY_LEVEL)


def test_broken_root_link_names_chain_and_its_row():
    from ministark_b200.validate import ConstraintViolation
    claim, trace = _case14()
    L = 8
    groups = M.updates_air_config(K14, DEPTH14).groups(len(trace))
    k = 37                                                   # write 37's old path rebuilt from another old leaf
    base = trace.base_columns()
    start = 16 * L * k
    cur = None
    for j in range(L):
        at = start + 8 * j
        state = [int(w) * pow(2**64, -1, P) % P for w in _host(base[:12, at])]
        bit = int(_host(base[12, at:at + 1])[0]) != 0
        if cur is None:
            cur = state[4:8] if bit else state[:4]
            cur[0] = (cur[0] + 1) % P
        sib = state[:4] if bit else state[4:8]
        states = R.round_states((sib + cur if bit else cur + sib) + [0] * 4)
        block = np.array([[w * 2**64 % P for w in st] for st in states], dtype=np.uint64).T
        base[:12, at:at + 8] = torch.from_numpy(np.ascontiguousarray(block).view(np.int64)).to(base.device)
        cur = states[-1][:4]
    chain_row = 16 * L * (k - 1) + 8 * L + 8 * DEPTH14 - 1  # write 36's new root, where write 37's old root is read
    with pytest.raises(ConstraintViolation) as e:
        GpuProver(0).prove(claim, M.OPTIONS, trace, validate=True)
    by_constraint = {v.constraint: v.first_row for v in e.value.violations}
    assert by_constraint and all(c in groups["CHAIN"] and r == chain_row for c, r in by_constraint.items()), by_constraint
    assert f"row {chain_row}" in str(e.value)


def test_sharded_prover_on_thread_ranks_gives_the_same_bytes():
    from test_gpu_sharded_one_gpu import _prove_on_thread_ranks
    claim, trace = _case14()
    single = GpuProver(0).prove(claim, M.OPTIONS, trace).to_bytes()
    proofs = _prove_on_thread_ranks(2, claim, M.OPTIONS, trace)
    assert all(p == [single, single] for p in proofs)
