"""GPU: examples/merkle with the tree and the path trace built on the device (csrc/rescue.cu, ms_rescue_merkle_tree and
ms_rescue_merkle_paths).

  * the device tree and trace equal tests/rescue_merkle_oracle.py word for word at D = 1, at D not a power of two and at
    depths that take the per-level kernel as well as the one-block top levels, with the heap in device or host memory;
    bad arguments are refused before anything is written;
  * at D = 16, K = 2^10 the heap, the root and the trace equal tests/golden/rescue_merkle_d16_k1024.json, which the
    restatement wrote (tests/golden/make_rescue_merkle_golden.py), and the proof verifies;
  * at D = 24 (the benchmark's 2^24-leaf tree) 64 random paths re-hash on the host to the device root;
  * at 2^14 rows the proof bytes from the device trace equal the CPU harness's (tests/cpu_device.py with
    tests/cpp/rescue_merkle_cpu_abi.c, in a spawned worker), resident and streamed, with validate=True;
  * a flipped sibling word raises ConstraintViolation naming LINK and the row that links its permutation onward;
  * ShardedProver with 2 and 4 ranks run as threads on one GPU gives the single-GPU bytes."""
import hashlib
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from make_rescue_merkle_golden import heap_sha256, indices, leaves  # noqa: E402
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


@pytest.mark.parametrize("depth,K", [(1, 4), (2, 2), (3, 8), (5, 16), (6, 4), (7, 64), (9, 32), (11, 8)])
def test_device_tree_and_trace_equal_oracle(depth, K):
    import rescue_merkle_oracle as MO
    lv, idx = leaves(depth, 7), indices(K, depth, 7)
    nodes = M.tree(lv, device=0)
    assert nodes.is_cuda and tuple(nodes.shape) == (2 << depth, 4)
    heap = MO.heap([[int(w) for w in leaf] for leaf in lv])
    got = _host(nodes)
    assert got[0].tolist() == [0, 0, 0, 0] and got[1:].tolist() == heap[1:]
    trace, got_leaves = M.gen_trace(nodes, depth, idx, device=0)
    base = trace.base_columns()
    L = 1 << (depth - 1).bit_length()
    assert base.is_cuda and tuple(base.shape) == (14, 8 * K * L)
    rows, want_leaves, roots = MO.paths_trace(heap, depth, [int(i) for i in idx])
    assert np.array_equal(_host(base), _mont_cols(rows))
    assert [list(v) for v in got_leaves] == want_leaves and all(r == heap[1] for r in roots)
    # the heap and the indices in host memory give the same trace
    from ministark_b200 import Context
    ctx, out = Context(0), torch.zeros_like(base)
    ctx.rescue_merkle_paths(np.ascontiguousarray(got), depth, idx, K, out)
    ctx.sync()
    assert torch.equal(out, base)


def test_device_refuses_bad_arguments():
    from ministark_b200 import Context, MsError
    ctx = Context(0)
    nodes = torch.zeros((16, 4), dtype=torch.int64, device="cuda")
    out = torch.zeros((14, 64), dtype=torch.int64, device="cuda")
    lv = torch.ones((8, 4), dtype=torch.int64, device="cuda")
    for args, msg in [((None, 3, nodes), "null argument"), ((lv, 0, nodes), "outside 1..32"),
                      ((lv, 33, nodes), "outside 1..32")]:
        with pytest.raises(MsError, match=msg):
            ctx.rescue_merkle_tree(*args)
    idx = torch.tensor([1, 7, 8, 2], dtype=torch.int64, device="cuda")
    for args, msg in [((nodes, 3, idx, 3), "not a power of two"), ((nodes, 3, None, 4), "null argument"),
                      ((nodes, 0, idx, 4), "outside 1..32"), ((nodes, 3, idx, 4), "index 8 of path 2 is not below 2\\^3"),
                      ((nodes, 1, idx, 1 << 30), "exceed 2\\^32")]:
        with pytest.raises(MsError, match=msg):
            ctx.rescue_merkle_paths(*args, out)
    ctx.sync()
    assert not nodes.any() and not out.any()                 # refused before anything was written


# ------------------------------------------------------------------------------------------ the golden shape
@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "rescue_merkle_d16_k1024.json")) as f:
        gold = json.load(f)
    depth, K, seed = gold["depth"], gold["K"], gold["seed"]
    nodes = M.tree(leaves(depth, seed), device=0)
    idx = indices(K, depth, seed)
    trace, lv = M.gen_trace(nodes, depth, idx, device=0)
    return gold, nodes, idx, trace, lv


def test_golden_tree_and_trace(golden):
    gold, nodes, idx, trace, _ = golden
    assert list(M.root(nodes)) == gold["root"]
    assert heap_sha256(_host(nodes)) == gold["heap_sha256"]
    assert hashlib.sha256(_host(trace.base_columns()).tobytes()).hexdigest() == gold["trace_sha256"]
    assert [int(i) for i in idx[:8]] == gold["first_indices"]


def test_golden_proof_verifies(golden):
    gold, nodes, idx, trace, lv = golden
    claim = M.MerklePathsClaim(gold["depth"], M.root(nodes), lv, idx)
    proof = GpuProver(0).prove(claim, M.OPTIONS, trace)
    claim.verify(proof.to_bytes(), M.SECURITY_LEVEL)


def test_benchmark_tree_paths_rehash_to_the_root():
    depth = 24
    nodes = M.tree(leaves(depth, 2), device=0)
    root = M.root(nodes)
    rng = random.Random(24)
    for index in [0, (1 << depth) - 1] + [rng.randrange(1 << depth) for _ in range(62)]:
        acc = tuple(int(w) for w in _host(nodes[(1 << depth) + index]))
        for j, sib in enumerate(M.path(nodes, depth, index)):
            acc = M.merge(sib, acc) if (index >> j) & 1 else M.merge(acc, sib)
        assert acc == root, index


# ------------------------------------------------------------------ device-trace proofs against the CPU harness's
DEPTH14, K14, SEED14 = 5, 256, 3    # L = 8: 2^14 rows


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
                     _lib._RESCUE_MERKLE_SIGS):
            _lib.bind(lib, sigs)
        _lib._lib = lib
        nodes = M.tree(leaves(DEPTH14, SEED14), device="cpu")
        idx = indices(K14, DEPTH14, SEED14)
        trace, lv = M.gen_trace(nodes, DEPTH14, idx, device="cpu")
        claim = M.MerklePathsClaim(DEPTH14, M.root(nodes), lv, idx)
        q.put(GpuProver(0).prove(claim, M.OPTIONS, trace).to_bytes())
    except Exception:
        import traceback
        q.put(traceback.format_exc())


def _case14():
    nodes = M.tree(leaves(DEPTH14, SEED14), device=0)
    idx = indices(K14, DEPTH14, SEED14)
    trace, lv = M.gen_trace(nodes, DEPTH14, idx, device=0)
    return M.MerklePathsClaim(DEPTH14, M.root(nodes), lv, idx), trace


def test_device_trace_proofs_equal_cpu_harness(tmp_path):
    import torch.multiprocessing as mp
    lib = str(tmp_path / "libms_rescue_merkle_cpu_abi.so")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "libms_cpu_abi.so"])
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", lib,
                           os.path.join(ROOT, "tests", "cpp", "rescue_merkle_cpu_abi.c")])
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
    est = peak_bytes(len(trace), 8, 14, 1, FQ3, 8, 8)
    for residency, budget in [("resident", None), ("streamed", (est["streamed"] + est["resident"]) // 2)]:
        prover = GpuProver(0, memory_budget=budget)
        got = prover.prove(claim, M.OPTIONS, trace, validate=True).to_bytes()
        assert prover.last_residency == residency
        assert got == want, residency
    claim.verify(want, M.SECURITY_LEVEL)


def test_flipped_sibling_names_link_and_its_row():
    from ministark_b200.validate import ConstraintViolation
    claim, trace = _case14()
    L = 8
    groups = M.air_config(K14, DEPTH14).groups(len(trace))
    k, j = 37, 2                                             # path 37, permutation 2 of 5
    base = trace.base_columns()
    start = 8 * (L * k + j)
    state = [int(w) * pow(2**64, -1, P) % P for w in _host(base[:12, start])]
    bit = int(_host(base[12, start:start + 1])[0]) != 0
    state[(0 if bit else 4) + 2] ^= 1                        # one word of the sibling half
    block = np.array([[w * 2**64 % P for w in st] for st in R.round_states(state)], dtype=np.uint64).T
    base[:12, start:start + 8] = torch.from_numpy(np.ascontiguousarray(block).view(np.int64)).to(base.device)
    link_row = start + 7                                     # permutation 2's output no longer feeds permutation 3
    with pytest.raises(ConstraintViolation) as e:
        GpuProver(0).prove(claim, M.OPTIONS, trace, validate=True)
    by_constraint = {v.constraint: v.first_row for v in e.value.violations}
    assert by_constraint and all(c in groups["LINK"] and r == link_row for c, r in by_constraint.items()), by_constraint
    assert f"row {link_row}" in str(e.value)


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_prover_on_thread_ranks_gives_the_same_bytes(world):
    from test_gpu_sharded_one_gpu import _prove_on_thread_ranks
    claim, trace = _case14()
    single = GpuProver(0).prove(claim, M.OPTIONS, trace).to_bytes()
    proofs = _prove_on_thread_ranks(world, claim, M.OPTIONS, trace)
    assert all(p == [single, single] for p in proofs)
