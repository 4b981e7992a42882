"""CPU-only: examples/merkle, K authentication paths in one Rescue-Prime Merkle tree proved against its root.

  * the host tree equals the restated tree (tests/rescue_merkle_oracle.py), and every sibling path() gives re-hashes to
    the root;
  * the CPU build of ms_rescue_merkle_tree and ms_rescue_merkle_paths (tests/cpp/rescue_merkle_cpu_abi.c, through
    `tree(..., device="cpu")` and `gen_trace(..., device="cpu")` on the CPU harness, tests/cpu_device.py) equals the
    restatement word for word, and bad arguments are refused before anything is written;
  * the restated trace satisfies every constraint (oracle/check_oracle.py, with R from oracle/extension_oracle.py) at
    L = 1, at D = L and at a D that is not a power of two (filler permutations); the constraint counts and the ce
    blow-up of 8; a flipped BIT, a flipped sibling word, a wrong IDX and a non-zero capacity word each break their group;
  * 2^12-row proofs verify with Stark.verify and oracle/stark_oracle.verify, resident and streamed give the same bytes,
    and a different root, a changed leaf word, a changed index and an index moved into the filler range are refused.
Harness cases run in spawned workers that install it themselves; the pytest process never does."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rescue_merkle_oracle as MO  # noqa: E402

P = 2**64 - 2**32 + 1
# (depth, K): L = 1; D = L = 2; D = 3 < L = 4 (one filler permutation); D = L = 4; D = 5 < L = 8 (three fillers)
SHAPES = [(1, 4), (2, 2), (3, 8), (4, 4), (5, 2)]


def leaves_of(depth, salt=0):
    """2^depth leaves of four canonical words, some near p"""
    rng = random.Random(1000 * depth + salt)
    return [tuple(P - 1 - rng.randrange(4) if rng.random() < 0.1 else rng.randrange(P) for _ in range(4))
            for _ in range(1 << depth)]


def indices_of(depth, K, salt=0):
    """K indices in 0..2^depth - 1, the first and last leaf and a repeat among them"""
    rng = random.Random(77 * depth + K + salt)
    idx = [rng.randrange(1 << depth) for _ in range(K)]
    idx[0] = (1 << depth) - 1
    if K > 2:
        idx[1], idx[2] = 0, idx[0]
    return idx


def _mont_cols(rows):
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T.copy()


# ------------------------------------------------------------------------------------------------------- the tree
def test_host_tree_equals_oracle():
    from ministark_b200.examples import merkle as M
    for depth in (1, 2, 3, 5, 6):
        leaves = leaves_of(depth)
        nodes = M.tree(leaves)
        want = MO.heap(leaves)
        assert len(nodes) == 2 << depth and nodes[0] == (0, 0, 0, 0)
        assert [list(v) for v in nodes[1:]] == want[1:], depth
        assert list(M.root(nodes)) == want[1]
    assert M.merge((1, 2, 3, 4), (5, 6, 7, 8)) == tuple(MO.compress([1, 2, 3, 4], [5, 6, 7, 8]))


def test_merge_is_one_permutation_not_the_padded_hash():
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rescue as R
    a, b = (1, 2, 3, 4), (5, 6, 7, 8)
    assert M.merge(a, b) == tuple(R.permute(list(a + b) + [0] * 4)[:4])
    assert M.merge(a, b) != R.hash(a + b)


def test_every_path_rehashes_to_the_root():
    from ministark_b200.examples import merkle as M
    depth = 6
    nodes = M.tree(leaves_of(depth))
    for index in range(1 << depth):
        acc = nodes[(1 << depth) + index]
        sibs = M.path(nodes, depth, index)
        assert len(sibs) == depth
        for j, sib in enumerate(sibs):
            acc = M.merge(sib, acc) if (index >> j) & 1 else M.merge(acc, sib)
        assert acc == M.root(nodes), index


def test_host_trace_equals_oracle():
    from ministark_b200.examples import merkle as M
    for depth, K in SHAPES:
        leaves = leaves_of(depth)
        idx = indices_of(depth, K)
        trace, got_leaves = M.gen_trace(M.tree(leaves), depth, idx)
        rows, want_leaves, roots = MO.paths_trace(MO.heap(leaves), depth, idx)
        assert np.array_equal(trace.base_columns(), _mont_cols(rows)), (depth, K)
        assert [list(v) for v in got_leaves] == want_leaves
        assert all(r == MO.heap(leaves)[1] for r in roots)


def test_bad_shapes_refused():
    from ministark_b200.examples import merkle as M
    nodes = M.tree(leaves_of(3))
    root, leaf = M.root(nodes), nodes[8]
    for depth, idx in [(3, [0, 1, 2]), (3, [8]), (3, [-1]), (0, [0]), (33, [0]), (3, [])]:
        with pytest.raises(ValueError):
            M.gen_trace(nodes, depth, idx)
        with pytest.raises(ValueError):
            M.MerklePathsClaim(depth, root, [leaf] * len(idx), idx)
    with pytest.raises(ValueError):
        M.air_config(1 << 30, 1)                                               # 8 K L = 2^33 rows
    with pytest.raises(ValueError):
        M.MerklePathsClaim(3, root, [leaf, leaf], [0])                         # two leaves, one index
    with pytest.raises(ValueError):
        M.MerklePathsClaim(3, (1, 2, 3, P), [leaf], [0])                       # root not canonical
    with pytest.raises(ValueError):
        M.MerklePathsClaim(3, root, [(0, 0, 0, P)], [0])                       # leaf not canonical
    for bad in ([(1, 2, 3, 4)] * 3, [(1, 2, 3, 4)], [(1, 2, 3, P)] * 2, [(1, 2, 3)] * 2):
        with pytest.raises(ValueError):
            M.tree(bad)
    with pytest.raises(ValueError):
        M.air_config(4, 3).constraints(8 * 4 * 2)                              # depth 3 takes L = 4, not 2
    assert M.air_config(4, 3) is M.air_config(4, 3)


# ------------------------------------------------------------------------------------------- the CPU stand-in
@pytest.fixture(scope="module")
def rescue_merkle_abi(tmp_path_factory, orc):
    """tests/cpp/rescue_merkle_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary
    directory"""
    out = str(tmp_path_factory.mktemp("rescue_merkle_abi") / "libms_rescue_merkle_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "cpp", "rescue_merkle_cpu_abi.c")])
    return out


def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS, _lib._RESCUE_SIGS, _lib._RESCUE_MERKLE_SIGS):
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


def _stand_in(shapes):
    from ministark_b200.examples import merkle as M
    out = []
    for depth, K in shapes:
        nodes = M.tree(np.array(leaves_of(depth), dtype=np.uint64), device="cpu")
        trace, leaves = M.gen_trace(nodes, depth, indices_of(depth, K), device="cpu")
        out.append((nodes.numpy().view(np.uint64).copy(), trace.base_columns().numpy().view(np.uint64).copy(), leaves))
    return out


def test_stand_in_tree_and_trace_equal_oracle(rescue_merkle_abi):
    got = _spawn(_worker, rescue_merkle_abi, _stand_in, (SHAPES,))
    assert isinstance(got, list), got
    for (depth, K), (nodes, cols, leaves) in zip(SHAPES, got):
        heap = MO.heap(leaves_of(depth))
        assert nodes[0].tolist() == [0, 0, 0, 0] and nodes[1:].tolist() == heap[1:], depth
        rows, want_leaves, _ = MO.paths_trace(heap, depth, indices_of(depth, K))
        assert np.array_equal(cols, _mont_cols(rows)), (depth, K)
        assert [list(v) for v in leaves] == want_leaves


def _stand_in_errors():
    from ministark_b200 import Context, MsError
    import torch
    ctx, msgs = Context(0), []
    nodes, out = torch.zeros((16, 4), dtype=torch.int64), torch.zeros((14, 64), dtype=torch.int64)
    leaves = np.arange(32, dtype=np.uint64).reshape(8, 4)
    for args in [(None, 3, nodes), (leaves, 0, nodes), (leaves, 33, nodes)]:
        try:
            ctx.rescue_merkle_tree(*args)
            msgs.append(None)
        except MsError as e:
            msgs.append(str(e))
    idx = np.array([1, 7, 8, 2], dtype=np.uint64)
    for args in [(nodes, 3, idx[:3], 3), (nodes, 3, None, 1), (nodes, 0, idx, 4), (nodes, 3, idx, 4),
                 (nodes, 1, idx, 1 << 30)]:                        # refused on its shape, before the indices
        try:
            ctx.rescue_merkle_paths(args[0], args[1], args[2], args[3], out)
            msgs.append(None)
        except MsError as e:
            msgs.append(str(e))
    return msgs, bool(nodes.any()), bool(out.any())


def test_stand_in_refuses_bad_arguments(rescue_merkle_abi):
    got = _spawn(_worker, rescue_merkle_abi, _stand_in_errors, ())
    assert isinstance(got, tuple), got
    msgs, nodes_written, out_written = got
    assert "null argument" in msgs[0] and "outside 1..32" in msgs[1] and "outside 1..32" in msgs[2]
    assert "not a power of two" in msgs[3] and "null argument" in msgs[4] and "outside 1..32" in msgs[5]
    assert "index 8 of path 2 is not below 2^3" in msgs[6] and "exceed 2^32" in msgs[7]
    assert not nodes_written and not out_written


# ------------------------------------------------------------------------------------------------------- the AIR
def _check(depth, rows, leaves, idx, root):
    from ministark_b200.examples import merkle as M
    from oracle import check_oracle, extension_oracle
    base = _mont_cols(rows)
    n = base.shape[1]
    claim = M.MerklePathsClaim(depth, root, leaves, idx)
    cfg = claim.AirConfig
    gamma = (123456789, 987654321, 55555)
    hints = cfg.gen_hints(n, claim, [gamma])
    ext = extension_oracle.builder(cfg, base, claim)([gamma])
    cons = [c.to_tuple() for c in cfg.constraints(n)]
    got = check_oracle.check(cons, n.bit_length() - 1, base, ext, 3, [gamma], hints)
    return [k for k, (first, _) in enumerate(got) if first is not None], ext, hints


@pytest.mark.parametrize("depth,K", SHAPES)
def test_oracle_trace_satisfies_every_constraint(depth, K):
    from ministark_b200.examples import merkle as M
    heap = MO.heap(leaves_of(depth))
    idx = indices_of(depth, K)
    rows, leaves, _ = MO.paths_trace(heap, depth, idx)
    failing, ext, hints = _check(depth, rows, leaves, idx, heap[1])
    assert failing == []
    n = len(rows)
    L = n // (8 * K)
    cfg = M.air_config(K, depth)
    groups = cfg.groups(n)
    # ROUND 12, CAP 4, LINK 4 (none at L = 1), BIT 2, IDX 3 (2 at L = 1), ROOT 4, R 4
    assert len(cfg.constraints(n)) == (28 if L == 1 else 33)
    assert ([len(groups[g]) for g in ("ROUND", "CAP", "LINK", "BIT", "IDX", "ROOT", "R")]
            == [12, 4, 0 if L == 1 else 4, 2, 2 if L == 1 else 3, 4, 4])
    # R's last row is the Horner evaluation gen_hints makes from the public (leaf, index) tuples
    last = tuple(int(w) * pow(2**64, -1, P) % P for w in ext[0, 3 * (n - 1):])
    assert last == tuple(hints[0])


def test_tuple_evaluation_is_horner_over_five_words():
    """digest_evaluation of 5-tuples equals acc <- acc gamma^5 + t_0 + gamma t_1 + ... + gamma^4 t_4"""
    from ministark_b200 import expr as E
    from ministark_b200.examples import rescue as R
    rng = random.Random(9)
    for K in (1, 2, 205, 1024, 1500):
        tuples = [tuple(rng.randrange(P) for _ in range(5)) for _ in range(K)]
        gamma = tuple(rng.randrange(P) for _ in range(3))
        gp = [(1, 0, 0)]
        for _ in range(5):
            gp.append(E.q_mul(gp[-1], gamma))
        acc = (0, 0, 0)
        for t in tuples:
            acc = E.q_mul(acc, gp[5])
            for w in range(5):
                acc = E.q_add(acc, E.q_mul(gp[w], (t[w], 0, 0)))
        assert R.digest_evaluation(tuples, gamma) == acc, K


def test_ce_blowup_is_8():
    from ministark_b200.examples import merkle as M
    from oracle import air_oracle
    for depth, K in SHAPES + [(16, 1 << 15), (24, 1 << 14), (32, 1 << 24), (1, 1 << 29)]:
        L = 1 << (depth - 1).bit_length()
        n = 8 * K * L
        if n < 16:                      # at 8 rows y = x^(n / 8) is x itself (as for the rescue AIRs)
            continue
        cons = [c.to_tuple() for c in M.air_config(K, depth).constraints(n)]
        assert air_oracle.composition_constraint(cons, n)[1] == 8, (depth, K)


def test_changes_break_their_constraints():
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rescue as R
    depth, K = 5, 4                                     # L = 8: 64 rows per path, permutations 5..7 are fillers
    heap = MO.heap(leaves_of(depth))
    idx = indices_of(depth, K)
    rows, leaves, _ = MO.paths_trace(heap, depth, idx)
    groups = M.air_config(K, depth).groups(len(rows))
    k, j = 2, 2
    base = 64 * k + 8 * j                               # permutation j of path k

    def fails(bad, group):
        failing, _, _ = _check(depth, bad, leaves, idx, heap[1])
        return any(c in groups[group] for c in failing), failing

    bad = [list(r) for r in rows]
    bad[base + 3][12] ^= 1                              # BIT on one row of the permutation
    assert fails(bad, "BIT")[0]
    bad = [list(r) for r in rows]
    bad[base + 5][13] = (bad[base + 5][13] + 1) % P     # IDX on one row
    assert fails(bad, "IDX")[0]
    bad = [list(r) for r in rows]
    bad[base][9] = 1                                    # a capacity word at r = 0
    assert fails(bad, "CAP")[0]
    # a sibling word flipped and permutation j recomputed from it: its output no longer feeds permutation j + 1
    bad = [list(r) for r in rows]
    b = bad[base][12]
    state = list(bad[base][:12])
    state[(0 if b else 4) + 1] ^= 1
    for r, st in enumerate(R.round_states(state)):
        bad[base + r][:12] = st
    ok, failing = fails(bad, "LINK")
    assert ok and all(c in groups["LINK"] for c in failing), failing


# ------------------------------------------------------------------------------------------------------ proofs
OPTS = (40, 8, 8, 8, 64)
DEPTH12, K12 = 5, 64                                   # L = 8: 2^12 rows


def _prove():
    from ministark_b200 import FQ3
    from ministark_b200.air import ProofOptions
    from ministark_b200.examples import merkle as M
    from ministark_b200.prover import GpuProver, peak_bytes
    nodes = M.tree(np.array(leaves_of(DEPTH12), dtype=np.uint64), device="cpu")
    trace, leaves = M.gen_trace(nodes, DEPTH12, indices_of(DEPTH12, K12), device="cpu")
    claim = M.MerklePathsClaim(DEPTH12, M.root(nodes), leaves, indices_of(DEPTH12, K12))
    got = {}
    for residency in ("resident", "streamed"):
        p = GpuProver(0)
        if residency == "streamed":
            est = peak_bytes(len(trace), 8, 14, 1, FQ3, 8, 8)
            p.memory_budget = (est["streamed"] + est["resident"]) // 2
        got[residency] = (p.prove(claim, ProofOptions(*OPTS), trace).to_bytes(), p.last_residency)
    return got, leaves, M.root(nodes)


def test_cpu_harness_proofs_verify(rescue_merkle_abi):
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.examples import merkle as M
    from ministark_b200.verifier import VerificationError
    from oracle import stark_oracle as SO
    got = _spawn(_worker, rescue_merkle_abi, _prove, ())
    assert isinstance(got, tuple), got
    proofs, leaves, root = got
    assert proofs["resident"][1] == "resident" and proofs["streamed"][1] == "streamed"
    assert proofs["resident"][0] == proofs["streamed"][0]
    idx = indices_of(DEPTH12, K12)
    assert root == tuple(MO.heap(leaves_of(DEPTH12))[1])
    claim = M.MerklePathsClaim(DEPTH12, root, leaves, idx)
    proof = proofs["resident"][0]
    claim.verify(proof, M.SECURITY_LEVEL)
    SO.verify(claim, proof, M.SECURITY_LEVEL, lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o)))
    other_root = (root[0], root[1], (root[2] + 1) % P, root[3])
    leaf_changed = [list(v) for v in leaves]
    leaf_changed[9][3] = (leaf_changed[9][3] + 1) % P
    index_changed = list(idx)
    index_changed[17] ^= 4
    # an index moved into the filler range: bit 5 set, which no public index of a depth-5 tree may have
    filler = M.MerklePathsClaim(DEPTH12, root, leaves, idx)
    filler.indices = list(idx)
    filler.indices[5] += 1 << DEPTH12
    for bad in (M.MerklePathsClaim(DEPTH12, other_root, leaves, idx), M.MerklePathsClaim(DEPTH12, root, leaf_changed, idx),
                M.MerklePathsClaim(DEPTH12, root, leaves, index_changed), filler):
        with pytest.raises(VerificationError):
            bad.verify(proof, M.SECURITY_LEVEL)


def test_header_bound_and_exported(rescue_merkle_abi):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.RESCUE_MERKLE_HEADER_PATH)
    assert declared == sorted(_lib._RESCUE_MERKLE_SIGS) == ["ms_rescue_merkle_paths", "ms_rescue_merkle_tree"]
    others = set(_lib.header_symbols())
    for path in (_lib.STREAM_HEADER_PATH, _lib.CHECK_HEADER_PATH, _lib.EXTENSION_HEADER_PATH, _lib.LOOKUP_HEADER_PATH,
                 _lib.BF_HEADER_PATH, _lib.DEVICE_HEADER_PATH, _lib.HOST_NODES_HEADER_PATH, _lib.RESCUE_HEADER_PATH,
                 _lib.RESCUE_HASH_HEADER_PATH):
        others |= set(_lib.header_symbols(path))
    assert not set(declared) & others
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(rescue_merkle_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)
