"""CPU-only: examples/merkle's ordered-write claim, K leaf writes that take one Rescue-Prime Merkle root to another.

  * merkle.update on the host equals the restatement (tests/rescue_merkle_updates_oracle.py): the trace, the K + 1
    roots and the final heap, at D = 1, at D not a power of two, at K = 1, with repeated indices, with consecutive writes
    to i and i ^ 1 and with a write of the leaf's current value; the final heap is tree() of the final leaves;
  * the CPU build of ms_rescue_merkle_updates (tests/cpp/rescue_merkle_updates_cpu_abi.c, through
    `update(..., device="cpu")` on the CPU harness, tests/cpu_device.py) equals the restatement, leaves the caller's
    heap alone, and refuses bad arguments before anything is written;
  * the restated trace satisfies every constraint (oracle/check_oracle.py) at those shapes; the constraint counts and
    the ce blow-up of 8; a sibling word changed in the new path only, a broken root link, a flipped bit, a wrong SIDE
    and a wrong capacity word each break their group;
  * the specialised evaluator's generated source (csrc/eval_jit.cu, compiled here by g++) and the CPU interpreter agree
    on the composition program, whose SIB and CHAIN constraints read the trace 8 L rows ahead;
  * 2^12-row proofs verify with Stark.verify and oracle/stark_oracle.verify, resident and streamed give the same bytes,
    and a wrong old root, new root, new leaf or index, and two writes to one leaf in swapped order, are refused.
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
import rescue_merkle_updates_oracle as UO  # noqa: E402

P = 2**64 - 2**32 + 1
# (depth, K, case): L = 1; D = 3 < L = 4; K = 1; D = L = 4; D = 5 < L = 8 with K = 4
SHAPES = [(1, 4, "repeat"), (3, 8, "siblings"), (3, 1, "single"), (4, 4, "same value"), (5, 4, "repeat"),
          (2, 16, "repeat")]


def leaves_of(depth, salt=0):
    """2^depth leaves of four canonical words, some near p"""
    rng = random.Random(1000 * depth + salt)
    return [tuple(P - 1 - rng.randrange(4) if rng.random() < 0.1 else rng.randrange(P) for _ in range(4))
            for _ in range(1 << depth)]


def writes_of(depth, K, case, salt=0):
    """(indices, new leaves): K writes with, by `case`, a repeated index, consecutive writes to i and i ^ 1, or a write
    of the value the leaf already holds"""
    rng = random.Random(31 * depth + K + salt)
    idx = [rng.randrange(1 << depth) for _ in range(K)]
    new = [tuple(rng.randrange(P) for _ in range(4)) for _ in range(K)]
    if case == "repeat" and K > 2:
        idx[K - 1] = idx[K - 3] = idx[0]
    elif case == "siblings" and K > 3:
        idx[2], idx[3] = idx[1], idx[1] ^ 1
        idx[4] = idx[1]
    elif case == "same value":
        new[1] = leaves_of(depth, salt)[idx[1]] if idx[1] not in idx[:1] else new[0]
    return idx, new


def _mont_cols(rows):
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T.copy()


def _final_leaves(depth, salt, idx, new):
    lv = list(leaves_of(depth, salt))
    for i, leaf in zip(idx, new):
        lv[i] = leaf
    return lv


# ------------------------------------------------------------------------------------------------- the host path
@pytest.mark.parametrize("depth,K,case", SHAPES)
def test_host_update_equals_oracle(depth, K, case):
    from ministark_b200.examples import merkle as M
    lv = leaves_of(depth)
    idx, new = writes_of(depth, K, case)
    nodes = M.tree(lv)
    before = list(nodes)
    trace, heap, roots = M.update(nodes, depth, idx, new)
    assert nodes == before                                          # the caller's heap is left alone
    rows, want_roots, want_heap = UO.updates_trace(MO.heap(lv), depth, idx, new)
    assert np.array_equal(trace.base_columns(), _mont_cols(rows)), (depth, K)
    assert [list(r) for r in roots] == want_roots and roots[0] == M.root(nodes)
    assert [list(v) for v in heap[1:]] == want_heap[1:]
    assert heap == M.tree(_final_leaves(depth, 0, idx, new))
    if case == "same value":
        assert roots[2] == roots[1]                                 # rewriting a leaf's value leaves the root


def test_bad_shapes_refused():
    from ministark_b200.examples import merkle as M
    nodes = M.tree(leaves_of(3))
    root, leaf = M.root(nodes), (1, 2, 3, 4)
    for depth, idx in [(3, [0, 1, 2]), (3, [8]), (3, [-1]), (0, [0]), (33, [0]), (3, [])]:
        with pytest.raises(ValueError):
            M.update(nodes, depth, idx, [leaf] * len(idx))
        with pytest.raises(ValueError):
            M.MerkleUpdatesClaim(depth, root, root, idx, [leaf] * len(idx))
    with pytest.raises(ValueError):
        M.update(nodes, 3, [0, 1], [leaf])                                     # two indices, one leaf
    with pytest.raises(ValueError):
        M.update(nodes, 3, [0], [(0, 0, 0, P)])                                # new leaf not canonical
    with pytest.raises(ValueError):
        M.update(nodes[:-2], 3, [0], [leaf])                                   # not a heap of depth 3
    with pytest.raises(ValueError):
        M.MerkleUpdatesClaim(3, root, (1, 2, 3, P), [0], [leaf])               # new root not canonical
    with pytest.raises(ValueError):
        M.updates_air_config(1 << 29, 1)                                       # 16 K L = 2^33 rows
    with pytest.raises(ValueError):
        M.updates_air_config(4, 3).constraints(16 * 4 * 2)                     # depth 3 takes L = 4, not 2
    assert M.updates_air_config(4, 3) is M.updates_air_config(4, 3)
    assert M.updates_air_config(4, 3) is not M.air_config(4, 3)


# ------------------------------------------------------------------------------------------- the CPU stand-in
@pytest.fixture(scope="module")
def updates_abi(tmp_path_factory, orc):
    """tests/cpp/rescue_merkle_updates_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary
    directory"""
    out = str(tmp_path_factory.mktemp("rescue_merkle_updates_abi") / "libms_rescue_merkle_updates_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "cpp", "rescue_merkle_updates_cpu_abi.c")])
    return out


def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS, _lib._RESCUE_SIGS, _lib._RESCUE_MERKLE_SIGS,
                 _lib._RESCUE_MERKLE_UPDATES_SIGS):
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
    for depth, K, case in shapes:
        nodes = M.tree(np.array(leaves_of(depth), dtype=np.uint64), device="cpu")
        before = nodes.clone()
        idx, new = writes_of(depth, K, case)
        trace, heap, roots = M.update(nodes, depth, idx, new, device="cpu")
        _, heap_from_list, roots_from_list = M.update(M.tree(leaves_of(depth)), depth, idx, new, device="cpu")
        out.append((trace.base_columns().numpy().view(np.uint64).copy(), heap.numpy().view(np.uint64).copy(), roots,
                    bool((nodes == before).all()), bool((heap_from_list == heap).all()) and roots_from_list == roots))
    return out


def test_stand_in_update_equals_oracle(updates_abi):
    got = _spawn(_worker, updates_abi, _stand_in, (SHAPES,))
    assert isinstance(got, list), got
    for (depth, K, case), (cols, heap, roots, untouched, same_from_list) in zip(SHAPES, got):
        idx, new = writes_of(depth, K, case)
        rows, want_roots, want_heap = UO.updates_trace(MO.heap(leaves_of(depth)), depth, idx, new)
        assert np.array_equal(cols, _mont_cols(rows)), (depth, K)
        assert [list(r) for r in roots] == want_roots
        assert heap[0].tolist() == [0, 0, 0, 0] and heap[1:].tolist() == want_heap[1:]
        assert untouched and same_from_list


def _stand_in_errors():
    from ministark_b200 import Context, MsError
    import torch
    from ministark_b200.examples import merkle as M
    ctx, msgs = Context(0), []
    nodes = M.tree(np.arange(32, dtype=np.uint64).reshape(8, 4), device="cpu")
    heap = nodes.clone()
    out, roots = torch.zeros((15, 256), dtype=torch.int64), torch.zeros((5, 4), dtype=torch.int64)
    idx = np.array([1, 7, 8, 2], dtype=np.uint64)
    lv = np.arange(16, dtype=np.uint64).reshape(4, 4)
    bad_lv = lv.copy()
    bad_lv[2, 1] = P
    for args in [(heap, 3, idx[:3], lv[:3], 3), (heap, 3, None, lv, 4), (heap, 0, idx, lv, 4), (heap, 33, idx, lv, 4),
                 (heap, 3, idx, lv, 4), (heap, 3, idx % 8, bad_lv, 4), (heap, 1, idx, lv, 1 << 30)]:
        try:
            ctx.rescue_merkle_updates(*args, out, roots)
            msgs.append(None)
        except MsError as e:
            msgs.append(str(e))
    return msgs, bool((heap == nodes).all()), bool(out.any()), bool(roots.any())


def test_stand_in_refuses_bad_arguments(updates_abi):
    got = _spawn(_worker, updates_abi, _stand_in_errors, ())
    assert isinstance(got, tuple), got
    msgs, heap_untouched, out_written, roots_written = got
    assert "not a power of two" in msgs[0] and "null argument" in msgs[1]
    assert "outside 1..32" in msgs[2] and "outside 1..32" in msgs[3]
    assert "index 8 of write 2 is not below 2^3" in msgs[4]
    assert f"word 1 of new leaf 2 ({P}) is not canonical" in msgs[5] and "exceed 2^32" in msgs[6]
    assert heap_untouched and not out_written and not roots_written


def test_header_bound_and_exported(updates_abi):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.RESCUE_MERKLE_UPDATES_HEADER_PATH)
    assert declared == sorted(_lib._RESCUE_MERKLE_UPDATES_SIGS) == ["ms_rescue_merkle_updates"]
    others = set(_lib.header_symbols())
    for path in (_lib.STREAM_HEADER_PATH, _lib.CHECK_HEADER_PATH, _lib.EXTENSION_HEADER_PATH, _lib.LOOKUP_HEADER_PATH,
                 _lib.PERMUTATION_HEADER_PATH, _lib.BF_HEADER_PATH, _lib.DEVICE_HEADER_PATH, _lib.HOST_NODES_HEADER_PATH,
                 _lib.RESCUE_HEADER_PATH, _lib.RESCUE_HASH_HEADER_PATH, _lib.RESCUE_MERKLE_HEADER_PATH):
        others |= set(_lib.header_symbols(path))
    assert not set(declared) & others
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(updates_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)


# ------------------------------------------------------------------------------------------------------- the AIR
def _check(depth, rows, roots, idx, new):
    from ministark_b200.examples import merkle as M
    from oracle import check_oracle, extension_oracle
    base = _mont_cols(rows)
    n = base.shape[1]
    claim = M.MerkleUpdatesClaim(depth, roots[0], roots[-1], idx, new)
    cfg = claim.AirConfig
    gamma = (123456789, 987654321, 55555)
    hints = cfg.gen_hints(n, claim, [gamma])
    ext = extension_oracle.builder(cfg, base, claim)([gamma])
    cons = [c.to_tuple() for c in cfg.constraints(n)]
    got = check_oracle.check(cons, n.bit_length() - 1, base, ext, 3, [gamma], hints)
    return {k: first for k, (first, _) in enumerate(got) if first is not None}, ext, hints


@pytest.mark.parametrize("depth,K,case", SHAPES)
def test_oracle_trace_satisfies_every_constraint(depth, K, case):
    from ministark_b200.examples import merkle as M
    idx, new = writes_of(depth, K, case)
    rows, roots, _ = UO.updates_trace(MO.heap(leaves_of(depth)), depth, idx, new)
    failing, ext, hints = _check(depth, rows, roots, idx, new)
    assert failing == {}
    n = len(rows)
    L = n // (16 * K)
    cfg = M.updates_air_config(K, depth)
    groups = cfg.groups(n)
    sizes = [12, 4, 0 if L == 1 else 4, 3, 5, 2, 2 if L == 1 else 3, 8, 0 if K == 1 else 4, 4]
    assert [len(groups[g]) for g in ("ROUND", "CAP", "LINK", "SIDE", "SIB", "BIT", "IDX", "ROOT", "CHAIN", "R")] == sizes
    assert len(cfg.constraints(n)) == sum(sizes)
    last = tuple(int(w) * pow(2**64, -1, P) % P for w in ext[0, 3 * (n - 1):])
    assert last == tuple(hints[0])


def test_ce_blowup_is_8_and_options_are_rescues():
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rescue as R
    from oracle import air_oracle
    assert M.OPTIONS is R.OPTIONS
    for depth, K in [(2, 2), (3, 8), (5, 32), (16, 1 << 15), (24, 1 << 14), (32, 1 << 23), (1, 1 << 28)]:
        L = 1 << (depth - 1).bit_length()
        n = 16 * K * L
        cons = [c.to_tuple() for c in M.updates_air_config(K, depth).constraints(n)]
        assert air_oracle.composition_constraint(cons, n)[1] == 8, (depth, K)


def test_changes_break_their_constraints():
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rescue as R
    depth, K = 5, 4                                     # L = 8: 64 rows per path, permutations 5..7 are fillers
    idx, new = writes_of(depth, K, "repeat")
    rows, roots, _ = UO.updates_trace(MO.heap(leaves_of(depth)), depth, idx, new)
    groups = M.updates_air_config(K, depth).groups(len(rows))
    k, j = 2, 2
    base = 128 * k + 8 * j                              # permutation j of write k's old path; its new path's is 64 on

    def failing(bad):
        return _check(depth, bad, roots, idx, new)[0]

    def rehash(bad, at, state):
        for r, st in enumerate(R.round_states(state)):
            bad[at + r][:12] = st
        return st[:4]

    bad = [list(r) for r in rows]
    bad[base + 3][12] ^= 1                              # BIT on one row of the permutation
    assert set(failing(bad)) & set(groups["BIT"])
    bad = [list(r) for r in rows]
    bad[base + 64][9] = 1                               # a capacity word of the new path at r = 0
    assert set(failing(bad)) & set(groups["CAP"])
    bad = [list(r) for r in rows]
    bad[base + 64 + 5][14] = 0                          # SIDE on one row of the new path
    assert set(failing(bad)) & set(groups["SIDE"])
    # a sibling word changed in the new path only, its permutation j recomputed from it
    bad = [list(r) for r in rows]
    state = list(bad[base + 64][:12])
    state[(0 if bad[base][12] else 4) + 1] ^= 1
    rehash(bad, base + 64, state)
    got = failing(bad)
    assert set(got) & set(groups["SIB"]) and got[groups["SIB"][1]] == base, got
    # a broken root link: write 1's old path rebuilt from another old leaf, consistent in itself
    bad = [list(r) for r in rows]
    cur = list(bad[128][0:4]) if not bad[128][12] else list(bad[128][4:8])
    cur[0] = (cur[0] + 1) % P
    for jj in range(8):
        at = 128 + 8 * jj
        b = bad[at][12]
        sib = list(bad[at][4:8]) if not b else list(bad[at][0:4])
        cur = rehash(bad, at, (sib + cur if b else cur + sib) + [0] * 4)
    got = failing(bad)
    assert got and all(c in groups["CHAIN"] for c in got), got
    assert set(got.values()) == {64 + 8 * depth - 1}    # write 0's new root, where write 1's old root is read 64 on


# ------------------------------------------------------------------------- the evaluator at a row offset of 8 L
def test_generated_kernel_source_reads_chain_offset_like_the_interpreter(tmp_path, orc):
    """the composition program of a K = 4, D = 3 AIR (CHAIN and SIB read 32 rows ahead), the generated kernel source
    against the CPU interpreter on random columns"""
    from test_eval_jit_source import GENERATOR, _host_kernel, _tables
    from ministark_b200.air import Air
    from ministark_b200.examples import merkle as M
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "libms_cpu_abi.so"])
    lib = C.CDLL(os.path.join(ROOT, "oracle", "libms_cpu_abi.so"))
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    rng = random.Random(5)
    depth, K = 3, 4
    claim = M.MerkleUpdatesClaim(depth, (1, 2, 3, 4), (5, 6, 7, 8), [1, 2, 3, 1], [(9, 9, 9, 9)] * K)
    air = Air(claim.AirConfig, 16 * K * 4, claim, M.OPTIONS)
    assert any(o == 32 for _, o in air.trace_arguments())
    q3 = lambda: tuple(rng.randrange(P) for _ in range(3))
    prog = air.composition_program().bind(challenges=[q3() for _ in range(32)], hints=[q3() for _ in range(256)],
                                          ccoefs=[q3() for _ in range(256)])
    log_m = air.log_n + air.ce_blowup_factor.bit_length() - 1
    m = 1 << log_m
    base = orc.rand_matrix(15, m, 1, seed=rng.randrange(1 << 30))
    ext = orc.rand_matrix(1, m, 3, seed=rng.randrange(1 << 30))
    cols = [np.ascontiguousarray(c) for c in base] + [np.ascontiguousarray(ext[0])]
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
OPTS = (40, 8, 8, 8, 64)
DEPTH12, K12 = 5, 32                                   # L = 8: 2^12 rows


def _writes12():
    idx, new = writes_of(DEPTH12, K12, "siblings", salt=12)
    idx[25] = idx[10]                                   # two writes to one leaf, with different values
    return idx, new


def _prove():
    from ministark_b200 import FQ3
    from ministark_b200.air import ProofOptions
    from ministark_b200.examples import merkle as M
    from ministark_b200.prover import GpuProver, peak_bytes
    nodes = M.tree(np.array(leaves_of(DEPTH12), dtype=np.uint64), device="cpu")
    idx, new = _writes12()
    trace, _, roots = M.update(nodes, DEPTH12, idx, new, device="cpu")
    claim = M.MerkleUpdatesClaim(DEPTH12, roots[0], roots[-1], idx, new)
    got = {}
    for residency in ("resident", "streamed"):
        p = GpuProver(0)
        if residency == "streamed":
            est = peak_bytes(len(trace), 8, 15, 1, FQ3, 8, 8)
            p.memory_budget = (est["streamed"] + est["resident"]) // 2
        got[residency] = (p.prove(claim, ProofOptions(*OPTS), trace).to_bytes(), p.last_residency)
    return got, roots


def test_cpu_harness_proofs_verify(updates_abi):
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.examples import merkle as M
    from ministark_b200.verifier import VerificationError
    from oracle import stark_oracle as SO
    got = _spawn(_worker, updates_abi, _prove, ())
    assert isinstance(got, tuple), got
    proofs, roots = got
    assert proofs["resident"][1] == "resident" and proofs["streamed"][1] == "streamed"
    assert proofs["resident"][0] == proofs["streamed"][0]
    idx, new = _writes12()
    _, want_roots, _ = UO.updates_trace(MO.heap(leaves_of(DEPTH12)), DEPTH12, idx, new)
    assert [list(r) for r in roots] == want_roots
    old, fresh = roots[0], roots[-1]
    claim = M.MerkleUpdatesClaim(DEPTH12, old, fresh, idx, new)
    proof = proofs["resident"][0]
    claim.verify(proof, M.SECURITY_LEVEL)
    SO.verify(claim, proof, M.SECURITY_LEVEL, lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o)))
    other = lambda r: (r[0], r[1], (r[2] + 1) % P, r[3])
    leaf_changed = [list(v) for v in new]
    leaf_changed[9][3] = (leaf_changed[9][3] + 1) % P
    index_changed = list(idx)
    index_changed[17] ^= 4
    swapped = list(new)                                 # the two writes to idx[10] in the other order
    swapped[10], swapped[25] = new[25], new[10]
    assert swapped != new
    for bad in (M.MerkleUpdatesClaim(DEPTH12, other(old), fresh, idx, new),
                M.MerkleUpdatesClaim(DEPTH12, old, other(fresh), idx, new),
                M.MerkleUpdatesClaim(DEPTH12, old, fresh, idx, leaf_changed),
                M.MerkleUpdatesClaim(DEPTH12, old, fresh, index_changed, new),
                M.MerkleUpdatesClaim(DEPTH12, old, fresh, idx, swapped)):
        with pytest.raises(VerificationError):
            bad.verify(proof, M.SECURITY_LEVEL)
