"""CPU-only: examples/rollup's transfer claim, K balance transfers that take one Rescue-Prime account root to another.

  * rollup.apply on the host equals the restatement (tests/rescue_rollup_oracle.py): the trace, the K + 1 roots and the
    final heap, at D = 1, at D not a power of two, at K = 1, with a self-transfer, a zero amount, repeated accounts, a
    sender left at 0 and a receiver brought to 2^32 - 1; the final heap is tree() of the final leaves;
  * the CPU build of ms_rescue_rollup (tests/cpp/rescue_rollup_cpu_abi.c, through `apply(..., device="cpu")` on the CPU
    harness, tests/cpu_device.py) equals the restatement, leaves the caller's heap alone, and refuses bad arguments and
    invalid batches before anything is written;
  * an overdraft and an overflow are refused by apply with the transfer and its step named, the heap untouched; bad
    shapes are refused;
  * the restated trace satisfies every constraint, the package's lookup constraints included (oracle/check_oracle.py)
    at those shapes; the constraint counts and the ce blow-up of 8; a wrong DELTA, a nonce + 2, a changed owner word, a
    limb of 256, a balance wrapped below zero and a broken TBL step each break their group;
  * the specialised evaluator's generated source (csrc/eval_jit.cu, compiled here by g++) and the CPU interpreter agree
    on the composition program, which reads the trace 1 + 8 L rows ahead;
  * 2^12-row proofs verify with Stark.verify and oracle/stark_oracle.verify, resident and streamed give the same bytes,
    and a wrong new root, a changed amount, two swapped transfers and a shorter transfer list are refused.
Harness cases run in spawned workers that install it themselves; the pytest process never does."""
import ctypes as C
import os
import random
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rescue_merkle_oracle as MO  # noqa: E402
import rescue_rollup_oracle as RO  # noqa: E402

P = 2**64 - 2**32 + 1
TOP = 2**32 - 1
# (depth, K, case): L = 1 with K L = 8; D = 3 < L = 4; K = 1 with D = 5 < L = 8; D = L = 4; D = 2 with 16 transfers
SHAPES = [(1, 8, "self"), (3, 2, "edges"), (5, 1, "single"), (4, 4, "self"), (2, 16, "edges")]


def accounts_of(depth, salt=0):
    """2^depth accounts: balances below 2^31 (account 0: 2^32 - 1), nonces some near p, owners any field elements; every
    fourth account empty"""
    rng = random.Random(1000 * depth + salt)
    lv = [(rng.randrange(2**31), P - 1 - rng.randrange(2) if rng.random() < 0.2 else rng.randrange(2**16),
           rng.randrange(P), rng.randrange(P)) for _ in range(1 << depth)]
    for i in range(1, len(lv), 4):
        lv[i] = (0, 0, 0, 0)
    lv[0] = (TOP, 7, 1, 2)
    return lv


def transfers_of(depth, K, case, salt=0):
    """K valid transfers over accounts_of(depth, salt); by `case`, a self-transfer, or a sender left at 0, a receiver
    brought to 2^32 - 1 and a zero amount, and always repeated accounts"""
    rng = random.Random(31 * depth + K + salt)
    lv = accounts_of(depth, salt)
    bal = {}
    get = lambda a: bal.get(a, lv[a][0])
    out = []
    for k in range(K):
        s, d = rng.randrange(1 << depth), rng.randrange(1 << depth)
        if k % 3 == 1:
            s = out[k - 1][1]                               # the previous receiver sends
        if case == "self" and k == K // 2:
            d = s
        bs, br = get(s), get(d)
        amount = rng.randrange(bs + 1)
        if s != d:
            amount = min(amount, TOP - br)
        if case == "edges" and K > 1:
            if k == 0:
                s, d = 1 + (1 << depth) // 2, 0
                bs, br = get(s), get(d)
                amount = 0                                  # a zero amount (account 0 holds 2^32 - 1 already)
            elif k == 1:
                d = 0 if s != 0 else 1
                bs, br = get(s), get(d)
                amount = bs                                 # the sender left at 0, account 0 gives back
                if br + amount > TOP:
                    s, d, bs, br, amount = 0, s, get(0), get(s), TOP - get(s)      # the receiver brought to 2^32 - 1
        bal[s] = bs - amount
        bal[d] = get(d) + amount
        out.append((s, d, amount))
    return out


def _mont_cols(rows):
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T.copy()


def _final_leaves(depth, salt, txs):
    lv = [list(a) for a in accounts_of(depth, salt)]
    for s, d, a in txs:
        lv[s][0] = (lv[s][0] - a) % P
        lv[s][1] = (lv[s][1] + 1) % P
        lv[d][0] = (lv[d][0] + a) % P
    return [tuple(v) for v in lv]


def test_cases_hold_their_edges():
    for depth, K, case in SHAPES:
        txs = transfers_of(depth, K, case)
        if case == "self" and K > 1:
            assert any(s == d for s, d, _ in txs)
    txs = transfers_of(3, 2, "edges")
    assert txs[0][2] == 0
    final = _final_leaves(3, 0, txs)
    assert 0 in [final[s][0] for s, _, _ in txs[1:]] or TOP in [final[d][0] for _, d, _ in txs[1:]]


# ------------------------------------------------------------------------------------------------- the host path
@pytest.mark.parametrize("depth,K,case", SHAPES)
def test_host_apply_equals_oracle(depth, K, case):
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rollup as RL
    lv = accounts_of(depth)
    txs = transfers_of(depth, K, case)
    nodes = M.tree(lv)
    before = list(nodes)
    trace, heap, roots = RL.apply(nodes, depth, txs)
    assert nodes == before                                          # the caller's heap is left alone
    rows, want_roots, want_heap = RO.rollup_trace(MO.heap(lv), depth, txs)
    assert trace.base_columns().shape == (23, 32 * K * (1 << (depth - 1).bit_length()))
    assert np.array_equal(trace.base_columns(), _mont_cols(rows)), (depth, K)
    assert [list(r) for r in roots] == want_roots and roots[0] == M.root(nodes) and len(roots) == K + 1
    assert [list(v) for v in heap[1:]] == want_heap[1:]
    assert heap == M.tree(_final_leaves(depth, 0, txs))


def test_leaf_helper():
    from ministark_b200.examples import rollup as RL
    assert RL.leaf(5) == (5, 0, 0, 0) and RL.leaf(5, 2, (3, 4)) == (5, 2, 3, 4)
    with pytest.raises(ValueError):
        RL.leaf(P)


def test_invalid_transfers_are_refused_and_named():
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rollup as RL
    lv = [RL.leaf(100, 0, (9, 9)), RL.leaf(TOP - 5), RL.leaf(0), RL.leaf(7)] * 2
    nodes = M.tree(lv)
    before = list(nodes)
    ok = (3, 2, 7)
    for txs, msg in [([ok, (0, 2, 101)], "the sender step of transfer 1 leaves account 0 with balance "
                      f"{(100 - 101) % P}, not below 2^32"),
                     ([(0, 1, 6), ok], f"the receiver step of transfer 0 leaves account 1 with balance {TOP + 1}, "
                      "not below 2^32"),
                     ([ok, (0, 1, 50), (0, 1, 1), ok], "the receiver step of transfer 1 leaves account 1"),
                     ([ok, (2, 2, 8)], "the sender step of transfer 1 leaves account 2")]:
        with pytest.raises(ValueError, match=re.escape(msg)):
            RL.apply(nodes, 3, txs)
        with pytest.raises(RO.InvalidTransfer, match=re.escape(msg)):
            RO.rollup_trace(MO.heap(lv), 3, txs)
    assert nodes == before
    # the edges themselves are valid: balance 0 and 2^32 - 1
    _, heap, _ = RL.apply(nodes, 3, [(0, 1, 5), (0, 2, 95)])
    assert heap[8][0] == 0 and heap[9][0] == TOP


def test_bad_shapes_refused():
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rollup as RL
    nodes = M.tree(accounts_of(3))
    root = M.root(nodes)
    for depth, txs in [(3, [(0, 1, 1)] * 3), (3, [(8, 1, 1)] * 2), (3, [(0, 8, 1)] * 2), (3, [(0, 1, 2**32)] * 2),
                       (3, [(0, -1, 1)] * 2), (0, [(0, 0, 0)] * 8), (33, [(0, 0, 0)] * 8), (3, []),
                       (3, [(0, 1, 1)]), (1, [(0, 1, 0)] * 4), (3, [(0, 1)] * 2)]:
        with pytest.raises(ValueError):
            RL.apply(nodes, depth, txs)
        with pytest.raises(ValueError):
            RL.TransfersClaim(depth, root, root, txs)
    with pytest.raises(ValueError, match="receiver 8 of transfer 1 is not below 2\\^3"):
        RL.apply(nodes, 3, [(0, 1, 1), (0, 8, 1)])
    with pytest.raises(ValueError, match="amount 4294967296 of transfer 0 is not below 2\\^32"):
        RL.apply(nodes, 3, [(0, 1, 2**32), (0, 1, 1)])
    with pytest.raises(ValueError, match="at least 256"):
        RL.rollup_air_config(1, 4)                                             # 32 K L = 128 rows
    with pytest.raises(ValueError):
        RL.apply(nodes[:-2], 3, [(0, 1, 1)] * 2)                               # not a heap of depth 3
    with pytest.raises(ValueError):
        RL.TransfersClaim(3, root, (1, 2, 3, P), [(0, 1, 1)] * 2)              # new root not canonical
    with pytest.raises(ValueError):
        RL.rollup_air_config(1 << 26, 4)                                       # 32 K L = 2^33 rows
    with pytest.raises(ValueError):
        RL.rollup_air_config(2, 3).constraints(32 * 2 * 2)                     # depth 3 takes L = 4, not 2
    assert RL.rollup_air_config(2, 3) is RL.rollup_air_config(2, 3)
    assert RL.rollup_air_config(2, 3) is not M.updates_air_config(4, 3)


# ------------------------------------------------------------------------------------------- the CPU stand-in
@pytest.fixture(scope="module")
def rollup_abi(tmp_path_factory, orc):
    """tests/cpp/rescue_rollup_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary
    directory"""
    out = str(tmp_path_factory.mktemp("rescue_rollup_abi") / "libms_rescue_rollup_cpu_abi.so")
    build_stand_in(out)
    return out


def build_stand_in(out):
    """tests/cpp/rescue_rollup_cpu_abi.c linked with tests/cpp/lookup_cpu_abi.c (the range lookup's multiplicities on
    the harness): both bring the same CPU build of the extension columns, whose second copy the linker drops"""
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "cpp", "rescue_rollup_cpu_abi.c"),
                           os.path.join(ROOT, "tests", "cpp", "lookup_cpu_abi.c"), "-Wl,--allow-multiple-definition"])


def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS, _lib._LOOKUP_SIGS, _lib._RESCUE_SIGS,
                 _lib._RESCUE_MERKLE_SIGS, _lib._RESCUE_MERKLE_UPDATES_SIGS, _lib._RESCUE_ROLLUP_SIGS):
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
    try:
        _install(lib_path)
        q.put(fn(*args))
    except Exception:                       # reported, not left for the queue's timeout
        import traceback
        q.put(traceback.format_exc())


def _stand_in(shapes):
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rollup as RL
    out = []
    for depth, K, case in shapes:
        nodes = M.tree(np.array(accounts_of(depth), dtype=np.uint64), device="cpu")
        before = nodes.clone()
        txs = transfers_of(depth, K, case)
        trace, heap, roots = RL.apply(nodes, depth, txs, device="cpu")
        _, heap_from_list, roots_from_list = RL.apply(M.tree(accounts_of(depth)), depth, txs, device="cpu")
        out.append((trace.base_columns().numpy().view(np.uint64).copy(), heap.numpy().view(np.uint64).copy(), roots,
                    bool((nodes == before).all()), bool((heap_from_list == heap).all()) and roots_from_list == roots))
    return out


def test_stand_in_apply_equals_oracle(rollup_abi):
    got = _spawn(_worker, rollup_abi, _stand_in, (SHAPES,))
    assert isinstance(got, list), got
    for (depth, K, case), (cols, heap, roots, untouched, same_from_list) in zip(SHAPES, got):
        txs = transfers_of(depth, K, case)
        rows, want_roots, want_heap = RO.rollup_trace(MO.heap(accounts_of(depth)), depth, txs)
        assert np.array_equal(cols, _mont_cols(rows)), (depth, K)
        assert [list(r) for r in roots] == want_roots
        assert heap[0].tolist() == [0, 0, 0, 0] and heap[1:].tolist() == want_heap[1:]
        assert untouched and same_from_list


def _stand_in_errors():
    from ministark_b200 import Context, MsError
    import torch
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rollup as RL
    ctx, msgs = Context(0), []
    lv = np.array([[100, 0, 9, 9], [TOP - 5, 0, 0, 0], [0, 0, 0, 0], [7, 0, 0, 0]] * 2, dtype=np.uint64)
    nodes = M.tree(lv, device="cpu")
    heap = nodes.clone()
    out, roots = torch.zeros((23, 256), dtype=torch.int64), torch.zeros((3, 4), dtype=torch.int64)
    ok = [3, 2, 7]
    for args in [(heap, 3, np.array([ok] * 3, dtype=np.uint64), 3), (heap, 3, None, 2),
                 (heap, 0, np.array([ok] * 2, dtype=np.uint64), 2), (heap, 3, np.array([ok, [1, 8, 0]], dtype=np.uint64), 2),
                 (heap, 3, np.array([[0, 1, 2**32], ok], dtype=np.uint64), 2), (heap, 1, np.array([ok] * 2), 1 << 30),
                 (heap, 3, np.array([ok], dtype=np.uint64), 1),
                 (heap, 3, np.array([ok, [0, 2, 101]], dtype=np.uint64), 2),
                 (heap, 3, np.array([[0, 1, 6], ok], dtype=np.uint64), 2)]:
        try:
            ctx.rescue_rollup(*args, out, roots)
            msgs.append(None)
        except MsError as e:
            msgs.append(str(e))
    try:
        RL.apply(nodes, 3, [ok, (0, 2, 101)], device="cpu")
        msgs.append(None)
    except ValueError as e:
        msgs.append(str(e))
    return msgs, bool((heap == nodes).all()), bool(out.any()), bool(roots.any())


def test_stand_in_refuses_bad_arguments_and_invalid_batches(rollup_abi):
    got = _spawn(_worker, rollup_abi, _stand_in_errors, ())
    assert isinstance(got, tuple), got
    msgs, heap_untouched, out_written, roots_written = got
    assert "not a power of two" in msgs[0] and "null argument" in msgs[1] and "outside 1..32" in msgs[2]
    assert "receiver 8 of transfer 1 is not below 2^3" in msgs[3]
    assert "amount 4294967296 of transfer 0 is not below 2^32" in msgs[4]
    assert "are not in 2^8..2^32" in msgs[5] and "are not in 2^8..2^32" in msgs[6]
    assert f"the sender step of transfer 1 leaves account 0 with balance {P - 1}, not below 2^32" in msgs[7]
    assert f"the receiver step of transfer 0 leaves account 1 with balance {TOP + 1}, not below 2^32" in msgs[8]
    assert msgs[9] == f"the sender step of transfer 1 leaves account 0 with balance {P - 1}, not below 2^32"
    assert heap_untouched and not out_written and not roots_written


def test_header_bound_and_exported(rollup_abi):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.RESCUE_ROLLUP_HEADER_PATH)
    assert declared == sorted(_lib._RESCUE_ROLLUP_SIGS) == ["ms_rescue_rollup"]
    others = set(_lib.header_symbols())
    for path in (_lib.STREAM_HEADER_PATH, _lib.CHECK_HEADER_PATH, _lib.EXTENSION_HEADER_PATH, _lib.LOOKUP_HEADER_PATH,
                 _lib.PERMUTATION_HEADER_PATH, _lib.BF_HEADER_PATH, _lib.DEVICE_HEADER_PATH, _lib.HOST_NODES_HEADER_PATH,
                 _lib.RESCUE_HEADER_PATH, _lib.RESCUE_HASH_HEADER_PATH, _lib.RESCUE_MERKLE_HEADER_PATH,
                 _lib.RESCUE_MERKLE_UPDATES_HEADER_PATH):
        others |= set(_lib.header_symbols(path))
    assert not set(declared) & others
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(rollup_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)


# ------------------------------------------------------------------------------------------------------- the AIR
GAMMA, ALPHA = (123456789, 987654321, 55555), (31337, 4242, 777)


def _check(depth, rows, roots, txs):
    """{constraint: first failing row} of the restated rows (multiplicities counted here, misses left out), and the
    extension columns and hints"""
    from ministark_b200.air import Air
    from ministark_b200.examples import rollup as RL
    from oracle import check_oracle, extension_oracle, lookup_oracle
    base = _mont_cols(rows)
    n = base.shape[1]
    claim = RL.TransfersClaim(depth, roots[0], roots[-1], txs)
    cfg = claim.AirConfig
    air = Air(cfg, n, claim, RL.OPTIONS)
    lk = cfg.lookups(n)[0]
    base[lk.multiplicity] = lookup_oracle.multiplicities(lk.table, lk.values, lk.selectors, base)[0]
    challenges = [GAMMA, ALPHA]
    hints = cfg.gen_hints(n, claim, challenges)
    decl = [(c.init, c.mul, c.add, c.inclusive) for c in air.extension_declaration]
    ext = extension_oracle.columns(decl, base, 3, challenges, hints)
    cons = [c.to_tuple() for c in air.constraints]
    got = check_oracle.check(cons, n.bit_length() - 1, base, ext, 3, challenges, hints)
    return {k: first for k, (first, _) in enumerate(got) if first is not None}, ext, hints


@pytest.mark.parametrize("depth,K,case", SHAPES)
def test_oracle_trace_satisfies_every_constraint(depth, K, case):
    from ministark_b200.air import Air
    from ministark_b200.examples import rollup as RL
    txs = transfers_of(depth, K, case)
    rows, roots, _ = RO.rollup_trace(MO.heap(accounts_of(depth)), depth, txs)
    failing, ext, hints = _check(depth, rows, roots, txs)
    assert failing == {}
    n = len(rows)
    L = n // (32 * K)
    cfg = RL.rollup_air_config(K, depth)
    groups = cfg.groups(n)
    names = ("ROUND", "CAP", "LINK", "SIDE", "SIB", "BIT", "IDX", "ROOT", "CHAIN", "BAL", "NONCE", "KEEP", "LIMB", "TBL",
             "R", "LOOKUP")
    sizes = [12, 4, 0 if L == 1 else 4, 3, 5, 2, 2 if L == 1 else 3, 8, 4, 1, 1, 2, 1, 3, 4, 3]
    assert list(groups) == list(names) and [len(groups[g]) for g in names] == sizes
    assert len(cfg.constraints(n)) == sum(sizes) - 3
    assert len(Air(cfg, n, None, RL.OPTIONS).constraints) == sum(sizes)
    last = tuple(int(w) * pow(2**64, -1, P) % P for w in ext[0, 3 * (n - 1):])
    assert last == tuple(hints[0])


def test_updates_constraints_are_reused_unchanged():
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rollup as RL
    K, depth = 4, 5
    n = 32 * K * 8
    own = [c.to_tuple() for c in RL.rollup_air_config(K, depth).constraints(n)]
    upd = [c.to_tuple() for c in M.updates_air_config(2 * K, depth).constraints(n)]
    assert own[:len(upd) - 4] == upd[:-4]


def test_ce_blowup_is_8_and_options_are_rescues():
    from ministark_b200.air import Air
    from ministark_b200.examples import rescue as R
    from ministark_b200.examples import rollup as RL
    assert RL.OPTIONS is R.OPTIONS
    for depth, K in [(1, 8), (3, 2), (5, 32), (16, 1 << 14), (24, 1 << 13), (32, 1 << 22), (1, 1 << 27)]:
        L = 1 << (depth - 1).bit_length()
        n = 32 * K * L
        air = Air(RL.rollup_air_config(K, depth), n, None, RL.OPTIONS)
        assert air.ce_blowup_factor == 8, (depth, K)


def test_composition_program_fits_the_evaluator():
    """every constraint, the lookup's included, compiles into the evaluator's registers (expr.MAX_REGS)"""
    from ministark_b200.air import Air
    from ministark_b200.examples import rollup as RL
    for depth, K in [(1, 8), (5, 4), (16, 1 << 14)]:
        n = 32 * K * (1 << (depth - 1).bit_length())
        air = Air(RL.rollup_air_config(K, depth), n, None, RL.OPTIONS)
        assert len(air.composition_program()) > 0
        assert any(o == 1 + 8 * (1 << (depth - 1).bit_length()) for _, o in air.trace_arguments())


def test_changes_break_their_constraints():
    from ministark_b200.examples import rollup as RL
    depth, K = 4, 4                                     # L = 4: write w's old path at rows 64 w, its new path 32 on
    txs = transfers_of(depth, K, "self")
    rows, roots, _ = RO.rollup_trace(MO.heap(accounts_of(depth)), depth, txs)
    groups = RL.rollup_air_config(K, depth).groups(len(rows))
    w = 3                                               # write 3 (transfer 1's receiver step), checked on row 64 w - 1
    at, end = 64 * w, 64 * w - 1

    def failing(bad):
        return _check(depth, bad, roots, txs)[0]

    def only(got, group, row=None):
        assert got and set(got) & set(groups[group]), (group, got)
        if row is not None:
            assert got[groups[group][0]] == row, (group, got)

    bad = [list(r) for r in rows]
    bad[at][15] = (bad[at][15] + 1) % P                 # a wrong DELTA (R binds it too)
    got = failing(bad)
    only(got, "BAL", end)
    assert set(got) & set(groups["R"])
    bad = [list(r) for r in rows]
    bad[at][16] = 2                                     # a nonce + 2 claimed
    only(failing(bad), "NONCE", end)
    # a changed owner word in the new path only, its first permutation recomputed from it
    from ministark_b200.examples import rescue as R
    bad = [list(r) for r in rows]
    new_at = at + 32
    state = list(bad[new_at][:12])
    b = bad[new_at][12]
    state[(4 if b else 0) + 2] = (state[(4 if b else 0) + 2] + 1) % P
    for r, st in enumerate(R.round_states(state)):
        bad[new_at + r][:12] = st
    only(failing(bad), "KEEP", end)
    bad = [list(r) for r in rows]
    bad[at][17] += 256                                  # a limb of 256 (and the balance it states is off by 256)
    bad[at][18] -= 1 if bad[at][18] else 0
    got = failing(bad)
    assert set(got) & (set(groups["LOOKUP"]) | set(groups["LIMB"])), got
    bad = [list(r) for r in rows]
    bad[at][17] = 256                                   # a limb of 256 alone: the lookup
    assert set(failing(bad)) & set(groups["LOOKUP"])
    bad = [list(r) for r in rows]
    bad[7][22] = (bad[7][22] + 1) % P                   # a broken TBL step
    got = failing(bad)
    assert got == {groups["TBL"][1]: 6}, got           # the step into row 7; the step out of it still holds


def test_wrapped_balance_is_named_by_limb_or_lookup():
    """an overdraft written into the trace with its wrapped balance: the old and new paths consistent, BAL holding, and
    limbs that cannot represent a balance above 2^32"""
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rollup as RL
    depth, K = 3, 2
    lv = [RL.leaf(100, 0, (9, 9)), RL.leaf(5)] + [RL.leaf(0)] * 6
    txs = [(0, 1, 101), (2, 3, 0)]                      # transfer 0 overdraws account 0 by 1
    nodes = MO.heap([list(v) for v in lv])
    # the restatement refuses it; build the rows with the wrapped balance by hand from the writes
    import rescue_merkle_updates_oracle as UO
    wrapped = (100 - 101) % P
    new = [[wrapped, 1, 9, 9], [106, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 0]]
    rows, wroots, _ = UO.updates_trace(nodes, depth, [0, 1, 2, 3], new)
    extra = [[P - 101, 1] + [wrapped >> 8 * q & 255 for q in range(4)], [101, 0, 106, 0, 0, 0], [0, 1, 0, 0, 0, 0],
             [0, 0, 0, 0, 0, 0]]
    rows = [r + (extra[i // 64] if i % 64 == 0 else [0] * 6) + [0, min(i, 255)] for i, r in enumerate(rows)]
    groups = RL.rollup_air_config(K, depth).groups(len(rows))
    got = _check(depth, rows, wroots[::2], txs)[0]
    assert got and set(got) <= set(groups["LIMB"]) | set(groups["LOOKUP"]), got
    assert got.get(groups["LIMB"][0]) == len(rows) - 1     # write 0 is checked on the last row
    assert M.root(M.tree(lv)) == tuple(wroots[0])


# ------------------------------------------------------------------------- the evaluator at a row offset of 1 + 8 L
def test_generated_kernel_source_reads_leaf_offset_like_the_interpreter(tmp_path, orc):
    """the composition program of a K = 2, D = 3 AIR (BAL, NONCE, KEEP and LIMB read 33 rows ahead, SIB and CHAIN 32),
    the generated kernel source against the CPU interpreter on random columns"""
    from test_eval_jit_source import GENERATOR, _host_kernel, _tables
    from ministark_b200.air import Air
    from ministark_b200.examples import rollup as RL
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "libms_cpu_abi.so"])
    lib = C.CDLL(os.path.join(ROOT, "oracle", "libms_cpu_abi.so"))
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    rng = random.Random(5)
    depth, K = 3, 2
    claim = RL.TransfersClaim(depth, (1, 2, 3, 4), (5, 6, 7, 8), [(1, 2, 3), (4, 5, 6)])
    air = Air(claim.AirConfig, 32 * K * 4, claim, RL.OPTIONS)
    offsets = {o for _, o in air.trace_arguments()}
    assert 33 in offsets and 32 in offsets
    q3 = lambda: tuple(rng.randrange(P) for _ in range(3))
    prog = air.composition_program().bind(challenges=[q3() for _ in range(32)], hints=[q3() for _ in range(256)],
                                          ccoefs=[q3() for _ in range(256)])
    log_m = air.log_n + air.ce_blowup_factor.bit_length() - 1
    m = 1 << log_m
    base = orc.rand_matrix(23, m, 1, seed=rng.randrange(1 << 30))
    ext = orc.rand_matrix(2, m, 3, seed=rng.randrange(1 << 30))
    cols = [np.ascontiguousarray(c) for c in base] + [np.ascontiguousarray(e) for e in ext]
    ptrs = (C.c_void_p * len(cols))(*[c.ctypes.data for c in cols])
    isq = (C.c_int * len(cols))(*([0] * 23 + [1, 1]))
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
DEPTH12, K12 = 5, 16                                   # L = 8: 2^12 rows


def _transfers12():
    txs = transfers_of(DEPTH12, K12, "edges", salt=12)
    return txs


def _prove():
    from ministark_b200 import FQ3
    from ministark_b200.air import ProofOptions
    from ministark_b200.examples import merkle as M
    from ministark_b200.examples import rollup as RL
    from ministark_b200.prover import GpuProver, peak_bytes
    nodes = M.tree(np.array(accounts_of(DEPTH12, 12), dtype=np.uint64), device="cpu")
    txs = _transfers12()
    trace, _, roots = RL.apply(nodes, DEPTH12, txs, device="cpu")
    claim = RL.TransfersClaim(DEPTH12, roots[0], roots[-1], txs)
    got = {}
    for residency in ("resident", "streamed"):
        p = GpuProver(0)
        if residency == "streamed":
            est = peak_bytes(len(trace), 8, 23, 2, FQ3, 8, 8)
            p.memory_budget = (est["streamed"] + est["resident"]) // 2
        got[residency] = (p.prove(claim, ProofOptions(*OPTS), trace).to_bytes(), p.last_residency)
    return got, roots


def test_cpu_harness_proofs_verify(rollup_abi):
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.examples import rollup as RL
    from ministark_b200.verifier import VerificationError
    from oracle import stark_oracle as SO
    got = _spawn(_worker, rollup_abi, _prove, ())
    assert isinstance(got, tuple), got
    proofs, roots = got
    assert proofs["resident"][1] == "resident" and proofs["streamed"][1] == "streamed"
    assert proofs["resident"][0] == proofs["streamed"][0]
    txs = _transfers12()
    _, want_roots, _ = RO.rollup_trace(MO.heap(accounts_of(DEPTH12, 12)), DEPTH12, txs)
    assert [list(r) for r in roots] == want_roots
    old, fresh = roots[0], roots[-1]
    claim = RL.TransfersClaim(DEPTH12, old, fresh, txs)
    proof = proofs["resident"][0]
    claim.verify(proof, RL.SECURITY_LEVEL)
    SO.verify(claim, proof, RL.SECURITY_LEVEL, lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o)))
    other = lambda r: (r[0], r[1], (r[2] + 1) % P, r[3])
    amount_changed = list(txs)
    s, d, a = txs[5]
    amount_changed[5] = (s, d, a + 1 if a < TOP else a - 1)
    # two transfers through one account, swapped
    i, j = next((i, j) for i in range(K12) for j in range(i + 1, K12)
                if set(txs[i][:2]) & set(txs[j][:2]) and txs[i] != txs[j])
    swapped = list(txs)
    swapped[i], swapped[j] = txs[j], txs[i]
    for bad in (RL.TransfersClaim(DEPTH12, old, other(fresh), txs),
                RL.TransfersClaim(DEPTH12, old, fresh, amount_changed),
                RL.TransfersClaim(DEPTH12, old, fresh, swapped)):
        with pytest.raises(VerificationError):
            bad.verify(proof, RL.SECURITY_LEVEL)
    with pytest.raises(ValueError):                     # one shorter: not a power of two, no claim at all
        RL.TransfersClaim(DEPTH12, old, fresh, txs[:-1])
    with pytest.raises((VerificationError, ValueError)):  # half the list: another AIR, another trace length
        RL.TransfersClaim(DEPTH12, old, fresh, txs[:K12 // 2]).verify(proof, RL.SECURITY_LEVEL)
