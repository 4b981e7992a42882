"""CPU-only: sorted-copy permutation arguments declared by the AIR (air.Permutation, AirConfig.permutations), their generated
constraints and running products, and their target columns filled by ms_permutation_fill.

  * Air rejects a malformed permutation with a ValueError naming the permutation and the problem, merges the generated
    running products into extension_columns by the rules of the lookup running sums, and assigns the challenges after
    the AIR's own and the lookups'; an AIR with lookups only keeps its challenges, constraints and proof bytes;
  * the generated constraints and running product are node for node the ones examples/memory.py's MemoryAirConfig writes;
  * ms_permutation_fill of the CPU build (tests/cpp/permutation_cpu_abi.c) equals oracle/permutation_oracle.py word for
    word for W = 1 to 4: random columns, duplicate tuples (stability), words 0 and p - 1, row offsets other than 0;
    malformed arguments are refused;
  * GpuProver on the CPU harness (tests/cpu_device.py), resident and streamed, and ShardedProver over gloo with two
    ranks: both memory AIRs prove to the bytes of oracle/stark_oracle.cpu_prove; a corrupted fill is named by
    validate=True as a generated constraint and refused by Stark.verify.
Prover cases run in spawned workers that install the harness themselves; the pytest process never does."""
import ctypes as C
import hashlib
import os
import re
import socket
import subprocess
import sys

import numpy as np
import pytest

from ministark_b200 import expr as E
from ministark_b200.air import Air, AirConfig, Lookup, Permutation, ProofOptions, RunningColumn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = E.P
_R = 2**64
OPTS = ProofOptions(16, 8, 4, 4, 8)
T = E.Trace


def _mont(v):
    return int(v) % P * _R % P


# ------------------------------------------------------------------------------------------- 1. declarations
def _config(perms, lookups=(), nbase=6, next_=1, ext=None):
    class Cfg(AirConfig):
        NUM_BASE_COLUMNS = nbase
        NUM_EXTENSION_COLUMNS = next_
        FQ_IS_FP = False

        @staticmethod
        def constraints(trace_len):
            return [(T(0) - E.Challenge(0) * E.Challenge(1)) / (E.X() - 1)]

        @staticmethod
        def extension_columns(trace_len):
            return ext

        @staticmethod
        def lookups(trace_len):
            return list(lookups)

        @staticmethod
        def permutations(trace_len):
            return perms
    return Cfg


def _pm(source=(T(0), T(1)), target=(2, 3), z=6):
    return Permutation(source, target, z)


LK = Lookup((T(0),), ((T(1),),), 5, 6)


@pytest.mark.parametrize("perms,lookups,next_,msg", [
    (["not a permutation"], (), 1, "permutation 0: expected a Permutation, got str"),
    ([_pm(source=(), target=())], (), 1, "permutation 0: source tuples of width 0; 1 to 4 are supported"),
    ([_pm(source=(T(0),) * 5, target=(1, 2, 3, 4, 5))], (), 1, "permutation 0: source tuples of width 5; 1 to 4"),
    ([_pm(target=(2,))], (), 1, "permutation 0: 1 target columns for source tuples of width 2"),
    ([_pm(target=(2, 6))], (), 1, "permutation 0: target column 6 is not a base column (0..5)"),
    ([_pm(target=(3, 3))], (), 1, "permutation 0: target column 3 is repeated"),
    ([_pm(), _pm(target=(4, 3), z=7)], (), 2, "permutation 1: target column 3 is also permutation 0's"),
    ([_pm(target=(2, 5), z=7)], (LK,), 2, "permutation 0: target column 5 is the multiplicity column of lookup 0"),
    ([_pm(z=5)], (), 1, "permutation 0: running-product column 5 is not an extension column (6..6)"),
    ([_pm(z=6)], (LK,), 1, "permutation 0: running-product column 6 is lookup 0's running sum"),
    ([_pm(), _pm(target=(4, 5), z=6)], (), 2, "permutation 1: running-product column 6 is also permutation 0's"),
    ([_pm(source=(T(0), T(2, 1)))], (), 1, "permutation 0: source[1] reads Trace(2, 1), a target column of permutation 0"),
    ([_pm(), _pm(source=(T(3, -1),), target=(4,), z=7)], (), 2,
     "permutation 1: source[0] reads Trace(3, -1), a target column of permutation 0"),
    ([_pm(source=(T(5), T(0)), z=7)], (LK,), 2, "permutation 0: source[0] reads Trace(5, 0), the multiplicity column"),
    ([_pm(source=(T(0) + E.Challenge(0), T(1)))], (), 1, "permutation 0: source[0] reads a challenge"),
    ([_pm(source=(T(0), E.Hint(0)))], (), 1, "permutation 0: source[1] reads a hint"),
    ([_pm(source=(E.Expr("ccoef", 0), T(1)))], (), 1, "permutation 0: source[0] reads a composition coefficient"),
    ([_pm(source=(E.Constant((1, 2, 3)), T(1)))], (), 1, "permutation 0: source[0] reads an extension-field constant"),
    ([_pm(source=(T(6), T(1)))], (), 1, "permutation 0: source[0] reads Trace(6, 0), which is not a base column (0..5)"),
])
def test_invalid_permutations_raise(perms, lookups, next_, msg):
    with pytest.raises(ValueError, match=re.escape(msg)):
        Air(_config(perms, lookups, next_=next_), 8, None, OPTS)


def test_extension_columns_merge_rules():
    rc = RunningColumn(1, E.Challenge(0) - T(0))
    lk = Lookup((T(0),), ((T(1),),), 5, 7)
    # a user column, a lookup's running sum and a permutation's running product
    air = Air(_config([_pm(z=8)], (lk,), next_=3, ext=[rc, None, None]), 8, None, OPTS)
    user, s, z = air.extension_declaration
    assert user.mul is rc.mul and s.init is E.Constant(0) and z.init is E.Constant(1) and z.add is E.Constant(0)
    ds, dt = air._permutation_denominators(0)
    assert z.mul is ds / dt
    bad = [([rc, None, rc], "extension column 8: permutation 0's running product is declared by the package"),
           ([rc, rc, None], "extension column 7: lookup 0's running sum is declared by the package"),
           ([None, None, None], "extension column 6: expected a RunningColumn, got NoneType"),
           (None, "extension_columns returned None, but only 2 of the 3 extension columns are lookup running sums or "
                  "permutation running products"),
           ([None, None], "extension_columns declares 2 columns but NUM_EXTENSION_COLUMNS is 3")]
    for ext, msg in bad:
        with pytest.raises(ValueError, match=re.escape(msg)):
            Air(_config([_pm(z=8)], (lk,), next_=3, ext=ext), 8, None, OPTS)
    # None as a whole when every extension column is generated
    air = Air(_config([_pm(), _pm(source=(T(1, 1),), target=(4,), z=7)], next_=2), 8, None, OPTS)
    assert [c.init for c in air.extension_declaration] == [E.Constant(1)] * 2


def test_challenge_indices_and_default():
    # the AIR's own constraints draw 2; lookup 0 (W = 1) takes 2; permutation 0 (W = 2) takes 3, 4, permutation 1 (W = 1) 5
    air = Air(_config([_pm(z=7), _pm(source=(T(1, 1),), target=(4,), z=8)], (LK,), next_=3), 8, None, OPTS)
    assert air.lookup_challenges == [(2, None)] and air.permutation_challenges == [(3, 4), (5, None)]
    assert air.num_challenges() == 6
    assert len(air.constraints) == 1 + 3 + 3 * 2
    assert AirConfig.permutations(8) == []
    assert air.permutation_programs() is air.permutation_programs()


def test_lookup_only_airs_keep_their_challenges_and_constraints():
    """an AIR without permutations builds the same Air as before: same challenges and constraint nodes"""
    from ministark_b200.examples import lookup as L

    class Explicit(L.SquareLookupAirConfig):
        @staticmethod
        def permutations(trace_len):
            return []
    for n in (8, 1 << 10):
        a, b = Air(L.SquareLookupAirConfig, n, None, OPTS), Air(Explicit, n, None, OPTS)
        assert a.permutations == [] and a.lookup_challenges == [(0, 1)] and a.num_challenges() == 2
        assert len(a.constraints) == 7 and all(x is y for x, y in zip(a.constraints, b.constraints))


def test_generated_constraints_are_the_hand_written_ones():
    from ministark_b200.examples import memory as MM
    for n in (8, 1 << 10):
        a, b = Air(MM.MemoryDeclaredAirConfig, n, None, OPTS), Air(MM.MemoryAirConfig, n, None, OPTS)
        assert len(a.constraints) == len(b.constraints) == 19
        assert all(x is y for x, y in zip(a.constraints, b.constraints))
        assert a.ce_blowup_factor == b.ce_blowup_factor and a.num_challenges() == b.num_challenges() == 4
        assert a.lookup_challenges == [(1, None)] and a.permutation_challenges == [(2, 3)]
        for x, y in zip(a.extension_declaration, b.extension_declaration):
            assert x.init is y.init and x.mul is y.mul and x.add is y.add and x.inclusive == y.inclusive


def test_permutation_program_slots():
    prog = E.compile_lookup_program((T(0), T(1, 1), E.X(), T(2, -3)), (), None, 4, 3)
    stores = sorted(int(w[1]) for w in prog.code if int(w[0]) & 0xff == E.OP_STORE)
    assert stores == [0, 1, 2, 3]


# ------------------------------------------------------------------------------------------------ 2. CPU ABI
@pytest.fixture(scope="module")
def perm_abi(tmp_path_factory, orc):
    """tests/cpp/permutation_cpu_abi.c compiled like the oracle's CPU ABI (oracle/Makefile), into a temporary directory"""
    out = str(tmp_path_factory.mktemp("permutation_abi") / "libms_permutation_cpu_abi.so")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "cpp", "permutation_cpu_abi.c")])
    return out


@pytest.fixture(scope="module")
def abi(perm_abi):
    from ministark_b200 import _lib
    lib = C.CDLL(perm_abi)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    _lib.bind(lib, _lib._PERMUTATION_SIGS)
    h = C.c_void_p()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    return lib, h


def run_abi(abi, source, base, log_n, code=None, width=None, ws_bytes=None, isq=None, targets=None):
    """returns (rc, error message, the (W, n) target words)"""
    from test_lookup_cpu import periodic_tables
    lib, h = abi
    prog = E.compile_lookup_program(source, (), None, base.shape[0], log_n)
    code = prog.code if code is None else np.ascontiguousarray(code, dtype=np.uint32)
    cols = [np.ascontiguousarray(c) for c in base] + periodic_tables(prog, log_n)
    ptrs = (C.c_void_p * max(len(cols), 1))(*[c.ctypes.data for c in cols])
    q = (C.c_int * max(len(cols), 1))(*([0] * len(cols) if isq is None else isq))
    W = width or len(source)
    need = C.c_size_t()
    assert lib.ms_permutation_workspace_bytes(min(log_n, 16), min(max(W, 1), 4), C.byref(need)) == 0
    work = np.zeros(need.value if ws_bytes is None else ws_bytes, dtype=np.uint8)
    out = np.zeros((max(W, 1), 1 << min(log_n, 16)), dtype=np.uint64)
    tp = [out[k].ctypes.data for k in range(max(W, 1))] if targets is None else targets(out)
    tgt = (C.c_void_p * max(len(tp), 1))(*tp)
    rc = lib.ms_permutation_fill(h, code.ctypes.data, code.shape[0], prog.consts.ctypes.data, prog.consts.shape[0], ptrs, q,
                                 len(cols), log_n, W, tgt, work.ctypes.data, work.size)
    return rc, lib.ms_last_error(h).decode() if rc else "", out


def _base(seed, log_n, nbase=4, hi=4):
    """random columns of small values (so duplicate tuples), with words 0 and p - 1 among them"""
    rng = np.random.default_rng(seed)
    n = 1 << log_n
    cols = rng.integers(0, hi, size=(nbase, n)).astype(object)
    cols[cols == hi - 1] = P - 1
    return np.array([[_mont(v) for v in c] for c in cols.tolist()], dtype=np.uint64)


def _check(abi, source, base):
    from oracle import permutation_oracle as PO
    log_n = base.shape[1].bit_length() - 1
    rc, err, got = run_abi(abi, source, base, log_n)
    assert rc == 0, err
    assert np.array_equal(got, PO.targets(source, base))


SOURCES = {
    1: (T(0, 1),),
    2: (T(1), T(0, -1)),
    3: (T(2, 3), T(0), T(1) * T(3) + E.Constant(P - 1)),
    4: (T(3), T(2, -2), T(1) + E.X() * 0, T(0, 5) + E.Periodic([1, 2], 4)),
}


@pytest.mark.parametrize("W,log_n,hi", [(1, 0, 4), (1, 6, 2**40), (2, 1, 3), (2, 9, 4), (3, 8, 3), (3, 12, 2**20), (4, 10, 3),
                                        (4, 16, 5)])
def test_cpu_abi_equals_oracle(abi, W, log_n, hi):
    _check(abi, SOURCES[W], _base(W * 100 + log_n, log_n, hi=hi))


def test_cpu_abi_is_stable_on_duplicates_and_edge_words(abi):
    """one repeated tuple, and tuples that differ only in the last word: equal tuples keep their row order, which for
    equal words means the output equals the oracle's stable sort (and every word is 0 or p - 1)"""
    log_n = 9
    n = 1 << log_n
    base = _base(3, log_n)
    base[0] = _mont(P - 1)
    base[1] = np.array([_mont(v) for v in np.random.default_rng(1).choice([0, P - 1], size=n).tolist()], dtype=np.uint64)
    for src in ((T(0),), (T(0), T(1)), (T(1), T(0), T(1, 1), T(0, -1))):
        _check(abi, src, base)
    rc, _, got = run_abi(abi, (T(0), T(1)), base, log_n)
    k = int((base[1] == 0).sum())
    assert rc == 0 and (got[1, :k] == 0).all() and (got[1, k:] == _mont(P - 1)).all()


def test_cpu_abi_rejects_malformed_arguments(abi):
    base = _base(5, 3)
    src = (T(0), T(1))
    prog = E.compile_lookup_program(src, (), None, 4, 3)
    assert run_abi(abi, src, base, 3)[0] == 0
    assert "domain too large" in run_abi(abi, src, base, 31)[1]
    assert "tuples of 5 words (1 to 4)" in run_abi(abi, src, base, 3, width=5)[1]
    assert "workspace of 100 bytes" in run_abi(abi, src, base, 3, ws_bytes=100)[1]
    assert "never stores slot 2 of 3" in run_abi(abi, src, base, 3, width=3)[1]
    assert "is not a base-field column" in run_abi(abi, src, base, 3, isq=[1, 0, 0, 0])[1]
    assert "targets 0 and 1 are the same column" in run_abi(abi, src, base, 3, targets=lambda o: [o[0].ctypes.data] * 2)[1]
    assert "target 1 is not a device pointer" in run_abi(abi, src, base, 3, targets=lambda o: [o[0].ctypes.data, None])[1]
    bad = prog.code.copy()
    st = [i for i, w in enumerate(bad) if int(w[0]) & 0xff == E.OP_STORE][-1]
    bad[st, 1] = 7
    assert "stores to slot 7 of 2" in run_abi(abi, src, base, 3, code=bad)[1]
    bad = prog.code.copy()
    bad[st, 0] |= 1 << 8
    assert "stores an extension-field value" in run_abi(abi, src, base, 3, code=bad)[1]
    bad = prog.code.copy()
    tr = [i for i, w in enumerate(bad) if int(w[0]) & 0xff == E.OP_TRACE][0]
    bad[tr, 2] = 9
    assert "column 9 out of range" in run_abi(abi, src, base, 3, code=bad)[1]
    lib, _ = abi
    out = C.c_size_t()
    assert lib.ms_permutation_workspace_bytes(31, 1, C.byref(out)) != 0
    assert lib.ms_permutation_workspace_bytes(10, 0, C.byref(out)) != 0
    assert lib.ms_permutation_workspace_bytes(10, 5, C.byref(out)) != 0
    assert lib.ms_permutation_workspace_bytes(10, 4, None) != 0


# ------------------------------------------------------------------------------------------------- 3. the prover
def _install(path):
    import cpu_device
    cpu_device.install()
    from ministark_b200 import _lib
    lib = C.CDLL(path)
    _lib.bind(lib, {k: v for k, v in _lib._SIGS.items() if hasattr(lib, k)})
    for sigs in (_lib._STREAM_SIGS, _lib._CHECK_SIGS, _lib._EXTENSION_SIGS, _lib._LOOKUP_SIGS, _lib._PERMUTATION_SIGS):
        _lib.bind(lib, sigs)
    _lib._lib = lib


MEM_N, MEM_A = 1 << 8, 16


class SortedCopyAirConfig(AirConfig):
    """a permutation and nothing else: columns 0, 1 random, 2, 3 their sorted copy by (column 1, column 0 one row on), 4
    the running product.  No constraint of the AIR's own reads the targets, so only the generated ones can fail"""
    NUM_BASE_COLUMNS = 4
    NUM_EXTENSION_COLUMNS = 1
    FQ_IS_FP = False

    @staticmethod
    def constraints(trace_len):
        return []

    @staticmethod
    def permutations(trace_len):
        return [Permutation((T(1), T(0, 1)), (2, 3), 4)]


def _make_case(which):
    """(claim, options, trace) of a named case"""
    from ministark_b200.examples import lookup as L
    from ministark_b200.examples import memory as MM
    from ministark_b200.prover import Stark, Trace
    opts = (16, 8, 4, 4, 8)
    if which == "memory_hand":
        trace, reads = MM.MemoryClaim.gen_trace(MEM_N, MEM_A, seed=4)
        return MM.MemoryClaim(reads), opts, trace
    if which == "memory":
        trace, reads = MM.MemoryDeclaredClaim.gen_trace(MEM_N, MEM_A, seed=4)
        return MM.MemoryDeclaredClaim(reads), opts, trace
    if which == "square":
        return L.SquareLookupClaim(), opts, L.SquareLookupClaim.gen_trace(1 << 6, seed=6)

    class SortedCopy(Stark):
        AirConfig = SortedCopyAirConfig

        def get_public_inputs(self):
            return []
    rng = np.random.default_rng(9)
    base = np.zeros((4, 1 << 6), dtype=np.uint64)
    base[:2] = L._to_mont(rng.integers(0, 50, size=(2, 1 << 6)).astype(np.uint64))
    return SortedCopy(), opts, Trace(base)


def _prove_worker(which, lib_path, residency, validate, corrupt, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    from ministark_b200 import FP, FQ3
    from ministark_b200.prover import GpuProver, peak_bytes
    from ministark_b200.validate import ConstraintViolation
    from ministark_b200.verifier import VerificationError
    claim, opts, trace = _make_case(which)
    before = np.array(trace.base_columns(), copy=True)

    class Corrupting(GpuProver):
        """a wrong fill injected after the kernels"""
        def _lookup_base(self, r, host_base):
            base = super()._lookup_base(r, host_base)
            if corrupt == "zero":
                base[2:4] = 0
            else:                       # two rows of one target column swapped: no longer a permutation of the source
                a, b = base[3, 5].item(), base[3, 40].item()
                base[3, 5], base[3, 40] = b, a
            return base

    p = Corrupting(0) if corrupt else GpuProver(0)
    if residency == "streamed":
        cfg, o, n = claim.AirConfig, ProofOptions(*opts), len(trace)
        est = peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, FP if cfg.FQ_IS_FP else FQ3,
                         Air(cfg, n, None, o).ce_blowup_factor, o.fri_folding_factor)
        p.memory_budget = (est["streamed"] + est["resident"]) // 2
    out = {}
    try:
        proof = p.prove(claim, ProofOptions(*opts), trace, validate=validate)
        out["bytes"] = proof.to_bytes()
        out["timed"] = sorted(k for k in ("permutation_fill", "lookup_multiplicities") if k in proof.timings)
        claim.verify(out["bytes"], 10)
        out["verified"] = True
    except ConstraintViolation as e:
        out["violations"] = [v.constraint for v in e.violations]
    except VerificationError as e:
        out["rejected"] = str(e)
    out["unchanged"] = bool(np.array_equal(np.asarray(trace.base_columns()), before))
    out["residency"] = p.last_residency
    q.put(out)


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


def _cpu_restatement(which):
    """cpu_prove with the oracles' targets and multiplicities in the oracle's trace, and the extension columns evaluated
    by the oracle"""
    from oracle import extension_oracle as XO
    from oracle import lookup_oracle as LO
    from oracle import permutation_oracle as PO
    from oracle import stark_oracle as SO
    claim, opts, trace = _make_case(which)
    cfg = claim.AirConfig
    mk = lambda n, o: Air(cfg, n, claim.get_public_inputs(), ProofOptions(*o))
    base = LO.fill(cfg, PO.fill(cfg, trace.base_columns()))          # targets first: the lookup reads them
    n = base.shape[1]
    decl = [(c.init, c.mul, c.add, c.inclusive) for c in mk(n, opts).extension_declaration]
    ext = lambda ch: XO.columns(decl, base, 1 if cfg.FQ_IS_FP else 3, ch, cfg.gen_hints(n, claim.get_public_inputs(), ch))
    want = SO.cpu_prove(claim, opts, base, mk, ext_builder=ext)
    SO.verify(claim, want, 10, mk)
    return want


@pytest.mark.parametrize("residency", ["resident", "streamed"])
def test_memory_airs_prove_to_the_restatement(orc, perm_abi, residency):
    out = _spawn(_prove_worker, "memory", perm_abi, residency, True, None)
    assert "violations" not in out, out
    assert out["residency"] == residency and out["verified"] and out["unchanged"]
    assert out["timed"] == ["lookup_multiplicities", "permutation_fill"]
    want = _cpu_restatement("memory")
    assert out["bytes"] == want
    hand = _spawn(_prove_worker, "memory_hand", perm_abi, residency, True, None)
    assert hand["bytes"] == want and hand["timed"] == []


def test_lookup_only_air_keeps_its_proof_bytes(orc, perm_abi):
    """SquareLookupClaim's 2^6-row proof: the bytes of the parent of this change, and no permutation fill timed"""
    out = _spawn(_prove_worker, "square", perm_abi, "resident", False, None)
    assert out["timed"] == ["lookup_multiplicities"]
    assert hashlib.sha256(out["bytes"]).hexdigest() == SQUARE_2P6_SHA256


SQUARE_2P6_SHA256 = "76ef4d1d6be068d3c827a0b6c0ab6bf427d353a7904c53c1448e78eabc318b5b"


@pytest.mark.parametrize("corrupt", ["zero", "swap"])
def test_corrupted_fill_is_refused(perm_abi, corrupt):
    out = _spawn(_prove_worker, "sorted_copy", perm_abi, "resident", True, None)
    assert out.get("verified"), out
    out = _spawn(_prove_worker, "sorted_copy", perm_abi, "resident", True, corrupt)
    assert out.get("violations") and all(k in (1, 2) for k in out["violations"]), out
    out = _spawn(_prove_worker, "sorted_copy", perm_abi, "resident", False, corrupt)
    assert "rejected" in out, out


def _sharded_worker(rank, world, port, which, lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.setdefault("OMP_NUM_THREADS", "2")
    _install(lib_path)
    import torch.distributed as dist
    from ministark_b200.prover_mgpu import ShardedProver
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        claim, opts, trace = _make_case(which)
        q.put((rank, ShardedProver(dist, rank).prove(claim, ProofOptions(*opts), trace).to_bytes()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("which", ["memory", "memory_hand"])
def test_sharded_prover_over_gloo(orc, perm_abi, which):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, which, perm_abi, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=900) for _ in range(2)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    want = _cpu_restatement("memory")
    for rank, b in got:
        assert b == want, f"rank {rank}"


def _own_builder_worker(lib_path, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    _install(lib_path)
    from ministark_b200.prover import GpuProver, ProvingError, Trace
    claim, opts, trace = _make_case("sorted_copy")
    try:
        GpuProver(0).prove(claim, ProofOptions(*opts), Trace(trace.base_columns(), lambda ch: None))
        q.put(None)
    except ProvingError as e:
        q.put(str(e))


def test_trace_with_its_own_extension_builder_is_refused(perm_abi):
    assert "the trace must not bring its own extension columns" in _spawn(_own_builder_worker, perm_abi)


# ---------------------------------------------------------------------------------------------------- 4. header
def test_permutation_header_is_bound_exported_and_separate(perm_abi):
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.PERMUTATION_HEADER_PATH)
    assert declared == sorted(_lib._PERMUTATION_SIGS) == ["ms_permutation_fill", "ms_permutation_workspace_bytes"]
    others = set(_lib.header_symbols()) | set(_lib.header_symbols(_lib.LOOKUP_HEADER_PATH)) | \
        set(_lib.header_symbols(_lib.EXTENSION_HEADER_PATH)) | set(_lib.header_symbols(_lib.CHECK_HEADER_PATH))
    assert not set(declared) & others
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(perm_abi)
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)
