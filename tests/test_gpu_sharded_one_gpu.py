"""GPU, one device: the call shapes only a real shard of ShardedProver (ministark_b200/prover_mgpu.py) passes to the
kernels, and the whole sharded prover with its ranks run as threads.

With one GPU the sharded prover otherwise runs at world size 1 only, where every rank offset is ONE and nothing is split,
and the NCCL tests (tests/test_gpu_multi.py) skip.  So this file pins:

  * ms_fri_fold at non-trivial coset offsets (ONE, the generator, the word p - 1, a random word, and every rank offset
    g_(2^ln)^bitrev(rank) of G = 2, 4, 8 ranks) against the C oracle word for word, the big-integer spec for small
    sizes, and, for the rank offsets, the slice of the whole codeword's fold at offset ONE: the G slab folds side by side
    are the whole fold, which is what fri_commit relies on;
  * ms_merkle_commit_rows_sha256 over G row slabs of a FRI layer, merged by top_levels / node_owner, against the same
    commitment over the whole layer, the oracle's tree and (leaves) hashlib;
  * ShardedProver with G = 2, 4, 8 thread ranks on cuda:0, each with its own Context and streams, exchanging through
    an in-process stand-in for torch.distributed: every rank's proof equals GpuProver's, the CPU restatement's
    (oracle/stark_oracle.cpu_prove) where one exists, and Stark.verify accepts it.  A second proof per prover runs on
    warm plans and scratch.  This also runs several contexts concurrently on one device from several threads."""
import hashlib
import pickle
import threading

import numpy as np
import pytest
import torch

import ministark_b200 as ms
from ministark_b200.air import ProofOptions, domain_generator
from ministark_b200.cosets import brev
from ministark_b200.prover import GpuProver
from ministark_b200.prover_mgpu import ShardedProver, node_owner, top_levels
from oracle import pyspec as S

pytestmark = pytest.mark.gpu

P, R = ms.P, 2**64


@pytest.fixture(scope="module")
def ctx():
    return ms.Context(0)


def _rank_offset(ln, rank, log_g):
    """the Montgomery word fri_commit folds rank `rank`'s slab of a 2^ln-entry layer with: ONE * g_(2^ln)^bitrev(rank)"""
    return pow(domain_generator(ln), brev(rank, log_g), P) * R % P


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()


def _host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint64)


def _fold(ctx, ev, field, log_n, log_ff, alpha, offset):
    """ms_fri_fold of a device codeword (a tensor or a slice of one) at `offset`; returns the host words"""
    out = torch.empty((field << log_n) >> log_ff, dtype=torch.int64, device="cuda")
    ctx.fri_fold(ev, out, field, log_n, log_ff, alpha, offset=offset)
    ctx.sync()
    return _host(out)


def _spec_fold(ev, field, log_n, log_ff, alpha, offset):
    """oracle/pyspec.fri_apply_drp on canonical integers, returned as Montgomery words"""
    canon = [S.from_mont(int(w)) for w in ev]
    elems = canon if field == 1 else [tuple(canon[3 * i:3 * i + 3]) for i in range(len(canon) // 3)]
    a = [S.from_mont(int(w)) for w in alpha]
    got = S.fri_apply_drp(elems, log_n, log_ff, a[0] if field == 1 else tuple(a), field, offset=S.from_mont(offset))
    flat = got if field == 1 else [x for e in got for x in e]
    return np.array([S.to_mont(x) for x in flat], dtype=np.uint64)


# ------------------------------------------------------------------ 1. FRI fold at the offsets a shard passes
NAMED_OFFSETS = {"one": ms.ONE, "generator": ms.GENERATOR, "p-1": P - 1, "random": 0x9C3E_51D2_07A4_B86F % P}


@pytest.mark.parametrize("field", [1, 3])
@pytest.mark.parametrize("log_ff", [1, 2, 3, 4])
@pytest.mark.parametrize("log_n", [4, 7, 11, 15, 20])
def test_fri_fold_at_offset(ctx, orc, field, log_ff, log_n):
    """ms_fri_fold at offsets other than ONE equals the oracle's apply_drp, and the spec's for log_n <= 8"""
    ev = orc.rand_matrix(1, 1 << log_n, field, seed=7 * log_n + log_ff)[0]
    alpha = orc.rand_matrix(1, 1, field, seed=31 + log_n)[0]
    d = _dev(ev)
    for name, off in NAMED_OFFSETS.items():
        got = _fold(ctx, d, field, log_n, log_ff, alpha, off)
        want = orc.fri_apply_drp(ev, field, log_n, log_ff, alpha, offset=off)
        assert np.array_equal(got, want), name
        if log_n <= 8:
            assert np.array_equal(got, _spec_fold(ev, field, log_n, log_ff, alpha, off)), name


@pytest.mark.parametrize("field", [1, 3])
@pytest.mark.parametrize("log_ff", [1, 2, 3, 4])
@pytest.mark.parametrize("log_n", [4, 7, 11, 15, 20])
def test_fri_fold_of_rank_slabs_is_the_whole_fold(ctx, orc, field, log_ff, log_n):
    """rank r of G holds entries [r 2^ln / G, (r + 1) 2^ln / G) of the bit-reversed layer: a bit-reversed codeword over
    the coset g_(2^ln)^bitrev(r) <g_(2^ln / G)>.  Folded at that offset, the G slabs side by side equal the whole layer
    folded at ONE, and each equals the oracle's (and, small, the spec's) apply_drp of the slab at that offset"""
    ev = orc.rand_matrix(1, 1 << log_n, field, seed=3 * log_n + log_ff)[0]
    alpha = orc.rand_matrix(1, 1, field, seed=77 + log_ff)[0]
    d = _dev(ev)
    whole = _fold(ctx, d, field, log_n, log_ff, alpha, ms.ONE)
    assert np.array_equal(whole, orc.fri_apply_drp(ev, field, log_n, log_ff, alpha))
    ran = 0
    for log_g in (1, 2, 3):
        ls = log_n - log_g                      # log2 of the slab's entries
        if ls < log_ff:
            continue
        G, words, out_words = 1 << log_g, field << ls, (field << ls) >> log_ff
        for rank in range(G):
            off = _rank_offset(log_n, rank, log_g)
            got = _fold(ctx, d[rank * words:(rank + 1) * words], field, ls, log_ff, alpha, off)
            assert np.array_equal(got, whole[rank * out_words:(rank + 1) * out_words]), (G, rank)
            slab = ev[rank * words:(rank + 1) * words]
            assert np.array_equal(got, orc.fri_apply_drp(slab, field, ls, log_ff, alpha, offset=off)), (G, rank)
            if ls <= 8:
                assert np.array_equal(got, _spec_fold(slab, field, ls, log_ff, alpha, off)), (G, rank)
            ran += 1
    assert ran or log_n - 1 < log_ff


@pytest.mark.parametrize("log_ff", [1, 2, 3, 4])
def test_fri_fold_structured_codewords_at_a_rank_offset(ctx, orc, log_ff):
    """few-valued codewords (constants, 2^63 / 2^62 pairs whose sums hit 2^64 exactly, 0/1 flags) folded at the offset
    of rank 3 of 4, as in test_gpu_commit_stages_fri.py's structured case at ONE"""
    log_n, log_g, rank = 12, 2, 3
    ls = log_n - log_g
    n = 1 << ls
    off = _rank_offset(log_n, rank, log_g)
    assert off != ms.ONE
    rng = np.random.default_rng(100 + log_ff)
    pool = np.array([0, ms.ONE, 2**63, 2**62, P - 1, P - 2**63, 2**32, 2**32 - 2], dtype=np.uint64)
    alpha = orc.rand_matrix(1, 1, 3, seed=19)[0]
    for lanes in (1, 3):
        a = alpha[:lanes]
        for pick in (pool[rng.integers(0, 4, size=n * lanes)], np.full(n * lanes, 2**63, dtype=np.uint64),
                     pool[(np.arange(n * lanes) // 3) % len(pool)]):
            ev = np.ascontiguousarray(pick, dtype=np.uint64)
            got = _fold(ctx, _dev(ev), lanes, ls, log_ff, a, off)
            assert np.array_equal(got, orc.fri_apply_drp(ev, lanes, ls, log_ff, a, offset=off))


# ------------------------------------------------------------------ 1b. slab commitments of a FRI layer
def _digests(t, n):
    return _host(t).view(np.uint8).reshape(n, 32)


def _commit_rows(ctx, rows, row_words, nrows):
    leaves, nodes = (torch.empty((nrows, 4), dtype=torch.int64, device="cuda") for _ in range(2))
    root = ctx.merkle_commit_rows(rows, row_words, nrows, leaves=leaves, nodes=nodes)
    ctx.sync()
    return root, _digests(leaves, nrows), _digests(nodes, nrows)


@pytest.mark.parametrize("fq", [1, 3])
@pytest.mark.parametrize("ff", [2, 4, 8, 16])
@pytest.mark.parametrize("G", [2, 4, 8])
@pytest.mark.parametrize("nloc", [2, 128])
def test_slab_commitments_merge_to_the_whole_tree(ctx, orc, fq, ff, G, nloc):
    """a layer of rows of ff * fq words committed as G row slabs (ms_merkle_commit_rows_sha256 on each), whose sub-roots
    are merged by top_levels: the root, the leaves and the node heap (read through node_owner) equal the commitment of
    the whole layer and the oracle's tree.  2 rows per rank is the smallest slab fri_commit keeps sharded."""
    nrows, rw = nloc * G, ff * fq
    layer = orc.rand_matrix(1, nrows * ff, fq, seed=ff * 10 + fq + G)[0]
    d = _dev(layer)
    root, leaves, nodes = _commit_rows(ctx, d, rw, nrows)
    subs = [_commit_rows(ctx, d[r * nloc * rw:(r + 1) * nloc * rw], rw, nloc) for r in range(G)]
    top = top_levels([s[0] for s in subs])
    assert top[1] == root
    assert np.array_equal(np.concatenate([s[1] for s in subs]), leaves)
    log_g = G.bit_length() - 1
    for k in range(1, nrows):
        owner, loc = node_owner(k, log_g)
        got = top[loc] if owner is None else subs[owner][2][loc].tobytes()
        assert got == nodes[k].tobytes(), k
    # the layer matrix of the reference: row k = ff consecutive entries (Matrix::from_arrays, src/fri.rs:199-216)
    cols = np.ascontiguousarray(layer.reshape(nrows, ff, fq).transpose(1, 0, 2)).reshape(ff, -1)
    want_leaves = orc.hash_rows(cols, fq)
    want_nodes = orc.merkle_nodes(want_leaves)
    assert np.array_equal(leaves, want_leaves)
    assert np.array_equal(nodes[1:], want_nodes[1:])
    assert root == want_nodes[1].tobytes()


@pytest.mark.parametrize("fq", [1, 3])
def test_slab_leaves_against_hashlib(ctx, orc, fq):
    """leaf = SHA-256 of the row's canonical words, 8 bytes little-endian each (src/hash.rs:92-99), for slabs of two
    rows of 4 ranks, with edge words in the layer; the tree above them by hashlib too"""
    ff, G, nloc = 4, 4, 2
    nrows, rw = G * nloc, ff * fq
    layer = orc.rand_matrix(1, nrows * ff, fq, seed=5 + fq)[0]
    layer[:6] = [0, ms.ONE, P - 1, S.to_mont(P - 1), S.to_mont(2**32), S.to_mont(2**63)]
    d = _dev(layer)
    subs = [_commit_rows(ctx, d[r * nloc * rw:(r + 1) * nloc * rw], rw, nloc) for r in range(G)]
    rows = layer.reshape(nrows, rw)
    want = [hashlib.sha256(b"".join(S.from_mont(int(w)).to_bytes(8, "little") for w in row)).digest() for row in rows]
    assert [lf.tobytes() for s in subs for lf in s[1]] == want
    assert top_levels([s[0] for s in subs])[1] == S.merkle_nodes(want)[1]


# ------------------------------------------------------------------ 2. the sharded prover on thread ranks
class _ThreadGroup:
    """An in-process stand-in for the torch.distributed calls ShardedProver makes, for G ranks that are G threads of
    this process on one device.  Ordered as NCCL orders a collective on the caller's current stream: a rank first
    waits for its stream (the prover issues collectives on its own stream), deposits its send buffer, and meets its
    peers at a barrier; each then copies the parts into its output on its own stream and waits for those copies before
    a second barrier, so no rank reuses or frees a buffer a peer still reads.  abort() breaks the barrier: every rank
    waiting at it, or arriving at it later, raises threading.BrokenBarrierError."""

    def __init__(self, world, timeout=300):
        self.world = world
        self.slots = [None] * world
        self.barrier = threading.Barrier(world, timeout=timeout)

    def rank(self, r):
        return _ThreadRank(self, r)

    def abort(self):
        self.barrier.abort()


class _ThreadRank:
    """torch.distributed as rank `r` of a _ThreadGroup sees it"""

    def __init__(self, group, r):
        self.g, self.r = group, r

    def get_world_size(self):
        return self.g.world

    def get_rank(self):
        return self.r

    def _exchange(self, send, collect):
        stream = torch.cuda.current_stream()
        stream.synchronize()
        self.g.slots[self.r] = send
        self.g.barrier.wait()
        try:
            collect(self.g.slots)
            stream.synchronize()
        finally:
            self.g.barrier.wait()

    def all_gather_into_tensor(self, out, inp):
        k = inp.numel()
        dst = out.view(-1)
        assert dst.numel() == k * self.g.world

        def collect(parts):
            for q, t in enumerate(parts):
                part = dst[q * k:(q + 1) * k]
                if part.data_ptr() != t.data_ptr():          # in place: this rank's part already sits in `out`
                    part.copy_(t.reshape(-1))
        self._exchange(inp, collect)

    def broadcast(self, tensor, src):
        def collect(parts):
            if self.r != src:
                tensor.copy_(parts[src])
        self._exchange(tensor, collect)

    def all_gather_object(self, out, obj):
        def collect(parts):
            out[:] = [pickle.loads(pickle.dumps(o)) for o in parts]
        self._exchange(obj, collect)


def _prove_on_thread_ranks(world, claim, opts, trace):
    """two proofs per rank by ShardedProver(rank of a _ThreadGroup, device 0), the ranks running as threads; returns
    [[first, second] bytes per rank], or raises the exception of the rank that failed first"""
    group = _ThreadGroup(world)
    proofs, errors = [None] * world, [None] * world

    def run(rank):
        try:
            prover = ShardedProver(group.rank(rank), 0)
            proofs[rank] = [prover.prove(claim, opts, trace).to_bytes() for _ in range(2)]
            prover.ctx.sync()
        except BaseException as e:          # handed to the test's thread below
            errors[rank] = e
            group.abort()

    threads = [threading.Thread(target=run, args=(r,), name=f"thread-rank-{r}", daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=900)
    if any(t.is_alive() for t in threads):
        group.abort()
        for t in threads:
            t.join(timeout=60)
        assert not any(t.is_alive() for t in threads), "a thread rank did not finish"
        pytest.fail("the thread ranks did not finish in time")
    torch.cuda.synchronize()
    failed = [e for e in errors if e is not None]
    if failed:          # the rank that failed, not the peers it released from a barrier
        raise next((e for e in failed if not isinstance(e, threading.BrokenBarrierError)), failed[0])
    return proofs


def _case(which):
    """(claim, ProofOptions, trace, CPU restatement bytes or None) of a named case; the fib, perm and brainfuck cases
    are the gloo suite's (tests/test_prover_cpu_device.py), memory is tests/test_permutation_cpu.py's"""
    if which == "memory":
        from test_permutation_cpu import _cpu_restatement, _make_case
    elif which == "rescue":             # K = 64 chains of L = 4 permutations: 2^11 rows, built on the device
        from ministark_b200.examples import rescue as RX
        trace, digests = RX.gen_trace([11, 22, 33, 44], 64, 4, device=0)
        torch.cuda.synchronize()
        return RX.RescueChainsClaim([11, 22, 33, 44], 64, 4, digests), RX.OPTIONS, trace, None
    else:
        from test_prover_cpu_device import _cpu_restatement, _make_case
    claim, opts, trace = _make_case(which)
    return claim, ProofOptions(*opts), trace, _cpu_restatement(which)


_CASES = {}


def _cached_case(which):
    if which not in _CASES:
        _CASES[which] = _case(which)
    return _CASES[which]


@pytest.mark.parametrize("world,which", [
    (2, "fib:7:16,4,4,8,16"), (4, "fib:7:16,4,4,8,16"),
    (2, "fib:10:32,4,8,8,64"), (4, "fib:9:32,4,8,8,64"),
    (2, "fib:6:10,2,0,2,8"),
    (8, "fib:8:16,8,3,4,8"),
    (2, "perm"), (4, "perm"),
    (2, "brainfuck"), (4, "brainfuck"),
    (2, "memory"), (4, "memory"),
    (2, "rescue"),
])
def test_sharded_prover_on_thread_ranks(orc, world, which):
    """every rank's two proofs are the same bytes, GpuProver's bytes, the CPU restatement's, and Stark.verify accepts them"""
    claim, opts, trace, want = _cached_case(which)
    proofs = _prove_on_thread_ranks(world, claim, opts, trace)
    single = GpuProver(0).prove(claim, opts, trace).to_bytes()
    for rank, (first, second) in enumerate(proofs):
        assert first == second == single, f"rank {rank} of {world}"
    if want is not None:
        assert single == want, "GpuProver differs from the CPU restatement"
    claim.verify(single, 10)


def test_a_failing_rank_ends_every_thread():
    """a rank that raises before its first collective aborts the group: every thread ends and the test sees that rank's
    exception, not its peers' BrokenBarrierError"""
    from ministark_b200.examples import fib

    class Boom(RuntimeError):
        pass

    class Witness:
        def __init__(self, t):
            self.t = t

        def __len__(self):
            return len(self.t)

        def base_columns(self):
            if threading.current_thread().name.endswith("-1"):
                raise Boom("rank 1 cannot read its trace")
            return self.t.base_columns()

        def build_extension_columns(self, challenges):
            return None

    trace, last = fib.gen_trace(8 << 7)
    before = threading.active_count()
    with pytest.raises(Boom, match="rank 1"):
        _prove_on_thread_ranks(4, fib.FibClaim(last), ProofOptions(16, 4, 4, 8, 16), Witness(trace))
    assert threading.active_count() == before
