"""prover_mgpu.py — `default_prove` (src/prover.rs:25-174) over G GPUs of one box, one process per GPU.

The reference has no multi-device code (one Metal device, gpu/src/plan.rs:465-469).  What makes the whole prover
shard — not just the first commitment — is the shape of the bit-reversed LDE (src/matrix.rs:225-234): it is
beta = lde_blowup_factor blocks of n rows, block q being the size-n transform of the SAME coefficients over the coset
h_q * <g_n>, h_q = offset * g_N^bitrev(q).  Every step after interpolation is local to a block:

  transform      block q of every column = one size-n coset NTT of the column's coefficients            (LDE)
  leaf hash      a leaf is one LDE row: rows of block q only                                           (src/merkle.rs:412-436)
  constraints    ce-domain point i and its neighbours i + ce_blowup * offset sit in the same block     (src/eval_cpu.rs:115-123)
  DEEP           pointwise over the LDE                                                                (src/composer.rs:89-188)
  FRI fold       a folded value needs ff CONSECUTIVE entries of the bit-reversed codeword               (src/fri.rs:199-231)
  queries        a row and its authentication path below the subtree root live where the row lives

so rank r owns blocks [r * beta/G, (r+1) * beta/G) — a contiguous slab of N/G LDE rows — of every matrix, for the whole
proof.  Only COEFFICIENTS are replicated (n values per column, 1/beta of the LDE): the interpolation of a matrix is
split by columns and the coefficient columns are all-gathered over NVLink (NCCL); no LDE data ever crosses a link.
Per commitment and per FRI layer the G subtree roots (32 bytes each) are all-gathered and every rank finishes the top
log2(G) levels of the tree (src/merkle.rs:485-508), so every rank holds the same transcript: the Fiat–Shamir channel,
the proof-of-work and the query positions are computed identically everywhere and nothing has to be broadcast.  The
proof bytes are identical to the single-GPU prover's (tests/test_gpu_multi.py), hence to the CPU restatement's.

A FRI layer is sharded while every rank still holds at least two of its rows; the remaining small layers are gathered
once and finished on every rank.  torch / torch.distributed are plumbing: buffers, the stream, the collectives.

ShardedProver is a GpuProver that runs GpuProver._default_prove with the _Sharded layout: only what depends on where
the LDE rows live is written here (the column-split interpolation, the slab LDE and commitment, the broadcast of the
ce-domain column, the sharded FRI layers and the query fetch plan).
"""
import hashlib

import numpy as np
import torch

from . import FP
from . import expr as E
from .air import domain_generator
from .cosets import brev as _brev, coset_offsets, merkle_walk
from .proof import LayerProof, MerkleView
from .prover import GpuProver, ProvingError, _Blocks, _Matrix, _Run, _canon_rows, _lift, _mont

P = E.P
_R = 2**64


def top_levels(sub_roots):
    """heap of the top log2(G) levels from the G subtree roots: top[G + r] = root of rank r's subtree, top[1] = the root"""
    g = len(sub_roots)
    top = [None] * (2 * g)
    for r, d in enumerate(sub_roots):
        top[g + r] = bytes(d)
    for k in range(g - 1, 0, -1):
        top[k] = hashlib.sha256(top[2 * k] + top[2 * k + 1]).digest()
    return top


def node_owner(k, log_g):
    """heap node k of the global tree -> (rank, heap index inside that rank's subtree), or (None, k) for the top levels"""
    d = k.bit_length() - 1
    if d < log_g:
        return None, k
    a = k >> (d - log_g)
    return a - (1 << log_g), (1 << (d - log_g)) + (k - (a << (d - log_g)))


class _ShardedTree:
    """rows [rank * n_local, (rank + 1) * n_local) of a tree with n_total leaves: local leaves / nodes + the shared top"""

    def __init__(self, leaves, nodes, n_local, n_total, top):
        self.leaves, self.nodes, self.n_local, self.n_total, self.top = leaves, nodes, n_local, n_total, top


class _FetchPlan:
    """The query phase needs ~30 LDE rows per matrix, ~30 rows per FRI layer and a few hundred path digests, each living
    on the rank that owns its row.  Requests are collected first (every rank builds the same plan, so every rank knows
    who owns what and how many bytes it is), every rank then fetches what it owns with one device gather per matrix /
    tree, and ONE fixed-layout NCCL all-gather of the packed pieces gives every rank everything."""

    def __init__(self, prover):
        self.p = prover
        self.groups = []          # (fetch(list of local indices) -> sequence of byte strings, [(item, local index)])
        self.items = []           # per handle: (owner rank or None for a literal, nbytes)
        self.literal = {}
        self.data = None

    def _new(self, owner, nbytes):
        self.items.append((owner, nbytes))
        return len(self.items) - 1

    def rows(self, gather_local, n_local, positions, row_words):
        """handles of the rows at global `positions`; gather_local(list of local row ids) -> (k, row_words) array"""
        mine, handles = [], []
        for p in positions:
            owner = p // n_local
            h = self._new(owner, 8 * row_words)
            handles.append(h)
            if owner == self.p.rank:
                mine.append((h, p - owner * n_local))
        if mine:
            self.groups.append((lambda loc, f=gather_local: [np.ascontiguousarray(r, dtype=np.uint64).tobytes() for r in f(loc)], mine))
        return handles

    def view(self, tree, positions):
        """handles of a MerkleView over a sharded tree: (path handles, initial-leaf handles, sibling-leaf handles, height)"""
        init, sib, path = merkle_walk(tree.n_total, positions)
        leaf_mine, node_mine = [], []

        def leaf(i):
            owner, loc = divmod(i, tree.n_local)
            h = self._new(owner, 32)
            if owner == self.p.rank:
                leaf_mine.append((h, loc))
            return h

        def node(k):
            owner, loc = node_owner(k, self.p.log_g)
            h = self._new(owner, 32)
            if owner is None:
                self.literal[h] = tree.top[loc] if loc else bytes(32)     # heap index 0: the unused default digest
            elif owner == self.p.rank:
                node_mine.append((h, loc))
            return h

        hi, hs, hp = [leaf(i) for i in init], [leaf(i) for i in sib], [node(k) for k in path]
        dev = self.p.device

        def fetch(t):
            return lambda loc: [r.tobytes() for r in t.index_select(0, torch.tensor(loc, dtype=torch.int64, device=dev)).cpu().numpy()]

        if leaf_mine:
            self.groups.append((fetch(tree.leaves), leaf_mine))
        if node_mine:
            self.groups.append((fetch(tree.nodes), node_mine))
        return hp, hi, hs, tree.n_total.bit_length() - 1

    def execute(self):
        G, rank = self.p.world, self.p.rank
        mine = {}
        for fn, lst in self.groups:
            for (h, _), v in zip(lst, fn([loc for _, loc in lst])):
                mine[h] = v
        # fixed layout: rank r's buffer = its items in handle order; every rank can compute every offset
        sizes = [0] * G
        offset = {}
        for h, (owner, nbytes) in enumerate(self.items):
            if owner is not None:
                offset[h] = sizes[owner]
                sizes[owner] += nbytes
        cap = max(max(sizes), 1)
        buf = bytearray(cap)
        for h, v in mine.items():
            assert len(v) == self.items[h][1]
            buf[offset[h]:offset[h] + len(v)] = v
        send = torch.frombuffer(buf, dtype=torch.uint8).to(self.p.device)
        recv = torch.empty(G * cap, dtype=torch.uint8, device=self.p.device)
        self.p.dist.all_gather_into_tensor(recv, send)
        raw = recv.cpu().numpy().tobytes()
        self.data = dict(self.literal)
        for h, (owner, nbytes) in enumerate(self.items):
            if owner is not None:
                o = owner * cap + offset[h]
                self.data[h] = raw[o:o + nbytes]
        assert len(self.data) == len(self.items), "a queried row or digest has no owner"

    def get_rows(self, handles):
        return np.frombuffer(b"".join(self.data[h] for h in handles), dtype=np.uint64) if handles else np.zeros(0, dtype=np.uint64)

    def get_view(self, v):
        hp, hi, hs, height = v
        return MerkleView([self.data[h] for h in hp], [self.data[h] for h in hi], [self.data[h] for h in hs], height)


class ShardedProver(GpuProver):
    def __init__(self, dist, device):
        super().__init__(device)
        self.dist = dist
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        if self.world & (self.world - 1):
            raise ValueError("world size must be a power of two")
        self.log_g = self.world.bit_length() - 1

    # ---- collectives (on the prover's stream: torch orders NCCL against the current stream)
    def _all_gather_bytes(self, b):
        t = torch.frombuffer(bytearray(b), dtype=torch.uint8).to(self.device)
        out = torch.empty(self.world * len(b), dtype=torch.uint8, device=self.device)
        self.dist.all_gather_into_tensor(out, t)
        raw = out.cpu().numpy().tobytes()
        return [raw[i * len(b):(i + 1) * len(b)] for i in range(self.world)]

    def _all_gather_objects(self, obj):
        out = [None] * self.world
        self.dist.all_gather_object(out, obj)
        return out

    # ---- building blocks
    def _interpolate(self, evals, field, ncols, log_n, from_host=False):
        """Matrix::interpolate (src/matrix.rs:101-116): the inverse transforms are split by columns, the coefficient
        columns all-gathered — every rank ends up with the whole (ncols, n) coefficient matrix.  from_host: `evals` is a
        host matrix of which only this rank's column block is uploaded."""
        n, G = 1 << log_n, self.world
        if ncols < G:
            polys = self._empty(ncols, n * field)
            self.ctx.ntt_batch_to(evals, polys, field, log_n, ncols, inverse=True)
            return polys
        per = (ncols + G - 1) // G
        pad = self._empty(G * per, n * field)
        lo, hi = min(self.rank * per, ncols), min((self.rank + 1) * per, ncols)
        if hi > lo:
            if from_host:
                pad[lo:hi].copy_(self._to_device(evals[lo:hi]))
                self.ctx.ntt_batch(pad[lo], field, log_n, hi - lo, inverse=True)
            else:
                self.ctx.ntt_batch_to(evals[lo], pad[lo], field, log_n, hi - lo, inverse=True)
        self.dist.all_gather_into_tensor(pad.view(-1), pad[self.rank * per:(self.rank + 1) * per].reshape(-1))
        return pad[:ncols]

    def _offsets(self, log_n, log_b):
        """Montgomery words of h_q = offset * g_N^bitrev(q) for this rank's blocks"""
        bpr = (1 << log_b) // self.world
        return coset_offsets(log_n, log_b, range(self.rank * bpr, (self.rank + 1) * bpr))

    def _lde_slab(self, polys, field, ncols, log_n, log_b):
        """this rank's blocks of the bit-reversed LDE of every column: (ncols, N/G) elements, block j at rows [j n, (j+1) n)"""
        n = 1 << log_n
        rows_per = (n << log_b) // self.world
        slab = self._empty(ncols, rows_per * field)
        for j, (_, h) in enumerate(self._offsets(log_n, log_b)):
            self.ctx.lde_batch(polys, slab.data_ptr() + j * n * field * 8, field, log_n, 0, ncols, in_stride=n,
                               out_stride=rows_per, offset=h, bitrev=True)
        return slab

    def _finish_tree(self, sub_root, leaves, nodes, n_local):
        top = top_levels(self._all_gather_bytes(sub_root))
        return _ShardedTree(leaves, nodes, n_local, n_local * self.world, top), top[1]

    def _commit_slab(self, slab, field, ncols, rows_per):
        leaves, nodes = self._empty(rows_per, 4), self._empty(rows_per, 4)
        sub = self.ctx.merkle_commit(slab, field, rows_per, ncols, col_stride=rows_per, leaves=leaves, nodes=nodes)
        return self._finish_tree(sub, leaves, nodes, rows_per)

    def _block_ptrs(self, slab, field, ncols, rows_per, j, n):
        return [slab.data_ptr() + (c * rows_per + j * n) * field * 8 for c in range(ncols)]

    def fri_commit(self, slab, log_n, fq, options, channel):
        """FriProver::build_layers (src/fri.rs:199-231) on a codeword sharded by rows: `slab` holds this rank's
        2^log_n / G consecutive entries of the bit-reversed codeword.  Per layer: rows of ff entries -> leaf hashes ->
        subtree -> all-gather of the G subtree roots -> channel; the fold is local (row k needs only row k).  Layers with
        fewer than 2 rows per rank are gathered once and finished on every rank by GpuProver._fri_layer.  Returns (sharded
        layers, gathered layers, last folded codeword (replicated), its log size); a layer is (evals, tree, root, rows in
        the layer), the tree of a sharded layer a _ShardedTree."""
        ctx, dist, G, rank = self.ctx, self.dist, self.world, self.rank
        ff = options.fri_folding_factor
        log_ff = ff.bit_length() - 1
        run = _Run(ctx=ctx, channel=channel, fq=fq, options=options)        # what _fri_layer reads
        layers, gathered = [], []
        cur, ln, sharded = slab, log_n, True
        for _ in range(options.fri_num_layers(1 << log_n)):
            nrows = 1 << (ln - log_ff)
            if sharded and nrows // G < 2:
                full = self._empty((1 << ln) * fq)
                dist.all_gather_into_tensor(full, cur)
                cur, sharded = full, False
            if sharded:
                nloc = nrows // G
                leaves, nodes = self._empty(nloc, 4), self._empty(nloc, 4)
                sub = ctx.merkle_commit_rows(cur, ff * fq, nloc, leaves=leaves, nodes=nodes)
                tree, root = self._finish_tree(sub, leaves, nodes, nloc)
                channel.commit_fri_layer(root)
                layers.append((cur, tree, root, nrows))
                alpha = channel.draw_fri_alpha()
                nxt = self._empty(nloc * fq)
                off = pow(domain_generator(ln), _brev(rank, self.log_g), P) * _R % P      # ONE * g_(2^ln)^bitrev(rank)
                ctx.fri_fold(cur, nxt, fq, ln - self.log_g, log_ff,
                             np.array([_mont(c) for c in _lift(alpha)], dtype=np.uint64), offset=off)
            else:
                layer, nxt = self._fri_layer(run, cur, ln)
                gathered.append(layer)
            cur, ln = nxt, ln - log_ff
        if sharded:
            full = self._empty((1 << ln) * fq)
            dist.all_gather_into_tensor(full, cur)
            cur = full
        return layers, gathered, cur, ln

    # ---- default_prove: GpuProver's sequence, with this rank's slab of every matrix
    def _prove(self, stark, options, witness, validate=False):
        if validate:
            raise ProvingError("the sharded prover does not validate the trace (its ranks need not hold the whole base "
                               "trace): validate with GpuProver")
        r = self._start(stark, options, witness, False)
        if r.beta % self.world or r.n < 16:
            raise ProvingError("the sharded prover needs a world size dividing the LDE blow-up factor and n >= 16")
        r.lap("init_air")
        return self._default_prove(r, _Sharded(self, r))


class _Sharded(_Blocks):
    """this rank's blocks of every matrix: a slab of N/G consecutive rows of the bit-reversed LDE, committed as this
    rank's subtree of the global tree"""

    def __init__(self, prover, r):
        super().__init__(prover, r)
        self.blocks = prover._offsets(r.log_n, r.log_b)
        self.rows_per = r.N // prover.world

    def commit_base(self):
        p, r = self.p, self.r
        host_base = p._base_columns(r)
        # extension columns are built from the whole base trace (on every rank); with lookups or permutations every
        # rank fills its own copy (each has an extension column)
        if r.next_ > 0 or r.nbase < p.world or (isinstance(host_base, torch.Tensor) and host_base.is_cuda):
            base = p._device_base(r, host_base)
            polys = p._interpolate(base, FP, r.nbase, r.log_n)
        else:
            base, polys = None, p._interpolate(host_base, FP, r.nbase, r.log_n, from_host=True)
        del host_base
        return base, self.commit_coeffs(polys, FP, r.nbase)

    def commit_evals(self, held, field, ncols):
        return self.commit_coeffs(self.p._interpolate(self.p._to_device(held[0]), field, ncols, self.r.log_n), field, ncols)

    def commit_coeffs(self, polys, field, ncols):
        slab = self.p._lde_slab(polys, field, ncols, self.r.log_n, self.r.log_b)
        tree, root = self.p._commit_slab(slab, field, ncols, self.rows_per)
        return _Matrix(polys, slab, field, ncols, tree, root)

    def _cols(self, j, h, mats):
        return [c for m in mats if m for c in self.p._block_ptrs(m.rows, m.field, m.ncols, self.rows_per, j, self.r.n)]

    def constraint_evals(self, base, ext, bind):
        """each block is evaluated where it lives, then the (small) evaluation column is shared"""
        comp_evals = super().constraint_evals(base, ext, bind)
        n, fq = self.r.n, self.r.fq
        for q in range(self.r.ce_blowup):
            self.p.dist.broadcast(comp_evals[q * n * fq:(q + 1) * n * fq], src=q // (self.r.beta // self.p.world))
        return comp_evals

    def composition_polys(self, held):
        """one small transform of the whole ce-domain column, done on every rank"""
        self.p.ctx.bit_reverse(held[0], self.r.fq, self.r.log_ce)
        return self.p._composition_columns(self.r, held[0])

    def fri(self, codeword):
        """layers sharded by rows while every rank keeps >= 2 rows of the layer, then gathered"""
        layers, gathered, cur, ln = self.p.fri_commit(codeword, self.r.log_N, self.r.fq, self.r.options, self.r.channel)
        self.p._fri_tail(self.r, cur, ln)
        return layers, gathered

    def open(self, layers, positions, mats):
        """rows and path digests come from the ranks that own them"""
        p, r, ctx = self.p, self.r, self.p.ctx
        layers, gathered = layers
        ff, fq, rows_per = r.options.fri_folding_factor, r.fq, self.rows_per
        pos_sorted = sorted(set(positions))
        plan = _FetchPlan(p)
        pending, folded = [], positions
        for evals, tree, root, nrows in layers:
            folded = sorted(set(q // ff for q in folded))
            nloc = nrows // p.world
            hr = plan.rows(lambda loc, e=evals, k=nloc: ctx.gather_rows_rowmajor(e, ff * fq, k, loc), nloc, folded, ff * fq)
            pending.append((root, hr, plan.view(tree, folded)))

        def trace_rows(m):
            # Queries::new keeps the caller's position order (sorted, deduplicated by draw_queries)
            return plan.rows(lambda loc: ctx.gather_rows(m.rows, m.field, rows_per, m.ncols, loc, col_stride=rows_per),
                             rows_per, positions, m.ncols * m.field)

        order = [k for k in (0, 2, 1) if mats[k]]          # base, composition, extension
        handles = {k: trace_rows(mats[k]) for k in order}
        views = {k: plan.view(mats[k].tree, pos_sorted) for k in order}
        plan.execute()
        fri_proof = p._fri_queries(r, gathered, folded)      # the gathered layers: on every rank
        fri_proof.layers[:0] = [LayerProof(_canon_rows(plan.get_rows(hr), fq), plan.get_view(hv), root) for root, hr, hv in pending]
        return fri_proof, [(plan.get_rows(handles[k]), plan.get_view(views[k])) if mats[k] else (None, None) for k in range(3)]
