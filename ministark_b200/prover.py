"""prover.py — `default_prove` (src/prover.rs:25-174) with every data-parallel step on the GPU.

Same order of commitments and Fiat–Shamir draws as the reference, so the transcript — and with it every
root, out-of-domain value, FRI layer and query in the proof — is determined by the same inputs.  What changes is
where the data lives and how each step is computed:

  reference (per step, host <-> unified memory)            here (resident in HBM, only digests/rows return)
  ---------------------------------------------------------------------------------------------------------
  Matrix::interpolate, bit_reversed_evaluate               ms_ntt_batch_to + ms_lde_batch (bit-reversed out)
  MerkleTree::from_matrix (CPU SHA-256)                    ms_merkle_commit_sha256, leaves + nodes stay on device
  bit_reverse_ce_trace x2 + eval_cpu::eval                 ms_eval_constraints on the bit-reversed LDE prefix
  into_polynomials + push loop + LDE                       ms_ntt_batch (ce coset) + ms_matrix_from_rows + ms_lde_batch
  horner_evaluate per column                               ms_poly_eval
  divide_out_points_into, sum_columns, degree adjust, LDE  one fused pointwise evaluation over the LDE (deep.py)
  apply_drp (iNTT + fold + NTT + 2 bit reversals)          ms_merkle_commit_rows_sha256 + ms_fri_fold per layer
  grind_proof_of_work (rayon find_any)                     ms_pow_grind_sha256 (smallest nonce)
  prove_rows / get_row                                     ms_merkle_prove_sha256 + ms_gather_rows(_rowmajor)

torch is used for device buffers and the stream only.  There is no CPU fallback: without the CUDA library the
Context constructor raises.
"""
import copy
import ctypes as C
import hashlib
import time
import weakref
from dataclasses import dataclass

import numpy as np
import torch

from . import FP, FQ3, GENERATOR as GEN_MONT, ONE, Context
from . import deep
from . import expr as E
from . import verifier
from .air import Air, _leaves, domain_generator
from .channel import ProverChannel, PublicCoin, serialize_element
from .cosets import block_program, coset_offsets, heap_location, merkle_walk
from .proof import FriProof, LayerProof, MerkleView, Proof, Queries

P = E.P
_R = 2**64
_RINV = pow(_R, -1, P)


class ProvingError(RuntimeError):
    pass


def _mont(v):
    return int(v) * _R % P


def _canon_rows(words, fq_words):
    """numpy Montgomery words -> flat list of canonical ints (fq_words == 1) or 3-tuples"""
    flat = [int(w) * _RINV % P for w in np.asarray(words, dtype=np.uint64).ravel()]
    if fq_words == 1:
        return flat
    return [tuple(flat[i:i + 3]) for i in range(0, len(flat), 3)]


def _lift(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (int(v), 0, 0)


class Trace:
    """src/trace.rs:13-35.  base_columns(): (ncols, n) uint64 Montgomery words — a numpy array or a cuda int64 tensor.
    build_extension_columns(challenges): None, or (ncols, n * fq_words) words of Fq elements."""

    def __init__(self, base, extension_builder=None):
        self._base, self._ext = base, extension_builder

    def base_columns(self):
        return self._base

    def __len__(self):
        return int(self._base.shape[1])

    def build_extension_columns(self, challenges):
        return None if self._ext is None else self._ext(challenges)


def declared_extension_columns(ctx, air, challenges, hints, base, device):
    """the extension columns `air` declares (AirConfig.extension_columns), built on the device from the natural-order base
    columns `base` ((NUM_BASE_COLUMNS, n) device tensor) by ms_extension_columns: the cached program bound with this
    proof's challenges and hints, each init evaluated on the host.  Returns a (K, n * fq) device tensor."""
    cfg = air.config
    fq = FP if cfg.FQ_IS_FP else FQ3
    decl, prog = air.extension_declaration, air.extension_program()
    for k, c in enumerate(decl):
        for e in (c.init, c.mul, c.add):
            for (i,) in sorted(_leaves(e, "hint")):
                if i >= len(hints):
                    raise ProvingError(f"extension column {cfg.NUM_BASE_COLUMNS + k} reads Hint({i}), but gen_hints "
                                       f"returned {len(hints)} hints")
    prog = prog.bind(challenges=challenges, hints=hints)
    init = np.array([[_mont(w) for w in E.evaluate_at(c.init, 0, challenges=challenges, hints=hints)[:fq]] for c in decl],
                    dtype=np.uint64)
    n = air.trace_len
    out = torch.empty((len(decl), n * fq), dtype=torch.int64, device=device)
    tables = E.periodic_tables(ctx, prog, air.log_n, 1, offset_canonical=1)
    try:
        ctx.extension_columns(prog, out, air.log_n, [base[c] for c in range(cfg.NUM_BASE_COLUMNS)] + [p for p, _ in tables],
                              [False] * cfg.NUM_BASE_COLUMNS + [q for _, q in tables], fq, init, [c.inclusive for c in decl])
    finally:
        if tables:
            ctx.sync()
        for p, _ in tables:
            ctx.free(p)
    return out


@dataclass(frozen=True)
class LookupMiss:
    """value tuple `tuple` of lookup `lookup` fails at `count` (row, tuple) pairs, the lowest row being `first_row`:
    kind "missing": its tuple is not in the table (count: rows of this tuple); kind "selector": its selector is neither 0
    nor 1 (count: such pairs over all of the lookup's tuples).  values: the tuple at first_row as canonical integers, and
    the selector for kind "selector"."""
    lookup: int
    tuple: int
    kind: str
    first_row: int
    count: int
    values: tuple
    selector: int = None

    def message(self):
        if self.kind == "missing":
            return (f"lookup {self.lookup}, value tuple {self.tuple}: {self.values} at row {self.first_row} is not in the "
                    f"table ({self.count} rows of this tuple are not)")
        return (f"lookup {self.lookup}, value tuple {self.tuple}: the selector is {self.selector} at row {self.first_row}, "
                f"neither 0 nor 1 ({self.count} (row, tuple) pairs of this lookup have such a selector); the tuple there is "
                f"{self.values}")


class LookupViolation(ProvingError):
    """a lookup of the AIR does not hold for the trace (raised before anything is committed): `misses` lists one LookupMiss
    per failing (lookup, value tuple); the message names the first"""

    def __init__(self, misses):
        self.misses = list(misses)
        more = f" (and {len(self.misses) - 1} more failing lookup tuples)" if len(self.misses) > 1 else ""
        super().__init__(self.misses[0].message() + more)


def _lookup_misses(ctx, air, base, l, missing, bad):
    """LookupMiss entries of lookup l from the kernel's status, with the named rows' tuples evaluated on the host from
    cells gathered off the device"""
    lk, n, nbase = air.lookups[l], air.trace_len, air.config.NUM_BASE_COLUMNS
    exprs = [e for v in lk.values for e in v] + list(lk.selectors or ())
    leaves = sorted(set().union(*(_leaves(e, "trace") for e in exprs)))
    g = domain_generator(air.log_n)

    def at(row):
        ids = sorted({(row + off) % n for _, off in leaves})
        got = ctx.gather_rows(base, FP, n, nbase, ids) if ids else None
        cells = {(c, off): int(got[ids.index((row + off) % n), c]) * _RINV % P for c, off in leaves}
        ev = lambda e: E.evaluate_at(e, pow(g, row, P), cells, trace_len=n)[0]
        return ([tuple(ev(w) for w in v) for v in lk.values],
                [1] * len(lk.values) if lk.selectors is None else [ev(s) for s in lk.selectors])

    out = []
    for q, (count, row) in enumerate(missing):
        if count:
            vals, _ = at(row)
            out.append(LookupMiss(l, q, "missing", row, count, vals[q]))
    if bad[0]:
        vals, sels = at(bad[1])
        out += [LookupMiss(l, q, "selector", bad[1], bad[0], vals[q], sels[q]) for q in range(len(sels)) if sels[q] not in (0, 1)]
    return sorted(out, key=lambda m: (m.tuple, m.kind))


def fill_lookup_multiplicities(ctx, air, base):
    """the multiplicity column of every lookup `air` declares (AirConfig.lookups), written into `base` ((NUM_BASE_COLUMNS,
    n) natural-order device tensor, the prover's own copy) by ms_lookup_multiplicities, one call per lookup with the
    cached programs.  Raises LookupViolation if a value tuple is not in its table or a selector is neither 0 nor 1."""
    nbase, log_n = air.config.NUM_BASE_COLUMNS, air.log_n
    misses = []
    for l, (lk, prog) in enumerate(zip(air.lookups, air.lookup_programs())):
        W, Q = len(lk.table), len(lk.values)
        work = torch.empty(ctx.lookup_workspace_bytes(log_n, W, Q), dtype=torch.uint8, device=base.device)
        tables = E.periodic_tables(ctx, prog, log_n, 1, offset_canonical=1)
        try:
            missing, bad = ctx.lookup_multiplicities(prog, base[lk.multiplicity], log_n,
                                                     [base[c] for c in range(nbase)] + [p for p, _ in tables], W, Q, work)
        finally:
            for p, _ in tables:
                ctx.free(p)
        del work
        if any(c for c, _ in missing) or bad[0]:
            misses += _lookup_misses(ctx, air, base, l, missing, bad)
    if misses:
        raise LookupViolation(misses)


def fill_permutation_targets(ctx, air, base):
    """the target columns of every permutation `air` declares (AirConfig.permutations), written into `base`
    ((NUM_BASE_COLUMNS, n) natural-order device tensor, the prover's own copy) by ms_permutation_fill, one call per
    permutation in declaration order with the cached programs"""
    nbase, log_n = air.config.NUM_BASE_COLUMNS, air.log_n
    for pm, prog in zip(air.permutations, air.permutation_programs()):
        W = len(pm.source)
        work = torch.empty(ctx.permutation_workspace_bytes(log_n, W), dtype=torch.uint8, device=base.device)
        tables = E.periodic_tables(ctx, prog, log_n, 1, offset_canonical=1)
        try:
            ctx.permutation_fill(prog, [base[t] for t in pm.target], log_n,
                                 [base[c] for c in range(nbase)] + [p for p, _ in tables], W, work)
        finally:
            if tables:
                ctx.sync()
            for p, _ in tables:
                ctx.free(p)
        del work                                # freed in stream order: the fill runs on the prover's stream


def check_lookup_trace(air, trace):
    """a trace that builds its own extension columns cannot know the columns the prover fills (lookup multiplicities,
    permutation targets): refused for an AIR with lookups or permutations, before anything is computed"""
    if (air.lookups or air.permutations) and (
            hasattr(trace, "build_extension_columns_device") or getattr(trace, "_ext", None) is not None
            or type(trace).build_extension_columns is not Trace.build_extension_columns):
        raise ProvingError("the AIR declares lookups or permutations, whose running columns the package builds from the "
                           "columns it fills; the trace must not bring its own extension columns")


class _Tree:
    def __init__(self, leaves, nodes, n):
        self.leaves, self.nodes, self.n = leaves, nodes, n


class Stark:
    """src/stark.rs:24-85.  Subclass: set AirConfig, implement get_public_inputs / generate_trace and, if the
    public inputs are not a single Fp, public_inputs_bytes()."""
    AirConfig = None

    def get_public_inputs(self):
        raise NotImplementedError

    def generate_trace(self, witness):
        return witness

    def public_inputs_bytes(self, public_inputs):
        """CanonicalSerialize of PublicInputs (compressed).  Default: one field element, or a tuple/list of them
        (ark-serialize writes tuple members back to back)."""
        if isinstance(public_inputs, list):
            return b"".join(serialize_element(v) for v in public_inputs)
        return serialize_element(public_inputs)

    def gen_public_coin(self, air):
        """examples/fib/main.rs:166-172: SHA-256(public inputs ‖ trace_len ‖ options), all serialize_compressed"""
        import hashlib
        seed = self.public_inputs_bytes(air.public_inputs) + int(air.trace_len).to_bytes(8, "little") + air.options.to_bytes()
        return PublicCoin(hashlib.sha256(seed).digest(), ext=not self.AirConfig.FQ_IS_FP)

    def gen_deep_coeffs(self, public_coin, air):
        """src/stark.rs:42-54"""
        ex = [public_coin.draw() for _ in range(len(air.trace_arguments()))]
        co = [public_coin.draw() for _ in range(air.ce_blowup_factor)]
        return ex, co, (public_coin.draw(), public_coin.draw())

    def prove(self, options, witness, device=0, validate=False):
        """Stark::prove (src/stark.rs:57-63).  The per-device prover (context, stream, compiled AIR programs) is created
        on first use and reused, like the reference's process-global Planner.  validate=True: check the trace against
        the AIR before the composition polynomial is computed (validate_constraints)."""
        return GpuProver.shared(device).prove(self, options, witness, validate=validate)

    def verify(self, proof, required_security_bits):
        """Stark::verify (src/stark.rs:78-84): default_verify of `proof` — a Proof, or its bytes (Proof.from_bytes with
        this claim's field) — against this claim, on the host (ministark_b200/verifier.py).  Returns the
        VerifierChannelArtifacts; raises verifier.VerificationError, or proof.ProofFormatError for bytes that are not a
        proof."""
        if isinstance(proof, (bytes, bytearray, memoryview)):
            proof = Proof.from_bytes(proof, self.AirConfig.FQ_IS_FP)
        return verifier.verify(self, proof, required_security_bits)

    def validate_constraints(self, air, challenges, hints, base_trace, extension_trace, ctx):
        """Stark::validate_constraints (src/stark.rs:65-75), called by `prove(..., validate=True)` right after the
        extension trace commitment (src/prover.rs:74-75) with the natural-order base and extension columns on the device.
        Default: every constraint at every row (ministark_b200/validate.py); raises ConstraintViolation if any fails."""
        from .validate import ConstraintViolation, validate_constraints
        violations = validate_constraints(ctx, air, challenges, hints, base_trace, extension_trace)
        if violations:
            raise ConstraintViolation(violations)


# Device memory torch does not see, kept free on top of either estimate: the NTT plans with their twiddle and scale
# tables (hundreds of MiB for 2^24-point LDEs), the NTT temporary (at most 1.125 GiB) and the context's scratch arenas.
MEMORY_RESERVE = 3 << 30


def peak_bytes(n, beta, nbase, next_, fq, ce_blowup, ff=2):
    """Peak bytes of one proof in each residency, from the shapes: {"resident": .., "streamed": .., "streamed_host": ..}
    on the device, and "host": the pinned host bytes of streamed_host.

    resident: every matrix's coefficients and bit-reversed LDE, and the leaf and node arrays of every tree, live until
    the queries, and so does the ce-domain composition column.  streamed: the coefficients, one coset block of every
    matrix and the node arrays (no leaves; one block's leaf digests in context scratch).  streamed_host: streamed with the
    node arrays in pinned host memory ("host"); the device holds two staging heaps of one block instead.  All hold the
    DEEP codeword and the FRI layers (folded codewords and trees, a geometric series in the folding factor ff), and
    16 MiB for the small buffers (block roots, top heaps, remainder, query rows) and the allocator's rounding."""
    N, M = n * beta, n * ce_blowup
    words = nbase + fq * (next_ + ce_blowup)                 # words per row over all matrices
    ntrees = 3 if next_ else 2
    fri = (8 * fq + 64) * N // (ff - 1)
    common = 8 * words * n + 8 * N * fq + fri + (16 << 20)
    blocks = common + 8 * words * n + 32 * n
    return {"resident": common + 8 * M * fq + 8 * words * N + 64 * ntrees * N,
            "streamed": blocks + 32 * ntrees * N,
            "streamed_host": blocks + 64 * n,
            "host": 32 * ntrees * N}


def _free_pinned(ctx, addr):
    ctx.sync()                  # the last block heaps may still be crossing into it
    ctx.free(addr)


def _gib(b):
    return f"{b / 2**30:.2f} GiB"


class _Run:
    """per-proof state shared by the phases of every residency (resident, streamed, sharded)"""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class _Matrix:
    """a committed matrix: its coefficients, its LDE rows where the residency keeps them (the whole bit-reversed LDE
    when resident, one coset-block buffer when streamed, this rank's slab when sharded), its Merkle tree and root"""

    def __init__(self, polys, rows, field, ncols, tree=None, root=None):
        self.polys, self.rows, self.field, self.ncols, self.tree, self.root = polys, rows, field, ncols, tree, root


class _Layout:
    """where one proof's LDE rows live: the steps of GpuProver._default_prove that depend on it"""

    def __init__(self, prover, r):
        self.p, self.r = prover, r

    def fri(self, codeword):
        """FRI layers (fri.rs:179-249), the remainder and the proof of work; returns the committed layers"""
        r = self.r
        log_ff = r.options.fri_folding_factor.bit_length() - 1
        layers = []
        cur, ln = codeword, r.log_N
        for _ in range(r.options.fri_num_layers(r.N)):
            layer, cur = self.p._fri_layer(r, cur, ln)
            layers.append(layer)
            ln -= log_ff
        self.p._fri_tail(r, cur, ln)
        return layers


class GpuProver:
    """owns the device context (one in-order stream) and runs default_prove.

    Three residencies, chosen per proof from the estimates of `peak_bytes` against `memory_available()` and
    `host_memory_budget`:
      resident       every LDE matrix and both arrays of every Merkle tree stay in HBM until the queries (the fastest);
      streamed       only coefficients and tree nodes stay; each coset block of the LDE is recomputed where it is needed
                     (commitment, constraint evaluation, DEEP) and query rows come from the coefficients (ms_lde_rows);
      streamed_host  streamed with every tree's node heap in pinned host memory: each block's subtree is copied out
                     while the next block's LDE runs, and the queries gather their path nodes on the host.
    All emit the same proof bytes.  The resident path runs whenever it fits, streamed_host only with a host budget."""
    _shared = {}
    memory_budget = None        # bytes one proof may use on the device; None: whatever the device has free
    host_memory_budget = None   # pinned host bytes one proof may hold (streamed_host's node heaps); None: none.  Heaps
                                # pinned under a larger budget are freed when the next proof starts
    last_residency = None       # "resident", "streamed" or "streamed_host": what the last proof ran
    _pinned = None              # (address, bytes, finalizer) of the pinned node heaps, kept for the next proof

    @classmethod
    def shared(cls, device=0):
        if device not in cls._shared:
            cls._shared[device] = cls(device)
        return cls._shared[device]

    def __init__(self, device=0, memory_budget=None, host_memory_budget=None):
        self.device = torch.device("cuda", device)
        self.stream = torch.cuda.Stream(device=self.device)
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self.ctx = Context(device, stream=self.stream.cuda_stream)
        self._airs = {}
        self.memory_budget = memory_budget
        self.host_memory_budget = host_memory_budget

    @property
    def pinned_bytes(self):
        """pinned host memory the prover holds for streamed_host's node heaps (0 before its first such proof)"""
        return self._pinned[1] if self._pinned else 0

    def release_host_memory(self):
        """free the pinned node heaps; the next streamed_host proof pins them again.  A prover that is dropped frees
        them too (a finalizer that keeps the context alive until it has run)"""
        if self._pinned:
            self._pinned[2]()
            self._pinned = None

    def _host_heaps(self, nbytes):
        """a uint8 view of at least nbytes of pinned host memory: the held allocation while it is large enough"""
        if self._pinned and self._pinned[1] < nbytes:
            self.release_host_memory()
        if not self._pinned:
            addr = self.ctx.alloc_host_pinned(nbytes)
            self._pinned = (addr, nbytes, weakref.finalize(self, _free_pinned, self.ctx, addr))
        return np.ctypeslib.as_array(C.cast(self._pinned[0], C.POINTER(C.c_uint8)), shape=(nbytes,))

    # ---- helpers
    def _to_device(self, a):
        if isinstance(a, torch.Tensor):
            return a.to(self.device)
        a = np.ascontiguousarray(a, dtype=np.uint64)
        return torch.from_numpy(a.view(np.int64)).to(self.device, non_blocking=False)

    def _own_copy(self, a):
        """a device copy of the (host or device) matrix `a` that shares no memory with it"""
        if not isinstance(a, torch.Tensor):
            a = torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64))
        return a.to(self.device, dtype=torch.int64, copy=True).contiguous()

    def _empty(self, *shape):
        return torch.empty(shape, dtype=torch.int64, device=self.device)

    def _view(self, tree, positions):
        nodes, init, sib, height = self.ctx.merkle_prove(tree.leaves, tree.nodes, tree.n, positions)
        return MerkleView(nodes, init, sib, height)

    # ---- residency
    def memory_available(self):
        """bytes a proof may allocate: free device memory as CUDA reports it, plus what torch's allocator holds unused,
        minus MEMORY_RESERVE, capped by memory_budget.  Off a CUDA device only memory_budget limits (None: no limit)."""
        cap = self.memory_budget
        if self.device.type != "cuda":
            return float("inf") if cap is None else cap
        free, _ = torch.cuda.mem_get_info(self.device)
        idle = torch.cuda.memory_reserved(self.device) - torch.cuda.memory_allocated(self.device)
        avail = free + idle - MEMORY_RESERVE
        return avail if cap is None else min(cap, avail)

    def choose_residency(self, est):
        """"resident" if its estimate fits, else "streamed" if that fits, else "streamed_host" if its device estimate fits
        and its node heaps fit host_memory_budget, else ProvingError (nothing is allocated yet)"""
        budget = self.memory_available()
        if est["resident"] <= budget:
            return "resident"
        if est["streamed"] <= budget:
            return "streamed"
        host = self.host_memory_budget
        if host is not None and est["streamed_host"] <= budget and est["host"] <= host:
            return "streamed_host"
        msg = (f"the proof does not fit on the device: it needs about {_gib(est['resident'])} resident or "
               f"{_gib(est['streamed'])} streamed, and {_gib(budget)} is available")
        if host is not None:
            msg += (f"; with the Merkle node heaps in pinned host memory it needs about {_gib(est['streamed_host'])} on the "
                    f"device and {_gib(est['host'])} of host memory, and {_gib(host)} of host memory is allowed")
        raise ProvingError(msg)

    # ---- default_prove
    def prove(self, stark, options, witness, validate=False):
        """default_prove.  validate=True: stark.validate_constraints checks the trace against the AIR once the extension
        trace is committed, and raises before anything after that commitment is computed; its time is recorded as
        timings["validate_constraints"].  The proof bytes do not depend on it.  (ShardedProver, whose ranks may not hold
        the whole base trace, refuses it with a ProvingError.)"""
        with torch.cuda.stream(self.stream):
            if validate:
                return self._prove(stark, options, witness, validate=True)
            return self._prove(stark, options, witness)

    def _prove(self, stark, options, witness, validate=False):
        r = self._start(stark, options, witness, validate)
        est = peak_bytes(r.n, r.beta, r.nbase, r.next_, r.fq, r.air.ce_blowup_factor, options.fri_folding_factor)
        if self.pinned_bytes > (self.host_memory_budget or 0):
            self.release_host_memory()          # heaps pinned under a larger budget are not held past a lower one
        residency = self.choose_residency(est)
        self.last_residency = residency
        r.lap("init_air")
        if residency == "resident":
            return self._default_prove(r, _Resident(self, r))
        host_heaps = None
        if residency == "streamed_host":
            # tree t's node heap: beta local heaps of n digests (base, extension if any, composition)
            host_heaps = self._host_heaps(est["host"])[:est["host"]].reshape(-1, r.beta, r.n, 32)
            r.lap("pin_host_memory")
        return self._default_prove(r, _Streamed(self, r, host_heaps))

    def _start(self, stark, options, witness, validate):
        """the set-up every residency shares: the trace, the cached Air with its compiled programs, this proof's public
        inputs, the shapes, the channel and the phase clock (r.lap).  Returns the _Run with the phase "init_air" open; the
        trace's columns are not read yet."""
        ctx = self.ctx
        cfg = stark.AirConfig
        timings = {}
        t_all = t0 = time.perf_counter()

        # NVTX range per prover phase (visible to nsys / ncu --nvtx): the range of phase k is closed and the range of
        # phase k + 1 opened where the reference prints its per-phase timings (src/prover.rs:40-170)
        phases = ["init_air", "base_trace_commitment", "extension_trace_commitment", "constraint_eval",
                  "composition_trace_commitment", "deep_composition", "fri", "proof_of_work", "queries"]
        torch.cuda.nvtx.range_push("prove:" + phases[0])

        def lap(name, since=None):
            nonlocal t0
            ctx.sync()
            t = time.perf_counter()
            if since is not None:           # permutation_fill, lookup_multiplicities: timed on their own, outside the phase
                timings[name] = t - since
                t0 += t - since
                return
            timings[name] = t - t0
            t0 = t
            if name not in phases:          # validate_constraints: timed, outside the fixed phases
                return
            torch.cuda.nvtx.range_pop()
            k = phases.index(name) + 1
            if k < len(phases):
                torch.cuda.nvtx.range_push("prove:" + phases[k])

        trace = stark.generate_trace(witness)
        n = len(trace)
        # the AIR bookkeeping and its two compiled evaluator programs depend on (AirConfig, trace length, options) only:
        # built once per prover, then shared by every proof (public inputs and verifier randomness are bound per proof)
        key = (cfg, n, options)
        if key not in self._airs:
            self._airs[key] = Air(cfg, n, None, options)
            self._airs[key].composition_program()
            self._airs[key].deep_program()
            self._airs[key].extension_program()
            self._airs[key].lookup_programs()
            self._airs[key].permutation_programs()
            self._airs[key].num_challenges(), self._airs[key].num_composition_constraint_coeffs(), self._airs[key].trace_arguments()
        air = copy.copy(self._airs[key])
        air.public_inputs = stark.get_public_inputs()
        check_lookup_trace(air, trace)
        fq = FP if cfg.FQ_IS_FP else FQ3
        log_n = air.log_n
        beta = options.lde_blowup_factor
        log_b = beta.bit_length() - 1
        nbase, next_ = cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS
        channel = ProverChannel(air, stark.gen_public_coin(air), ctx)
        ce_blowup = air.ce_blowup_factor
        return _Run(ctx=ctx, stark=stark, options=options, trace=trace, air=air, channel=channel, fq=fq, n=n, log_n=log_n,
                    beta=beta, log_b=log_b, log_N=log_n + log_b, N=n * beta, nbase=nbase, next_=next_,
                    ce_blowup=ce_blowup, log_ce=log_n + ce_blowup.bit_length() - 1, lap=lap, timings=timings,
                    t_all=t_all, cached_air=self._airs[key], validate=validate)

    def _base_columns(self, r):
        """the trace's base columns, refused unless they are (NUM_BASE_COLUMNS, n)"""
        base = r.trace.base_columns()
        if tuple(base.shape) != (r.nbase, r.n):
            raise ProvingError(f"expected {r.nbase} base columns of {r.n} rows")
        return base

    def _default_prove(self, r, rows):
        """default_prove (src/prover.rs:40-174) after the set-up: every commitment, Fiat–Shamir draw and phase in the
        reference's order, for every residency.  `rows` (_Resident, _Streamed, prover_mgpu._Sharded) does the steps that
        depend on where the LDE rows live: the commitments, the evaluations over the LDE, FRI and the queried rows."""
        air, channel, lap, fq = r.air, r.channel, r.lap, r.fq

        # ---- base trace commitment (prover.rs:46-55)
        base, base_m = rows.commit_base()
        channel.commit_base_trace(base_m.root)
        lap("base_trace_commitment")
        challenges = [channel.public_coin.draw() for _ in range(air.num_challenges())]
        hints = air.gen_hints(challenges)

        # ---- extension trace commitment (prover.rs:56-72)
        ext = self._extension_columns(r, challenges, hints, base)
        # with validation: the natural-order base columns and the extension columns on the device (a host-built extension
        # matrix uploaded once, for the check and the commitment), kept until the check has run
        check = (base, None if ext is None else self._to_device(ext)) if r.validate else None
        del base
        ext_m = None
        if ext is not None:
            # large buffers are handed to the layout in a list it may empty: the streamed layout frees them as soon as it
            # has their coefficients, the others when this list goes
            ext = [check[1] if check else ext]          # with validation: the one device copy serves both
            ext_m = rows.commit_evals(ext, fq, r.next_)
            channel.commit_extension_trace(ext_m.root)
        del ext
        lap("extension_trace_commitment")
        if check is not None:                   # Stark::validate_constraints at the reference's position (src/prover.rs:74-75)
            air._check_program = r.cached_air.check_program()        # compiled once per AIR and trace length
            r.stark.validate_constraints(air, challenges, hints, check[0], check[1], r.ctx)
            lap("validate_constraints")
        del check

        # ---- constraint evaluation over the ce domain (prover.rs:75-108)
        composition_coeffs = [channel.public_coin.draw() for _ in range(air.num_composition_constraint_coeffs())]
        comp_evals = [rows.constraint_evals(base_m, ext_m, dict(challenges=challenges, hints=hints, ccoefs=composition_coeffs))]
        lap("constraint_eval")

        # ---- composition trace (prover.rs:110-125)
        comp_m = rows.commit_coeffs(rows.composition_polys(comp_evals), fq, r.ce_blowup)
        channel.commit_composition_trace(comp_m.root)
        lap("composition_trace_commitment")

        # ---- DEEP composition polynomial, evaluated straight over the LDE domain (composer.rs:89-188 in evaluation form)
        mats = (base_m, ext_m, comp_m)
        dprog = self._bind_deep(r, base_m.polys, ext_m.polys if ext_m else None, comp_m.polys)
        codeword = rows.deep_codeword(dprog, mats)
        lap("deep_composition")

        layers = rows.fri(codeword)             # FRI layers, the remainder and the proof of work (fri.rs:179-249)

        # ---- queries (fri.rs:151-177, trace.rs:115-157)
        positions = channel.get_fri_query_positions()
        fri_proof, opened = rows.open(layers, positions, mats)
        (base_rows, base_view), (ext_rows, ext_view), (comp_rows, comp_view) = opened
        queries = Queries(_canon_rows(base_rows, 1), _canon_rows(ext_rows, fq) if ext_m else [], _canon_rows(comp_rows, fq),
                          base_view, ext_view, comp_view)
        return self._finish(r, fri_proof, queries)

    # ---- phases the sequence and the layouts share (ShardedProver included)
    def _lookup_base(self, r, host_base):
        """the prover's own device copy of the base columns (the caller's trace, host or device, is never written) with the
        columns the AIR leaves to the package filled: every permutation's targets first, in declaration order, then every
        lookup's multiplicity column (a lookup may read a target).  Timed as timings["permutation_fill"] and
        timings["lookup_multiplicities"]"""
        base = self._own_copy(host_base)
        r.ctx.sync()
        if r.air.permutations:
            t = time.perf_counter()
            fill_permutation_targets(r.ctx, r.air, base)
            r.lap("permutation_fill", since=t)
        if r.air.lookups:
            t = time.perf_counter()
            fill_lookup_multiplicities(r.ctx, r.air, base)
            r.lap("lookup_multiplicities", since=t)
        return base

    def _device_base(self, r, host_base):
        """the base columns on the device: the prover's own filled copy when the AIR has lookups or permutations"""
        return self._lookup_base(r, host_base) if r.air.lookups or r.air.permutations else self._to_device(host_base)

    def _extension_columns(self, r, challenges, hints, base):
        """the trace's own builder first (device or host); without one, the columns the AIR declares, built on the device"""
        if hasattr(r.trace, "build_extension_columns_device"):
            # running products / evaluations as device scans over the resident base trace (SURVEY.md §8f rank 3)
            ext = r.trace.build_extension_columns_device(challenges, r.ctx, base)
        else:
            ext = r.trace.build_extension_columns(challenges)
            if ext is None and r.air.extension_declaration:
                ext = declared_extension_columns(r.ctx, r.air, challenges, hints, base, self.device)
        release = getattr(r.trace, "release_base_columns", None)
        if release is not None:     # the natural-order base matrix is not read from the trace again in this proof
            release()
        num_ext = 0 if ext is None else int(ext.shape[0])
        if num_ext != r.next_:
            raise ProvingError(f"expected {r.next_} extension columns, got {num_ext}")
        return ext

    def _composition_columns(self, r, comp_evals):
        """the natural-order ce-domain column `comp_evals` (transformed in place) as its coefficients over the ce coset in
        ce_blowup columns, column i = coefficients = i mod ce_blowup"""
        r.ctx.ntt_batch(comp_evals, r.fq, r.log_ce, 1, inverse=True, offset=GEN_MONT)
        if r.ce_blowup == 1:
            return comp_evals.view(1, r.n * r.fq)
        comp_polys = self._empty(r.ce_blowup, r.n * r.fq)
        r.ctx.matrix_from_rows(comp_evals, comp_polys, r.fq, r.n, r.ce_blowup)
        return comp_polys

    def _bind_deep(self, r, base_polys, ext_polys, comp_polys):
        """out-of-domain evaluations (composer.rs:43-86) from the coefficients, sent to the channel; then the DEEP
        coefficients are drawn and bound into the DEEP program"""
        ctx, air, channel, stark, fq, n = r.ctx, r.air, r.channel, r.stark, r.fq, r.n
        nbase, next_, ce_blowup = r.nbase, r.next_, air.ce_blowup_factor
        z = channel.get_ood_point()
        zq = _lift(z)
        trace_arguments = air.trace_arguments()
        offsets = sorted(set(o for _, o in trace_arguments))
        z_points, z_m = deep.ood_points(zq, r.log_n, offsets, ce_blowup)
        pts = np.array([[_mont(c) for c in z_points[o]] for o in offsets], dtype=np.uint64).reshape(-1, 3)
        base_ood = ctx.poly_eval(base_polys, FP, n, nbase, pts)
        ext_ood = ctx.poly_eval(ext_polys, fq, n, next_, pts) if next_ else None
        comp_ood = ctx.poly_eval(comp_polys, fq, n, ce_blowup, np.array([[_mont(c) for c in z_m]], dtype=np.uint64))

        def unlift(w3):
            t = tuple(int(w) * _RINV % P for w in w3)
            if fq == FP:
                if t[1] or t[2]:
                    raise ProvingError("out-of-domain value left the base field although Fq = Fp")
                return t[0]
            return t

        execution_trace_oods = []
        for col, off in trace_arguments:
            k = offsets.index(off)
            if col < nbase:
                execution_trace_oods.append(unlift(base_ood[col, k]))
            elif col < nbase + next_:
                execution_trace_oods.append(unlift(ext_ood[col - nbase, k]))
            else:
                raise ProvingError(f"column is {col} but there are only {nbase + next_} columns")
        composition_trace_oods = [unlift(comp_ood[j, 0]) for j in range(ce_blowup)]
        channel.send_ood_evals(execution_trace_oods, composition_trace_oods)

        ex_alphas, co_alphas, (d_alpha, d_beta) = stark.gen_deep_coeffs(channel.public_coin, air)
        dprog_sym, dkeys = air.deep_program()
        return dprog_sym.bind(hints=deep.deep_hint_values(
            dkeys, z_points, z_m, [_lift(v) for v in execution_trace_oods], [_lift(v) for v in composition_trace_oods],
            [_lift(v) for v in ex_alphas], [_lift(v) for v in co_alphas], _lift(d_alpha), _lift(d_beta),
            trace_arguments=trace_arguments))

    def _fri_layer(self, r, cur, ln):
        """one FRI layer of the whole codeword `cur` (2^ln entries): commit its rows of ff entries, draw alpha, fold.
        Returns the layer (evals, tree, root, rows) and the folded codeword."""
        ctx, channel, fq = r.ctx, r.channel, r.fq
        ff = r.options.fri_folding_factor
        log_ff = ff.bit_length() - 1
        nrows = 1 << (ln - log_ff)
        leaves, nodes = self._empty(nrows, 4), self._empty(nrows, 4)
        root = ctx.merkle_commit_rows(cur, ff * fq, nrows, leaves=leaves, nodes=nodes)   # Matrix::from_arrays + from_matrix
        channel.commit_fri_layer(root)
        alpha = channel.draw_fri_alpha()
        nxt = self._empty(nrows * fq)
        ctx.fri_fold(cur, nxt, fq, ln, log_ff, np.array([_mont(c) for c in _lift(alpha)], dtype=np.uint64))   # apply_drp, offset ONE
        return (cur, _Tree(leaves, nodes, nrows), root, nrows), nxt

    def _fri_tail(self, r, cur, ln):
        """set_remainder (fri.rs:233-249) from the last folded codeword `cur` (2^ln entries), then the proof of work"""
        ctx, channel, options, fq, beta = r.ctx, r.channel, r.options, r.fq, r.beta
        rem_size = 1 << ln
        if rem_size > options.fri_max_remainder_coeffs * beta:
            raise ProvingError("remainder domain too large")
        rem = cur.clone()
        ctx.bit_reverse(rem, fq, ln)
        ctx.ntt_batch(rem, fq, ln, 1, inverse=True, offset=ONE)
        ctx.sync()
        rem_coeffs = _canon_rows(rem.cpu().numpy().view(np.uint64), fq)
        keep = rem_size // beta
        zero = 0 if fq == FP else (0, 0, 0)
        if any(c != zero for c in rem_coeffs[keep:]):
            raise ProvingError("FRI remainder is not low degree: the trace does not satisfy the AIR (fri.rs:246)")
        channel.commit_remainder(rem_coeffs[:keep])
        r.lap("fri")

        channel.grind_fri_commitments()
        r.lap("proof_of_work")

    def _fri_queries(self, r, layers, positions):
        """FRI layer rows and paths at the folded query positions (fri.rs:151-177)"""
        ff, fq = r.options.fri_folding_factor, r.fq
        fri_layers, folded = [], positions
        for evals, tree, root, nrows in layers:
            folded = sorted(set(p // ff for p in folded))                                    # fold_positions
            rows = r.ctx.gather_rows_rowmajor(evals, ff * fq, nrows, folded)
            fri_layers.append(LayerProof(_canon_rows(rows, fq), self._view(tree, folded), root))
        return FriProof(fri_layers, r.channel.fri_remainder_coeffs)

    def _finish(self, r, fri_proof, queries):
        r.lap("queries")
        r.timings["total"] = time.perf_counter() - r.t_all
        c = r.channel
        return Proof(r.options, r.n, c.base_trace_commitment, c.extension_trace_commitment, c.composition_trace_commitment,
                     fri_proof, c.pow_nonce, queries, c.execution_trace_ood_evals, c.composition_trace_ood_evals, r.timings)


class _Resident(_Layout):
    """every LDE matrix and both arrays of every Merkle tree in HBM until the queries"""

    def commit_base(self):
        """A host trace is uploaded in column chunks on a second stream while the previous chunk is interpolated and
        extended (columns are independent until the row hash); a pinned trace — the analogue of the reference's
        GpuAllocator-backed columns — makes the copies asynchronous."""
        p, r, ctx = self.p, self.r, self.p.ctx
        n, N, nbase = r.n, r.N, r.nbase
        host_base = p._base_columns(r)
        if r.air.lookups or r.air.permutations or (isinstance(host_base, torch.Tensor) and host_base.is_cuda):
            # the filled columns are written before the commitment, so the upload cannot overlap the transforms here
            base = p._device_base(r, host_base)
            return base, self.commit_evals([base], FP, nbase)
        if not isinstance(host_base, torch.Tensor):
            host_base = torch.from_numpy(np.ascontiguousarray(host_base, dtype=np.uint64).view(np.int64))
        base, base_polys, base_lde = p._empty(nbase, n), p._empty(nbase, n), p._empty(nbase, N)
        chunk = max(1, min(nbase, (64 << 20) // (8 * n) or 1))            # ~64 MiB per copy
        p.copy_stream.wait_stream(p.stream)
        events = []
        with torch.cuda.stream(p.copy_stream):
            for c0 in range(0, nbase, chunk):
                c1 = min(c0 + chunk, nbase)
                base[c0:c1].copy_(host_base[c0:c1], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(p.copy_stream)
                events.append((c0, c1, ev))
        for c0, c1, ev in events:
            p.stream.wait_event(ev)
            ctx.ntt_batch_to(base[c0], base_polys[c0], FP, r.log_n, c1 - c0, inverse=True)
            ctx.lde_batch(base_polys[c0], base_lde[c0], FP, r.log_n, r.log_b, c1 - c0, offset=GEN_MONT, bitrev=True)
        leaves, nodes = p._empty(N, 4), p._empty(N, 4)
        root = ctx.merkle_commit(base_lde, FP, N, nbase, leaves=leaves, nodes=nodes)
        return base, _Matrix(base_polys, base_lde, FP, nbase, _Tree(leaves, nodes, N), root)

    def commit_evals(self, held, field, ncols):
        """Matrix::interpolate over the trace domain, then commit_coeffs"""
        evals = self.p._to_device(held[0])
        polys = self.p._empty(ncols, self.r.n * field)
        self.p.ctx.ntt_batch_to(evals, polys, field, self.r.log_n, ncols, inverse=True)
        return self.commit_coeffs(polys, field, ncols)

    def commit_coeffs(self, polys, field, ncols):
        """bit-reversed LDE + Merkle commit of a column-major coefficient matrix"""
        p, N = self.p, self.r.N
        lde = p._empty(ncols, N * field)
        p.ctx.lde_batch(polys, lde, field, self.r.log_n, self.r.log_b, ncols, offset=GEN_MONT, bitrev=True)
        leaves, nodes = p._empty(N, 4), p._empty(N, 4)
        root = p.ctx.merkle_commit(lde, field, N, ncols, leaves=leaves, nodes=nodes)
        return _Matrix(polys, lde, field, ncols, _Tree(leaves, nodes, N), root)

    def constraint_evals(self, base, ext, bind):
        """The first M entries of a bit-reversed LDE column ARE the ce-coset evaluations in bit-reversed order, so they
        are read in place (trace_bitrev); the output is in natural order"""
        r = self.r
        prog = r.air.composition_program().bind(**bind)
        comp_evals = self.p._empty(r.n * r.ce_blowup * r.fq)
        self.p.ctx.eval_constraints(prog, comp_evals, r.log_ce, base_cols=base.rows, nbase=r.nbase, base_stride=r.N,
                                    ext_cols=ext.rows if ext else None, next_=r.next_, ext_stride=r.N, fq_field=r.fq,
                                    offset=GEN_MONT, trace_bitrev=True)
        return comp_evals

    def composition_polys(self, held):
        return self.p._composition_columns(self.r, held[0])

    def deep_codeword(self, dprog, mats):
        r = self.r
        cols = [m.rows.data_ptr() + c * r.N * 8 * m.field for m in mats if m for c in range(m.ncols)]
        codeword = self.p._empty(r.N * r.fq)
        self.p.ctx.eval_constraints_ptrs(dprog, codeword, r.log_N, cols, [False] * r.nbase + [True] * (len(cols) - r.nbase),
                                         fq_field=r.fq, offset=GEN_MONT, trace_bitrev=True, out_bitrev=True)
        return codeword

    def open(self, layers, positions, mats):
        p, r = self.p, self.r
        fri_proof = p._fri_queries(r, layers, positions)
        rows = [p.ctx.gather_rows(m.rows, m.field, r.N, m.ncols, positions) if m else None for m in mats]
        views = [p._view(m.tree, positions) if m else None for m in mats]
        return fri_proof, list(zip(rows, views))


class _Blocks(_Layout):
    """a layout that evaluates coset block by coset block with the block-local program: self.blocks lists the (q, h_q)
    it evaluates, block j at entries [j n, (j+1) n) of its codeword, and self._cols(j, h_q, mats) gives block j's columns"""

    def constraint_evals(self, base, ext, bind):
        """the blocks q < ce_blowup of the LDE are the ce domain; the column comes out bit-reversed"""
        r = self.r
        n, fq = r.n, r.fq
        prog = block_program(r.cached_air).bind(**bind)
        comp_evals = self.p._empty(n * r.ce_blowup * fq)
        is_fq = [False] * r.nbase + [True] * r.next_
        for j, (q, h) in enumerate(self.blocks):
            if q < r.ce_blowup:
                self.p.ctx.eval_constraints_ptrs(prog, comp_evals[q * n * fq:(q + 1) * n * fq], r.log_n,
                                                 self._cols(j, h, (base, ext)), is_fq, fq_field=fq, offset=h,
                                                 trace_bitrev=True, out_bitrev=True)
        return comp_evals

    def deep_codeword(self, dprog, mats):
        r = self.r
        n, fq = r.n, r.fq
        codeword = self.p._empty(len(self.blocks) * n * fq)
        is_fq = [False] * r.nbase + [True] * (r.next_ + r.ce_blowup)
        for j, (q, h) in enumerate(self.blocks):
            self.p.ctx.eval_constraints_ptrs(dprog, codeword[j * n * fq:(j + 1) * n * fq], r.log_n, self._cols(j, h, mats),
                                             is_fq, fq_field=fq, offset=h, trace_bitrev=True, out_bitrev=True)
        return codeword


class _Streamed(_Blocks):
    """only the coefficients and the tree nodes stay; each coset block of the LDE is recomputed into one block buffer
    per matrix where it is needed, and query rows come from the coefficients.  host_heaps ((ntrees, beta, n, 32) bytes
    of pinned host memory, streamed_host): the node heaps of the trees, in commitment order"""

    def __init__(self, prover, r, host_heaps):
        super().__init__(prover, r)
        self.blocks = coset_offsets(r.log_n, r.log_b)
        self.host_heaps = host_heaps
        self.heaps = iter([None] * 3 if host_heaps is None else host_heaps)

    def commit_base(self):
        base = self.p._device_base(self.r, self.p._base_columns(self.r))
        return base, self.commit_evals([base], FP, self.r.nbase)

    def commit_evals(self, held, field, ncols):
        evals = held.pop()
        polys = self.p._empty(ncols, self.r.n * field)
        self.p.ctx.ntt_batch_to(self.p._to_device(evals), polys, field, self.r.log_n, ncols, inverse=True)
        del evals
        return self.commit_coeffs(polys, field, ncols)

    def commit_coeffs(self, polys, field, ncols):
        """Merkle commitment of the bit-reversed LDE, one coset block at a time: block q is transformed into the block
        buffer and hashed into its subtree of the node heap; the top log_b levels come from the block roots.  With a host
        heap ((beta, n, 32) bytes), block q's subtree is its local heap host_heap[q] and the tree is (top heap of 2 beta
        digests on the host, host_heap): the split layout of include/ministark_host_nodes.h."""
        ctx, r = self.p.ctx, self.r
        beta, host_heap = r.beta, next(self.heaps)
        m = _Matrix(polys, self.p._empty(ncols, r.n * field), field, ncols)
        if host_heap is None:
            nodes, roots = self.p._empty(beta << r.log_n, 4), self.p._empty(beta, 4)
        else:
            nodes = self.p._empty(2 * beta, 4)
            roots = nodes[beta:]
        for q, h in self.blocks:
            self._block(m, h)
            if host_heap is None:
                ctx.merkle_commit_block(m.rows, field, r.log_n, r.log_b, q, ncols, nodes, roots[q])
            else:
                ctx.merkle_commit_block_host(m.rows, field, r.log_n, ncols, host_heap[q], roots[q])
        if beta > 1:
            ctx.merkle_nodes(roots, nodes, beta)
        nodes[0].zero_()                        # the unused default digest (named by a walk over a 2-leaf tree)
        m.root = nodes[1].cpu().numpy().tobytes()
        m.tree = nodes if host_heap is None else (nodes.cpu().numpy().view(np.uint8), host_heap)
        return m

    def _block(self, m, h):
        """coset block with offset h of the bit-reversed LDE of every column of `m`, into its block buffer.  Its NTT plan
        is dropped at once: every block has its own offset, and beta cached plans with their full tables (up to GiBs each
        at 2^24 points) would take back the memory streaming saves"""
        self.p.ctx.lde_batch(m.polys, m.rows, m.field, self.r.log_n, 0, m.ncols, offset=h, bitrev=True)
        self.p.ctx.set_option("drop_plans", 1)

    def _cols(self, j, h, mats):
        """block j (offset h) of every column of `mats`, recomputed into their block buffers"""
        cols = []
        for m in mats:
            if m:
                self._block(m, h)
                cols += [m.rows[c] for c in range(m.ncols)]
        return cols

    def composition_polys(self, held):
        ctx, r = self.p.ctx, self.r
        comp_evals = held.pop()
        ctx.bit_reverse(comp_evals, r.fq, r.log_ce)
        if self.host_heaps is not None:
            # the size-M transform's temporary (as large as the column: 12 GiB at 2^25 rows) is the context's own
            # allocation and cannot reuse blocks torch's allocator keeps cached from the trace and extension columns
            torch.cuda.empty_cache()
        comp_polys = self.p._composition_columns(r, comp_evals)
        del comp_evals                          # (when ce_blowup == 1, comp_polys is a view of it and keeps it)
        ctx.set_option("drop_scratch", 1)       # the size-M transform's temporary: as large as the column itself
        return comp_polys

    def deep_codeword(self, dprog, mats):
        """every block of the three matrices recomputed once more; the block buffers are released afterwards"""
        codeword = super().deep_codeword(dprog, mats)
        for m in mats:
            if m:
                m.rows = None
        return codeword

    def open(self, layers, positions, mats):
        fri_proof = self.p._fri_queries(self.r, layers, positions)
        opened = {k: self._query(mats[k], positions) for k in (0, 2, 1) if mats[k]}      # base, composition, extension
        return fri_proof, [opened.get(k, (None, None)) for k in range(3)]

    def _query(self, m, positions):
        """the rows at `positions` and their MerkleView without the LDE: rows and leaf digests from the coefficients
        (ms_lde_rows), path nodes gathered from the node heap"""
        ctx, r = self.p.ctx, self.r
        init, sib, path = merkle_walk(r.N, positions)
        k = len(positions)
        rows = ctx.lde_rows(m.polys, m.field, r.log_n, r.log_b, m.ncols, list(positions) + init + sib)

        def leaf(row):                         # hash_rows: canonical words, 8 bytes little-endian each
            return hashlib.sha256(b"".join((int(w) * _RINV % P).to_bytes(8, "little") for w in row)).digest()

        digests = [leaf(row) for row in rows[k:]]
        if isinstance(m.tree, tuple):           # split heap: the top heap, then each block's local heap
            top, blocks = m.tree
            ctx.sync()                          # the last blocks' copies to host memory
            path_nodes = []
            for i in path:
                b, j = heap_location(i, r.log_b)
                path_nodes.append((top[j] if b is None else blocks[b, j]).tobytes())
        else:
            path_nodes = [d.tobytes() for d in ctx.gather_rows_rowmajor(m.tree, 4, r.N, path)] if path else []
        return rows[:k], MerkleView(path_nodes, digests[:len(init)], digests[len(init):], r.N.bit_length() - 1)
