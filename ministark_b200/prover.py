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
    """per-proof state shared by the phases of every driver (resident, streamed, sharded)"""

    def __init__(self, **kw):
        self.__dict__.update(kw)


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

    def _commit_columns(self, polys_in, field, log_n, log_b, ncols, is_evals):
        """interpolate (if is_evals) + bit-reversed LDE + Merkle commit of a column-major matrix.
        Returns (polys, lde, tree, root)."""
        ctx, n, N = self.ctx, 1 << log_n, 1 << (log_n + log_b)
        if is_evals:
            polys = self._empty(ncols, n * field)
            ctx.ntt_batch_to(polys_in, polys, field, log_n, ncols, inverse=True)      # Matrix::interpolate over the trace domain
        else:
            polys = polys_in
        lde = self._empty(ncols, N * field)
        ctx.lde_batch(polys, lde, field, log_n, log_b, ncols, offset=GEN_MONT, bitrev=True)
        leaves, nodes = self._empty(N, 4), self._empty(N, 4)
        root = ctx.merkle_commit(lde, field, N, ncols, leaves=leaves, nodes=nodes)
        return polys, lde, _Tree(leaves, nodes, N), root

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
            return self._prove_resident(r)
        if residency == "streamed_host":
            # tree t's node heap: beta local heaps of n digests (base, extension if any, composition)
            r.host_heaps = self._host_heaps(est["host"])[:est["host"]].reshape(-1, r.beta, r.n, 32)
            r.lap("pin_host_memory")
        return self._prove_streamed(r)

    def _start(self, stark, options, witness, validate):
        """the set-up every driver shares: the trace, the cached Air with its compiled programs, this proof's public
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
        return _Run(ctx=ctx, stark=stark, options=options, trace=trace, air=air, channel=channel, fq=fq, n=n, log_n=log_n,
                    beta=beta, log_b=log_b, log_N=log_n + log_b, N=n * beta, nbase=nbase, next_=next_, lap=lap,
                    timings=timings, t_all=t_all, cached_air=self._airs[key], validate=validate, host_heaps=None)

    def _base_columns(self, r):
        """the trace's base columns, refused unless they are (NUM_BASE_COLUMNS, n)"""
        base = r.trace.base_columns()
        if tuple(base.shape) != (r.nbase, r.n):
            raise ProvingError(f"expected {r.nbase} base columns of {r.n} rows")
        return base

    def _prove_resident(self, r):
        ctx, air, channel, lap = r.ctx, r.air, r.channel, r.lap
        fq, n, log_n, log_b, N, nbase, next_ = r.fq, r.n, r.log_n, r.log_b, r.N, r.nbase, r.next_

        # ---- base trace commitment (prover.rs:46-55).  A host trace is uploaded in column chunks on a second stream
        # while the previous chunk is interpolated and extended (columns are independent until the row hash); a
        # pinned trace — the analogue of the reference's GpuAllocator-backed columns — makes the copies asynchronous.
        host_base = self._base_columns(r)
        if air.lookups or air.permutations:
            # the filled columns are written before the commitment, so the upload cannot overlap the transforms here
            base = self._lookup_base(r, host_base)
            base_polys, base_lde, base_tree, base_root = self._commit_columns(base, FP, log_n, log_b, nbase, True)
        elif isinstance(host_base, torch.Tensor) and host_base.is_cuda:
            base = host_base.to(self.device)
            base_polys, base_lde, base_tree, base_root = self._commit_columns(base, FP, log_n, log_b, nbase, True)
        else:
            if not isinstance(host_base, torch.Tensor):
                host_base = torch.from_numpy(np.ascontiguousarray(host_base, dtype=np.uint64).view(np.int64))
            base, base_polys, base_lde = self._empty(nbase, n), self._empty(nbase, n), self._empty(nbase, N)
            chunk = max(1, min(nbase, (64 << 20) // (8 * n) or 1))            # ~64 MiB per copy
            self.copy_stream.wait_stream(self.stream)
            events = []
            with torch.cuda.stream(self.copy_stream):
                for c0 in range(0, nbase, chunk):
                    c1 = min(c0 + chunk, nbase)
                    base[c0:c1].copy_(host_base[c0:c1], non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(self.copy_stream)
                    events.append((c0, c1, ev))
            for c0, c1, ev in events:
                self.stream.wait_event(ev)
                ctx.ntt_batch_to(base[c0], base_polys[c0], FP, log_n, c1 - c0, inverse=True)
                ctx.lde_batch(base_polys[c0], base_lde[c0], FP, log_n, log_b, c1 - c0, offset=GEN_MONT, bitrev=True)
            leaves, nodes = self._empty(N, 4), self._empty(N, 4)
            base_root = ctx.merkle_commit(base_lde, FP, N, nbase, leaves=leaves, nodes=nodes)
            base_tree = _Tree(leaves, nodes, N)
        del host_base                           # held no longer than `base`: see release_base_columns below
        channel.commit_base_trace(base_root)
        lap("base_trace_commitment")
        challenges = [channel.public_coin.draw() for _ in range(air.num_challenges())]
        hints = air.gen_hints(challenges)

        # ---- extension trace commitment (prover.rs:56-72)
        ext = self._extension_columns(r, challenges, hints, base)
        check = self._keep_for_check(r, base, ext)
        del base
        ext_polys = ext_lde = ext_tree = None
        if ext is not None:
            ext = check[1] if check else ext           # with validation: the one device copy serves both
            ext_polys, ext_lde, ext_tree, ext_root = self._commit_columns(self._to_device(ext), fq, log_n, log_b, next_, True)
            channel.commit_extension_trace(ext_root)
        del ext
        lap("extension_trace_commitment")
        self._check(r, challenges, hints, check)
        del check

        # ---- constraint evaluation over the ce domain (prover.rs:75-108).  The first M entries of a bit-reversed LDE
        # column ARE the ce-coset evaluations in bit-reversed order, so they are read in place (trace_bitrev).
        ce_blowup = air.ce_blowup_factor
        log_ce = log_n + ce_blowup.bit_length() - 1
        M = n * ce_blowup
        composition_coeffs = [channel.public_coin.draw() for _ in range(air.num_composition_constraint_coeffs())]
        prog = air.composition_program().bind(challenges=challenges, hints=hints, ccoefs=composition_coeffs)
        comp_evals = self._empty(M * fq)
        ctx.eval_constraints(prog, comp_evals, log_ce, base_cols=base_lde, nbase=nbase, base_stride=N,
                             ext_cols=ext_lde, next_=next_, ext_stride=N, fq_field=fq, offset=GEN_MONT, trace_bitrev=True)
        lap("constraint_eval")

        # ---- composition trace (prover.rs:110-125): coefficients over the ce coset, column i = coefficients = i mod ce_blowup
        ctx.ntt_batch(comp_evals, fq, log_ce, 1, inverse=True, offset=GEN_MONT)
        comp_polys = self._composition_columns(r, comp_evals)
        _, comp_lde, comp_tree, comp_root = self._commit_columns(comp_polys, fq, log_n, log_b, ce_blowup, False)
        channel.commit_composition_trace(comp_root)
        lap("composition_trace_commitment")

        # ---- DEEP composition polynomial, evaluated straight over the LDE domain (composer.rs:89-188 in evaluation form)
        dprog = self._bind_deep(r, base_polys, ext_polys, comp_polys)
        ncols_all = nbase + next_ + ce_blowup
        sz = N * 8
        cols = [base_lde.data_ptr() + c * sz for c in range(nbase)]
        cols += [ext_lde.data_ptr() + c * sz * fq for c in range(next_)]
        cols += [comp_lde.data_ptr() + c * sz * fq for c in range(ce_blowup)]
        deep_lde = self._empty(N * fq)
        ctx.eval_constraints_ptrs(dprog, deep_lde, r.log_N, cols, [False] * nbase + [True] * (ncols_all - nbase), fq_field=fq,
                                  offset=GEN_MONT, trace_bitrev=True, out_bitrev=True)
        lap("deep_composition")

        layers = self._fri(r, deep_lde)

        # ---- queries (fri.rs:151-177, trace.rs:115-157)
        positions = channel.get_fri_query_positions()
        fri_proof = self._fri_queries(r, layers, positions)
        queries = Queries(
            _canon_rows(ctx.gather_rows(base_lde, FP, N, nbase, positions), 1),
            _canon_rows(ctx.gather_rows(ext_lde, fq, N, next_, positions), fq) if next_ else [],
            _canon_rows(ctx.gather_rows(comp_lde, fq, N, ce_blowup, positions), fq),
            self._view(base_tree, positions),
            self._view(ext_tree, positions) if next_ else None,
            self._view(comp_tree, positions))
        return self._finish(r, fri_proof, queries)

    # ---- streamed residency: coefficients and tree nodes stay, coset blocks are recomputed
    def _commit_blocks(self, polys, blk, field, ncols, log_n, log_b, offsets, host_heap=None):
        """Merkle commitment of the bit-reversed LDE of `polys`, one coset block at a time: block q is transformed into
        `blk` and hashed into its subtree of the node heap; the top log_b levels come from the block roots.
        Returns (nodes, root).  With host_heap ((beta, n, 32) bytes of pinned host memory), block q's subtree is its local
        heap host_heap[q] and nodes is (top heap of 2 beta digests on the host, host_heap): the split layout of
        include/ministark_host_nodes.h."""
        ctx, beta = self.ctx, 1 << log_b
        if host_heap is None:
            nodes, roots = self._empty(beta << log_n, 4), self._empty(beta, 4)
        else:
            nodes = self._empty(2 * beta, 4)
            roots = nodes[beta:]
        for q, h in offsets:
            self._block(polys, blk, field, ncols, log_n, h)
            if host_heap is None:
                ctx.merkle_commit_block(blk, field, log_n, log_b, q, ncols, nodes, roots[q])
            else:
                ctx.merkle_commit_block_host(blk, field, log_n, ncols, host_heap[q], roots[q])
        if beta > 1:
            ctx.merkle_nodes(roots, nodes, beta)
        nodes[0].zero_()                        # the unused default digest (named by a walk over a 2-leaf tree)
        root = nodes[1].cpu().numpy().tobytes()
        if host_heap is not None:
            nodes = (nodes.cpu().numpy().view(np.uint8), host_heap)
        return nodes, root

    def _block(self, polys, blk, field, ncols, log_n, h):
        """coset block with offset h of the bit-reversed LDE of every column of `polys`, into `blk`.  Its NTT plan is
        dropped at once: every block has its own offset, and beta cached plans with their full tables (up to GiBs each
        at 2^24 points) would take back the memory streaming saves"""
        self.ctx.lde_batch(polys, blk, field, log_n, 0, ncols, offset=h, bitrev=True)
        self.ctx.set_option("drop_plans", 1)

    def _streamed_queries(self, polys, field, ncols, nodes, log_n, log_b, positions):
        """the rows at `positions` and their MerkleView without the LDE: rows and leaf digests from the coefficients
        (ms_lde_rows), path nodes gathered from the resident node heap"""
        N = 1 << (log_n + log_b)
        init, sib, path = merkle_walk(N, positions)
        k = len(positions)
        rows = self.ctx.lde_rows(polys, field, log_n, log_b, ncols, list(positions) + init + sib)

        def leaf(row):                         # hash_rows: canonical words, 8 bytes little-endian each
            return hashlib.sha256(b"".join((int(w) * _RINV % P).to_bytes(8, "little") for w in row)).digest()

        digests = [leaf(row) for row in rows[k:]]
        if isinstance(nodes, tuple):            # split heap: the top heap, then each block's local heap
            top, blocks = nodes
            self.ctx.sync()                     # the last blocks' copies to host memory
            path_nodes = []
            for i in path:
                b, j = heap_location(i, log_b)
                path_nodes.append((top[j] if b is None else blocks[b, j]).tobytes())
        else:
            path_nodes = [d.tobytes() for d in self.ctx.gather_rows_rowmajor(nodes, 4, N, path)] if path else []
        return rows[:k], MerkleView(path_nodes, digests[:len(init)], digests[len(init):], N.bit_length() - 1)

    def _prove_streamed(self, r):
        ctx, air, channel, lap = r.ctx, r.air, r.channel, r.lap
        fq, n, log_n, log_b, N, nbase, next_ = r.fq, r.n, r.log_n, r.log_b, r.N, r.nbase, r.next_
        offsets = coset_offsets(log_n, log_b)

        # ---- base trace commitment: coefficients stay, the LDE passes through one block buffer
        host_base = self._base_columns(r)
        base = self._lookup_base(r, host_base) if air.lookups or air.permutations else self._to_device(host_base)
        del host_base                           # held no longer than `base`: see release_base_columns below
        base_polys, base_blk = self._empty(nbase, n), self._empty(nbase, n)
        ctx.ntt_batch_to(base, base_polys, FP, log_n, nbase, inverse=True)
        heaps = r.host_heaps if r.host_heaps is not None else [None] * 3
        base_nodes, base_root = self._commit_blocks(base_polys, base_blk, FP, nbase, log_n, log_b, offsets, heaps[0])
        channel.commit_base_trace(base_root)
        lap("base_trace_commitment")
        challenges = [channel.public_coin.draw() for _ in range(air.num_challenges())]
        hints = air.gen_hints(challenges)

        # ---- extension trace commitment
        ext = self._extension_columns(r, challenges, hints, base)
        check = self._keep_for_check(r, base, ext)
        del base
        ext_polys = ext_blk = ext_nodes = None
        if ext is not None:
            ext = check[1] if check else ext
            ext_polys = self._empty(next_, n * fq)
            ctx.ntt_batch_to(self._to_device(ext), ext_polys, fq, log_n, next_, inverse=True)
            del ext
            ext_blk = self._empty(next_, n * fq)
            ext_nodes, ext_root = self._commit_blocks(ext_polys, ext_blk, fq, next_, log_n, log_b, offsets, heaps[1])
            channel.commit_extension_trace(ext_root)
        lap("extension_trace_commitment")
        self._check(r, challenges, hints, check)
        del check

        def trace_block(h):
            self._block(base_polys, base_blk, FP, nbase, log_n, h)
            cols = [base_blk[c] for c in range(nbase)]
            if next_:
                self._block(ext_polys, ext_blk, fq, next_, log_n, h)
                cols += [ext_blk[c] for c in range(next_)]
            return cols

        # ---- constraint evaluation, block by block: the blocks q < ce_blowup of the LDE are the ce domain
        ce_blowup = air.ce_blowup_factor
        log_ce = log_n + ce_blowup.bit_length() - 1
        M = n * ce_blowup
        composition_coeffs = [channel.public_coin.draw() for _ in range(air.num_composition_constraint_coeffs())]
        prog = block_program(r.cached_air).bind(challenges=challenges, hints=hints, ccoefs=composition_coeffs)
        comp_evals = self._empty(M * fq)
        is_fq = [False] * nbase + [True] * next_
        for q, h in offsets[:ce_blowup]:
            ctx.eval_constraints_ptrs(prog, comp_evals[q * n * fq:(q + 1) * n * fq], log_n, trace_block(h), is_fq, fq_field=fq,
                                      offset=h, trace_bitrev=True, out_bitrev=True)
        lap("constraint_eval")

        # ---- composition trace: the bit-reversed ce-domain column -> coefficients -> ce_blowup columns
        ctx.bit_reverse(comp_evals, fq, log_ce)
        if r.host_heaps is not None:
            # the size-M transform's temporary (as large as the column: 12 GiB at 2^25 rows) is the context's own
            # allocation and cannot reuse blocks torch's allocator keeps cached from the trace and extension columns
            torch.cuda.empty_cache()
        ctx.ntt_batch(comp_evals, fq, log_ce, 1, inverse=True, offset=GEN_MONT)
        comp_polys = self._composition_columns(r, comp_evals)
        del comp_evals                          # (when ce_blowup == 1, comp_polys is a view of it and keeps it)
        ctx.set_option("drop_scratch", 1)       # the size-M transform's temporary: as large as the column itself
        comp_blk = self._empty(ce_blowup, n * fq)
        comp_nodes, comp_root = self._commit_blocks(comp_polys, comp_blk, fq, ce_blowup, log_n, log_b, offsets, heaps[-1])
        channel.commit_composition_trace(comp_root)
        lap("composition_trace_commitment")

        # ---- DEEP composition polynomial: every block of the three matrices recomputed once more
        dprog = self._bind_deep(r, base_polys, ext_polys, comp_polys)
        deep_lde = self._empty(N * fq)
        is_fq = [False] * nbase + [True] * (next_ + ce_blowup)
        for q, h in offsets:
            cols = trace_block(h)
            self._block(comp_polys, comp_blk, fq, ce_blowup, log_n, h)
            cols += [comp_blk[c] for c in range(ce_blowup)]
            ctx.eval_constraints_ptrs(dprog, deep_lde[q * n * fq:(q + 1) * n * fq], log_n, cols, is_fq, fq_field=fq, offset=h,
                                      trace_bitrev=True, out_bitrev=True)
        del base_blk, ext_blk, comp_blk
        lap("deep_composition")

        layers = self._fri(r, deep_lde)

        # ---- queries: rows and leaf digests from the coefficients, path nodes from the node heaps
        positions = channel.get_fri_query_positions()
        fri_proof = self._fri_queries(r, layers, positions)
        base_rows, base_view = self._streamed_queries(base_polys, FP, nbase, base_nodes, log_n, log_b, positions)
        comp_rows, comp_view = self._streamed_queries(comp_polys, fq, ce_blowup, comp_nodes, log_n, log_b, positions)
        ext_rows, ext_view = (self._streamed_queries(ext_polys, fq, next_, ext_nodes, log_n, log_b, positions) if next_
                              else (None, None))
        queries = Queries(_canon_rows(base_rows, 1), _canon_rows(ext_rows, fq) if next_ else [], _canon_rows(comp_rows, fq),
                          base_view, ext_view, comp_view)
        return self._finish(r, fri_proof, queries)

    # ---- phases every driver shares (ShardedProver included)
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

    def _keep_for_check(self, r, base, ext):
        """with validation: the natural-order base columns and the extension columns on the device (a host-built
        extension matrix uploaded once, for the check and the commitment), kept until the check has run"""
        if not r.validate:
            return None
        return base, None if ext is None else self._to_device(ext)

    def _check(self, r, challenges, hints, check):
        """Stark::validate_constraints at the reference's position (src/prover.rs:74-75)"""
        if check is not None:
            r.air._check_program = r.cached_air.check_program()      # compiled once per AIR and trace length
            r.stark.validate_constraints(r.air, challenges, hints, check[0], check[1], r.ctx)
            r.lap("validate_constraints")

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

    def _composition_columns(self, r, comp_coeffs):
        """the composition coefficients over the ce coset as ce_blowup columns, column i = coefficients = i mod ce_blowup"""
        ce_blowup = r.air.ce_blowup_factor
        if ce_blowup == 1:
            return comp_coeffs.view(1, r.n * r.fq)
        comp_polys = self._empty(ce_blowup, r.n * r.fq)
        r.ctx.matrix_from_rows(comp_coeffs, comp_polys, r.fq, r.n, ce_blowup)
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

    def _fri(self, r, deep_lde):
        """FRI layers (fri.rs:179-249), the remainder and the proof of work; returns the committed layers"""
        log_ff = r.options.fri_folding_factor.bit_length() - 1
        layers = []
        cur, ln = deep_lde, r.log_N
        for _ in range(r.options.fri_num_layers(r.N)):
            layer, cur = self._fri_layer(r, cur, ln)
            layers.append(layer)
            ln -= log_ff
        self._fri_tail(r, cur, ln)
        return layers

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
