"""ministark_b200 — H100 (sm_90a) implementation of miniSTARK's gpu-poly hot path.

Python host-side mirror of the reference's Rust interface for this path (the Rust toolchain
is not available in the build image; the C ABI in include/ministark_b200.h is the drop-in
boundary, see INTEGRATION.md):

    reference (Rust)                                   here
    -------------------------------------------------  -----------------------------------
    get_planner() / Planner   gpu/src/plan.rs:327-350  Context
    GpuFft / GpuIfft          gpu/src/plan.rs:236-325  GpuFft / GpuIfft (.encode / .execute)
    Radix2EvaluationDomain    ark-poly                 Domain(log_n, offset)
    Matrix<F>                 src/matrix.rs            Matrix (interpolate, evaluate,
                                                       bit_reversed_evaluate, sum_columns, ...)
    MatrixMerkleTreeImpl      src/merkle.rs:316-386    MatrixMerkleTree.from_matrix
    *Stage (14 types)         gpu/src/stage.rs         Context.pointwise / pointwise_const
    apply_drp                 src/fri.rs:526-567       Context.fri_fold

Arrays are numpy uint64 (host, staged through the device inside each call) or anything with a
CUDA `data_ptr()` (torch tensors; resident, no copies).  Words are Montgomery residues exactly
as the reference stores them.  Errors raise MsError (the reference panics).
There is no CPU fallback anywhere in this package.
"""
import ctypes as C

import numpy as np

from . import _lib

FP = 1
FQ3 = 3
FORWARD = 0
INVERSE = 1
ONE = 4294967295            # Montgomery form of 1
P = 2**64 - 2**32 + 1
_R = 2**64
GENERATOR = 7 * _R % P      # Fp::GENERATOR (coset offset, src/air.rs:42-44), Montgomery form
OPS = dict(mul=0, add=1, convert=2, inv=3, exp=4, neg=5, mulpow=6, fill=7, sub=8)


class MsError(RuntimeError):
    pass


def to_mont(x):
    return int(x) % P * _R % P


def from_mont(w):
    return int(w) * pow(_R, -1, P) % P


def root_of_unity(log_n):
    """ark-ff get_root_of_unity(2^log_n), Montgomery form."""
    return to_mont(pow(pow(7, (P - 1) >> 32, P), 1 << (32 - log_n), P))


def _ptr(x):
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        if not x.flags["C_CONTIGUOUS"]:
            raise MsError("numpy arrays must be C-contiguous")
        return x.ctypes.data
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    if isinstance(x, int):
        return x
    raise MsError(f"unsupported buffer type {type(x)}")


class Context:
    """Device context: one device, one in-order stream (Planner, gpu/src/plan.rs:327-350)."""

    def __init__(self, device=0, stream=None):
        self.lib = _lib.load()
        h = C.c_void_p()
        rc = self.lib.ms_ctx_create(device, C.byref(h))
        if rc != 0:
            raise MsError(f"ms_ctx_create(device={device}) failed with {rc} "
                          "(no CUDA device? this package has no CPU fallback)")
        self.h = h
        if stream is not None:
            self.set_stream(stream)

    def close(self):
        if getattr(self, "h", None):
            self.lib.ms_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise MsError(f"[{rc}] {self.lib.ms_last_error(self.h).decode()}")

    def set_stream(self, cuda_stream):
        self._ck(self.lib.ms_ctx_set_stream(self.h, cuda_stream))

    def sync(self):
        self._ck(self.lib.ms_ctx_sync(self.h))

    def set_option(self, name, value):
        """kernel tuning / A-B switches (ms_set_option), e.g. ("ntt_tma", 0) selects the one-tile-per-CTA NTT passes"""
        self._ck(self.lib.ms_set_option(self.h, name.encode(), int(value)))

    @property
    def launches(self):
        return int(self.lib.ms_launch_count(self.h))

    # ---- transforms
    def ntt_batch(self, data, field, log_n, ncols=1, col_stride=None, inverse=False, offset=ONE):
        col_stride = (1 << log_n) if col_stride is None else col_stride
        self._ck(self.lib.ms_ntt_batch(self.h, field, _ptr(data), col_stride, ncols, log_n,
                                       INVERSE if inverse else FORWARD, offset))

    def ntt_batch_to(self, src, dst, field, log_n, ncols=1, src_stride=None, dst_stride=None, inverse=False,
                     offset=ONE):
        src_stride = (1 << log_n) if src_stride is None else src_stride
        dst_stride = (1 << log_n) if dst_stride is None else dst_stride
        self._ck(self.lib.ms_ntt_batch_to(self.h, field, _ptr(src), src_stride, _ptr(dst), dst_stride, ncols, log_n,
                                          INVERSE if inverse else FORWARD, offset))

    def lde_batch(self, coeffs, evals, field, log_n, log_blowup, ncols=1, in_stride=None, out_stride=None,
                  offset=GENERATOR, bitrev=True):
        in_stride = (1 << log_n) if in_stride is None else in_stride
        out_stride = (1 << (log_n + log_blowup)) if out_stride is None else out_stride
        self._ck(self.lib.ms_lde_batch(self.h, field, _ptr(coeffs), in_stride, _ptr(evals), out_stride, ncols,
                                       log_n, log_blowup, offset, int(bitrev)))

    def lde_batch_scatter(self, coeffs, work, field, log_n, log_blowup, ncols, block_ptrs, block_col_stride, dup_ptrs=None,
                          dup_col_stride=0, in_stride=None, work_stride=None, offset=GENERATOR):
        """bit-reversed coset LDE whose last pass stores coset block q of the local columns at block_ptrs[q] (raw
        device addresses, possibly peer memory) and optionally a second copy at dup_ptrs[q] (multi-GPU fused exchange)"""
        nb = 1 << log_blowup
        n = 1 << log_n
        bp = (C.c_void_p * nb)(*[int(p) for p in block_ptrs])
        dp = (C.c_void_p * nb)(*[int(p) if p else None for p in dup_ptrs]) if dup_ptrs is not None else None
        self._ck(self.lib.ms_lde_batch_scatter(self.h, field, _ptr(coeffs), n if in_stride is None else in_stride, ncols, log_n,
                                               log_blowup, offset, _ptr(work), (n << log_blowup) if work_stride is None else work_stride,
                                               bp, block_col_stride, dp, dup_col_stride))

    # ---- raw device buffers and CUDA IPC (peer slabs of the multi-GPU commit)
    def alloc_device(self, nbytes):
        out = C.c_void_p()
        self._ck(self.lib.ms_alloc_device(self.h, nbytes, C.byref(out)))
        return int(out.value)

    def alloc_host_pinned(self, nbytes):
        out = C.c_void_p()
        self._ck(self.lib.ms_alloc_host_pinned(self.h, nbytes, C.byref(out)))
        return int(out.value)

    def free(self, ptr):
        self._ck(self.lib.ms_free(self.h, ptr))

    def ipc_export(self, ptr):
        h = (C.c_uint8 * 64)()
        self._ck(self.lib.ms_ipc_export(self.h, ptr, h))
        return bytes(h)

    def ipc_open(self, handle):
        out = C.c_void_p()
        self._ck(self.lib.ms_ipc_open(self.h, (C.c_uint8 * 64).from_buffer_copy(bytes(handle)), C.byref(out)))
        return int(out.value)

    def ipc_close(self, ptr):
        self._ck(self.lib.ms_ipc_close(self.h, ptr))

    def bit_reverse(self, data, field, log_n, ncols=1, col_stride=None):
        col_stride = (1 << log_n) if col_stride is None else col_stride
        self._ck(self.lib.ms_bit_reverse(self.h, field, _ptr(data), col_stride, ncols, log_n))

    # ---- pointwise stages
    def pointwise(self, op, dst, dfield, lhs, lfield, rhs=None, rfield=FP, n=None, shift=0, exponent=0):
        self._ck(self.lib.ms_pointwise(self.h, OPS[op], dfield, _ptr(dst), lfield, _ptr(lhs), rfield, _ptr(rhs),
                                       n, shift, exponent))

    def pointwise_const(self, op, dst, dfield, lhs, lfield, const, cfield, n):
        k = np.ascontiguousarray(const, dtype=np.uint64)
        self._ck(self.lib.ms_pointwise_const(self.h, OPS[op], dfield, _ptr(dst), lfield, _ptr(lhs), cfield,
                                             k.ctypes.data, n))

    def sum_columns(self, cols, acc, field, n, ncols, col_stride=None):
        col_stride = n if col_stride is None else col_stride
        self._ck(self.lib.ms_sum_columns(self.h, field, _ptr(cols), col_stride, ncols, n, _ptr(acc)))

    # ---- commitments
    def hash_rows(self, cols, digests, field, nrows, ncols, col_stride=None):
        col_stride = nrows if col_stride is None else col_stride
        self._ck(self.lib.ms_hash_rows_sha256(self.h, field, _ptr(cols), col_stride, ncols, nrows, _ptr(digests)))

    def merkle_nodes(self, leaves, nodes, n):
        self._ck(self.lib.ms_merkle_nodes_sha256(self.h, _ptr(leaves), n, _ptr(nodes)))

    def merkle_commit(self, cols, field, nrows, ncols, col_stride=None, leaves=None, nodes=None):
        """MatrixMerkleTree::from_matrix; returns the 32-byte root."""
        col_stride = nrows if col_stride is None else col_stride
        root = np.zeros(32, dtype=np.uint8)
        self._ck(self.lib.ms_merkle_commit_sha256(self.h, field, _ptr(cols), col_stride, ncols, nrows,
                                                  _ptr(leaves), _ptr(nodes), root.ctypes.data))
        return root.tobytes()

    def merkle_commit_rows(self, rows, row_words, nrows, leaves=None, nodes=None):
        """commit a row-major matrix (a FRI layer: rows of ff consecutive evaluations, src/fri.rs:199-216)"""
        root = np.zeros(32, dtype=np.uint8)
        self._ck(self.lib.ms_merkle_commit_rows_sha256(self.h, _ptr(rows), row_words, nrows, _ptr(leaves), _ptr(nodes),
                                                       root.ctypes.data))
        return root.tobytes()

    def merkle_commit_block(self, cols, field, log_block_rows, log_blocks, block, ncols, nodes, block_root, col_stride=None):
        """hash one coset block (2^log_block_rows rows at `cols`) and write its subtree into `nodes`, the heap of the
        whole 2^(log_block_rows + log_blocks)-leaf tree; the subtree root goes to `block_root` (32 bytes)"""
        col_stride = (1 << log_block_rows) if col_stride is None else col_stride
        self._ck(self.lib.ms_merkle_commit_block_sha256(self.h, field, _ptr(cols), col_stride, ncols, log_block_rows,
                                                        log_blocks, block, _ptr(nodes), _ptr(block_root)))

    def merkle_commit_block_host(self, cols, field, log_block_rows, ncols, host_subtree, block_root, col_stride=None):
        """hash one coset block (2^log_block_rows rows at `cols`) and copy its local heap to `host_subtree` (pinned host
        memory, 2^log_block_rows x 32 bytes; complete after sync()); the block root goes to `block_root` (32 bytes)"""
        col_stride = (1 << log_block_rows) if col_stride is None else col_stride
        self._ck(self.lib.ms_merkle_commit_block_sha256_host(self.h, field, _ptr(cols), col_stride, ncols, log_block_rows,
                                                             _ptr(host_subtree), _ptr(block_root)))

    def lde_rows(self, coeffs, field, log_n, log_blowup, ncols, positions, offset=GENERATOR, col_stride=None, out=None):
        """rows `positions` of the bit-reversed coset LDE of `coeffs`, evaluated from the coefficients; returns
        (len(positions), ncols * field) words laid out like gather_rows (or fills `out`, e.g. a device tensor)"""
        ids = np.ascontiguousarray(positions, dtype=np.uint64)
        if out is None:
            out = np.empty((ids.size, ncols * field), dtype=np.uint64)
        self._ck(self.lib.ms_lde_rows(self.h, field, _ptr(coeffs), (1 << log_n) if col_stride is None else col_stride, ncols,
                                      log_n, log_blowup, offset, ids.ctypes.data, ids.size, _ptr(out)))
        return out

    def pow_grind(self, seed, bits):
        """smallest nonce >= 1 with leading_zeros(SHA-256(seed || nonce_be8)) >= bits (src/random.rs:48-55)"""
        sd = (C.c_uint8 * 32).from_buffer_copy(bytes(seed))
        out = C.c_uint64()
        self._ck(self.lib.ms_pow_grind_sha256(self.h, sd, bits, C.byref(out)))
        return int(out.value)

    def merkle_prove(self, leaves, nodes, n_leaves, indices):
        """MerkleTreeImpl::prove (src/merkle.rs:149-207) on a resident tree.  Returns the reference's MerkleView as
        (nodes, initial_leaves, sibling_leaves, height): three lists of 32-byte digests and log2(n_leaves)."""
        ids = np.ascontiguousarray(indices, dtype=np.uint64)
        height = int(n_leaves).bit_length() - 1
        k = max(int(ids.size), 1)
        init = np.empty((k, 32), dtype=np.uint8)
        sib = np.empty((k, 32), dtype=np.uint8)
        path = np.empty((k * max(height, 1), 32), dtype=np.uint8)
        counts = (C.c_uint * 3)()
        self._ck(self.lib.ms_merkle_prove_sha256(self.h, _ptr(leaves), _ptr(nodes), n_leaves, ids.ctypes.data, ids.size,
                                                 init.ctypes.data, sib.ctypes.data, path.ctypes.data, counts))
        as_list = lambda a, m: [a[i].tobytes() for i in range(m)]
        return as_list(path, counts[2]), as_list(init, counts[0]), as_list(sib, counts[1]), height

    def matrix_from_rows(self, rows, cols, field, n, k, col_stride=None):
        self._ck(self.lib.ms_matrix_from_rows(self.h, field, _ptr(rows), n, k, _ptr(cols), n if col_stride is None else col_stride))

    def gather_rows(self, cols, field, nrows, ncols, row_ids, col_stride=None):
        ids = np.ascontiguousarray(row_ids, dtype=np.uint64)
        out = np.empty((ids.size, ncols * field), dtype=np.uint64)
        self._ck(self.lib.ms_gather_rows(self.h, field, _ptr(cols), nrows if col_stride is None else col_stride, ncols,
                                         nrows, ids.ctypes.data, ids.size, out.ctypes.data))
        return out

    def gather_rows_rowmajor(self, rows, row_words, nrows, row_ids):
        """rows of a committed FRI layer (query_layer, src/fri.rs:650-664); returns (len(row_ids), row_words) words"""
        ids = np.ascontiguousarray(row_ids, dtype=np.uint64)
        out = np.empty((ids.size, row_words), dtype=np.uint64)
        self._ck(self.lib.ms_gather_rows_rowmajor(self.h, _ptr(rows), row_words, nrows, ids.ctypes.data, ids.size,
                                                  out.ctypes.data))
        return out

    def scan_affine(self, out, field, n, init, a=None, a_field=FP, a_const=None, b=None, b_field=FP, inclusive=False):
        """x_0 = init, x_(i+1) = x_i * a_i + b_i; out[i] = x_i (or x_(i+1) if inclusive) — running products and
        running evaluations of trace columns as one parallel scan (examples/brainfuck/trace.rs:108-279)."""
        w = lambda v: None if v is None else np.ascontiguousarray(v, dtype=np.uint64)
        ini, ac = w(init), w(a_const)
        self._ck(self.lib.ms_scan_affine(self.h, field, _ptr(a), a_field, None if ac is None else ac.ctypes.data,
                                         _ptr(b), b_field, n, ini.ctypes.data, int(inclusive), _ptr(out)))

    # ---- FRI
    def fri_fold(self, evals, out, field, log_n, log_ff, alpha, offset=ONE):
        a = np.ascontiguousarray(alpha, dtype=np.uint64)
        self._ck(self.lib.ms_fri_fold(self.h, field, _ptr(evals), log_n, log_ff, offset, a.ctypes.data, _ptr(out)))

    # ---- constraint evaluation
    def eval_constraints(self, program, out, log_m, base_cols=None, nbase=0, base_stride=None, ext_cols=None, next_=0,
                         ext_stride=None, fq_field=FP, offset=GENERATOR, trace_bitrev=False, out_bitrev=False):
        """AirConfig::eval_constraint (src/air.rs:86-128): `program` from expr.compile_program."""
        m = 1 << log_m
        self._ck(self.lib.ms_eval_constraints(
            self.h, program.code.ctypes.data, len(program), program.consts.ctypes.data, program.consts.shape[0],
            _ptr(base_cols), m if base_stride is None else base_stride, nbase,
            _ptr(ext_cols), m if ext_stride is None else ext_stride, next_, fq_field, log_m, offset,
            int(trace_bitrev), int(out_bitrev), _ptr(out)))

    def eval_constraints_ptrs(self, program, out, log_m, cols, cols_are_fq, fq_field=FP, offset=GENERATOR,
                              trace_bitrev=False, out_bitrev=False):
        """same evaluator over a list of resident columns (device buffers) that may live in different matrices"""
        k = len(cols)
        ptrs = (C.c_void_p * max(k, 1))(*[_ptr(c) for c in cols])
        isq = (C.c_int * max(k, 1))(*[int(bool(q)) for q in cols_are_fq])
        self._ck(self.lib.ms_eval_constraints_ptrs(self.h, program.code.ctypes.data, len(program),
                                                   program.consts.ctypes.data, program.consts.shape[0], ptrs, isq, k,
                                                   fq_field, log_m, offset, int(trace_bitrev), int(out_bitrev), _ptr(out)))

    def check_constraints(self, program, cols, cols_are_fq, fq_field, log_n, nconstraints):
        """Constraint::check (src/constraints.rs:168-249) of constraints 0..nconstraints-1 of a checked `program`
        (expr.compile_check_program, bound) at every row of the trace domain 2^log_n; `cols`: natural-order device
        columns, then the program's periodic tables.  Returns (first_row, fail_count), numpy uint64 arrays of
        nconstraints: the lowest failing row (2^64 - 1 where none fails) and the number of failing rows."""
        k = len(cols)
        ptrs = (C.c_void_p * max(k, 1))(*[_ptr(c) for c in cols])
        isq = (C.c_int * max(k, 1))(*[int(bool(q)) for q in cols_are_fq])
        first_row = np.empty(nconstraints, dtype=np.uint64)
        fail_count = np.empty(nconstraints, dtype=np.uint64)
        self._ck(self.lib.ms_check_constraints(self.h, program.code.ctypes.data, len(program), program.consts.ctypes.data,
                                               program.consts.shape[0], ptrs, isq, k, fq_field, log_n, nconstraints,
                                               first_row.ctypes.data, fail_count.ctypes.data))
        return first_row, fail_count

    def extension_columns(self, program, out, log_n, cols, cols_are_fq, fq_field, init, inclusive):
        """the declared extension columns of an AIR (include/ministark_extension.h): column k is x_0 = init[k],
        x_(i+1) = x_i * mul_k(i) + add_k(i) over the trace domain 2^log_n, with mul_k / add_k slots 2k / 2k + 1 of `program`
        (expr.compile_extension_program, bound); row i holds x_(i+1) where inclusive[k], else x_i.  `cols`: natural-order
        device columns, then the program's periodic tables; init: (K, fq_field) Montgomery words; out: a device matrix of K
        columns of 2^log_n Fq elements."""
        k = len(cols)
        ptrs = (C.c_void_p * max(k, 1))(*[_ptr(c) for c in cols])
        isq = (C.c_int * max(k, 1))(*[int(bool(q)) for q in cols_are_fq])
        ini = np.ascontiguousarray(init, dtype=np.uint64).reshape(-1)
        inc = (C.c_int * max(len(inclusive), 1))(*[int(bool(v)) for v in inclusive])
        self._ck(self.lib.ms_extension_columns(self.h, program.code.ctypes.data, len(program), program.consts.ctypes.data,
                                               program.consts.shape[0], ptrs, isq, k, fq_field, log_n, len(inclusive),
                                               ini.ctypes.data, inc, _ptr(out)))

    def lookup_workspace_bytes(self, log_n, width, ntuples):
        """bytes of the workspace lookup_multiplicities needs (ms_lookup_workspace_bytes; arithmetic only)"""
        out = C.c_size_t()
        rc = self.lib.ms_lookup_workspace_bytes(log_n, width, ntuples, C.byref(out))
        if rc != 0:
            raise MsError(f"[{rc}] ms_lookup_workspace_bytes: log_n={log_n}, width={width}, ntuples={ntuples} out of range")
        return int(out.value)

    def lookup_multiplicities(self, program, out, log_n, cols, width, ntuples, workspace):
        """the multiplicity column of one LogUp lookup (include/ministark_lookup.h) into `out` (2^log_n Montgomery words on
        the device): `program` from expr.compile_lookup_program, `cols`: natural-order base columns (device), then the
        program's periodic tables; workspace: a device buffer of lookup_workspace_bytes(log_n, width, ntuples) bytes.
        Returns (missing, bad): per value tuple (number of rows whose tuple is not in the table, lowest such row), and
        (number of (row, tuple) pairs whose selector is neither 0 nor 1, lowest such row); a lowest row is None where
        there is none."""
        k = len(cols)
        ptrs = (C.c_void_p * max(k, 1))(*[_ptr(c) for c in cols])
        isq = (C.c_int * max(k, 1))()
        status = np.zeros(2 * ntuples + 2, dtype=np.uint64)
        nbytes = workspace.numel() * workspace.element_size() if hasattr(workspace, "numel") else workspace.nbytes
        self._ck(self.lib.ms_lookup_multiplicities(self.h, program.code.ctypes.data, len(program), program.consts.ctypes.data,
                                                   program.consts.shape[0], ptrs, isq, k, log_n, width, ntuples,
                                                   _ptr(workspace), nbytes, _ptr(out), status.ctypes.data))
        pairs = [(int(status[2 * q]), None if int(status[2 * q + 1]) == 2**64 - 1 else int(status[2 * q + 1]))
                 for q in range(ntuples + 1)]
        return pairs[:ntuples], pairs[ntuples]

    def permutation_workspace_bytes(self, log_n, width):
        """bytes of the workspace permutation_fill needs (ms_permutation_workspace_bytes; arithmetic only)"""
        out = C.c_size_t()
        rc = self.lib.ms_permutation_workspace_bytes(log_n, width, C.byref(out))
        if rc != 0:
            raise MsError(f"[{rc}] ms_permutation_workspace_bytes: log_n={log_n}, width={width} out of range")
        return int(out.value)

    def permutation_fill(self, program, targets, log_n, cols, width, workspace):
        """the target columns of one sorted-copy permutation (include/ministark_permutation.h): `targets`, width device
        columns of 2^log_n Montgomery words, receive the source tuples of `program` (expr.compile_lookup_program with no
        value tuples) sorted lexicographically, stably.  `cols`: natural-order base columns (device), then the program's
        periodic tables; workspace: a device buffer of permutation_workspace_bytes(log_n, width) bytes.  Asynchronous on
        the context's stream."""
        k = len(cols)
        ptrs = (C.c_void_p * max(k, 1))(*[_ptr(c) for c in cols])
        isq = (C.c_int * max(k, 1))()
        tgt = (C.c_void_p * max(len(targets), 1))(*[_ptr(t) for t in targets])
        nbytes = workspace.numel() * workspace.element_size() if hasattr(workspace, "numel") else workspace.nbytes
        self._ck(self.lib.ms_permutation_fill(self.h, program.code.ctypes.data, len(program), program.consts.ctypes.data,
                                              program.consts.shape[0], ptrs, isq, k, log_n, width, tgt, _ptr(workspace),
                                              nbytes))

    def poly_eval(self, coeffs, field, n, ncols, points, col_stride=None):
        """horner_evaluate of every column at every point (get_ood_evals, src/composer.rs:43-86).
        points: (k, 3) Montgomery words; returns (ncols, k, 3) numpy uint64."""
        pts = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 3)
        out = np.empty((ncols, pts.shape[0], 3), dtype=np.uint64)
        self._ck(self.lib.ms_poly_eval(self.h, field, _ptr(coeffs), n if col_stride is None else col_stride, ncols, n,
                                       pts.ctypes.data, pts.shape[0], out.ctypes.data))
        return out

    def fill_random(self, dst, nwords, seed):
        self._ck(self.lib.ms_fill_random(self.h, _ptr(dst), nwords, seed))

    # ---- examples/brainfuck execution trace (include/ministark_bf.h)
    def bf_trace_sizes(self, program, program_len, log, nrec):
        """table lengths of the trace of a run (ms_bf_trace_sizes): dict with proc_rows, instr_rows, mem_rows, reads,
        writes, n and work_bytes (the workspace bf_trace_fill needs).  program: uint32 words; log: nrec records"""
        s = np.zeros(len(BF_SIZES), dtype=np.uint64)
        self._ck(self.lib.ms_bf_trace_sizes(self.h, _ptr(program), program_len, _ptr(log), nrec, s.ctypes.data))
        return dict(zip(BF_SIZES, (int(v) for v in s)))

    def bf_trace_fill(self, program, program_len, log, nrec, sizes, work, out):
        """fill `out`, the (17, n) base matrix, from the same program and log (ms_bf_trace_fill); work: device buffer of
        sizes["work_bytes"] bytes"""
        s = np.array([sizes[k] for k in BF_SIZES], dtype=np.uint64)
        self._ck(self.lib.ms_bf_trace_fill(self.h, _ptr(program), program_len, _ptr(log), nrec, s.ctypes.data, _ptr(work),
                                           _ptr(out)))

    def bf_helper_columns(self, base, n, aux):
        """the eight helper columns of BrainfuckTrace.helper_columns() from a (17, n) base matrix into (8, n) `aux`"""
        self._ck(self.lib.ms_bf_helper_columns(self.h, _ptr(base), n, _ptr(aux)))

    # ---- examples/rescue trace (include/ministark_rescue.h)
    def rescue_chains(self, seed, K, L, out):
        """write `out`, the (12, 8 K L) matrix of K chains of L Rescue-Prime permutations from the four canonical seed
        words (ms_rescue_chains); not synchronised"""
        s = np.array([int(v) for v in seed], dtype=np.uint64)
        if s.size != 4:
            raise MsError("ms_rescue_chains: the seed is four words")
        self._ck(self.lib.ms_rescue_chains(self.h, s.ctypes.data, int(K), int(L), _ptr(out)))

    # ---- examples/rescue hash trace (include/ministark_rescue_hash.h)
    def rescue_hash(self, messages, K, length, out):
        """write `out`, the (13, 8 K L) sponge trace of K messages of `length` canonical words (`messages`: K x length,
        row-major, host or device; ms_rescue_hash); not synchronised"""
        self._ck(self.lib.ms_rescue_hash(self.h, _ptr(messages), int(K), int(length), _ptr(out)))

    # ---- examples/merkle tree and paths (include/ministark_rescue_merkle.h)
    def rescue_merkle_tree(self, leaves, depth, nodes):
        """write `nodes`, the (2^(D + 1), 4) heap of the Rescue-Prime Merkle tree over `leaves` ((2^D, 4) canonical
        words, host or device; ms_rescue_merkle_tree); not synchronised when both are device memory"""
        self._ck(self.lib.ms_rescue_merkle_tree(self.h, _ptr(leaves), int(depth), _ptr(nodes)))

    def rescue_merkle_paths(self, nodes, depth, indices, K, out):
        """write `out`, the (14, 8 K L) trace of the K authentication paths of `indices` (K uint64 words, host or
        device) through the heap `nodes` of depth D (host or device; ms_rescue_merkle_paths); synchronises"""
        self._ck(self.lib.ms_rescue_merkle_paths(self.h, _ptr(nodes), int(depth), _ptr(indices), int(K), _ptr(out)))

    def rescue_merkle_updates(self, nodes, depth, indices, new_leaves, K, out, roots):
        """apply K leaf writes in order to the heap `nodes` of depth D, in place: leaf indices[k] (K uint64 words) becomes
        new_leaves[k] ((K, 4) canonical words); write `out`, the (15, 16 K L) trace of the old and the new paths, and
        `roots`, the (K + 1, 4) roots before the first write and after each (all host or device;
        ms_rescue_merkle_updates); synchronises"""
        self._ck(self.lib.ms_rescue_merkle_updates(self.h, _ptr(nodes), int(depth), _ptr(indices), _ptr(new_leaves),
                                                   int(K), _ptr(out), _ptr(roots)))

    def rescue_rollup(self, nodes, depth, transfers, K, out, roots):
        """apply K transfers in order to the accounts of the heap `nodes` of depth D, in place: transfers is (K, 3)
        uint64 words (sender, receiver, amount); write `out`, the (23, 32 K L) trace, and `roots`, the (K + 1, 4) roots
        before the first transfer and after each (all host or device; ms_rescue_rollup); synchronises.  An invalid
        batch raises MsError naming its first failing transfer and writes nothing"""
        self._ck(self.lib.ms_rescue_rollup(self.h, _ptr(nodes), int(depth), _ptr(transfers), int(K), _ptr(out),
                                           _ptr(roots)))

    def rescue_wots_sign(self, secrets, seeds, messages, K, signatures, public_keys):
        """sign messages[k] (K x 4 words) with the key of secrets[k] (K x 4) and seeds[k] (K x 2): write `signatures`
        (K x 67 x 4 words) and `public_keys` (K x 6: the seed, then the root) (all host or device;
        ms_rescue_wots_sign)"""
        self._ck(self.lib.ms_rescue_wots_sign(self.h, _ptr(secrets), _ptr(seeds), _ptr(messages), int(K),
                                              _ptr(signatures), _ptr(public_keys)))

    def rescue_wots_trace(self, public_keys, messages, signatures, K, out):
        """write `out`, the (15, 128 B) trace of K signatures (public_keys K x 6, messages K x 4, signatures K x 67 x 4
        words; all host or device; ms_rescue_wots_trace); synchronises.  A signature that does not verify raises
        MsError naming the lowest such k and writes nothing"""
        self._ck(self.lib.ms_rescue_wots_trace(self.h, _ptr(public_keys), _ptr(messages), _ptr(signatures), int(K),
                                               _ptr(out)))


BF_SIZES = ("proc_rows", "instr_rows", "mem_rows", "reads", "writes", "n", "work_bytes")     # MS_BF_* of ministark_bf.h


def bf_run(program, input_bytes=b"", max_cycles=1 << 26):
    """ms_bf_run: the brainfuck VM over a compiled program (uint32 words) on the host.  Returns (log, output bytes): the
    uint64 records of the cycles + 1 processor rows (include/ministark_bf.h).  Raises MsError when the memory pointer
    leaves the tape, the input runs out or max_cycles cycles do not reach the end of the program."""
    lib = _lib.load()
    prog = np.ascontiguousarray(program, dtype=np.uint32)
    inp = np.frombuffer(bytes(input_bytes), dtype=np.uint8).copy()
    log = np.empty(max_cycles + 1, dtype=np.uint64)         # pages the run does not reach are never touched
    out = np.empty(max(max_cycles, 1), dtype=np.uint8)
    counts = np.zeros(2, dtype=np.uint64)
    rc = lib.ms_bf_run(prog.ctypes.data, prog.size, inp.ctypes.data, inp.size, max_cycles, log.ctypes.data,
                       out.ctypes.data, counts.ctypes.data)
    if rc != 0:
        raise MsError(f"[{rc}] {lib.ms_last_error(None).decode()}")
    cycles, nout = int(counts[0]), int(counts[1])
    return log[:cycles + 1].copy(), out[:nout].tobytes()


_default_ctx = None


def get_planner():
    """process-global lazily created context (get_planner(), gpu/src/plan.rs:465-469)."""
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(0)
    return _default_ctx


class Domain:
    """Radix2EvaluationDomain: size 2^log_n, coset offset (Montgomery word)."""

    def __init__(self, log_n, offset=ONE):
        self.log_n, self.offset = log_n, offset

    def size(self):
        return 1 << self.log_n


class _FftBase:
    MIN_SIZE = 2048  # gpu/src/plan.rs:246,292 (kept for interface parity; not enforced)
    _direction = FORWARD

    def __init__(self, domain, field=FP, ctx=None):
        self.ctx = ctx or get_planner()
        self.domain, self.field = domain, field
        h = C.c_void_p()
        self.ctx._ck(self.ctx.lib.ms_ntt_plan_create(self.ctx.h, field, domain.log_n, self._direction,
                                                     domain.offset, C.byref(h)))
        self.h = h
        self._keep = []

    def encode(self, column):
        """enqueue an in-place transform of one column of exactly domain.size() elements
        (GpuFft::encode, gpu/src/plan.rs:254-267)."""
        if isinstance(column, np.ndarray) and column.size != self.domain.size() * self.field:
            raise MsError("column length must equal the domain size")  # assert_eq!, plan.rs:257
        self._keep.append(column)
        self.ctx._ck(self.ctx.lib.ms_ntt_encode(self.h, _ptr(column)))

    def execute(self):
        """run everything encoded and block until done (FftEncoder::execute, plan.rs:229-232)."""
        self.ctx._ck(self.ctx.lib.ms_ntt_execute(self.h))
        self._keep = []

    def __del__(self):
        try:
            if self.h:
                self.ctx.lib.ms_ntt_plan_destroy(self.h)
                self.h = None
        except Exception:
            pass


class GpuFft(_FftBase):
    _direction = FORWARD


class GpuIfft(_FftBase):
    _direction = INVERSE


class Matrix:
    """Column-major matrix of field elements (src/matrix.rs:26): numpy (ncols, nrows*field) uint64."""

    def __init__(self, cols, field=FP, ctx=None):
        self.cols = np.ascontiguousarray(cols, dtype=np.uint64)
        if self.cols.ndim == 1:
            self.cols = self.cols.reshape(1, -1)
        self.field = field
        self.ctx = ctx or get_planner()

    def num_cols(self):
        return self.cols.shape[0]

    def num_rows(self):
        return self.cols.shape[1] // self.field

    def _log_rows(self):
        n = self.num_rows()
        if n & (n - 1):
            raise MsError("number of rows must be a power of two")
        return n.bit_length() - 1

    def interpolate(self, domain):
        """Matrix::interpolate (src/matrix.rs:157-163): iNTT of every column."""
        out = self.cols.copy()
        self.ctx.ntt_batch(out, self.field, domain.log_n, self.num_cols(), inverse=True, offset=domain.offset)
        return Matrix(out, self.field, self.ctx)

    def evaluate(self, domain):
        """Matrix::evaluate (src/matrix.rs:237-243): zero-pad to the domain and NTT, natural order."""
        return self._lde(domain, False)

    def bit_reversed_evaluate(self, domain):
        """Matrix::bit_reversed_evaluate (src/matrix.rs:245-251)."""
        return self._lde(domain, True)

    def _lde(self, domain, bitrev):
        log_n = self._log_rows()
        if domain.log_n < log_n:
            raise MsError("domain smaller than the polynomial")
        out = np.empty((self.num_cols(), domain.size() * self.field), dtype=np.uint64)
        self.ctx.lde_batch(self.cols, out, self.field, log_n, domain.log_n - log_n, self.num_cols(),
                           offset=domain.offset, bitrev=bitrev)
        return Matrix(out, self.field, self.ctx)

    def bit_reverse_rows(self):
        self.ctx.bit_reverse(self.cols, self.field, self._log_rows(), self.num_cols())

    def sum_columns(self):
        acc = np.empty(self.cols.shape[1], dtype=np.uint64)
        self.ctx.sum_columns(self.cols, acc, self.field, self.num_rows(), self.num_cols())
        return Matrix(acc.reshape(1, -1), self.field, self.ctx)

    def hash_rows(self):
        d = np.empty((self.num_rows(), 32), dtype=np.uint8)
        self.ctx.hash_rows(self.cols, d, self.field, self.num_rows(), self.num_cols())
        return d

    def get_row(self, i):
        f = self.field
        return self.cols[:, i * f:(i + 1) * f].copy()


class MatrixMerkleTree:
    """MatrixMerkleTreeImpl<Sha256HashFn> (src/merkle.rs:316-386): heap-layout nodes, root = nodes[1]."""

    def __init__(self, leaves, nodes):
        self.leaves, self.nodes = leaves, nodes

    @classmethod
    def from_matrix(cls, m):
        n = m.num_rows()
        leaves = np.empty((n, 32), dtype=np.uint8)
        nodes = np.empty((n, 32), dtype=np.uint8)
        m.ctx.merkle_commit(m.cols, m.field, n, m.num_cols(), leaves=leaves, nodes=nodes)
        return cls(leaves, nodes)

    def root(self):
        return self.nodes[1].tobytes()
