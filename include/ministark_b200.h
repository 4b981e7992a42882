/*
 * ministark_b200.h — C ABI of libministark_b200.so: the H100 (sm_90a) replacement for
 * the Metal backend of andrewmilson/ministark's `ministark-gpu` crate and for the CPU
 * steps that sit between its GPU calls in the prover hot path (SURVEY.md §8).
 *
 * The reference has no FFI of its own (it reaches the device through the `metal`
 * crate); each entry point below names the reference interface it replaces
 * (file:line under /root/reference).  A Rust `extern "C"` binding for these symbols is
 * shown in INTEGRATION.md; include/ministark_gpu.hpp is the C++ mirror of the Rust
 * item set (GpuFft, GpuIfft, Planner, *Stage, Matrix, MatrixMerkleTree).
 *
 * Conventions
 *   - Field elements are raw 64-bit Montgomery words, canonical (< p), R = 2^64, exactly
 *     as ark-ff-optimized keeps them in memory (gpu/src/metal/felt_u64.h.metal:118,127).
 *     MS_FIELD_FP  : 1 word / element.   MS_FIELD_FQ3 : 3 words (c0,c1,c2), X^3 = 2
 *     (gpu/src/fields.rs:52-53,78-97).
 *   - A matrix is column-major: column c starts at base + c * col_stride_elems elements
 *     (src/matrix.rs:26, Vec<GpuVec<F>>).
 *   - Every pointer argument may be a device pointer, a pinned/managed host pointer or a
 *     pageable host pointer; host buffers are staged through device scratch inside the
 *     call (the reference relies on Apple unified memory: gpu/src/utils.rs:106-134).
 *   - All functions return 0 on success, a negative MS_ERR_* otherwise; the reference
 *     panics on any failure (gpu/src/stage.rs:55-75, gpu/src/plan.rs:255-257), the
 *     Rust/C++ shims turn non-zero into panic!/throw.  ms_last_error() gives the text.
 *   - A context is not re-entrant; all work is issued on its stream in order
 *     (one in-order Metal queue in the reference, gpu/src/plan.rs:327-350).
 *   - There is no CPU fallback: without a CUDA device ms_ctx_create fails.
 */
#ifndef MINISTARK_B200_H
#define MINISTARK_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MS_OK 0
#define MS_ERR_INVALID (-1)   /* bad argument (size not a power of two, out of range, …) */
#define MS_ERR_CUDA (-2)      /* CUDA runtime failure */
#define MS_ERR_NOMEM (-3)
#define MS_ERR_NODEVICE (-4)

#define MS_FIELD_FP 1   /* Goldilocks base field, kernel suffix "p18446744069414584321_fp"  (gpu/src/fields.rs:55-61) */
#define MS_FIELD_FQ3 3  /* cubic extension,        kernel suffix "p18446744069414584321_fq3" (gpu/src/fields.rs:211-217) */

#define MS_NTT_FORWARD 0 /* FftDirection::Forward (gpu/src/plan.rs:176-183) */
#define MS_NTT_INVERSE 1 /* FftDirection::Inverse */

/* pointwise stage opcodes (gpu/src/metal/evaluation_shaders.h.metal:11-168) */
#define MS_OP_MUL 0     /* MulInto / MulAssign                     :58-66,79-88  */
#define MS_OP_ADD 1     /* AddInto / AddAssign                     :68-76,90-99  */
#define MS_OP_CONVERT 2 /* ConvertInto (Fp -> Fq3 embed)           :121-127      */
#define MS_OP_INV 3     /* InverseInto / InverseInPlace            :11-16,33-39  */
#define MS_OP_EXP 4     /* ExpInto / ExpInPlace                    :18-24,41-48  */
#define MS_OP_NEG 5     /* NegInto / NegInPlace                    :26-31,50-56  */
#define MS_OP_MULPOW 6  /* MulPow                                  :149-161      */
#define MS_OP_FILL 7    /* FillBuff                                :163-168      */
#define MS_OP_SUB 8     /* (not a reference stage; used by the fused evaluator) */

typedef struct ms_ctx ms_ctx;
typedef struct ms_ntt_plan ms_ntt_plan;

/* ---- context: replaces Planner / get_planner() (gpu/src/plan.rs:327-350,465-469) ---- */
int ms_ctx_create(int device, ms_ctx **out);
int ms_ctx_destroy(ms_ctx *ctx);
/* use an existing cudaStream_t (e.g. torch's current stream); NULL = the context's own */
int ms_ctx_set_stream(ms_ctx *ctx, void *cuda_stream);
int ms_ctx_sync(ms_ctx *ctx);
const char *ms_last_error(ms_ctx *ctx);
const char *ms_version(void);
/* tuning / A-B switches of the kernels (process-wide; no reference counterpart): "ntt_tma" 0|1 selects the persistent
 * TMA pipeline for the 256 x 16 tile NTT passes (default 1), "ntt_tma_groups" 2|3 consumer groups per CTA,
 * "ntt_tma_stages" 3..8 cap on its shared-memory ring; "drop_plans" (any value) frees this context's cached NTT plans and
 * their twiddle / scale tables (hundreds of MiB for 2^24-point LDE plans; rebuilt on demand); "drop_scratch" (any value)
 * frees its scratch arenas (e.g. the temporary of a large single-column transform; regrown on demand).  Test switches:
 * "ntt_table_words" (per context, -1 = built-in limits) caps in words each full twiddle / scale table of new plans and
 * drops the cached plans; "ntt_wide_index" 0|1 makes the tile passes use their 64-bit-offset instantiations at every size. */
int ms_set_option(ms_ctx *ctx, const char *name, int64_t value);
/* number of kernels this context has launched so far (bench.py "gpu_launches") */
uint64_t ms_launch_count(ms_ctx *ctx);

/* ---- memory: backs GpuAllocator / GpuVec (src/utils.rs:438-493) and
 *      page_aligned_uninit_vector (gpu/src/utils.rs:208-220) ---- */
int ms_alloc_device(ms_ctx *ctx, size_t bytes, void **out);
int ms_alloc_host_pinned(ms_ctx *ctx, size_t bytes, void **out);
int ms_free(ms_ctx *ctx, void *ptr); /* either kind */
int ms_copy(ms_ctx *ctx, void *dst, const void *src, size_t bytes); /* any direction, stream-ordered + sync */

/* ---- GpuFft / GpuIfft (gpu/src/plan.rs:236-325): plan, encode many columns, execute ----
 * log_n in [0, 32].  offset_mont = domain.offset as a Montgomery word (ONE = 4294967295
 * for a subgroup).  Forward: out[i] = sum_j c_j (offset*g^i)^j, natural order in place.
 * Inverse: the inverse map incl. 1/n and offset^-j (gpu/src/plan.rs:404-424).
 * GpuFft::MIN_SIZE (2048, plan.rs:246) is NOT enforced: smaller sizes also run on device. */
int ms_ntt_plan_create(ms_ctx *ctx, int field, unsigned log_n, int direction, uint64_t offset_mont,
                       ms_ntt_plan **out);
int ms_ntt_encode(ms_ntt_plan *plan, void *column);   /* exactly 2^log_n elements, transformed in place */
int ms_ntt_execute(ms_ntt_plan *plan);                /* runs everything encoded; blocks; clears the queue */
int ms_ntt_plan_destroy(ms_ntt_plan *plan);

/* ---- resident batched forms used by Matrix::{into_polynomials,into_evaluations,
 *      into_bit_reversed_evaluations} (src/matrix.rs:101-251) ---- */
int ms_ntt_batch(ms_ctx *ctx, int field, void *data, size_t col_stride_elems, unsigned ncols,
                 unsigned log_n, int direction, uint64_t offset_mont);
/* out-of-place form (Matrix::interpolate = clone + into_polynomials, src/matrix.rs:157-163, without
 * the clone): src is left untouched; src == dst is allowed. */
int ms_ntt_batch_to(ms_ctx *ctx, int field, const void *src, size_t src_stride_elems, void *dst,
                    size_t dst_stride_elems, unsigned ncols, unsigned log_n, int direction, uint64_t offset_mont);
/* coefficients (2^log_n per column) -> evaluations over offset*<g_N>, N = 2^(log_n+log_blowup),
 * bit-reversed row order when bitrev_out != 0 (no zero padding, no separate bit-reverse pass). */
int ms_lde_batch(ms_ctx *ctx, int field, const void *coeffs, size_t in_stride_elems, void *evals,
                 size_t out_stride_elems, unsigned ncols, unsigned log_n, unsigned log_blowup,
                 uint64_t offset_mont, int bitrev_out);

/* ---- bit_reverse (gpu/src/utils.rs:32-78, BitReverseGpuStage stage.rs:280-332) ---- */
int ms_bit_reverse(ms_ctx *ctx, int field, void *data, size_t col_stride_elems, unsigned ncols, unsigned log_n);

/* ---- pointwise stages (gpu/src/stage.rs, 14 stage types; evaluation_shaders.h.metal) ----
 * dst[i] = lhs[i] OP rhs[(i + shift) % n].  dst may alias lhs (the ...Assign and ...InPlace forms).
 * Unary ops (INV, EXP, NEG, CONVERT) ignore rhs.  exponent is used by EXP / MULPOW. */
int ms_pointwise(ms_ctx *ctx, int op, int dst_field, void *dst, int lhs_field, const void *lhs,
                 int rhs_field, const void *rhs, size_t n, size_t shift, uint64_t exponent);
/* dst[i] = lhs[i] OP constant (the *Const stages); MS_OP_FILL ignores lhs */
int ms_pointwise_const(ms_ctx *ctx, int op, int dst_field, void *dst, int lhs_field, const void *lhs,
                       int const_field, const uint64_t *constant, size_t n);
/* Matrix::sum_columns (src/matrix.rs:322-394): acc[i] = sum_c col_c[i] in ONE pass */
int ms_sum_columns(ms_ctx *ctx, int field, const void *cols, size_t col_stride_elems, unsigned ncols,
                   size_t n, void *acc);

/* ---- Merkle commitment: hash_rows + build_merkle_nodes (src/merkle.rs:412-508,
 *      Sha256HashFn src/hash.rs:58-100) ----
 * leaf_i = SHA-256( ||_c LE64(canonical(col_c[i])) ), Fq3 = c0||c1||c2.  digests: nrows x 32 B. */
int ms_hash_rows_sha256(ms_ctx *ctx, int field, const void *cols, size_t col_stride_elems, unsigned ncols,
                        size_t nrows, void *digests);
/* nodes: n x 32 B heap layout, nodes[0] = zero digest, nodes[1] = root, nodes[n/2+i] = H(leaf 2i || leaf 2i+1) */
int ms_merkle_nodes_sha256(ms_ctx *ctx, const void *leaves, size_t n, void *nodes);
/* MatrixMerkleTree::from_matrix in one call; nodes may be NULL (root only); root: 32 B (host or device) */
int ms_merkle_commit_sha256(ms_ctx *ctx, int field, const void *cols, size_t col_stride_elems, unsigned ncols,
                            size_t nrows, void *leaves, void *nodes, void *root);

/* commitment of a ROW-MAJOR matrix (nrows rows of row_words contiguous words): a FRI layer commits rows of
 * ff consecutive evaluations (src/fri.rs:199-216, Matrix::from_arrays + from_matrix) — hashed in place */
int ms_merkle_commit_rows_sha256(ms_ctx *ctx, const void *rows, unsigned row_words, size_t nrows, void *leaves,
                                 void *nodes, void *root);

/* ---- proof of work: PublicCoin::grind_proof_of_work (src/random.rs:48-55,129-132; src/channel.rs:76-93) ----
 * smallest nonce >= 1 with leading_zeros(SHA-256(seed[32] || nonce as 8 big-endian bytes)) >= bits
 * (deterministic, unlike the reference's rayon find_any) */
int ms_pow_grind_sha256(ms_ctx *ctx, const uint8_t *seed, unsigned bits, uint64_t *nonce_out);

/* ---- query phase: MerkleTreeImpl::prove / MatrixMerkleTree::prove_rows (src/merkle.rs:149-207,301-303) ----
 * batched authentication paths (the reference's MerkleView) for `indices` (any order, duplicates allowed) from the
 * resident leaf and node arrays of a committed tree.  Outputs (host): initial_leaves and sibling_leaves hold up to
 * n_indices digests each, path_nodes up to n_indices * log2(n_leaves); counts = {initial, sibling, path} digests written */
int ms_merkle_prove_sha256(ms_ctx *ctx, const void *leaves, const void *nodes, size_t n_leaves, const uint64_t *indices,
                           unsigned n_indices, uint8_t *initial_leaves, uint8_t *sibling_leaves, uint8_t *path_nodes,
                           unsigned counts[3]);

/* ---- matrix plumbing ----
 * Matrix::from_arrays / from_rows (src/matrix.rs:33-64) and the composition split (src/prover.rs:113-120):
 * n rows of k elements (row-major) -> k columns of n elements */
int ms_matrix_from_rows(ms_ctx *ctx, int field, const void *rows, size_t n, unsigned k, void *cols,
                        size_t col_stride_elems);
/* Matrix::get_row for a list of rows (src/matrix.rs:288-294; Queries::new src/trace.rs:115-157):
 * out[q * ncols + c] = cols[c][row_ids[q]]; row_ids is a host array */
int ms_gather_rows(ms_ctx *ctx, int field, const void *cols, size_t col_stride_elems, unsigned ncols, size_t nrows,
                   const uint64_t *row_ids, unsigned nq, void *out);
/* query_layer (src/fri.rs:650-664): rows of a ROW-MAJOR matrix (a committed FRI layer); out[q] = rows[row_ids[q]] */
int ms_gather_rows_rowmajor(ms_ctx *ctx, const void *rows, unsigned row_words, size_t nrows, const uint64_t *row_ids,
                            unsigned nq, void *out);

/* ---- multi-GPU: LDE fused with the exchange into row slabs (SURVEY.md §8e) ----
 * one process per GPU; the bit-reversed LDE is 2^log_blowup coset blocks of n rows and, with G | 2^log_blowup GPUs,
 * the row slab a GPU hashes is a run of whole blocks.  The last NTT pass stores block q of every local column at
 * block_ptrs[q] + column * block_col_stride_elems (element units) — block_ptrs[q] may point into a PEER GPU's slab
 * (mapped with ms_ipc_open), so the all-to-all disappears into the LDE's own stores over NVLink.  dup_ptrs (or NULL;
 * entries may be NULL): a second copy of block q, e.g. the local ce-domain prefix.  work: ncols x work_stride_elems
 * resident scratch for the earlier passes.  The caller synchronises the ranks (barrier) before reading a slab. */
int ms_lde_batch_scatter(ms_ctx *ctx, int field, const void *coeffs, size_t in_stride_elems, unsigned ncols, unsigned log_n,
                         unsigned log_blowup, uint64_t offset_mont, void *work, size_t work_stride_elems,
                         void *const *block_ptrs, size_t block_col_stride_elems, void *const *dup_ptrs,
                         size_t dup_col_stride_elems);
/* CUDA IPC: export a buffer obtained from ms_alloc_device (handle: 64 bytes), map / unmap a peer's buffer */
int ms_ipc_export(ms_ctx *ctx, const void *dev_ptr, uint8_t *handle64);
int ms_ipc_open(ms_ctx *ctx, const uint8_t *handle64, void **peer_ptr);
int ms_ipc_close(ms_ctx *ctx, void *peer_ptr);

/* ---- trace generation: running products / running evaluations as a parallel scan (SURVEY.md §8f rank 3) ----
 * the sequential column builders of examples/brainfuck/trace.rs:108-279 and examples/fib/main.rs:175-222:
 *     x_0 = init,  x_(i+1) = x_i * a_i + b_i,      out[i] = x_i (inclusive == 0) or x_(i+1) (inclusive != 0)
 * field: type of x / out / init (MS_FIELD_FP or MS_FIELD_FQ3).  a: n elements of a_field (Fp or `field`), or NULL for
 * the constant multiplier a_const (one element of `field`).  b: n elements of b_field, or NULL for 0. */
int ms_scan_affine(ms_ctx *ctx, int field, const void *a, int a_field, const uint64_t *a_const, const void *b, int b_field,
                   size_t n, const uint64_t *init, int inclusive, void *out);

/* ---- FRI: apply_drp (src/fri.rs:526-567) evaluated per coset, bit-reversed order in and out ----
 * evals: 2^log_n elements; out: 2^(log_n-log_ff).  alpha: one element of `field`.
 * Equals bit_reverse ∘ NTT ∘ fold ∘ (·ff) ∘ iNTT ∘ bit_reverse of the reference, in one pass. */
int ms_fri_fold(ms_ctx *ctx, int field, const void *evals, unsigned log_n, unsigned log_ff,
                uint64_t offset_mont, const uint64_t *alpha, void *out);

/* ---- constraint evaluation: AirConfig::eval_constraint -> eval_cpu::eval (src/air.rs:86-128,
 *      src/eval_cpu.rs:33-150; dead GPU twin src/eval_gpu.rs:46-131) as ONE fused kernel ----
 * program: nprog x 4 uint32 words, the linear form of the composition-constraint DAG produced by
 * ministark_b200/expr.py::compile_program (opcodes in csrc/eval.cu); consts: nconsts x 3 Montgomery
 * words.  base_cols: nbase Fp columns, ext_cols: next columns of `fq_field` elements, each holding the
 * M = 2^log_m evaluations over the ce coset offset*<g_M> — in natural order, or (trace_bitrev != 0) as
 * the first M entries of a bit-reversed LDE column (what src/prover.rs:86-91 un-permutes on the CPU).
 * out: M elements of fq_field (one Fq value per domain point), natural order, or — out_bitrev != 0 together
 * with trace_bitrev — in the same bit-reversed order as the inputs (used by the DEEP composition, whose
 * result feeds FRI in bit-reversed order, src/prover.rs:146-148). */
int ms_eval_constraints(ms_ctx *ctx, const uint32_t *program, unsigned nprog, const uint64_t *consts,
                        unsigned nconsts, const void *base_cols, size_t base_stride_elems, unsigned nbase,
                        const void *ext_cols, size_t ext_stride_elems, unsigned next, int fq_field,
                        unsigned log_m, uint64_t offset_mont, int trace_bitrev, int out_bitrev, void *out);

/* same evaluator over an explicit table of DEVICE column pointers (columns from different matrices);
 * col_is_fq[i] = 0: base-field column, 1: column of `fq_field` elements; out must be a device pointer */
int ms_eval_constraints_ptrs(ms_ctx *ctx, const uint32_t *program, unsigned nprog, const uint64_t *consts,
                             unsigned nconsts, const void *const *col_ptrs, const int *col_is_fq, unsigned ncols,
                             int fq_field, unsigned log_m, uint64_t offset_mont, int trace_bitrev, int out_bitrev,
                             void *out);

/* diagnostic (tests only): the lazy field primitives of the NTT butterflies, element-wise over ANY 64-bit words:
 * out[k*n + i], k = 0 add_lc(a, canon b), 1 sub_lc(a, canon b), 2 add_ll(a, b), 3 sub_ll(a, b), 4 mul(a, canon b) */
int ms_debug_lazy_ops(ms_ctx *ctx, const uint64_t *a, const uint64_t *b, size_t n, uint64_t *out);

/* diagnostic, needs no GPU: generate the run-time specialised evaluation kernel for a program (csrc/eval_jit.cu)
 * and compile it with NVRTC for sm_90a.  0 = ok, 1 = NVRTC not installed (the interpreter kernel is used),
 * -1 = compile error (log_out receives the NVRTC log) */
int ms_eval_jit_check(const uint32_t *program, unsigned nprog, const uint64_t *consts, unsigned nconsts, int fq_field,
                      char *log_out, size_t log_cap);

/* ---- DEEP: out-of-domain evaluations, DeepPolyComposer::get_ood_evals (src/composer.rs:43-86) =
 *      horner_evaluate (src/utils.rs:124-131) of every column at every point, as a parallel reduction ----
 * coeffs: ncols columns of n coefficients of `field`; points: npoints Fq3 elements (3 words each);
 * out[(col * npoints + k) * 3 ..] = P_col(points[k]) as Fq3.  The DEEP quotients themselves are evaluated
 * pointwise over the LDE by ms_eval_constraints (program built by ministark_b200/deep.py). */
int ms_poly_eval(ms_ctx *ctx, int field, const void *coeffs, size_t col_stride_elems, unsigned ncols, size_t n,
                 const uint64_t *points, unsigned npoints, uint64_t *out);

/* ---- synthetic data (SURVEY.md §8d): splitmix64, reject >= p, store x*2^64 mod p ---- */
int ms_fill_random(ms_ctx *ctx, void *dst, size_t nwords, uint64_t seed);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_B200_H */
