/*
 * ministark_permutation.h — target columns of the sorted-copy permutation arguments an AIR declares, filled on the device
 * from the base trace.  Conventions as in ministark_b200.h (Montgomery words, 0 on success, a negative MS_ERR_* otherwise).
 *
 * A permutation (ministark_b200/air.py, Permutation) has a source tuple s(i) of W expressions over the base trace at every
 * row i = 0..n-1, and W target columns.  Row j of target column k holds word k of the j-th source tuple in ascending
 * lexicographic order of the canonical integers, word 0 first; equal tuples keep their row order (a stable sort).
 */
#ifndef MINISTARK_PERMUTATION_H
#define MINISTARK_PERMUTATION_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The workspace ms_permutation_fill needs for one permutation of width words per tuple over a trace domain of 2^log_n
 * rows (log_n <= 30, 1 <= width <= 4), in *bytes.  Arithmetic only: no device is touched, so the caller can allocate it
 * where its allocator accounts for it. */
int ms_permutation_workspace_bytes(unsigned log_n, unsigned width, size_t *bytes);

/* Fills the target columns of one permutation.  program: an evaluator program of nprog 4-word instructions
 * (ministark_b200/expr.py::compile_lookup_program with no value tuples) over the base field whose OP_STORE k stores source
 * word k, k < width; evaluated at row i with X = g_n^i, Trace(col, off) = column[(i + off) mod 2^log_n] and periodic
 * tables over <g_n>.  consts: nconsts Fq3 constants.  col_ptrs / col_is_fq: ncols device columns (natural order, all of
 * Fp words).  targets: width distinct device columns of 2^log_n Montgomery words, natural order; every source word is
 * evaluated before any target is written, so a target may be a column the program reads.  workspace: device memory of
 * workspace_bytes >= ms_permutation_workspace_bytes(log_n, width).  Asynchronous on the context's stream. */
int ms_permutation_fill(ms_ctx *ctx, const uint32_t *program, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                        const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, unsigned log_n, unsigned width,
                        void *const *targets, void *workspace, size_t workspace_bytes);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_PERMUTATION_H */
