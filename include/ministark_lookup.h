/*
 * ministark_lookup.h — multiplicity columns of the LogUp lookups an AIR declares, filled on the device from the base trace.
 * Conventions as in ministark_b200.h (Montgomery words, 0 on success, a negative MS_ERR_* otherwise).
 *
 * A lookup (ministark_b200/air.py, Lookup) says that at every row i the value tuples v_q(i) whose selector is 1 are rows of
 * the table, the tuple t(j) at row j for j = 0..n-1; all of them are expressions over the base trace.  Its multiplicity
 * column holds, at row j, the number of (row, value tuple) pairs that look up t(j); a tuple that occurs more than once in
 * the table counts at its lowest row, the others get 0.  Tuples are matched exactly, word for word, with no hashing.
 */
#ifndef MINISTARK_LOOKUP_H
#define MINISTARK_LOOKUP_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The workspace ms_lookup_multiplicities needs for one lookup of width words per tuple and ntuples value tuples over a
 * trace domain of 2^log_n rows (log_n <= 30, 1 <= width <= 4, 1 <= ntuples <= 4), in *bytes.  Arithmetic only: no device
 * is touched, so the caller can allocate it where its allocator accounts for it. */
int ms_lookup_workspace_bytes(unsigned log_n, unsigned width, unsigned ntuples, size_t *bytes);

/* Fills the multiplicity column of one lookup.  program: an evaluator program of nprog 4-word instructions
 * (ministark_b200/expr.py::compile_lookup_program) over the base field whose OP_STORE s stores slot s: table word k is
 * slot k, value tuple q's selector slot width + q * (width + 1) and its word k the slot k + 1 after it; evaluated at row i
 * with X = g_n^i, Trace(col, off) = column[(i + off) mod 2^log_n] and periodic tables over <g_n>.  consts: nconsts Fq3
 * constants.  col_ptrs / col_is_fq: ncols device columns (natural order, all of Fp words).  workspace: device memory of
 * workspace_bytes >= ms_lookup_workspace_bytes(log_n, width, ntuples).  out: the device multiplicity column, 2^log_n
 * Montgomery words in natural order; it may be one of the trace columns the program does not read.
 * status: 2 * ntuples + 2 host words: for value tuple q, status[2q] rows whose tuple is not in the table and status[2q + 1]
 * the lowest of them; then the number of (row, tuple) pairs whose selector is neither 0 nor 1 and the lowest such row.
 * A lowest row is 2^64 - 1 where there is none.  Rows with a missing tuple or a bad selector add nothing to out.
 * Synchronizes with the host once, to fill status. */
int ms_lookup_multiplicities(ms_ctx *ctx, const uint32_t *program, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                             const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, unsigned log_n, unsigned width,
                             unsigned ntuples, void *workspace, size_t workspace_bytes, void *out, uint64_t *status);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_LOOKUP_H */
