/*
 * ministark_extension.h — extension columns declared by the AIR, built on the device from the base trace.
 * Conventions as in ministark_b200.h (Montgomery words, 0 on success, a negative MS_ERR_* otherwise).
 *
 * The reference builds its extension columns (running products, running evaluations, running sums) with hand-written
 * host loops (src/trace.rs, examples/brainfuck/trace.rs:108-279).  Here an AIR declares column k as the recurrence
 *     x_0 = init_k,   x_(i+1) = x_i * mul_k(i) + add_k(i)
 * with mul_k and add_k expressions over the base trace (ministark_b200/air.py, RunningColumn), and all columns of one
 * AIR are built by one evaluation-and-scan pass over the resident natural-order trace.
 */
#ifndef MINISTARK_EXTENSION_H
#define MINISTARK_EXTENSION_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Builds ncolumns extension columns over the trace domain of size 2^log_n (log_n <= 32, 1 <= ncolumns <= 8).
 * program: an evaluator program of nprog 4-word instructions (ministark_b200/expr.py::compile_extension_program, bound)
 * whose OP_STORE s stores slot s: slot 2k is mul_k, slot 2k + 1 is add_k, evaluated at row i with X = g_n^i,
 * Trace(col, off) = column[(i + off) mod 2^log_n] and periodic tables over <g_n>; a zero inverse is 0.  consts: nconsts
 * Fq3 constants.  col_ptrs / col_is_fq: ncols device columns (natural order), col_is_fq[i] != 0 for a column of fq_field
 * elements.  init: ncolumns * fq_field canonical Montgomery words; inclusive[k] != 0: row i of column k holds x_(i+1),
 * else x_i.  out: device matrix of ncolumns columns of 2^log_n elements of fq_field (MS_FIELD_FP or MS_FIELD_FQ3), column
 * k at out + k * 2^log_n * fq_field words. */
int ms_extension_columns(ms_ctx *ctx, const uint32_t *program, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                         const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, int fq_field, unsigned log_n,
                         unsigned ncolumns, const uint64_t *init, const int *inclusive, void *out);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_EXTENSION_H */
