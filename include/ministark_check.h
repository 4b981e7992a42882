/*
 * ministark_check.h — the constraint check of libministark_b200.so: does a trace satisfy its AIR, and where not?
 * Conventions as in ministark_b200.h (Montgomery words, 0 on success, a negative MS_ERR_* otherwise).
 *
 * The reference calls Stark::validate_constraints in debug builds right after the extension trace commitment
 * (src/prover.rs:74-75, src/stark.rs:65-75) and leaves its body (src/debug.rs) unfinished; this is that body's
 * data-parallel part.
 */
#ifndef MINISTARK_CHECK_H
#define MINISTARK_CHECK_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Constraint::check (src/constraints.rs:168-249) of constraints 0..nconstraints-1 at every row of the trace domain of size
 * 2^log_n; columns are natural-order trace columns (device pointers).  first_row / fail_count: host arrays of nconstraints.
 * program: a checked program (ministark_b200/expr.py::compile_check_program) of nprog 4-word instructions; consts: nconsts
 * Fq3 constants; col_is_fq[i] != 0 marks a column of fq_field (MS_FIELD_FP or MS_FIELD_FQ3) elements, 0 a base-field
 * column.  Constraint k fails at row i where its value is None: first_row[k] receives the lowest such row (UINT64_MAX if
 * none) and fail_count[k] the number of such rows. */
int ms_check_constraints(ms_ctx *ctx, const uint32_t *program, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                         const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, int fq_field, unsigned log_n,
                         unsigned nconstraints, uint64_t *first_row, uint64_t *fail_count);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_CHECK_H */
