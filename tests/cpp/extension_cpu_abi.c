/*
 * extension_cpu_abi.c — CPU build of the declared extension columns (include/ministark_extension.h).  TEST
 * INFRASTRUCTURE ONLY, compiled by tests/test_extension_cpu.py into a temporary directory.
 *
 * The CPU build of the constraint check (tests/cpp/check_cpu_abi.c, itself the oracle's CPU ABI plus the streamed
 * residency) is extended by ms_extension_columns, so that both residencies of `GpuProver` and the sharded prover run on
 * AIRs that declare their extension columns on the CPU harness (tests/cpu_device.py).  The program is interpreted row by
 * row with the evaluator's instruction set, then every column's recurrence runs serially.  The product never loads this
 * library.
 */
#include "check_cpu_abi.c"
#include "../../include/ministark_extension.h"

#define EXT_MAX_COLUMNS 8

int ms_extension_columns(ms_ctx *c, const uint32_t *prog, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                         const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, int fq_field, unsigned log_n,
                         unsigned ncolumns, const uint64_t *init, const int *inclusive, void *out) {
    if (!c || !prog || !consts || nprog == 0 || (ncols && (!col_ptrs || !col_is_fq)) || !init || !inclusive || !out)
        return MS_ERR_INVALID;
    if (bad_field(fq_field)) return fail(c, MS_ERR_INVALID, "ms_extension_columns: bad Fq field id");
    if (log_n > 32) return fail(c, MS_ERR_INVALID, "ms_extension_columns: domain too large");
    if (ncolumns == 0 || ncolumns > EXT_MAX_COLUMNS)
        return fail(c, MS_ERR_INVALID, "ms_extension_columns: %u columns (1 to %d)", ncolumns, EXT_MAX_COLUMNS);
    for (unsigned k = 0; k < ncolumns * (unsigned)fq_field; k++)
        if (init[k] >= GL_P) return fail(c, MS_ERR_INVALID, "ms_extension_columns: non-canonical init of column %u", k / fq_field);
    const unsigned nout = 2 * ncolumns;
    {
        char defined[CK_REGS] = {0}, stored[2 * EXT_MAX_COLUMNS] = {0};
        for (unsigned k = 0; k < nprog; k++) {
            const uint32_t *ins = prog + 4 * k, op = ins[0] & 0xff;
            if (op > CK_PERIODIC || ins[1] >= CK_REGS) return fail(c, MS_ERR_INVALID, "ms_extension_columns: bad instruction %u", k);
            if (op == CK_CONST && ins[2] >= nconsts) return fail(c, MS_ERR_INVALID, "ms_extension_columns: constant index out of range");
            if (op == CK_TRACE || op == CK_PERIODIC) {
                if (ins[2] >= ncols) return fail(c, MS_ERR_INVALID, "ms_extension_columns: column %u out of range", ins[2]);
                if (!col_ptrs[ins[2]]) return fail(c, MS_ERR_INVALID, "ms_extension_columns: column %u is not a device pointer", ins[2]);
                if ((col_is_fq[ins[2]] ? 1 : 0) != (int)((ins[0] >> 8) & 1))
                    return fail(c, MS_ERR_INVALID, "ms_extension_columns: column %u has the wrong field", ins[2]);
                if (op == CK_PERIODIC && ins[3] > log_n) return fail(c, MS_ERR_INVALID, "ms_extension_columns: periodic table longer than the domain");
            }
            if (op == CK_STORE && ins[1] >= nout)
                return fail(c, MS_ERR_INVALID, "ms_extension_columns: instruction %u stores to slot %u of %u", k, ins[1], nout);
            const int unary = op == CK_NEG || op == CK_INV || op == CK_POW || op == CK_STORE, binary = op == CK_ADD || op == CK_SUB || op == CK_MUL;
            if ((unary || binary) && (ins[2] >= CK_REGS || !defined[ins[2]]))
                return fail(c, MS_ERR_INVALID, "ms_extension_columns: instruction %u reads register %u before it is written", k, ins[2]);
            if (binary && (ins[3] >= CK_REGS || !defined[ins[3]]))
                return fail(c, MS_ERR_INVALID, "ms_extension_columns: instruction %u reads register %u before it is written", k, ins[3]);
            if (op == CK_STORE) stored[ins[1]] = 1;
            else defined[ins[1]] = 1;
        }
        for (unsigned s = 0; s < nout; s++)
            if (!stored[s]) return fail(c, MS_ERR_INVALID, "ms_extension_columns: program never stores slot %u of %u", s, nout);
    }
    const double t0 = now_s();
    const size_t n = (size_t)1 << log_n;
    const int fq3m = fq_field == 3;
    const u64 g = orc_root_of_unity(log_n);
    fq3 x[EXT_MAX_COLUMNS], slot[2 * EXT_MAX_COLUMNS], r[CK_REGS];
    for (unsigned k = 0; k < ncolumns; k++) {
        x[k] = fq3_zero();
        memcpy(x[k].c, init + (size_t)k * fq_field, 8 * (size_t)fq_field);
    }
    u64 *o = (u64 *)out;
    u64 xi = GL_ONE;                                 /* g^i */
    for (size_t i = 0; i < n; i++, xi = fp_mul(xi, g)) {
        for (unsigned pc = 0; pc < nprog; pc++) {
            const uint32_t *ins = prog + 4 * pc, op = ins[0] & 0xff, d = ins[1], a = ins[2], b = ins[3];
            const int qa = ((ins[0] >> 8) & 1) && fq3m;
            fq3 v = fq3_zero();
            switch (op) {
            case CK_X: v.c[0] = xi; break;
            case CK_CONST: v.c[0] = consts[3 * (size_t)a]; if (qa) { v.c[1] = consts[3 * (size_t)a + 1]; v.c[2] = consts[3 * (size_t)a + 2]; } break;
            case CK_TRACE:
            case CK_PERIODIC: {
                const size_t pos = op == CK_TRACE ? (i + b) & (n - 1) : i & (((size_t)1 << b) - 1);
                const u64 *col = (const u64 *)col_ptrs[a];
                if ((ins[0] >> 8) & 1) memcpy(v.c, col + pos * fq_field, 8 * (size_t)fq_field);
                else v.c[0] = col[pos];
                break;
            }
            /* registers of Fp type hold zero upper words, so the Fq3 operations give the evaluator's values */
            case CK_NEG: v = fq3_sub(fq3_zero(), r[a]); break;
            case CK_ADD: v = fq3_add(r[a], r[b]); break;
            case CK_SUB: v = fq3_sub(r[a], r[b]); break;
            case CK_MUL: v = fq3_mul(r[a], r[b]); break;
            case CK_INV: v = qa ? fq3_inv(r[a]) : fq3_from_fp(fp_inv(r[a].c[0])); break;
            case CK_POW: v = qa ? fq3_pow(r[a], b) : fq3_from_fp(fp_pow(r[a].c[0], b)); break;
            case CK_STORE: slot[d] = qa ? r[a] : fq3_from_fp(r[a].c[0]); continue;
            default: continue;
            }
            r[d] = v;
        }
        for (unsigned k = 0; k < ncolumns; k++) {
            u64 *dst = o + ((size_t)k * n + i) * fq_field;
            if (!inclusive[k]) memcpy(dst, x[k].c, 8 * (size_t)fq_field);
            x[k] = fq3_add(fq3_mul(x[k], slot[2 * k]), slot[2 * k + 1]);
            if (inclusive[k]) memcpy(dst, x[k].c, 8 * (size_t)fq_field);
        }
    }
    return done(c, "ms_extension_columns", t0);
}
