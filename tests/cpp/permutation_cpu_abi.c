/*
 * permutation_cpu_abi.c — CPU build of the permutation target fill (include/ministark_permutation.h).  TEST
 * INFRASTRUCTURE ONLY, compiled by tests/test_permutation_cpu.py into a temporary directory.
 *
 * The CPU build of the lookup fill (tests/cpp/lookup_cpu_abi.c) is extended by both permutation entry points, so that
 * `GpuProver` and `ShardedProver` run AIRs with permutations (and lookups) on the CPU harness (tests/cpu_device.py).  The
 * program is interpreted row by row into the workspace's slot columns as canonical words, the (tuple, row) records are
 * sorted with qsort, ties broken by row (a stable sort), and written to the targets as Montgomery words.  The product
 * never loads this library.
 */
#include "lookup_cpu_abi.c"
#include "../../include/ministark_permutation.h"

#define PM_MAX_WIDTH 4
#define PM_MAX_LOG 30

/* the layout of csrc/permutation.cu: slots, two key buffers, two permutations */
static size_t pm_bytes(unsigned log_n, unsigned W) {
    const size_t n = (size_t)1 << log_n;
    return lk_align((size_t)W * n * 8) + lk_align(2 * n * 8) + lk_align(2 * n * 4);
}

int ms_permutation_workspace_bytes(unsigned log_n, unsigned width, size_t *bytes) {
    if (!bytes || log_n > PM_MAX_LOG || width < 1 || width > PM_MAX_WIDTH) return MS_ERR_INVALID;
    *bytes = pm_bytes(log_n, width);
    return MS_OK;
}

int ms_permutation_fill(ms_ctx *c, const uint32_t *prog, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                        const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, unsigned log_n, unsigned width,
                        void *const *targets, void *workspace, size_t workspace_bytes) {
    if (!c || !prog || !consts || nprog == 0 || (ncols && (!col_ptrs || !col_is_fq)) || !targets || !workspace)
        return MS_ERR_INVALID;
    if (log_n > PM_MAX_LOG) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: domain too large (at most 2^%u rows)", PM_MAX_LOG);
    if (width < 1 || width > PM_MAX_WIDTH)
        return fail(c, MS_ERR_INVALID, "ms_permutation_fill: tuples of %u words (1 to %u)", width, PM_MAX_WIDTH);
    const size_t need = pm_bytes(log_n, width);
    if (workspace_bytes < need)
        return fail(c, MS_ERR_INVALID, "ms_permutation_fill: workspace of %zu bytes, %zu needed", workspace_bytes, need);
    for (unsigned k = 0; k < width; k++) {
        if (!targets[k]) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: target %u is not a device pointer", k);
        for (unsigned j = 0; j < k; j++)
            if (targets[j] == targets[k]) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: targets %u and %u are the same column", j, k);
    }
    {
        char defined[CK_REGS] = {0}, stored[PM_MAX_WIDTH] = {0};
        for (unsigned k = 0; k < ncols; k++) {
            if (!col_ptrs[k]) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: column %u is not a device pointer", k);
            if (col_is_fq[k]) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: column %u is not a base-field column", k);
        }
        for (unsigned k = 0; k < nprog; k++) {
            const uint32_t *ins = prog + 4 * k, op = ins[0] & 0xff;
            if (op > CK_PERIODIC || ins[1] >= CK_REGS) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: bad instruction %u", k);
            if (op == CK_CONST && ins[2] >= nconsts) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: constant index out of range");
            if (op == CK_TRACE || op == CK_PERIODIC) {
                if (ins[2] >= ncols) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: column %u out of range", ins[2]);
                if ((ins[0] >> 8) & 1) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: column %u has the wrong field", ins[2]);
                if (op == CK_PERIODIC && ins[3] > log_n) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: periodic table longer than the domain");
            }
            if (op == CK_STORE && ins[1] >= width)
                return fail(c, MS_ERR_INVALID, "ms_permutation_fill: instruction %u stores to slot %u of %u", k, ins[1], width);
            if (op == CK_STORE && ((ins[0] >> 8) & 1))
                return fail(c, MS_ERR_INVALID, "ms_permutation_fill: instruction %u stores an extension-field value", k);
            const int unary = op == CK_NEG || op == CK_INV || op == CK_POW || op == CK_STORE, binary = op == CK_ADD || op == CK_SUB || op == CK_MUL;
            if ((unary || binary) && (ins[2] >= CK_REGS || !defined[ins[2]]))
                return fail(c, MS_ERR_INVALID, "ms_permutation_fill: instruction %u reads register %u before it is written", k, ins[2]);
            if (binary && (ins[3] >= CK_REGS || !defined[ins[3]]))
                return fail(c, MS_ERR_INVALID, "ms_permutation_fill: instruction %u reads register %u before it is written", k, ins[3]);
            if (op == CK_STORE) stored[ins[1]] = 1;
            else defined[ins[1]] = 1;
        }
        for (unsigned s = 0; s < width; s++)
            if (!stored[s]) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: program never stores slot %u of %u", s, width);
    }
    const double t0 = now_s();
    const size_t n = (size_t)1 << log_n;
    const u64 g = orc_root_of_unity(log_n);
    u64 *slots = (u64 *)workspace, r[CK_REGS];
    u64 xi = GL_ONE;                                 /* g^i */
    for (size_t i = 0; i < n; i++, xi = fp_mul(xi, g)) {
        for (unsigned pc = 0; pc < nprog; pc++) {
            const uint32_t *ins = prog + 4 * pc, op = ins[0] & 0xff, d = ins[1], a = ins[2], b = ins[3];
            u64 v = 0;
            switch (op) {
            case CK_X: v = xi; break;
            case CK_CONST: v = consts[3 * (size_t)a]; break;
            case CK_TRACE: v = ((const u64 *)col_ptrs[a])[(i + b) & (n - 1)]; break;
            case CK_PERIODIC: v = ((const u64 *)col_ptrs[a])[i & (((size_t)1 << b) - 1)]; break;
            case CK_NEG: v = fp_neg(r[a]); break;
            case CK_ADD: v = fp_add(r[a], r[b]); break;
            case CK_SUB: v = fp_sub(r[a], r[b]); break;
            case CK_MUL: v = fp_mul(r[a], r[b]); break;
            case CK_INV: v = fp_inv(r[a]); break;
            case CK_POW: v = fp_pow(r[a], b); break;
            case CK_STORE: slots[(size_t)d * n + i] = fp_to_canon(r[a]); continue;
            default: continue;
            }
            r[d] = v;
        }
    }
    lk_rec *rec = (lk_rec *)malloc(n * sizeof(lk_rec));
    if (!rec) return fail(c, MS_ERR_NOMEM, "ms_permutation_fill: out of host memory");
    for (size_t j = 0; j < n; j++) {
        memset(rec[j].w, 0, sizeof rec[j].w);
        for (unsigned k = 0; k < width; k++) rec[j].w[k] = slots[(size_t)k * n + j];
        rec[j].row = j;
    }
    lk_width = width;
    qsort(rec, n, sizeof(lk_rec), lk_cmp_rec);
    for (unsigned k = 0; k < width; k++) {
        u64 *t = (u64 *)targets[k];
        for (size_t j = 0; j < n; j++) t[j] = fp_from_canon(rec[j].w[k]);
    }
    free(rec);
    return done(c, "ms_permutation_fill", t0);
}
