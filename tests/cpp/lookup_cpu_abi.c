/*
 * lookup_cpu_abi.c — CPU build of the lookup multiplicity fill (include/ministark_lookup.h).  TEST INFRASTRUCTURE ONLY,
 * compiled by tests/test_lookup_cpu.py into a temporary directory.
 *
 * The CPU build of the declared extension columns (tests/cpp/extension_cpu_abi.c) is extended by both lookup entry points,
 * so that `GpuProver` and `ShardedProver` run AIRs with lookups on the CPU harness (tests/cpu_device.py).  The program is
 * interpreted row by row into the workspace's slot columns as canonical words, the table's (tuple, row) records are
 * sorted with qsort, and every looked-up tuple is found with bsearch, then walked back to the first record of its run
 * (the lowest row of that tuple).  The product never loads this library.
 */
#include "extension_cpu_abi.c"
#include "../../include/ministark_lookup.h"

#define LK_MAX_WIDTH 4
#define LK_MAX_TUPLES 4
#define LK_MAX_LOG 30

static size_t lk_align(size_t b) { return (b + 255) & ~(size_t)255; }

/* the layout of csrc/lookup.cu: slots, sorted table, two key buffers, two permutations, status */
static size_t lk_bytes(unsigned log_n, unsigned W, unsigned Q) {
    const size_t n = (size_t)1 << log_n, S = (size_t)W + (size_t)Q * (W + 1);
    return lk_align(S * n * 8) + lk_align((size_t)W * n * 8) + lk_align(2 * n * 8) + lk_align(2 * n * 4) +
           lk_align((2 * LK_MAX_TUPLES + 2) * 8);
}

int ms_lookup_workspace_bytes(unsigned log_n, unsigned width, unsigned ntuples, size_t *bytes) {
    if (!bytes || log_n > LK_MAX_LOG || width < 1 || width > LK_MAX_WIDTH || ntuples < 1 || ntuples > LK_MAX_TUPLES)
        return MS_ERR_INVALID;
    *bytes = lk_bytes(log_n, width, ntuples);
    return MS_OK;
}

typedef struct {
    u64 w[LK_MAX_WIDTH];
    u64 row;
} lk_rec;

static unsigned lk_width;

static int lk_cmp_tuple(const void *a, const void *b) {
    const lk_rec *x = (const lk_rec *)a, *y = (const lk_rec *)b;
    for (unsigned k = 0; k < lk_width; k++)
        if (x->w[k] != y->w[k]) return x->w[k] < y->w[k] ? -1 : 1;
    return 0;
}

static int lk_cmp_rec(const void *a, const void *b) {
    const int t = lk_cmp_tuple(a, b);
    if (t) return t;
    const lk_rec *x = (const lk_rec *)a, *y = (const lk_rec *)b;
    return x->row < y->row ? -1 : x->row > y->row;
}

int ms_lookup_multiplicities(ms_ctx *c, const uint32_t *prog, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                             const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, unsigned log_n, unsigned width,
                             unsigned ntuples, void *workspace, size_t workspace_bytes, void *out, uint64_t *status) {
    if (!c || !prog || !consts || nprog == 0 || (ncols && (!col_ptrs || !col_is_fq)) || !workspace || !out || !status)
        return MS_ERR_INVALID;
    if (log_n > LK_MAX_LOG) return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: domain too large (at most 2^%u rows)", LK_MAX_LOG);
    if (width < 1 || width > LK_MAX_WIDTH)
        return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: tuples of %u words (1 to %u)", width, LK_MAX_WIDTH);
    if (ntuples < 1 || ntuples > LK_MAX_TUPLES)
        return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: %u value tuples (1 to %u)", ntuples, LK_MAX_TUPLES);
    const size_t need = lk_bytes(log_n, width, ntuples);
    if (workspace_bytes < need)
        return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: workspace of %zu bytes, %zu needed", workspace_bytes, need);
    const unsigned nout = width + ntuples * (width + 1);
    {
        char defined[CK_REGS] = {0}, stored[LK_MAX_WIDTH + LK_MAX_TUPLES * (LK_MAX_WIDTH + 1)] = {0};
        for (unsigned k = 0; k < ncols; k++) {
            if (!col_ptrs[k]) return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: column %u is not a device pointer", k);
            if (col_is_fq[k]) return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: column %u is not a base-field column", k);
        }
        for (unsigned k = 0; k < nprog; k++) {
            const uint32_t *ins = prog + 4 * k, op = ins[0] & 0xff;
            if (op > CK_PERIODIC || ins[1] >= CK_REGS) return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: bad instruction %u", k);
            if (op == CK_CONST && ins[2] >= nconsts) return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: constant index out of range");
            if (op == CK_TRACE || op == CK_PERIODIC) {
                if (ins[2] >= ncols) return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: column %u out of range", ins[2]);
                if ((ins[0] >> 8) & 1) return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: column %u has the wrong field", ins[2]);
                if (op == CK_PERIODIC && ins[3] > log_n) return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: periodic table longer than the domain");
            }
            if (op == CK_STORE && ins[1] >= nout)
                return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: instruction %u stores to slot %u of %u", k, ins[1], nout);
            if (op == CK_STORE && ((ins[0] >> 8) & 1))
                return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: instruction %u stores an extension-field value", k);
            const int unary = op == CK_NEG || op == CK_INV || op == CK_POW || op == CK_STORE, binary = op == CK_ADD || op == CK_SUB || op == CK_MUL;
            if ((unary || binary) && (ins[2] >= CK_REGS || !defined[ins[2]]))
                return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: instruction %u reads register %u before it is written", k, ins[2]);
            if (binary && (ins[3] >= CK_REGS || !defined[ins[3]]))
                return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: instruction %u reads register %u before it is written", k, ins[3]);
            if (op == CK_STORE) stored[ins[1]] = 1;
            else defined[ins[1]] = 1;
        }
        for (unsigned s = 0; s < nout; s++)
            if (!stored[s]) return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: program never stores slot %u of %u", s, nout);
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
    lk_rec *table = (lk_rec *)malloc(n * sizeof(lk_rec));
    if (!table) return fail(c, MS_ERR_NOMEM, "ms_lookup_multiplicities: out of host memory");
    for (size_t j = 0; j < n; j++) {
        memset(table[j].w, 0, sizeof table[j].w);
        for (unsigned k = 0; k < width; k++) table[j].w[k] = slots[(size_t)k * n + j];
        table[j].row = j;
    }
    lk_width = width;
    qsort(table, n, sizeof(lk_rec), lk_cmp_rec);
    u64 *counts = (u64 *)out;
    memset(counts, 0, n * 8);
    for (unsigned k = 0; k <= ntuples; k++) {
        status[2 * k] = 0;
        status[2 * k + 1] = ~0ull;
    }
    for (unsigned q = 0; q < ntuples; q++) {
        const size_t base = width + (size_t)q * (width + 1);
        for (size_t i = 0; i < n; i++) {
            const u64 sel = slots[base * n + i];
            if (sel == 0) continue;
            if (sel != 1) {
                status[2 * ntuples]++;
                if (i < status[2 * ntuples + 1]) status[2 * ntuples + 1] = i;
                continue;
            }
            lk_rec key;
            memset(&key, 0, sizeof key);
            for (unsigned k = 0; k < width; k++) key.w[k] = slots[(base + 1 + k) * n + i];
            const lk_rec *hit = (const lk_rec *)bsearch(&key, table, n, sizeof(lk_rec), lk_cmp_tuple);
            if (!hit) {
                status[2 * q]++;
                if (i < status[2 * q + 1]) status[2 * q + 1] = i;
                continue;
            }
            while (hit > table && lk_cmp_tuple(hit - 1, &key) == 0) hit--;
            counts[hit->row]++;
        }
    }
    free(table);
    for (size_t j = 0; j < n; j++) counts[j] = fp_from_canon(counts[j]);
    return done(c, "ms_lookup_multiplicities", t0);
}
