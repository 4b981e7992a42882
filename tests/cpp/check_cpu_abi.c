/*
 * check_cpu_abi.c — CPU build of the constraint check (include/ministark_check.h).  TEST INFRASTRUCTURE ONLY, compiled by
 * tests/test_validate_cpu.py into a temporary directory.
 *
 * The CPU build of the streamed-residency entry points (tests/cpp/stream_cpu_abi.c, itself the oracle's CPU ABI plus
 * include/ministark_stream.h) is extended by ms_check_constraints, so that both residencies of `GpuProver` run with
 * validate=True on the CPU harness (tests/cpu_device.py).  The checked program is interpreted row by row with a None
 * flag per register, as csrc/check.cu does it.  The product never loads this library.
 */
#include "stream_cpu_abi.c"
#include "../../include/ministark_check.h"

enum { CK_X = 0, CK_CONST, CK_TRACE, CK_NEG, CK_ADD, CK_SUB, CK_MUL, CK_INV, CK_POW, CK_STORE, CK_PERIODIC, CK_DIV, CK_CHECK };
#define CK_REGS 48

static int ck_zero(fq3 v, int q) { return q ? !(v.c[0] | v.c[1] | v.c[2]) : !v.c[0]; }

int ms_check_constraints(ms_ctx *c, const uint32_t *prog, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                         const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, int fq_field, unsigned log_n,
                         unsigned nconstraints, uint64_t *first_row, uint64_t *fail_count) {
    if (!c || !prog || !consts || nprog == 0 || (ncols && (!col_ptrs || !col_is_fq)) || !first_row || !fail_count)
        return MS_ERR_INVALID;
    if (bad_field(fq_field)) return fail(c, MS_ERR_INVALID, "ms_check_constraints: bad Fq field id");
    if (log_n > 32) return fail(c, MS_ERR_INVALID, "ms_check_constraints: domain too large");
    if (nconstraints == 0) return fail(c, MS_ERR_INVALID, "ms_check_constraints: no constraints");
    {
        char defined[CK_REGS] = {0};
        for (unsigned k = 0; k < nprog; k++) {
            const uint32_t *ins = prog + 4 * k, op = ins[0] & 0xff;
            if (op > CK_CHECK || ins[1] >= CK_REGS) return fail(c, MS_ERR_INVALID, "ms_check_constraints: bad instruction %u", k);
            if (op == CK_STORE || op == CK_INV)
                return fail(c, MS_ERR_INVALID, "ms_check_constraints: instruction %u: %s has no place in a checked program", k,
                            op == CK_STORE ? "STORE" : "INV");
            if (op == CK_CONST && ins[2] >= nconsts) return fail(c, MS_ERR_INVALID, "ms_check_constraints: constant index out of range");
            if (op == CK_TRACE || op == CK_PERIODIC) {
                if (ins[2] >= ncols) return fail(c, MS_ERR_INVALID, "ms_check_constraints: column %u out of range", ins[2]);
                if (!col_ptrs[ins[2]]) return fail(c, MS_ERR_INVALID, "ms_check_constraints: column %u is NULL", ins[2]);
                if ((col_is_fq[ins[2]] ? 1 : 0) != (int)((ins[0] >> 8) & 1))
                    return fail(c, MS_ERR_INVALID, "ms_check_constraints: column %u has the wrong field", ins[2]);
                if (op == CK_PERIODIC && ins[3] > log_n) return fail(c, MS_ERR_INVALID, "ms_check_constraints: periodic table longer than the domain");
            }
            if (op == CK_CHECK && ins[3] >= nconstraints)
                return fail(c, MS_ERR_INVALID, "ms_check_constraints: instruction %u checks constraint %u of %u", k, ins[3], nconstraints);
            const int unary = op == CK_NEG || op == CK_POW || op == CK_CHECK, binary = op == CK_ADD || op == CK_SUB || op == CK_MUL || op == CK_DIV;
            if ((unary || binary) && (ins[2] >= CK_REGS || !defined[ins[2]]))
                return fail(c, MS_ERR_INVALID, "ms_check_constraints: instruction %u reads register %u before it is written", k, ins[2]);
            if (binary && (ins[3] >= CK_REGS || !defined[ins[3]]))
                return fail(c, MS_ERR_INVALID, "ms_check_constraints: instruction %u reads register %u before it is written", k, ins[3]);
            if (op != CK_CHECK) defined[ins[1]] = 1;
        }
    }
    const double t0 = now_s();
    const size_t n = (size_t)1 << log_n;
    const int fq3m = fq_field == 3;
    const u64 g = orc_root_of_unity(log_n);
    for (unsigned k = 0; k < nconstraints; k++) { first_row[k] = UINT64_MAX; fail_count[k] = 0; }
    fq3 r[CK_REGS];
    int none[CK_REGS];
    u64 x = GL_ONE;                                  /* g^i */
    for (size_t i = 0; i < n; i++, x = fp_mul(x, g)) {
        for (unsigned pc = 0; pc < nprog; pc++) {
            const uint32_t *ins = prog + 4 * pc, op = ins[0] & 0xff, d = ins[1], a = ins[2], b = ins[3];
            const int qa = ((ins[0] >> 8) & 1) && fq3m, qb = ((ins[0] >> 9) & 1) && fq3m;
            fq3 v = fq3_zero();
            int vn = 0;
            switch (op) {
            case CK_X: v.c[0] = x; break;
            case CK_CONST: v.c[0] = consts[3 * (size_t)a]; if (qa) { v.c[1] = consts[3 * (size_t)a + 1]; v.c[2] = consts[3 * (size_t)a + 2]; } break;
            case CK_TRACE:
            case CK_PERIODIC: {
                const size_t pos = op == CK_TRACE ? (i + b) & (n - 1) : i & (((size_t)1 << b) - 1);
                const u64 *col = (const u64 *)col_ptrs[a];
                if ((ins[0] >> 8) & 1) memcpy(v.c, col + pos * fq_field, 8 * (size_t)fq_field);
                else v.c[0] = col[pos];
                break;
            }
            case CK_NEG: vn = none[a]; v = fq3_sub(fq3_zero(), qa ? r[a] : fq3_from_fp(r[a].c[0])); break;
            case CK_ADD:
            case CK_SUB: {
                const fq3 x_ = qa ? r[a] : fq3_from_fp(r[a].c[0]), y = qb ? r[b] : fq3_from_fp(r[b].c[0]);
                vn = none[a] || none[b];
                v = op == CK_ADD ? fq3_add(x_, y) : fq3_sub(x_, y);
                break;
            }
            case CK_MUL:
            case CK_DIV: {
                const fq3 x_ = qa ? r[a] : fq3_from_fp(r[a].c[0]), y = qb ? r[b] : fq3_from_fp(r[b].c[0]);
                const int za = ck_zero(x_, 1), zb = ck_zero(y, 1);
                if (none[a] && none[b]) vn = 1;
                else if (none[a]) vn = !zb;
                else if (none[b]) vn = !za;
                else if (op == CK_MUL) v = fq3_mul(x_, y);
                else if (zb) vn = !za;
                else v = fq3_mul(x_, qb ? fq3_inv(y) : fq3_from_fp(fp_inv(y.c[0])));
                break;
            }
            case CK_POW: vn = none[a]; v = qa ? fq3_pow(r[a], b) : fq3_from_fp(fp_pow(r[a].c[0], b)); break;
            case CK_CHECK:
                if (none[a]) {
                    if (!fail_count[b]++) first_row[b] = i;
                }
                continue;
            default: continue;
            }
            r[d] = v;
            none[d] = vn;
        }
    }
    return done(c, "ms_check_constraints", t0);
}
