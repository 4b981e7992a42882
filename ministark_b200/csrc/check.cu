// check.cu — Constraint::check (src/constraints.rs:168-249) of every constraint at every row of the trace domain.
//
// The reference's debug builds call Stark::validate_constraints right after the extension trace commitment
// (src/prover.rs:74-75, src/stark.rs:65-75); its body (src/debug.rs) is left as a comment: evaluate each constraint at
// each row with Option-valued arithmetic, where a division by zero with a non-zero numerator gives None, and report
// the first row where a constraint is None.  On the host that is rows x DAG nodes, ~10^10 node evaluations for the
// brainfuck AIR at 2^24 rows; here it is one pass over the resident natural-order trace.
//
// The program is a checked program from expr.compile_check_program (all constraints, shared subexpressions once).  One
// thread evaluates it at one row i, natural order; beside its register file a 64-bit mask marks the registers that
// hold None.  Leaves: X = g_n^i (no coset offset), Trace(col, off) = column[(i + off) mod n], constants and bound
// challenges / hints from the pool, periodic columns from tables over <g_n> (offset 1).  Operations follow
// src/constraints.rs:181-246 exactly; "zero" is all three coordinates for an Fq3 value.  OP_CHECK k, r: a ballot over
// the warp of "register r is None", then one atomicAdd to the failure count and one atomicMin to the first failing row
// per warp that has a failure.  Every thread runs the same program, so control flow at the ballot is uniform; threads
// past the end of a domain smaller than a warp evaluate row 0 and vote false.
//
// Its own kernel, not a mode of eval_kernel: the composition evaluator (and its run-time specialised twin, eval_jit.cu)
// stays free of the None bookkeeping.
#include "eval.cuh"
#include "../../include/ministark_check.h"

#include <vector>

namespace ms {

using gl::Fq3;

struct CheckParams {
    const uint4 *prog;
    u32 nprog;
    const u64 *consts;          // [k][3] Montgomery words
    const u64 *const *col_ptr;  // natural-order trace columns, then periodic tables
    u32 fq_words;               // 1: Fq = Fp, 3: Fq = Fq3
    u32 log_n;
    const u64 *tw_lo, *tw_hi;   // g_n^e two-level table
    u32 hi_len;
    unsigned long long *first_row, *fail_count;   // per constraint
};

__device__ __forceinline__ bool ck_zero(const u64 *v, bool q) { return q ? (v[0] | v[1] | v[2]) == 0 : v[0] == 0; }

__global__ void __launch_bounds__(128) check_kernel(const CheckParams p) {
    const u64 n = 1ull << p.log_n;
    const u64 t = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    const bool live = t < n;
    const u64 i = live ? t : 0;
    const unsigned lane = threadIdx.x & 31;
    const bool fq3 = p.fq_words == 3;
    u64 r[kMaxRegs][3];
    u64 none = 0;                                   // bit d: register d holds None

    for (u32 pc = 0; pc < p.nprog; pc++) {
        const uint4 ins = __ldg(p.prog + pc);
        const u32 op = ins.x & 0xff;
        const bool qa = ((ins.x >> 8) & 1) && fq3, qb = ((ins.x >> 9) & 1) && fq3;
        const u32 d = ins.y;
        const bool na = (none >> (ins.z & 63)) & 1, nb = (none >> (ins.w & 63)) & 1;
        u64 v0 = 0, v1 = 0, v2 = 0;                 // the result, written to r[d] after the operands are read
        bool vn = false;                            // the result is None
        switch (op) {
            case OP_X: {
                v0 = p.tw_lo[i & 4095];
                if (p.hi_len > 1) v0 = gl::mul(p.tw_hi[i >> 12], v0);
                break;
            }
            case OP_CONST: {
                const u64 *k = p.consts + 3 * (u64)ins.z;
                v0 = k[0];
                if (qa) { v1 = k[1]; v2 = k[2]; }
                break;
            }
            case OP_TRACE:
            case OP_PERIODIC: {
                const u64 pos = op == OP_TRACE ? (i + (u64)ins.w) & (n - 1) : i & ((1ull << ins.w) - 1);
                const u64 *col = p.col_ptr[ins.z];
                if ((ins.x >> 8) & 1) {
                    const u64 *c = col + pos * p.fq_words;
                    v0 = c[0];
                    if (fq3) { v1 = c[1]; v2 = c[2]; }
                } else {
                    v0 = col[pos];
                }
                break;
            }
            case OP_NEG: {
                vn = na;
                v0 = gl::neg(r[ins.z][0]);
                if (qa) { v1 = gl::neg(r[ins.z][1]); v2 = gl::neg(r[ins.z][2]); }
                break;
            }
            case OP_ADD:
            case OP_SUB: {
                vn = na || nb;
                const u64 a1 = qa ? r[ins.z][1] : 0, a2 = qa ? r[ins.z][2] : 0;
                const u64 b1 = qb ? r[ins.w][1] : 0, b2 = qb ? r[ins.w][2] : 0;
                if (op == OP_ADD) {
                    v0 = gl::add(r[ins.z][0], r[ins.w][0]); v1 = gl::add(a1, b1); v2 = gl::add(a2, b2);
                } else {
                    v0 = gl::sub(r[ins.z][0], r[ins.w][0]); v1 = gl::sub(a1, b1); v2 = gl::sub(a2, b2);
                }
                break;
            }
            case OP_MUL:
            case OP_DIV: {
                const bool za = ck_zero(r[ins.z], qa), zb = ck_zero(r[ins.w], qb);
                if (na || nb) {
                    // Some(x) * None, None * Some(x), Some(x) / None, None / Some(x): Some(0) if x = 0; None / None: None
                    vn = !(na != nb && (na ? zb : za));
                } else if (op == OP_DIV && zb) {
                    vn = !za;                       // 0 / 0 = Some(0), a / 0 = None
                } else {
                    const Fq3 A{r[ins.z][0], qa ? r[ins.z][1] : 0, qa ? r[ins.z][2] : 0};
                    Fq3 c;
                    if (op == OP_MUL) {
                        if (qa && qb) c = gl::mul(A, Fq3{r[ins.w][0], r[ins.w][1], r[ins.w][2]});
                        else if (qb) c = gl::mul(Fq3{r[ins.w][0], r[ins.w][1], r[ins.w][2]}, A.c0);
                        else c = qa ? gl::mul(A, r[ins.w][0]) : gl::fq3(gl::mul(A.c0, r[ins.w][0]));
                    } else if (qb) {
                        const Fq3 ib = gl::inv(Fq3{r[ins.w][0], r[ins.w][1], r[ins.w][2]});
                        c = qa ? gl::mul(A, ib) : gl::mul(ib, A.c0);
                    } else {
                        const u64 ib = gl::inv(r[ins.w][0]);
                        c = qa ? gl::mul(A, ib) : gl::fq3(gl::mul(A.c0, ib));
                    }
                    v0 = c.c0; v1 = c.c1; v2 = c.c2;
                }
                break;
            }
            case OP_POW: {
                vn = na;
                if (qa) {
                    const Fq3 c = gl::pow(Fq3{r[ins.z][0], r[ins.z][1], r[ins.z][2]}, (u64)ins.w);
                    v0 = c.c0; v1 = c.c1; v2 = c.c2;
                } else {
                    v0 = gl::pow(r[ins.z][0], (u64)ins.w);
                }
                break;
            }
            case OP_CHECK: {
                const unsigned m = __ballot_sync(0xffffffffu, live && na);
                if (m && lane == 0) {
                    atomicAdd(p.fail_count + ins.w, (unsigned long long)__popc(m));
                    atomicMin(p.first_row + ins.w, (unsigned long long)(t - lane + (unsigned)(__ffs(m) - 1)));
                }
                continue;                           // writes no register
            }
            default: continue;
        }
        r[d][0] = v0; r[d][1] = v1; r[d][2] = v2;
        none = vn ? (none | (1ull << d)) : (none & ~(1ull << d));
    }
}

}  // namespace ms

using namespace ms;

extern "C" int ms_check_constraints(ms_ctx *c, const uint32_t *program, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                                    const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, int fq_field, unsigned log_n,
                                    unsigned nconstraints, uint64_t *first_row, uint64_t *fail_count) {
    if (!c || !program || !consts || nprog == 0 || (ncols && (!col_ptrs || !col_is_fq)) || !first_row || !fail_count)
        return MS_ERR_INVALID;
    if (fq_field != MS_FIELD_FP && fq_field != MS_FIELD_FQ3) return fail(c, MS_ERR_INVALID, "ms_check_constraints: bad Fq field id");
    if (log_n > 32) return fail(c, MS_ERR_INVALID, "ms_check_constraints: domain too large");
    if (nconstraints == 0) return fail(c, MS_ERR_INVALID, "ms_check_constraints: no constraints");
    cudaSetDevice(c->device);
    std::vector<const u64 *> cols;
    std::vector<int> isq;
    for (unsigned k = 0; k < ncols; k++) {
        if (!col_ptrs[k] || !is_device_ptr(col_ptrs[k])) return fail(c, MS_ERR_INVALID, "ms_check_constraints: column %u is not a device pointer", k);
        cols.push_back((const u64 *)col_ptrs[k]);
        isq.push_back(col_is_fq[k] ? 1 : 0);
    }
    int rc = validate_program(c, "ms_check_constraints", program, nprog, nconsts, isq, log_n, nconstraints);
    if (rc) return rc;
    // program, constants, column table and the two result arrays: one scratch block
    void *meta;
    const size_t prog_bytes = (size_t)nprog * 16, const_bytes = (size_t)nconsts * 24, ptr_bytes = (size_t)ncols * 8;
    const size_t res_bytes = (size_t)nconstraints * 8, res_off = (prog_bytes + const_bytes + ptr_bytes + 15) & ~(size_t)15;
    if ((rc = scratch_get(c, 3, res_off + 2 * res_bytes + 64, &meta))) return rc;
    char *m = (char *)meta;
    MS_CUDA(c, cudaMemcpyAsync(m, program, prog_bytes, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaMemcpyAsync(m + prog_bytes, consts, const_bytes, cudaMemcpyDefault, c->stream));
    if (ptr_bytes) MS_CUDA(c, cudaMemcpyAsync(m + prog_bytes + const_bytes, cols.data(), ptr_bytes, cudaMemcpyHostToDevice, c->stream));
    MS_CUDA(c, cudaMemsetAsync(m + res_off, 0xff, res_bytes, c->stream));             // first row: UINT64_MAX
    MS_CUDA(c, cudaMemsetAsync(m + res_off + res_bytes, 0, res_bytes, c->stream));    // failure count: 0
    const u64 *tw_lo, *tw_hi;
    u32 hi_len;
    if ((rc = ntt_plan_tables(c, log_n, &tw_lo, &tw_hi, &hi_len))) return rc;
    CheckParams p;
    p.prog = (const uint4 *)m;
    p.nprog = nprog;
    p.consts = (const u64 *)(m + prog_bytes);
    p.col_ptr = (const u64 *const *)(m + prog_bytes + const_bytes);
    p.fq_words = (u32)fq_field;
    p.log_n = log_n;
    p.tw_lo = tw_lo;
    p.tw_hi = tw_hi;
    p.hi_len = hi_len;
    p.first_row = (unsigned long long *)(m + res_off);
    p.fail_count = (unsigned long long *)(m + res_off + res_bytes);
    const size_t n = (size_t)1 << log_n;
    check_kernel<<<(unsigned)((n + 127) / 128), 128, 0, c->stream>>>(p);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    MS_CUDA(c, cudaMemcpyAsync(first_row, m + res_off, res_bytes, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaMemcpyAsync(fail_count, m + res_off + res_bytes, res_bytes, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));   // the results are host arrays the caller reads next
    return MS_OK;
}
