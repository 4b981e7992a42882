// eval.cuh — the instruction set of the flattened constraint programs (ministark_b200/expr.py) and their validation,
// shared by the fused evaluator (eval.cu, ms_eval_constraints*) and the constraint check (check.cu,
// ms_check_constraints).  Instruction words: [op | a_is_fq << 8 | b_is_fq << 9, dst, a, b].
#pragma once
#include "ctx.cuh"

namespace ms {

// OP_DIV and OP_CHECK belong to checked programs only; the evaluator rejects them, the check rejects OP_INV and OP_STORE
enum { OP_X = 0, OP_CONST, OP_TRACE, OP_NEG, OP_ADD, OP_SUB, OP_MUL, OP_INV, OP_POW, OP_STORE, OP_PERIODIC, OP_DIV, OP_CHECK };
constexpr int kMaxRegs = 48;

// validates a program against the register file, the constant pool and the column table: every source register must
// have been written by an earlier instruction.  nconstraints == 0: an evaluator program whose OP_STORE s needs
// s < nout, every slot stored at least once; otherwise a checked program whose OP_CHECK k needs k < nconstraints.
// Error messages start with `who`.
int validate_program(ms_ctx *c, const char *who, const uint32_t *program, unsigned nprog, unsigned nconsts,
                     const std::vector<int> &col_is_q, unsigned log_m, unsigned nconstraints, unsigned nout = 1);

// One evaluation point of an evaluator program (OP_X .. OP_PERIODIC), shared by the fused evaluator (eval.cu) and the
// extension-column scan (extension.cu).  p supplies prog, nprog, consts, col_ptr, fq_words, log_m, trace_bitrev, tw_lo,
// tw_hi, hi_len and offset; i is the point index of the domain of size M = 2^p.log_m, r the register file.  OP_STORE s, r
// hands register r to store(s, r, r_is_fq): the caller decides where slot s goes.
template <class Params, class Store>
__device__ __forceinline__ void eval_point(const Params &p, const u64 M, const u64 i, u64 (*r)[3], Store &&store) {
    const u32 lm = p.log_m;
    const bool fq3 = p.fq_words == 3;
    for (u32 pc = 0; pc < p.nprog; pc++) {
        const uint4 ins = __ldg(p.prog + pc);
        const u32 op = ins.x & 0xff;
        const bool qa = ((ins.x >> 8) & 1) && fq3, qb = ((ins.x >> 9) & 1) && fq3;
        const u32 d = ins.y;
        switch (op) {
            case OP_X: {
                u64 w = p.tw_lo[i & 4095];
                if (p.hi_len > 1) w = gl::mul(p.tw_hi[i >> 12], w);
                r[d][0] = gl::mul(w, p.offset);
                break;
            }
            case OP_CONST: {
                const u64 *k = p.consts + 3 * (u64)ins.z;
                r[d][0] = k[0];
                if (qa) { r[d][1] = k[1]; r[d][2] = k[2]; }
                break;
            }
            case OP_TRACE: {
                u64 pos = (i + (u64)ins.w) & (M - 1);
                if (p.trace_bitrev && lm) pos = __brevll(pos) >> (64 - lm);
                const u64 *col = p.col_ptr[ins.z];
                if ((ins.x >> 8) & 1) {  // Fq column
                    const u64 *c = col + pos * p.fq_words;
                    r[d][0] = c[0];
                    if (fq3) { r[d][1] = c[1]; r[d][2] = c[2]; }
                } else {
                    r[d][0] = col[pos];
                }
                break;
            }
            case OP_NEG: {
                const u64 a0 = r[ins.z][0];
                if (qa) {
                    const u64 a1 = r[ins.z][1], a2 = r[ins.z][2];
                    r[d][1] = gl::neg(a1);
                    r[d][2] = gl::neg(a2);
                }
                r[d][0] = gl::neg(a0);
                break;
            }
            case OP_ADD: {
                const u64 a0 = r[ins.z][0], b0 = r[ins.w][0];
                if (qa || qb) {
                    const u64 a1 = qa ? r[ins.z][1] : 0, a2 = qa ? r[ins.z][2] : 0;
                    const u64 b1 = qb ? r[ins.w][1] : 0, b2 = qb ? r[ins.w][2] : 0;
                    r[d][1] = gl::add(a1, b1);
                    r[d][2] = gl::add(a2, b2);
                }
                r[d][0] = gl::add(a0, b0);
                break;
            }
            case OP_SUB: {
                const u64 a0 = r[ins.z][0], b0 = r[ins.w][0];
                if (qa || qb) {
                    const u64 a1 = qa ? r[ins.z][1] : 0, a2 = qa ? r[ins.z][2] : 0;
                    const u64 b1 = qb ? r[ins.w][1] : 0, b2 = qb ? r[ins.w][2] : 0;
                    r[d][1] = gl::sub(a1, b1);
                    r[d][2] = gl::sub(a2, b2);
                }
                r[d][0] = gl::sub(a0, b0);
                break;
            }
            case OP_PERIODIC: {
                // periodic column (src/constraints.rs:107-146, src/eval_cpu.rs:234-256): a table of 2^ins.w evaluations
                // over the coset of size interval * lde_step, repeated along the ce domain; natural order
                const u64 pos = i & ((1ull << ins.w) - 1);
                const u64 *col = p.col_ptr[ins.z];
                if ((ins.x >> 8) & 1) {
                    const u64 *c = col + pos * p.fq_words;
                    r[d][0] = c[0];
                    if (fq3) { r[d][1] = c[1]; r[d][2] = c[2]; }
                } else {
                    r[d][0] = col[pos];
                }
                break;
            }
            case OP_MUL: {
                if (!qa && !qb) {
                    r[d][0] = gl::mul(r[ins.z][0], r[ins.w][0]);
                } else if (qa && qb) {
                    const gl::Fq3 a{r[ins.z][0], r[ins.z][1], r[ins.z][2]}, b{r[ins.w][0], r[ins.w][1], r[ins.w][2]};
                    const gl::Fq3 c = gl::mul(a, b);
                    r[d][0] = c.c0; r[d][1] = c.c1; r[d][2] = c.c2;
                } else {
                    const u32 q = qa ? ins.z : ins.w, s = qa ? ins.w : ins.z;
                    const gl::Fq3 a{r[q][0], r[q][1], r[q][2]};
                    const gl::Fq3 c = gl::mul(a, r[s][0]);
                    r[d][0] = c.c0; r[d][1] = c.c1; r[d][2] = c.c2;
                }
                break;
            }
            case OP_INV: {
                if (qa) {
                    const gl::Fq3 c = gl::inv(gl::Fq3{r[ins.z][0], r[ins.z][1], r[ins.z][2]});
                    r[d][0] = c.c0; r[d][1] = c.c1; r[d][2] = c.c2;
                } else {
                    r[d][0] = gl::inv(r[ins.z][0]);
                }
                break;
            }
            case OP_POW: {
                if (qa) {
                    const gl::Fq3 c = gl::pow(gl::Fq3{r[ins.z][0], r[ins.z][1], r[ins.z][2]}, (u64)ins.w);
                    r[d][0] = c.c0; r[d][1] = c.c1; r[d][2] = c.c2;
                } else {
                    r[d][0] = gl::pow(r[ins.z][0], (u64)ins.w);
                }
                break;
            }
            case OP_STORE: {
                store(d, r[ins.z], qa);
                break;
            }
            default: break;
        }
    }
}

}  // namespace ms
