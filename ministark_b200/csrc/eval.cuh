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
// have been written by an earlier instruction.  nconstraints == 0: an evaluator program (ends in OP_STORE); otherwise a
// checked program whose OP_CHECK k needs k < nconstraints.  Error messages start with `who`.
int validate_program(ms_ctx *c, const char *who, const uint32_t *program, unsigned nprog, unsigned nconsts,
                     const std::vector<int> &col_is_q, unsigned log_m, unsigned nconstraints);

}  // namespace ms
