// eval.cu — fused symbolic constraint evaluation.
//
// Reference: AirConfig::eval_constraint -> eval_cpu::eval (src/air.rs:86-128,
// src/eval_cpu.rs:33-150) evaluates the composition-constraint DAG over the ce domain in
// 512-element chunks on the CPU; its GPU version (src/eval_gpu.rs:46-217, disabled in
// src/air.rs:104-117 as "currently slower than CPU") issues one dispatch + barrier per DAG node
// out of 35 pointwise stages, every one a full round trip through device memory.
//
// Here the whole DAG is ONE kernel: the host flattens it (ministark_b200/expr.py) into a typed
// linear program; every thread evaluates the program for one point of the ce domain with all
// temporaries in its own register file (local memory, L1 resident), reading each trace column
// exactly once per referenced row offset and writing one Fq element.  Algorithmic traffic:
// (sum of distinct input columns * element size + output element) * M bytes (SURVEY.md §8d).
//
//  * Leaves: X is h * g^i from the two-level twiddle table of the ce-domain plan (the reference
//    materialises an x_lde vector, src/prover.rs:95); Constant / Challenge / Hint come from a
//    constant pool; Trace(col, off) reads column[(i + step*off) mod M] (eval_cpu.rs:119-134).
//  * The columns may be given in the bit-reversed LDE order the commitments use: the first M
//    entries of a bit-reversed LDE column are the bit-reversed evaluations over the ce coset
//    (src/prover.rs:86-91 bit-reverses them back on the CPU, twice per proof).  With
//    trace_bitrev the thread for storage position t evaluates point i = bitrev(t), so loads stay
//    coalesced and neither CPU permutation is needed.
//  * Div is a per-point field inversion (Fermat chain); eval_cpu uses batch inversion per chunk
//    (eval_cpu.rs:280-295) — the same field element either way.
#include "eval.cuh"

namespace ms {

using gl::Fq3;

struct EvalParams {
    const uint4 *prog;
    u32 nprog;
    const u64 *consts;          // [k][3] Montgomery words
    const u64 *const *col_ptr;  // one device pointer per column (base columns first, then Fq columns)
    u32 fq_words;               // 1: Fq = Fp, 3: Fq = Fq3
    u32 log_m;                  // ce domain size M = 2^log_m
    u32 trace_bitrev;
    u32 out_bitrev;             // store the result at the storage position t instead of the point index i
    const u64 *tw_lo, *tw_hi;   // g_M^e two-level table
    u32 hi_len;
    u64 offset;                 // domain offset h (Montgomery)
    u64 *out;                   // M elements of fq_words words, natural order
};

__global__ void __launch_bounds__(128) eval_kernel(const EvalParams p) {
    const u64 M = 1ull << p.log_m;
    const u64 t = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    if (t >= M) return;
    const u32 lm = p.log_m;
    const u64 i = (p.trace_bitrev && lm) ? (__brevll(t) >> (64 - lm)) : t;   // evaluation point index
    const bool fq3 = p.fq_words == 3;
    u64 r[kMaxRegs][3];
    eval_point(p, M, i, r, [&](u32, const u64 *v, bool qa) {
        u64 *o = p.out + (p.out_bitrev ? t : i) * p.fq_words;
        o[0] = v[0];
        if (fq3) {
            o[1] = qa ? v[1] : 0;
            o[2] = qa ? v[2] : 0;
        }
    });
}

int validate_program(ms_ctx *c, const char *who, const uint32_t *program, unsigned nprog, unsigned nconsts,
                     const std::vector<int> &col_is_q, unsigned log_m, unsigned nconstraints, unsigned nout) {
    const bool checked = nconstraints > 0;
    std::vector<char> defined(kMaxRegs, 0), stored(checked ? 0 : nout, 0);
    for (unsigned k = 0; k < nprog; k++) {
        const uint32_t *ins = program + 4 * k;
        const uint32_t op = ins[0] & 0xff;
        if (op > (checked ? (uint32_t)OP_CHECK : (uint32_t)OP_PERIODIC) || ins[1] >= (uint32_t)kMaxRegs)
            return fail(c, MS_ERR_INVALID, "%s: bad instruction %u", who, k);
        if (checked && (op == OP_STORE || op == OP_INV))
            return fail(c, MS_ERR_INVALID, "%s: instruction %u: %s has no place in a checked program", who, k, op == OP_STORE ? "STORE" : "INV");
        if (op == OP_CONST && ins[2] >= nconsts) return fail(c, MS_ERR_INVALID, "%s: constant index out of range", who);
        if (op == OP_TRACE || op == OP_PERIODIC) {
            const int is_q = (ins[0] >> 8) & 1;
            if (ins[2] >= col_is_q.size()) return fail(c, MS_ERR_INVALID, "%s: column %u out of range", who, ins[2]);
            if (col_is_q[ins[2]] != is_q) return fail(c, MS_ERR_INVALID, "%s: column %u has the wrong field", who, ins[2]);
            if (op == OP_PERIODIC && ins[3] > log_m) return fail(c, MS_ERR_INVALID, "%s: periodic table longer than the domain", who);
        }
        if (op == OP_STORE && ins[1] >= nout)
            return fail(c, MS_ERR_INVALID, "%s: instruction %u stores to slot %u of %u", who, k, ins[1], nout);
        if (op == OP_CHECK && ins[3] >= nconstraints)
            return fail(c, MS_ERR_INVALID, "%s: instruction %u checks constraint %u of %u", who, k, ins[3], nconstraints);
        const bool unary = op == OP_NEG || op == OP_INV || op == OP_POW || op == OP_STORE || op == OP_CHECK;
        const bool binary = op == OP_ADD || op == OP_SUB || op == OP_MUL || op == OP_DIV;
        if (unary || binary) {
            if (ins[2] >= (uint32_t)kMaxRegs || !defined[ins[2]])
                return fail(c, MS_ERR_INVALID, "%s: instruction %u reads register %u before it is written", who, k, ins[2]);
        }
        if (binary) {
            if (ins[3] >= (uint32_t)kMaxRegs || !defined[ins[3]])
                return fail(c, MS_ERR_INVALID, "%s: instruction %u reads register %u before it is written", who, k, ins[3]);
        }
        if (op == OP_STORE) stored[ins[1]] = 1;
        else if (op != OP_CHECK) defined[ins[1]] = 1;
    }
    for (unsigned s = 0; s < stored.size(); s++) {
        if (stored[s]) continue;
        if (nout == 1) return fail(c, MS_ERR_INVALID, "%s: program stores no result", who);
        return fail(c, MS_ERR_INVALID, "%s: program never stores slot %u of %u", who, s, nout);
    }
    return MS_OK;
}

int eval_launch_jit(ms_ctx *c, const uint32_t *program, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                    const u64 *const *dev_col_ptr, const u64 *dev_consts, int fq_field, unsigned log_m, uint64_t offset_mont,
                    int trace_bitrev, int out_bitrev, const u64 *tw_lo, const u64 *tw_hi, u32 hi_len, u64 *out_dev);

}  // namespace ms

using namespace ms;

static int eval_launch(ms_ctx *c, const uint32_t *program, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                       const std::vector<const u64 *> &cols, const std::vector<int> &col_is_q, int fq_field, unsigned log_m,
                       uint64_t offset_mont, int trace_bitrev, int out_bitrev, u64 *out_dev) {
    const size_t M = (size_t)1 << log_m;
    int rc = validate_program(c, "ms_eval_constraints", program, nprog, nconsts, col_is_q, log_m, 0);
    if (rc) return rc;
    // program, constants and the column pointer table are tiny: always copied to the device
    void *meta;
    const size_t prog_bytes = (size_t)nprog * 16, const_bytes = (size_t)nconsts * 24, ptr_bytes = cols.size() * 8;
    rc = scratch_get(c, 3, prog_bytes + const_bytes + ptr_bytes + 64, &meta);
    if (rc) return rc;
    MS_CUDA(c, cudaMemcpyAsync(meta, program, prog_bytes, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaMemcpyAsync((char *)meta + prog_bytes, consts, const_bytes, cudaMemcpyDefault, c->stream));
    if (ptr_bytes)
        MS_CUDA(c, cudaMemcpyAsync((char *)meta + prog_bytes + const_bytes, cols.data(), ptr_bytes, cudaMemcpyHostToDevice, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));  // the host buffers may be temporaries of the caller
    const u64 *tw_lo, *tw_hi;
    u32 hi_len;
    if ((rc = ntt_plan_tables(c, log_m, &tw_lo, &tw_hi, &hi_len))) return rc;
    // run-time specialised kernel first (eval_jit.cu); the interpreter below is the fallback
    {
        const int jrc = eval_launch_jit(c, program, nprog, consts, nconsts, (const u64 *const *)((char *)meta + prog_bytes + const_bytes),
                                        (const u64 *)((char *)meta + prog_bytes), fq_field, log_m, offset_mont, trace_bitrev, out_bitrev, tw_lo, tw_hi, hi_len, out_dev);
        if (jrc == MS_OK) return MS_OK;
        if (jrc == MS_ERR_CUDA) return jrc;
    }
    EvalParams p;
    p.prog = (const uint4 *)meta;
    p.nprog = nprog;
    p.consts = (const u64 *)((char *)meta + prog_bytes);
    p.col_ptr = (const u64 *const *)((char *)meta + prog_bytes + const_bytes);
    p.fq_words = (u32)fq_field;
    p.log_m = log_m;
    p.trace_bitrev = trace_bitrev ? 1 : 0;
    p.out_bitrev = (out_bitrev && trace_bitrev) ? 1 : 0;
    p.tw_lo = tw_lo;
    p.tw_hi = tw_hi;
    p.hi_len = hi_len;
    p.offset = offset_mont;
    p.out = out_dev;
    eval_kernel<<<(unsigned)((M + 127) / 128), 128, 0, c->stream>>>(p);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    return MS_OK;
}

extern "C" int ms_eval_constraints(ms_ctx *c, const uint32_t *program, unsigned nprog, const uint64_t *consts,
                                   unsigned nconsts, const void *base_cols, size_t base_stride_elems, unsigned nbase,
                                   const void *ext_cols, size_t ext_stride_elems, unsigned next, int fq_field,
                                   unsigned log_m, uint64_t offset_mont, int trace_bitrev, int out_bitrev, void *out) {
    if (!c || !program || !consts || !out || nprog == 0) return MS_ERR_INVALID;
    if (fq_field != MS_FIELD_FP && fq_field != MS_FIELD_FQ3) return fail(c, MS_ERR_INVALID, "ms_eval_constraints: bad Fq field id");
    if (log_m > 32) return fail(c, MS_ERR_INVALID, "ms_eval_constraints: domain too large");
    if (offset_mont >= gl::P || offset_mont == 0) return fail(c, MS_ERR_INVALID, "offset must be a non-zero canonical word");
    const size_t M = (size_t)1 << log_m;
    if ((nbase && !base_cols) || (next && !ext_cols)) return fail(c, MS_ERR_INVALID, "ms_eval_constraints: missing columns");
    if (nbase > 1 && base_stride_elems < M) return fail(c, MS_ERR_INVALID, "ms_eval_constraints: base stride < domain");
    if (next > 1 && ext_stride_elems < M) return fail(c, MS_ERR_INVALID, "ms_eval_constraints: ext stride < domain");
    Staged B(c, nbase ? base_cols : nullptr, nbase ? ((size_t)(nbase - 1) * base_stride_elems + M) * 8 : 0, true, false);
    if (B.rc) return B.rc;
    Staged E(c, next ? ext_cols : nullptr, next ? ((size_t)(next - 1) * ext_stride_elems + M) * fq_field * 8 : 0, true, false);
    if (E.rc) return E.rc;
    Staged O(c, out, M * fq_field * 8, false, true);
    if (O.rc) return O.rc;
    std::vector<const u64 *> cols;
    std::vector<int> isq;
    for (unsigned i = 0; i < nbase; i++) { cols.push_back(B.as<u64>() + (size_t)i * base_stride_elems); isq.push_back(0); }
    for (unsigned i = 0; i < next; i++) { cols.push_back(E.as<u64>() + (size_t)i * ext_stride_elems * fq_field); isq.push_back(1); }
    int rc = eval_launch(c, program, nprog, consts, nconsts, cols, isq, fq_field, log_m, offset_mont, trace_bitrev, out_bitrev,
                         O.as<u64>());
    if (rc) return rc;
    if ((rc = B.finish())) return rc;
    if ((rc = E.finish())) return rc;
    return O.finish();
}

// Same evaluator over an explicit table of DEVICE column pointers (columns living in different matrices:
// base trace LDE, extension trace LDE, composition trace LDE — as the DEEP composition needs).
// col_fields[i] = MS_FIELD_FP for a base-field column, anything else = a column of `fq_field` elements.
extern "C" int ms_eval_constraints_ptrs(ms_ctx *c, const uint32_t *program, unsigned nprog, const uint64_t *consts,
                                        unsigned nconsts, const void *const *col_ptrs, const int *col_is_fq, unsigned ncols,
                                        int fq_field, unsigned log_m, uint64_t offset_mont, int trace_bitrev, int out_bitrev,
                                        void *out) {
    if (!c || !program || !consts || !out || nprog == 0 || (ncols && (!col_ptrs || !col_is_fq))) return MS_ERR_INVALID;
    if (fq_field != MS_FIELD_FP && fq_field != MS_FIELD_FQ3) return fail(c, MS_ERR_INVALID, "ms_eval_constraints: bad Fq field id");
    if (log_m > 32) return fail(c, MS_ERR_INVALID, "ms_eval_constraints: domain too large");
    if (offset_mont >= gl::P || offset_mont == 0) return fail(c, MS_ERR_INVALID, "offset must be a non-zero canonical word");
    cudaSetDevice(c->device);
    std::vector<const u64 *> cols;
    std::vector<int> isq;
    for (unsigned i = 0; i < ncols; i++) {
        if (!col_ptrs[i] || !is_device_ptr(col_ptrs[i])) return fail(c, MS_ERR_INVALID, "ms_eval_constraints_ptrs: column %u is not a device pointer", i);
        cols.push_back((const u64 *)col_ptrs[i]);
        isq.push_back(col_is_fq[i] ? 1 : 0);
    }
    if (!is_device_ptr(out)) return fail(c, MS_ERR_INVALID, "ms_eval_constraints_ptrs: out must be a device pointer");
    return eval_launch(c, program, nprog, consts, nconsts, cols, isq, fq_field, log_m, offset_mont, trace_bitrev, out_bitrev,
                       (u64 *)out);
}
