// tuples.cuh — the evaluate-and-sort stages shared by the lookup multiplicity fill (lookup.cu) and the permutation fill
// (permutation.cu): W-word tuples, one per row of the trace domain, evaluated from the base trace and ordered
// lexicographically.
//
//   tuple_evaluate: one evaluator program (expr.py, compile_lookup_program) stores S slots per row; eval.cuh's eval_point
//                   interprets it over the trace domain, one thread per row, and every output is written as a canonical
//                   integer (never a lazy or Montgomery word), so equal field elements are equal words;
//   tuple_sort:     W stable cub radix sorts of (word k gathered through the current permutation, row), from the last word
//                   to the first — an LSD lexicographic sort, so equal tuples end adjacent and in row order.
// Rows and offsets into the slot columns are 64-bit throughout; the permutation is 32-bit (at most 2^30 rows).
// Everything here has internal linkage: each translation unit that includes it compiles its own copy of the kernels.
#pragma once
#include "eval.cuh"

#include <cub/cub.cuh>
#include <vector>

namespace ms {
namespace {

constexpr int kTupleThreads = 256;

struct TupleEvalParams {
    // the fields eval_point reads
    const uint4 *prog;
    u32 nprog;
    const u64 *consts;
    const u64 *const *col_ptr;
    u32 fq_words;               // 1: every expression is over Fp
    u32 log_m;
    u32 trace_bitrev;           // 0: natural order
    const u64 *tw_lo, *tw_hi;
    u32 hi_len;
    u64 offset;                 // ONE: X is g_n^i
    u64 *slots;                 // slot s of row i at slots[s * n + i], canonical
};

__global__ void __launch_bounds__(kTupleThreads) tuple_eval_kernel(const TupleEvalParams p) {
    const u64 n = 1ull << p.log_m;
    const u64 i = (u64)blockIdx.x * kTupleThreads + threadIdx.x;
    if (i >= n) return;
    u64 r[kMaxRegs][3];
    eval_point(p, n, i, r, [&](u32 s, const u64 *v, bool) { p.slots[(u64)s * n + i] = gl::canon(gl::from_mont(v[0])); });
}

// key[j] = word[perm[j]] (perm == nullptr: key[j] = word[j] and perm_out[j] = j)
__global__ void __launch_bounds__(kTupleThreads) tuple_gather_kernel(const u64 *word, const u32 *perm, u64 *key, u32 *perm_out,
                                                                     u64 n) {
    const u64 j = (u64)blockIdx.x * kTupleThreads + threadIdx.x;
    if (j >= n) return;
    if (perm) {
        key[j] = word[perm[j]];
    } else {
        key[j] = word[j];
        perm_out[j] = (u32)j;
    }
}

// workspace regions are 256-byte aligned
size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

unsigned tuple_blocks(u64 n) { return (unsigned)((n + kTupleThreads - 1) / kTupleThreads); }

// Checks the columns and the program (an evaluator program over the base field storing slots 0..nslots-1), stages them
// in scratch arena 3 and launches the evaluation into `slots` ([nslots][2^log_n] canonical words).  Error messages
// start with `who`.
int tuple_evaluate(ms_ctx *c, const char *who, const uint32_t *program, unsigned nprog, const uint64_t *consts,
                   unsigned nconsts, const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, unsigned log_n,
                   unsigned nslots, u64 *slots) {
    std::vector<const u64 *> cols;
    std::vector<int> isq;
    for (unsigned k = 0; k < ncols; k++) {
        if (!col_ptrs[k] || !is_device_ptr(col_ptrs[k])) return fail(c, MS_ERR_INVALID, "%s: column %u is not a device pointer", who, k);
        if (col_is_fq[k]) return fail(c, MS_ERR_INVALID, "%s: column %u is not a base-field column", who, k);
        cols.push_back((const u64 *)col_ptrs[k]);
        isq.push_back(0);
    }
    int rc = validate_program(c, who, program, nprog, nconsts, isq, log_n, 0, nslots);
    if (rc) return rc;
    for (unsigned k = 0; k < nprog; k++)
        if ((program[4 * k] & 0xff) == OP_STORE && ((program[4 * k] >> 8) & 1))
            return fail(c, MS_ERR_INVALID, "%s: instruction %u stores an extension-field value", who, k);
    void *meta;
    const size_t prog_bytes = (size_t)nprog * 16, const_bytes = (size_t)nconsts * 24, ptr_bytes = (size_t)ncols * 8;
    if ((rc = scratch_get(c, 3, prog_bytes + const_bytes + ptr_bytes + 64, &meta))) return rc;
    char *m = (char *)meta;
    // pageable host sources: each copy returns once its source is staged, so the caller's buffers are free afterwards
    MS_CUDA(c, cudaMemcpyAsync(m, program, prog_bytes, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaMemcpyAsync(m + prog_bytes, consts, const_bytes, cudaMemcpyDefault, c->stream));
    if (ptr_bytes) MS_CUDA(c, cudaMemcpyAsync(m + prog_bytes + const_bytes, cols.data(), ptr_bytes, cudaMemcpyHostToDevice, c->stream));

    TupleEvalParams p;
    if ((rc = ntt_plan_tables(c, log_n, &p.tw_lo, &p.tw_hi, &p.hi_len))) return rc;
    p.prog = (const uint4 *)m;
    p.nprog = nprog;
    p.consts = (const u64 *)(m + prog_bytes);
    p.col_ptr = (const u64 *const *)(m + prog_bytes + const_bytes);
    p.fq_words = 1;
    p.log_m = log_n;
    p.trace_bitrev = 0;
    p.offset = gl::ONE;
    p.slots = slots;
    tuple_eval_kernel<<<tuple_blocks(1ull << log_n), kTupleThreads, 0, c->stream>>>(p);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    return MS_OK;
}

// LSD lexicographic sort of the n tuples whose word k is slots[k * n + row], k < width: stable passes from the last word
// to the first.  keys0/keys1 (n words each) and perm0/perm1 (n entries each) are the double buffers; *order receives the
// one of perm0/perm1 that maps sorted position -> row.  cub's temporary storage is scratch arena 2.
int tuple_sort(ms_ctx *c, const u64 *slots, unsigned width, u64 n, u64 *keys0, u64 *keys1, u32 *perm0, u32 *perm1,
               const u32 **order) {
    const unsigned nblk = tuple_blocks(n);
    cub::DoubleBuffer<u64> keys(keys0, keys1);
    cub::DoubleBuffer<u32> perm(perm0, perm1);
    size_t tb = 0;
    MS_CUDA(c, cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, perm, (int)n, 0, 64, c->stream));
    void *temp;
    int rc = scratch_get(c, 2, tb, &temp);
    if (rc) return rc;
    for (int k = (int)width - 1; k >= 0; k--) {
        const bool first = k == (int)width - 1;
        tuple_gather_kernel<<<nblk, kTupleThreads, 0, c->stream>>>(slots + (u64)k * n, first ? nullptr : perm.Current(),
                                                                  keys.Current(), perm.Current(), n);
        c->launches++;
        MS_CHECK_LAUNCH(c);
        MS_CUDA(c, cub::DeviceRadixSort::SortPairs(temp, tb, keys, perm, (int)n, 0, 64, c->stream));
    }
    *order = perm.Current();
    return MS_OK;
}

}  // namespace
}  // namespace ms
