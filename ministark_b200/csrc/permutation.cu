// permutation.cu — the target columns of a sorted-copy permutation argument an AIR declares (ministark_b200/air.py,
// Permutation): the source tuples of every row, sorted lexicographically, written back as base columns.
//
// One call handles one permutation of W words per tuple (1..4) over n = 2^log_n rows:
//   1. evaluate (tuples.cuh, tuple_evaluate): the program stores the W source words of every row as canonical integers in
//      the workspace's slot columns;
//   2. order (tuples.cuh, tuple_sort): W stable radix passes over (word, row), from the last word to the first, give the
//      sorted position -> row map; equal tuples keep their row order;
//   3. write: target k at position j is slot k at that row, converted to a Montgomery word.
// Rows and offsets are 64-bit throughout.  Traffic per row: the cells the program reads, the W slot words written once
// and read twice (one key gather, one write gather), 16 bytes of keys and 8 of permutation per radix digit pass
// (8 digit passes of 8 bits per word), and the W target words written.
#include "tuples.cuh"
#include "../../include/ministark_permutation.h"

namespace ms {

constexpr unsigned kMaxPermutationWidth = 4, kMaxPermutationLog = 30;

// workspace layout (byte offsets, each region 256-byte aligned)
struct PermutationWork {
    size_t slots, keys, perm, total;
};

static PermutationWork permutation_layout(unsigned log_n, unsigned W) {
    const size_t n = (size_t)1 << log_n;
    PermutationWork w;
    w.slots = 0;
    w.keys = w.slots + align256((size_t)W * n * 8);
    w.perm = w.keys + align256(2 * n * 8);
    w.total = w.perm + align256(2 * n * 4);
    return w;
}

struct PermutationTargets {
    u64 *col[kMaxPermutationWidth];
};

// target k at sorted position j: Montgomery form of source word k of row order[j]; blockIdx.y is k
__global__ void __launch_bounds__(kTupleThreads) permutation_write_kernel(const u64 *slots, const u32 *order,
                                                                          const PermutationTargets t, u64 n) {
    const u64 j = (u64)blockIdx.x * kTupleThreads + threadIdx.x;
    if (j >= n) return;
    const u32 k = blockIdx.y;
    u64 *col = k == 0 ? t.col[0] : k == 1 ? t.col[1] : k == 2 ? t.col[2] : t.col[3];     // no local copy of t
    col[j] = gl::to_mont(slots[(u64)k * n + order[j]]);
}

}  // namespace ms

using namespace ms;

extern "C" int ms_permutation_workspace_bytes(unsigned log_n, unsigned width, size_t *bytes) {
    if (!bytes || log_n > kMaxPermutationLog || width < 1 || width > kMaxPermutationWidth) return MS_ERR_INVALID;
    *bytes = permutation_layout(log_n, width).total;
    return MS_OK;
}

extern "C" int ms_permutation_fill(ms_ctx *c, const uint32_t *program, unsigned nprog, const uint64_t *consts,
                                   unsigned nconsts, const void *const *col_ptrs, const int *col_is_fq, unsigned ncols,
                                   unsigned log_n, unsigned width, void *const *targets, void *workspace,
                                   size_t workspace_bytes) {
    if (!c || !program || !consts || nprog == 0 || (ncols && (!col_ptrs || !col_is_fq)) || !targets || !workspace)
        return MS_ERR_INVALID;
    if (log_n > kMaxPermutationLog)
        return fail(c, MS_ERR_INVALID, "ms_permutation_fill: domain too large (at most 2^%u rows)", kMaxPermutationLog);
    if (width < 1 || width > kMaxPermutationWidth)
        return fail(c, MS_ERR_INVALID, "ms_permutation_fill: tuples of %u words (1 to %u)", width, kMaxPermutationWidth);
    const PermutationWork w = permutation_layout(log_n, width);
    if (workspace_bytes < w.total)
        return fail(c, MS_ERR_INVALID, "ms_permutation_fill: workspace of %zu bytes, %zu needed", workspace_bytes, w.total);
    cudaSetDevice(c->device);
    if (!is_device_ptr(workspace)) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: the workspace must be device memory");
    PermutationTargets t;
    for (unsigned k = 0; k < width; k++) {
        if (!targets[k] || !is_device_ptr(targets[k]))
            return fail(c, MS_ERR_INVALID, "ms_permutation_fill: target %u is not a device pointer", k);
        for (unsigned j = 0; j < k; j++)
            if (targets[j] == targets[k]) return fail(c, MS_ERR_INVALID, "ms_permutation_fill: targets %u and %u are the same column", j, k);
        t.col[k] = (u64 *)targets[k];
    }
    const u64 n = 1ull << log_n;
    char *wb = (char *)workspace;
    u64 *slots = (u64 *)(wb + w.slots), *keys0 = (u64 *)(wb + w.keys), *keys1 = keys0 + n;
    u32 *perm0 = (u32 *)(wb + w.perm), *perm1 = perm0 + n;

    // 1. evaluate
    int rc = tuple_evaluate(c, "ms_permutation_fill", program, nprog, consts, nconsts, col_ptrs, col_is_fq, ncols, log_n,
                            width, slots);
    if (rc) return rc;
    // 2. order
    const u32 *order;
    if ((rc = tuple_sort(c, slots, width, n, keys0, keys1, perm0, perm1, &order))) return rc;
    // 3. write
    permutation_write_kernel<<<dim3(tuple_blocks(n), width), kTupleThreads, 0, c->stream>>>(slots, order, t, n);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    return MS_OK;
}
