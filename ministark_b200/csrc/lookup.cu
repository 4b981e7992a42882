// lookup.cu — the multiplicity column of a LogUp lookup an AIR declares (ministark_b200/air.py, Lookup), filled from the
// base trace with exact tuple matching.
//
// One call handles one lookup of W words per tuple (1..4) and Q value tuples (1..4) over n = 2^log_n rows:
//   1. evaluate (tuples.cuh, tuple_evaluate): one evaluator program (expr.py, compile_lookup_program) stores the W table
//      words and, per value tuple, its selector and W words, as canonical integers in the workspace's slot columns;
//   2. order the table (tuples.cuh, tuple_sort): an LSD lexicographic sort of W stable radix passes, so equal tuples end
//      adjacent and in row order, the first row of a run being the lowest row holding that tuple; the sorted tuples are
//      then gathered word by word;
//   3. match: one thread per (row, value tuple).  Selector 0: nothing.  A selector that is neither 0 nor 1 is counted as
//      bad.  Otherwise a lexicographic lower-bound binary search in the sorted table; a hit adds 1 to the 64-bit counter of
//      the run's first row (threads of a warp that hit the same row add once, together), a miss is counted for the tuple;
//   4. write: the counters (at most Q n, far below p) become Montgomery words in `out`.
// Rows and offsets into the workspace are 64-bit throughout.  Traffic per row: the cells the program reads, the S =
// W + Q (W + 1) slot words written once and read once or twice, 16 W bytes of keys and 8 W of permutation per sort pass
// (plus cub's 8-bit digit passes), and W sorted words per search step (log2 n steps, cached near the root).
#include "tuples.cuh"
#include "../../include/ministark_lookup.h"

namespace ms {

constexpr unsigned kMaxLookupWidth = 4, kMaxLookupTuples = 4, kMaxLookupLog = 30;
constexpr int kLookupThreads = kTupleThreads;

// workspace layout (byte offsets, each region 256-byte aligned)
struct LookupWork {
    size_t slots, sorted, keys, perm, status, total;
};

static LookupWork lookup_layout(unsigned log_n, unsigned W, unsigned Q) {
    const size_t n = (size_t)1 << log_n, S = (size_t)W + (size_t)Q * (W + 1);
    LookupWork w;
    w.slots = 0;
    w.sorted = w.slots + align256(S * n * 8);
    w.keys = w.sorted + align256((size_t)W * n * 8);
    w.perm = w.keys + align256(2 * n * 8);
    w.status = w.perm + align256(2 * n * 4);
    w.total = w.status + align256((2 * kMaxLookupTuples + 2) * 8);
    return w;
}

template <int W>
struct LookupMatchParams {
    const u64 *slots;           // [S][n]
    const u64 *sorted;          // [W][n]: the table tuples in lexicographic order
    const u32 *perm;            // sorted position -> row
    u64 n;
    u32 ntuples;
    u64 *counts;                // n counters (the out column, zeroed)
    u64 *status;                // [2 Q + 2]
};

// lexicographic compare of the sorted tuple at position j with v: < 0, 0, > 0
template <int W>
__device__ __forceinline__ int lookup_cmp(const u64 *sorted, u64 n, u64 j, const u64 (&v)[W]) {
#pragma unroll
    for (int k = 0; k < W; k++) {
        const u64 t = sorted[(u64)k * n + j];
        if (t != v[k]) return t < v[k] ? -1 : 1;
    }
    return 0;
}

template <int W>
__global__ void __launch_bounds__(kLookupThreads) lookup_match_kernel(const LookupMatchParams<W> p) {
    const u64 n = p.n, i = (u64)blockIdx.x * kLookupThreads + threadIdx.x;
    const u32 q = blockIdx.y;
    const u64 base = (u64)W + (u64)q * (W + 1);
    u64 target = ~0ull;                         // the row whose counter this (row, tuple) adds to
    if (i < n) {
        const u64 sel = p.slots[base * n + i];
        if (sel == 1) {
            u64 v[W];
#pragma unroll
            for (int k = 0; k < W; k++) v[k] = p.slots[(base + 1 + k) * n + i];
            u64 lo = 0, hi = n;                 // lower bound: the first sorted position whose tuple is >= v
            while (lo < hi) {
                const u64 mid = lo + ((hi - lo) >> 1);
                if (lookup_cmp<W>(p.sorted, n, mid, v) < 0) lo = mid + 1;
                else hi = mid;
            }
            if (lo < n && lookup_cmp<W>(p.sorted, n, lo, v) == 0) {
                target = p.perm[lo];
            } else {
                atomicAdd(p.status + 2 * q, 1ull);
                atomicMin(p.status + 2 * q + 1, i);
            }
        } else if (sel != 0) {
            atomicAdd(p.status + 2 * p.ntuples, 1ull);
            atomicMin(p.status + 2 * p.ntuples + 1, i);
        }
    }
    // every lane of the warp reaches this point: lanes hitting the same row add once (a table of few distinct tuples
    // would otherwise serialise n atomics on one counter)
    const unsigned same = __match_any_sync(0xffffffffu, target);
    if (target != ~0ull && (threadIdx.x & 31) == (unsigned)(__ffs(same) - 1)) atomicAdd(p.counts + target, (u64)__popc(same));
}

__global__ void __launch_bounds__(kLookupThreads) lookup_write_kernel(u64 *out, u64 n) {
    const u64 j = (u64)blockIdx.x * kLookupThreads + threadIdx.x;
    if (j < n) out[j] = gl::to_mont(out[j]);
}

template <int W>
static int lookup_match(ms_ctx *c, const u64 *slots, const u64 *sorted, const u32 *perm, u64 n, unsigned Q, u64 *counts,
                        u64 *status) {
    LookupMatchParams<W> p{slots, sorted, perm, n, Q, counts, status};
    const dim3 grid((unsigned)((n + kLookupThreads - 1) / kLookupThreads), Q);
    lookup_match_kernel<W><<<grid, kLookupThreads, 0, c->stream>>>(p);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    return MS_OK;
}

}  // namespace ms

using namespace ms;

extern "C" int ms_lookup_workspace_bytes(unsigned log_n, unsigned width, unsigned ntuples, size_t *bytes) {
    if (!bytes || log_n > kMaxLookupLog || width < 1 || width > kMaxLookupWidth || ntuples < 1 || ntuples > kMaxLookupTuples)
        return MS_ERR_INVALID;
    *bytes = lookup_layout(log_n, width, ntuples).total;
    return MS_OK;
}

extern "C" int ms_lookup_multiplicities(ms_ctx *c, const uint32_t *program, unsigned nprog, const uint64_t *consts,
                                        unsigned nconsts, const void *const *col_ptrs, const int *col_is_fq, unsigned ncols,
                                        unsigned log_n, unsigned width, unsigned ntuples, void *workspace,
                                        size_t workspace_bytes, void *out, uint64_t *status) {
    if (!c || !program || !consts || nprog == 0 || (ncols && (!col_ptrs || !col_is_fq)) || !workspace || !out || !status)
        return MS_ERR_INVALID;
    if (log_n > kMaxLookupLog) return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: domain too large (at most 2^%u rows)", kMaxLookupLog);
    if (width < 1 || width > kMaxLookupWidth)
        return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: tuples of %u words (1 to %u)", width, kMaxLookupWidth);
    if (ntuples < 1 || ntuples > kMaxLookupTuples)
        return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: %u value tuples (1 to %u)", ntuples, kMaxLookupTuples);
    const LookupWork w = lookup_layout(log_n, width, ntuples);
    if (workspace_bytes < w.total)
        return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: workspace of %zu bytes, %zu needed", workspace_bytes, w.total);
    cudaSetDevice(c->device);
    if (!is_device_ptr(workspace) || !is_device_ptr(out))
        return fail(c, MS_ERR_INVALID, "ms_lookup_multiplicities: workspace and out must be device pointers");
    const u64 n = 1ull << log_n;
    const unsigned nblk = tuple_blocks(n);
    char *wb = (char *)workspace;
    u64 *slots = (u64 *)(wb + w.slots), *sorted = (u64 *)(wb + w.sorted), *st = (u64 *)(wb + w.status);
    u64 *keys0 = (u64 *)(wb + w.keys), *keys1 = keys0 + n;
    u32 *perm0 = (u32 *)(wb + w.perm), *perm1 = perm0 + n;
    u64 *counts = (u64 *)out;

    // 1. evaluate
    int rc = tuple_evaluate(c, "ms_lookup_multiplicities", program, nprog, consts, nconsts, col_ptrs, col_is_fq, ncols, log_n,
                            width + ntuples * (width + 1), slots);
    if (rc) return rc;
    std::vector<u64> init(2 * ntuples + 2);
    for (unsigned k = 0; k < ntuples + 1; k++) {
        init[2 * k] = 0;
        init[2 * k + 1] = ~0ull;
    }
    MS_CUDA(c, cudaMemcpyAsync(st, init.data(), init.size() * 8, cudaMemcpyHostToDevice, c->stream));
    MS_CUDA(c, cudaMemsetAsync(counts, 0, n * 8, c->stream));

    // 2. order the table, then gather its tuples word by word
    const u32 *order;
    if ((rc = tuple_sort(c, slots, width, n, keys0, keys1, perm0, perm1, &order))) return rc;
    for (unsigned k = 0; k < width; k++) {
        tuple_gather_kernel<<<nblk, kTupleThreads, 0, c->stream>>>(slots + (u64)k * n, order, sorted + (u64)k * n, nullptr, n);
        c->launches++;
    }
    MS_CHECK_LAUNCH(c);

    // 3. match
    switch (width) {
        case 1: rc = lookup_match<1>(c, slots, sorted, order, n, ntuples, counts, st); break;
        case 2: rc = lookup_match<2>(c, slots, sorted, order, n, ntuples, counts, st); break;
        case 3: rc = lookup_match<3>(c, slots, sorted, order, n, ntuples, counts, st); break;
        default: rc = lookup_match<4>(c, slots, sorted, order, n, ntuples, counts, st); break;
    }
    if (rc) return rc;

    // 4. write
    lookup_write_kernel<<<nblk, kLookupThreads, 0, c->stream>>>(counts, n);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    MS_CUDA(c, cudaMemcpyAsync(status, st, (2 * ntuples + 2) * 8, cudaMemcpyDeviceToHost, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    return MS_OK;
}
