// extension.cu — the extension columns an AIR declares (ministark_b200/air.py, RunningColumn), built from the base trace.
//
// Every declared column is a first-order recurrence  x_0 = init_k,  x_(i+1) = x_i * mul_k(i) + add_k(i)  whose row maps
// are expressions over the base trace: the running products, running evaluations and running sums the reference builds
// with host loops (src/trace.rs, examples/brainfuck/trace.rs:108-279).  One evaluator program (expr.py,
// compile_extension_program) computes all 2K row values of a row, mul_k into slot 2k and add_k into slot 2k + 1, with
// subexpressions shared between them; the per-point interpreter is eval.cu's (eval.cuh, eval_point) over the trace
// domain (X = g_n^i, Trace(col, off) = column[(i + off) mod n]).  The scan is scan.cu's three phases, with the row maps
// evaluated where scan.cu loads them, so no mul/add column is ever written:
//   1. every CTA evaluates its 2048 rows (8 per thread), composes each column's maps and writes K tile aggregates;
//   2. scan_tile_prefix_kernel turns each column's tile aggregates into exclusive prefixes (K one-CTA launches);
//   3. every CTA evaluates its rows again (keeping the thread's 8 rows of maps in its stack frame), scans the thread
//      aggregates of each column, applies tile prefix ∘ thread prefix to init_k and walks its rows writing x_i or x_(i+1).
// Traffic per row: the base cells the program reads, twice, and K Fq elements written; scratch: K * ceil(n / 2048) maps.
// No decoupled look-back: no CTA ever waits on another.
#include "eval.cuh"
#include "scan.cuh"
#include "../../include/ministark_extension.h"

#include <vector>

namespace ms {

constexpr int kMaxExtColumns = 8;

struct ExtParams {
    // the fields eval_point reads
    const uint4 *prog;
    u32 nprog;
    const u64 *consts;          // [k][3] Montgomery words
    const u64 *const *col_ptr;  // natural-order trace columns, then periodic tables
    u32 fq_words;               // 1: Fq = Fp, 3: Fq = Fq3
    u32 log_m;                  // trace domain n = 2^log_m
    u32 trace_bitrev;           // always 0: natural order
    const u64 *tw_lo, *tw_hi;   // g_n^e two-level table
    u32 hi_len;
    u64 offset;                 // ONE: X is g_n^i
    // the columns
    u32 ncolumns;
    u32 inclusive;              // bit k: column k is inclusive
    u64 init[kMaxExtColumns][3];
    u64 *out;                   // column k at out + k * n * fq_words
    size_t ntiles;
};

template <int L>
__device__ __forceinline__ El<L> ext_value(const u64 *v, bool q) {
    if constexpr (L == 1) {
        (void)q;
        return El<1>{v[0]};
    } else {
        return El<3>{gl::Fq3{v[0], q ? v[1] : 0, q ? v[2] : 0}};
    }
}

// row i's maps: slot 2k = mul_k, slot 2k + 1 = add_k
template <int L>
__device__ __forceinline__ void ext_row(const ExtParams &p, u64 n, u64 i, u64 (*r)[3], El<L> *slot) {
    eval_point(p, n, i, r, [&](u32 s, const u64 *v, bool q) { slot[s] = ext_value<L>(v, q); });
}

template <int L>
__global__ void __launch_bounds__(kScanThreads) ext_aggregate_kernel(const ExtParams p, Map<L> *agg) {
    extern __shared__ unsigned char scan_sm_raw[];
    Map<L> *sm = reinterpret_cast<Map<L> *>(scan_sm_raw);
    const u64 n = 1ull << p.log_m;
    const size_t first = (size_t)blockIdx.x * kScanTile + (size_t)threadIdx.x * kScanPerThread;
    u64 r[kMaxRegs][3];
    El<L> v[2 * kMaxExtColumns];
    Map<L> m[kMaxExtColumns];
    for (u32 k = 0; k < p.ncolumns; k++) m[k] = Map<L>::identity();
    for (int j = 0; j < kScanPerThread; j++) {
        if (first + j >= n) break;
        ext_row<L>(p, n, first + j, r, v);
        for (u32 k = 0; k < p.ncolumns; k++) m[k] = m[k].then(Map<L>{v[2 * k], v[2 * k + 1]});
    }
    for (u32 k = 0; k < p.ncolumns; k++) {
        if (k) __syncthreads();                     // the previous column's total has been read from sm
        block_scan<L, kScanThreads>(m[k], sm);
        if (threadIdx.x == 0) agg[k * p.ntiles + blockIdx.x] = sm[kScanThreads - 1];
    }
}

template <int L>
__global__ void __launch_bounds__(kScanThreads) ext_apply_kernel(const ExtParams p, const Map<L> *prefix) {
    extern __shared__ unsigned char scan_sm_raw[];
    Map<L> *sm = reinterpret_cast<Map<L> *>(scan_sm_raw);
    const u64 n = 1ull << p.log_m;
    const size_t first = (size_t)blockIdx.x * kScanTile + (size_t)threadIdx.x * kScanPerThread;
    u64 r[kMaxRegs][3];
    El<L> v[kScanPerThread][2 * kMaxExtColumns];    // this thread's rows of maps, walked again below
    const int rows = first >= n ? 0 : (n - first < (u64)kScanPerThread ? (int)(n - first) : kScanPerThread);
    for (int j = 0; j < rows; j++) ext_row<L>(p, n, first + j, r, v[j]);
    for (u32 k = 0; k < p.ncolumns; k++) {
        Map<L> m = Map<L>::identity();
        for (int j = 0; j < rows; j++) m = m.then(Map<L>{v[j][2 * k], v[j][2 * k + 1]});
        if (k) __syncthreads();                     // every thread has read the previous column's prefix from sm
        block_scan<L, kScanThreads>(m, sm);
        Map<L> before = prefix[k * p.ntiles + blockIdx.x];
        if (threadIdx.x) before = before.then(sm[threadIdx.x - 1]);
        El<L> x = before.apply(El<L>::load(p.init[k], L, 0));
        u64 *out = p.out + (size_t)k * n * L;
        const bool inclusive = (p.inclusive >> k) & 1;
        for (int j = 0; j < rows; j++) {
            if (!inclusive) x.store(out, first + j);
            x = Map<L>{v[j][2 * k], v[j][2 * k + 1]}.apply(x);
            if (inclusive) x.store(out, first + j);
        }
    }
}

template <int L>
static int ext_run(ms_ctx *c, const ExtParams &p) {
    void *agg;
    if (int rc = scratch_get(c, 2, p.ncolumns * p.ntiles * sizeof(Map<L>), &agg)) return rc;
    static bool attr[64][2] = {{false}};
    int dev = 0;
    cudaGetDevice(&dev);
    const size_t sm1 = kScanThreads * sizeof(Map<L>), sm2 = 1024 * sizeof(Map<L>);
    if (dev >= 0 && dev < 64 && !attr[dev][L == 3]) {
        MS_CUDA(c, cudaFuncSetAttribute(scan_tile_prefix_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
        attr[dev][L == 3] = true;
    }
    ext_aggregate_kernel<L><<<(unsigned)p.ntiles, kScanThreads, sm1, c->stream>>>(p, (Map<L> *)agg);
    for (u32 k = 0; k < p.ncolumns; k++)
        scan_tile_prefix_kernel<L><<<1, 1024, sm2, c->stream>>>((Map<L> *)agg + k * p.ntiles, p.ntiles);
    ext_apply_kernel<L><<<(unsigned)p.ntiles, kScanThreads, sm1, c->stream>>>(p, (const Map<L> *)agg);
    c->launches += 2 + p.ncolumns;
    MS_CHECK_LAUNCH(c);
    return MS_OK;
}

}  // namespace ms

using namespace ms;

extern "C" int ms_extension_columns(ms_ctx *c, const uint32_t *program, unsigned nprog, const uint64_t *consts, unsigned nconsts,
                                    const void *const *col_ptrs, const int *col_is_fq, unsigned ncols, int fq_field, unsigned log_n,
                                    unsigned ncolumns, const uint64_t *init, const int *inclusive, void *out) {
    if (!c || !program || !consts || nprog == 0 || (ncols && (!col_ptrs || !col_is_fq)) || !init || !inclusive || !out)
        return MS_ERR_INVALID;
    if (fq_field != MS_FIELD_FP && fq_field != MS_FIELD_FQ3) return fail(c, MS_ERR_INVALID, "ms_extension_columns: bad Fq field id");
    if (log_n > 32) return fail(c, MS_ERR_INVALID, "ms_extension_columns: domain too large");
    if (ncolumns == 0 || ncolumns > (unsigned)kMaxExtColumns)
        return fail(c, MS_ERR_INVALID, "ms_extension_columns: %u columns (1 to %d)", ncolumns, kMaxExtColumns);
    for (unsigned k = 0; k < ncolumns * (unsigned)fq_field; k++)
        if (init[k] >= gl::P) return fail(c, MS_ERR_INVALID, "ms_extension_columns: non-canonical init of column %u", k / fq_field);
    cudaSetDevice(c->device);
    std::vector<const u64 *> cols;
    std::vector<int> isq;
    for (unsigned k = 0; k < ncols; k++) {
        if (!col_ptrs[k] || !is_device_ptr(col_ptrs[k])) return fail(c, MS_ERR_INVALID, "ms_extension_columns: column %u is not a device pointer", k);
        cols.push_back((const u64 *)col_ptrs[k]);
        isq.push_back(col_is_fq[k] ? 1 : 0);
    }
    if (!is_device_ptr(out)) return fail(c, MS_ERR_INVALID, "ms_extension_columns: out must be a device pointer");
    int rc = validate_program(c, "ms_extension_columns", program, nprog, nconsts, isq, log_n, 0, 2 * ncolumns);
    if (rc) return rc;
    void *meta;
    const size_t prog_bytes = (size_t)nprog * 16, const_bytes = (size_t)nconsts * 24, ptr_bytes = (size_t)ncols * 8;
    if ((rc = scratch_get(c, 3, prog_bytes + const_bytes + ptr_bytes + 64, &meta))) return rc;
    char *m = (char *)meta;
    MS_CUDA(c, cudaMemcpyAsync(m, program, prog_bytes, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaMemcpyAsync(m + prog_bytes, consts, const_bytes, cudaMemcpyDefault, c->stream));
    if (ptr_bytes) MS_CUDA(c, cudaMemcpyAsync(m + prog_bytes + const_bytes, cols.data(), ptr_bytes, cudaMemcpyHostToDevice, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));   // the host buffers may be temporaries of the caller
    ExtParams p;
    if ((rc = ntt_plan_tables(c, log_n, &p.tw_lo, &p.tw_hi, &p.hi_len))) return rc;
    p.prog = (const uint4 *)m;
    p.nprog = nprog;
    p.consts = (const u64 *)(m + prog_bytes);
    p.col_ptr = (const u64 *const *)(m + prog_bytes + const_bytes);
    p.fq_words = (u32)fq_field;
    p.log_m = log_n;
    p.trace_bitrev = 0;
    p.offset = gl::ONE;
    p.ncolumns = ncolumns;
    p.inclusive = 0;
    for (unsigned k = 0; k < (unsigned)kMaxExtColumns; k++) {
        if (k < ncolumns && inclusive[k]) p.inclusive |= 1u << k;
        for (int w = 0; w < 3; w++) p.init[k][w] = (k < ncolumns && w < fq_field) ? init[k * fq_field + w] : 0;
    }
    p.out = (u64 *)out;
    p.ntiles = (((size_t)1 << log_n) + kScanTile - 1) / kScanTile;
    return fq_field == MS_FIELD_FP ? ext_run<1>(c, p) : ext_run<3>(c, p);
}
