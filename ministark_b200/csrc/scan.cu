// scan.cu — running products / running evaluations over trace rows as a parallel scan.
//
// The reference builds its extension columns with one sequential loop per column
// (examples/brainfuck/trace.rs:108-279: permutation running products  p <- p * (alpha - a*ip - b*ci - c*ni),
// evaluation arguments  e <- e * gamma + v), and the fib trace with a serial recurrence
// (examples/fib/main.rs:175-222).  All of them are instances of
//        x_0 = init,      x_(i+1) = x_i * a_i + b_i
// and the affine maps  x -> x*a + b  compose associatively:  (a1,b1) then (a2,b2) = (a1*a2, b1*a2 + b2).
// SURVEY.md §8(f) rank 3.  Three phases, all on the context's stream:
//   1. tile aggregates: every CTA composes the maps of its 2048 rows (thread-serial over 8 rows, then a
//      Kogge-Stone scan over the 256 thread aggregates in shared memory);
//   2. one CTA turns the tile aggregates into exclusive tile prefixes;
//   3. every CTA re-reads its tile, scans the thread aggregates again, applies tile prefix ∘ thread prefix
//      to `init` and walks its 8 rows writing x_i (exclusive) or x_(i+1) (inclusive).
// Traffic: a and b are read twice, out written once; the arithmetic is Fq3 (or Fp) multiplications.
#include "scan.cuh"

namespace ms {

struct ScanArgs {
    const u64 *a;      // n elements of field fa, or nullptr
    const u64 *b;      // n elements of field fb, or nullptr
    int fa, fb;
    u64 a_const[3];    // used when a == nullptr
    u64 init[3];
    size_t n;
    int inclusive;
    u64 *out;
};

template <int L>
__device__ __forceinline__ Map<L> row_map(const ScanArgs &s, const El<L> &ac, size_t i) {
    Map<L> m;
    m.a = s.a ? El<L>::load(s.a, s.fa, i) : ac;
    m.b = s.b ? El<L>::load(s.b, s.fb, i) : El<L>::zero();
    return m;
}

template <int L>
__global__ void __launch_bounds__(kScanThreads) scan_tile_aggregate_kernel(ScanArgs s, Map<L> *agg) {
    extern __shared__ unsigned char scan_sm_raw[];
    Map<L> *sm = reinterpret_cast<Map<L> *>(scan_sm_raw);
    const El<L> ac = El<L>::load(s.a_const, L, 0);
    const size_t first = (size_t)blockIdx.x * kScanTile + (size_t)threadIdx.x * kScanPerThread;
    Map<L> m = Map<L>::identity();
    for (int k = 0; k < kScanPerThread; k++)
        if (first + k < s.n) m = m.then(row_map<L>(s, ac, first + k));
    block_scan<L, kScanThreads>(m, sm);
    if (threadIdx.x == 0) agg[blockIdx.x] = sm[kScanThreads - 1];
}

template <int L>
__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(ScanArgs s, const Map<L> *prefix) {
    extern __shared__ unsigned char scan_sm_raw[];
    Map<L> *sm = reinterpret_cast<Map<L> *>(scan_sm_raw);
    const El<L> ac = El<L>::load(s.a_const, L, 0);
    const size_t first = (size_t)blockIdx.x * kScanTile + (size_t)threadIdx.x * kScanPerThread;
    Map<L> m = Map<L>::identity();
    for (int k = 0; k < kScanPerThread; k++)
        if (first + k < s.n) m = m.then(row_map<L>(s, ac, first + k));
    block_scan<L, kScanThreads>(m, sm);
    Map<L> before = prefix[blockIdx.x];
    if (threadIdx.x) before = before.then(sm[threadIdx.x - 1]);
    El<L> x = before.apply(El<L>::load(s.init, L, 0));
    for (int k = 0; k < kScanPerThread; k++) {
        const size_t i = first + k;
        if (i >= s.n) break;
        if (!s.inclusive) x.store(s.out, i);
        x = row_map<L>(s, ac, i).apply(x);
        if (s.inclusive) x.store(s.out, i);
    }
}

template <int L>
static int scan_run(ms_ctx *c, const ScanArgs &s) {
    const size_t ntiles = (s.n + kScanTile - 1) / kScanTile;
    void *agg;
    if (int rc = scratch_get(c, 2, ntiles * sizeof(Map<L>), &agg)) return rc;
    static bool attr[64][2] = {{false}};
    int dev = 0;
    cudaGetDevice(&dev);
    const size_t sm1 = kScanThreads * sizeof(Map<L>), sm2 = 1024 * sizeof(Map<L>);
    if (dev >= 0 && dev < 64 && !attr[dev][L == 3]) {
        MS_CUDA(c, cudaFuncSetAttribute(scan_tile_prefix_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
        attr[dev][L == 3] = true;
    }
    scan_tile_aggregate_kernel<L><<<(unsigned)ntiles, kScanThreads, sm1, c->stream>>>(s, (Map<L> *)agg);
    scan_tile_prefix_kernel<L><<<1, 1024, sm2, c->stream>>>((Map<L> *)agg, ntiles);
    scan_apply_kernel<L><<<(unsigned)ntiles, kScanThreads, sm1, c->stream>>>(s, (const Map<L> *)agg);
    c->launches += 3;
    MS_CHECK_LAUNCH(c);
    return MS_OK;
}

}  // namespace ms

using namespace ms;

extern "C" int ms_scan_affine(ms_ctx *c, int field, const void *a, int a_field, const uint64_t *a_const, const void *b, int b_field,
                              size_t n, const uint64_t *init, int inclusive, void *out) {
    if (!c || !init || !out) return MS_ERR_INVALID;
    if (field != 1 && field != 3) return fail(c, MS_ERR_INVALID, "ms_scan_affine: bad field id");
    if (a && a_field != 1 && a_field != field) return fail(c, MS_ERR_INVALID, "ms_scan_affine: a must be Fp or the output field");
    if (b && b_field != 1 && b_field != field) return fail(c, MS_ERR_INVALID, "ms_scan_affine: b must be Fp or the output field");
    if (!a && !a_const) return fail(c, MS_ERR_INVALID, "ms_scan_affine: need a or a_const");
    if (n == 0) return MS_OK;
    cudaSetDevice(c->device);
    Staged A(c, a, a ? n * a_field * 8 : 0, true, false);
    if (A.rc) return A.rc;
    Staged B(c, b, b ? n * b_field * 8 : 0, true, false);
    if (B.rc) return B.rc;
    Staged O(c, out, n * field * 8, false, true);
    if (O.rc) return O.rc;
    ScanArgs s;
    s.a = a ? A.as<u64>() : nullptr;
    s.b = b ? B.as<u64>() : nullptr;
    s.fa = a_field;
    s.fb = b_field;
    for (int i = 0; i < 3; i++) {
        s.a_const[i] = (a_const && i < field) ? a_const[i] : (i == 0 && !a_const ? gl::ONE : 0);
        s.init[i] = i < field ? init[i] : 0;
        if (s.a_const[i] >= gl::P || s.init[i] >= gl::P) return fail(c, MS_ERR_INVALID, "ms_scan_affine: non-canonical constant");
    }
    s.n = n;
    s.inclusive = inclusive;
    s.out = O.as<u64>();
    int rc = field == 1 ? scan_run<1>(c, s) : scan_run<3>(c, s);
    if (rc) return rc;
    if ((rc = A.finish())) return rc;
    if ((rc = B.finish())) return rc;
    return O.finish();
}
