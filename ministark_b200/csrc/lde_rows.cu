// lde_rows.cu — chosen rows of a bit-reversed coset LDE, straight from the coefficients.
//
// Row r of ms_lde_batch(..., bitrev_out = 1) holds P_c(x_r), x_r = offset * g_N^bitrev(r), for every column c.  The
// streaming prover keeps coefficients and not the LDE, so its query phase asks for a few dozen such rows.  x_r is a
// BASE-field point: an Fp column needs only Fp products and an Fq3 column Fq3 x Fp (3 products per coefficient), where
// ms_poly_eval (Fq3 points) spends an Fq3 x Fq3 product (6) on every coefficient of every column.
//
// Pass 1: block (span b, column c, point group) stages the span's coefficients in shared memory, one tile of L at a time,
// and evaluates them at up to 256 / G points: G threads per point, thread g running Horner in y = x^G over the
// coefficients j = g (mod G) and weighting its sum by x^g, so consecutive threads read consecutive words.  The block's G
// sums give the span's value relative to its first coefficient.  Every coefficient leaves HBM once per point group,
// i.e. once for up to 64 points.
// Pass 2: per (column, point), the span values are a polynomial in x^(span length): strided Horner per thread, x^t
// weights, tree sum.
#include "ctx.cuh"
#include "../../include/ministark_stream.h"

#include <vector>

namespace ms {

using gl::Fq3;

constexpr int kLrThreads = 256;
template <int F> struct LrChunk;
template <> struct LrChunk<1> { static constexpr int L = 2048; };   // 16 KiB of shared memory
template <> struct LrChunk<3> { static constexpr int L = 1024; };   // 24 KiB

template <int F> struct El;
template <> struct El<1> {
    u64 v;
    __device__ __forceinline__ static El zero() { return El{0}; }
    __device__ __forceinline__ static El load(const u64 *p) { return El{p[0]}; }
    __device__ __forceinline__ void store(u64 *p) const { p[0] = v; }
    __device__ __forceinline__ El mul(u64 x) const { return El{gl::mul(v, x)}; }
    __device__ __forceinline__ El add(El o) const { return El{gl::add(v, o.v)}; }
};
template <> struct El<3> {
    Fq3 v;
    __device__ __forceinline__ static El zero() { return El{gl::fq3(0)}; }
    __device__ __forceinline__ static El load(const u64 *p) { return El{Fq3{p[0], p[1], p[2]}}; }
    __device__ __forceinline__ void store(u64 *p) const { p[0] = v.c0; p[1] = v.c1; p[2] = v.c2; }
    __device__ __forceinline__ El mul(u64 x) const { return El{gl::mul(v, x)}; }
    __device__ __forceinline__ El add(El o) const { return El{gl::add(v, o.v)}; }
};

// partials[(col * npoints + k) * nspans + span] (F words each) = sum_{j < R L} c[span * R L + j] * x_k^j, the span's R
// tiles of L coefficients staged one after the other (highest first: each thread's Horner runs on across tiles)
template <int F>
__global__ void __launch_bounds__(kLrThreads) lde_rows_chunk_kernel(const u64 *__restrict__ coeffs, size_t col_stride_words,
                                                                     size_t n, unsigned tiles_per_span, const u64 *__restrict__ points,
                                                                     unsigned npoints, unsigned log_g, u64 *__restrict__ partials) {
    constexpr int L = LrChunk<F>::L;
    __shared__ u64 tile[L * F];
    __shared__ u64 red[kLrThreads * F];
    const unsigned t = threadIdx.x, span = blockIdx.x, col = blockIdx.y, nspans = gridDim.x;
    const unsigned G = 1u << log_g, per_block = kLrThreads >> log_g;
    const unsigned g = t & (G - 1);
    const unsigned k = blockIdx.z * per_block + (t >> log_g);
    const bool live = k < npoints;
    const u64 x = live ? points[k] : gl::ONE;
    const u64 y = gl::pow(x, (u64)G);
    const u64 *src_col = coeffs + (size_t)col * col_stride_words;
    const size_t ntiles = (n + L - 1) / L, first = (size_t)span * tiles_per_span;
    const size_t end = first + tiles_per_span < ntiles ? first + tiles_per_span : ntiles;
    El<F> acc = El<F>::zero();
    for (size_t tl = end; tl-- > first;) {
        const size_t start = tl * L;
        const size_t avail = (n - start < (size_t)L ? n - start : (size_t)L) * F;
        const u64 *src = src_col + start * F;
        __syncthreads();                                   // the previous tile is consumed
        for (unsigned w = t; w < L * F; w += kLrThreads) tile[w] = w < avail ? src[w] : 0;
        __syncthreads();
#pragma unroll 4
        for (int j = L / (int)G - 1; j >= 0; j--) acc = acc.mul(y).add(El<F>::load(tile + ((size_t)j * G + g) * F));
    }
    acc = acc.mul(gl::pow(x, (u64)g));
    acc.store(red + t * F);
    __syncthreads();
    for (unsigned s = G / 2; s > 0; s >>= 1) {   // the G consecutive threads of one point
        if (g < s) El<F>::load(red + t * F).add(El<F>::load(red + (t + s) * F)).store(red + t * F);
        __syncthreads();
    }
    if (live && g == 0) El<F>::load(red + t * F).store(partials + (((size_t)col * npoints + k) * nspans + span) * F);
}

// out[(k * ncols + col) * F ..] = sum_b partials[(col * npoints + k) * nspans + b] * x_k^(b span_len)
template <int F>
__global__ void __launch_bounds__(kLrThreads) lde_rows_combine_kernel(const u64 *__restrict__ partials, unsigned nspans,
                                                                       u64 span_len, const u64 *__restrict__ points,
                                                                       unsigned npoints, unsigned ncols, u64 *__restrict__ out) {
    __shared__ u64 red[kLrThreads * F];
    const unsigned t = threadIdx.x, k = blockIdx.x, col = blockIdx.y;
    const u64 X = gl::pow(points[k], span_len);
    const u64 z = gl::pow(X, (u64)kLrThreads);
    const u64 *p = partials + ((size_t)col * npoints + k) * nspans * F;
    El<F> acc = El<F>::zero();
    if (t < nspans) {
        const unsigned last = (nspans - 1 - t) / kLrThreads;
        for (int m = (int)last; m >= 0; m--) acc = acc.mul(z).add(El<F>::load(p + ((size_t)m * kLrThreads + t) * F));
        acc = acc.mul(gl::pow(X, (u64)t));
    }
    acc.store(red + t * F);
    __syncthreads();
    for (unsigned s = kLrThreads / 2; s > 0; s >>= 1) {
        if (t < s) El<F>::load(red + t * F).add(El<F>::load(red + (t + s) * F)).store(red + t * F);
        __syncthreads();
    }
    if (t == 0) El<F>::load(red).store(out + ((size_t)k * ncols + col) * F);
}

// spans of R tiles: about 256 spans per column, so the partial sums stay small and the grid stays full
template <int F>
static unsigned lr_tiles_per_span(size_t n) {
    const size_t ntiles = (n + LrChunk<F>::L - 1) / LrChunk<F>::L;
    return (unsigned)((ntiles + 255) / 256);
}
template <int F>
static int lde_rows_run(ms_ctx *c, const u64 *coeffs, size_t col_stride_elems, unsigned ncols, size_t n, const u64 *dpts,
                        unsigned npoints, u64 *partials, u64 *out) {
    constexpr int L = LrChunk<F>::L;
    const unsigned R = lr_tiles_per_span<F>(n);
    const size_t ntiles = (n + L - 1) / L;
    const unsigned nspans = (unsigned)((ntiles + R - 1) / R);
    // G threads per point: as many points per block as there are (up to 64), the rest of the block splits each tile
    unsigned kp = 1;
    while (kp < npoints && kp < 64) kp <<= 1;
    unsigned log_g = 0;
    while ((kLrThreads >> log_g) > kp) log_g++;
    const unsigned per_block = kLrThreads >> log_g;
    dim3 g1(nspans, ncols, (npoints + per_block - 1) / per_block);
    lde_rows_chunk_kernel<F><<<g1, kLrThreads, 0, c->stream>>>(coeffs, col_stride_elems * F, n, R, dpts, npoints, log_g, partials);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    dim3 g2(npoints, ncols);
    lde_rows_combine_kernel<F><<<g2, kLrThreads, 0, c->stream>>>(partials, nspans, (u64)R * L, dpts, npoints, ncols, out);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    return MS_OK;
}

static u64 lr_root_of_unity(unsigned log_n) {
    u64 r = gl::to_mont(1753635133440165772ULL);
    for (unsigned i = log_n; i < 32; i++) r = gl::sqr(r);
    return r;
}

}  // namespace ms

using namespace ms;

extern "C" int ms_lde_rows(ms_ctx *c, int field, const void *coeffs, size_t col_stride_elems, unsigned ncols, unsigned log_n,
                           unsigned log_blowup, uint64_t offset_mont, const uint64_t *positions, unsigned npos, void *out) {
    if (!c || !coeffs || !positions || !out) return MS_ERR_INVALID;
    if (field != MS_FIELD_FP && field != MS_FIELD_FQ3) return fail(c, MS_ERR_INVALID, "unknown field id %d", field);
    if (log_n + log_blowup > 32) return fail(c, MS_ERR_INVALID, "ms_lde_rows: log_n + log_blowup > 32");
    if (offset_mont >= gl::P || offset_mont == 0) return fail(c, MS_ERR_INVALID, "offset must be a non-zero canonical word");
    if (ncols == 0 || ncols > 65535 || npos > 65535) return fail(c, MS_ERR_INVALID, "ms_lde_rows: bad sizes");
    const size_t n = (size_t)1 << log_n;
    if (ncols > 1 && col_stride_elems < n) return fail(c, MS_ERR_INVALID, "ms_lde_rows: stride < 2^log_n");
    if (npos == 0) return MS_OK;
    const unsigned log_N = log_n + log_blowup;
    const u64 N = (u64)1 << log_N;
    // the points offset * g_N^bitrev(pos): a handful, built on the host
    std::vector<u64> pos(positions, positions + npos), pts(npos);
    const u64 gN = lr_root_of_unity(log_N);
    for (unsigned k = 0; k < npos; k++) {
        if (pos[k] >= N) return fail(c, MS_ERR_INVALID, "ms_lde_rows: row %llu out of range", (unsigned long long)pos[k]);
        u64 r = 0, v = pos[k];
        for (unsigned b = 0; b < log_N; b++, v >>= 1) r = (r << 1) | (v & 1);
        pts[k] = gl::mul(offset_mont, gl::pow(gN, r));
    }
    Staged in(c, coeffs, ((size_t)(ncols - 1) * col_stride_elems + n) * field * 8, true, false);
    if (in.rc) return in.rc;
    Staged o(c, out, (size_t)npos * ncols * field * 8, false, true);
    if (o.rc) return o.rc;
    const size_t L = field == 1 ? LrChunk<1>::L : LrChunk<3>::L;
    const size_t R = field == 1 ? lr_tiles_per_span<1>(n) : lr_tiles_per_span<3>(n);
    const size_t nspans = ((n + L - 1) / L + R - 1) / R;
    void *scr;
    int rc = scratch_get(c, 3, (npos + (size_t)ncols * npos * nspans * field) * 8, &scr);
    if (rc) return rc;
    u64 *dpts = (u64 *)scr, *partials = dpts + npos;
    MS_CUDA(c, cudaMemcpyAsync(dpts, pts.data(), (size_t)npos * 8, cudaMemcpyHostToDevice, c->stream));
    rc = field == 1 ? lde_rows_run<1>(c, in.as<u64>(), col_stride_elems, ncols, n, dpts, npos, partials, o.as<u64>())
                    : lde_rows_run<3>(c, in.as<u64>(), col_stride_elems, ncols, n, dpts, npos, partials, o.as<u64>());
    if (rc) return rc;
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if ((rc = in.finish())) return rc;
    return o.finish();
}
