// scan.cuh — the affine maps x -> x*a + b over Fp (L = 1) or Fq3 (L = 3), their block-wide scan and the one-CTA scan of
// tile aggregates: the pieces shared by the scan of given columns (scan.cu, ms_scan_affine) and the scan of declared
// extension columns (extension.cu, ms_extension_columns).  (a1,b1) then (a2,b2) = (a1*a2, b1*a2 + b2).
#pragma once
#include "ctx.cuh"

namespace ms {

template <int L>
struct El;
template <>
struct El<1> {
    u64 v;
    __device__ __forceinline__ static El one() { return El{gl::ONE}; }
    __device__ __forceinline__ static El zero() { return El{0}; }
    __device__ __forceinline__ static El load(const u64 *p, int f, size_t i) { (void)f; return El{p[i]}; }
    __device__ __forceinline__ void store(u64 *p, size_t i) const { p[i] = v; }
    __device__ __forceinline__ El mul(El o) const { return El{gl::mul(v, o.v)}; }
    __device__ __forceinline__ El add(El o) const { return El{gl::add(v, o.v)}; }
};
template <>
struct El<3> {
    gl::Fq3 v;
    __device__ __forceinline__ static El one() { return El{gl::Fq3{gl::ONE, 0, 0}}; }
    __device__ __forceinline__ static El zero() { return El{gl::Fq3{0, 0, 0}}; }
    __device__ __forceinline__ static El load(const u64 *p, int f, size_t i) {
        return f == 1 ? El{gl::Fq3{p[i], 0, 0}} : El{gl::Fq3{p[3 * i], p[3 * i + 1], p[3 * i + 2]}};
    }
    __device__ __forceinline__ void store(u64 *p, size_t i) const { p[3 * i] = v.c0; p[3 * i + 1] = v.c1; p[3 * i + 2] = v.c2; }
    __device__ __forceinline__ El mul(El o) const { return El{gl::mul(v, o.v)}; }
    __device__ __forceinline__ El add(El o) const { return El{gl::add(v, o.v)}; }
};

template <int L>
struct Map {      // x -> x*a + b
    El<L> a, b;
    __device__ __forceinline__ static Map identity() { return Map{El<L>::one(), El<L>::zero()}; }
    // this first, then o
    __device__ __forceinline__ Map then(const Map &o) const { return Map{a.mul(o.a), b.mul(o.a).add(o.b)}; }
    __device__ __forceinline__ El<L> apply(El<L> x) const { return x.mul(a).add(b); }
};

constexpr int kScanThreads = 256, kScanPerThread = 8, kScanTile = kScanThreads * kScanPerThread;

// inclusive Kogge-Stone scan of one Map per thread; returns this thread's inclusive value, total in sm[T-1]
template <int L, int T>
__device__ __forceinline__ Map<L> block_scan(Map<L> mine, Map<L> *sm) {
    const int tid = threadIdx.x;
    sm[tid] = mine;
    __syncthreads();
#pragma unroll 1
    for (int d = 1; d < T; d <<= 1) {
        Map<L> prev;
        const bool on = tid >= d;
        if (on) prev = sm[tid - d];
        __syncthreads();
        if (on) {
            mine = prev.then(mine);
            sm[tid] = mine;
        }
        __syncthreads();
    }
    return mine;
}

// exclusive prefixes of the tile aggregates, in place (one CTA; each thread owns a contiguous chunk)
template <int L>
__global__ void __launch_bounds__(1024) scan_tile_prefix_kernel(Map<L> *agg, size_t ntiles) {
    extern __shared__ unsigned char scan_sm_raw[];
    Map<L> *sm = reinterpret_cast<Map<L> *>(scan_sm_raw);
    const size_t chunk = (ntiles + 1023) / 1024;
    const size_t lo = (size_t)threadIdx.x * chunk, hi = lo + chunk < ntiles ? lo + chunk : ntiles;
    Map<L> m = Map<L>::identity();
    for (size_t t = lo; t < hi; t++) m = m.then(agg[t]);
    block_scan<L, 1024>(m, sm);
    Map<L> run = threadIdx.x ? sm[threadIdx.x - 1] : Map<L>::identity();
    for (size_t t = lo; t < hi; t++) {
        const Map<L> cur = agg[t];
        agg[t] = run;
        run = run.then(cur);
    }
}

}  // namespace ms
