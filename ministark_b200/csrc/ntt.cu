// ntt.cu — multi-pass radix-2^k number-theoretic transform over Goldilocks for sm_90a.
//
// Replaces the reference's FftSingle / FftMultiple / BitReverse / MulAssign kernel chain
// (gpu/src/metal/fft_shaders.h.metal:13-101, encoded by gpu/src/plan.rs:427-450), which
// makes log2(n)-10 global passes + a threadgroup pass + a bit-reverse pass + a scale pass.
// Here a 2^24-point column takes THREE global passes in total and nothing else:
//
//   N = R_1 * R_2 * ... * R_m  (digits of <= 8 bits; a single digit of <= 12 bits if N <= 4096)
//   pass k: each CTA stages a [R_k][W] tile (<= 4096 elements) in shared memory, runs W
//           R_k-point sub-NTTs with radix-16/8/4/2 in-register butterflies (DIT networks,
//           lazy 64-bit arithmetic, twiddles of the in-register levels are compile-time
//           constants), multiplies by the inter-pass twiddles omega_{N_k}^(i_k * lower) generated
//           per thread as a geometric progression from a two-level table, and writes back.
//   * coset scaling (offset^j on the way in) and inverse scaling (n^-1 offset^-i on the way out)
//     are fused into the first / last pass; the reference's extra MulAssign pass
//     (ScaleAndNormalizeGpuStage, gpu/src/stage.rs:235-277) and its CPU-built n-entry scale
//     vector disappear.
//   * natural-order output: the last pass writes transposed (digit-reversed) tiles, so no
//     BitReverse pass.  bit-reversed output (what commitments use, src/matrix.rs:225-234):
//     every pass is position-preserving and the digit is left bit-reversed, so the
//     reference's GPU bit-reverse followed by a CPU bit-reverse vanish as well.
//
// Integer ALU bound (64-bit modular arithmetic on 32-bit lanes); tensor cores do not apply.
#include "ntt.cuh"

#include "dft.cuh"

#include <cstdio>
#include <type_traits>

namespace msntt {

using namespace gl;

// ------------------------------------------------------------------------------------------
__device__ __forceinline__ u32 brev_rt(u32 k, int bits) { return bits ? (__brev(k) >> (32 - bits)) : 0; }

__device__ __forceinline__ u32 padi(u32 i) { return i + (i >> 4); }

struct TileCtx {
    u64 in_base, out_base, low_base;
    const u64 *sc_lo, *sc_hi;
    const u64 *pre_tab;
    const u64 *sm2;   // last-step multiplier tile prefetched into shared memory (or nullptr)
    u64 pre_step;
    u64 *dst2;        // second destination of this CTA's outputs (LDE scatter: local copy of a block) or nullptr
};

__device__ __forceinline__ void cp_async8(u64 *smem_dst, const u64 *gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ u64 tw_lookup(const u64 *lo, const u64 *hi, u32 hi_len, u64 e) {
    u64 t = lo[e & 4095];
    if (hi_len > 1) t = mul(hi[e >> 12], t);
    return t;
}

// One radix-2^B step of the CTA-level sub-NTT.  f = bit position of the field inside the linear
// tile index (r * W + c); lbits = number of r-bits below the field; B1/B2 describe the fields
// already transformed (needed by the last step only).  LW >= 0 fixes log2(W) at compile time so all
// shared-memory offsets fold into immediates.
//   din : the first step reads its 16 inputs straight from global memory (lane-contiguous tiles), the
//         coset pre-scale factor is applied on the way in;
//   dout: the last step writes its 16 outputs straight to global memory.
template <int B, bool INV, bool FIRST, bool LAST, int B1, int B2, int LOGR, int LW>
__device__ __forceinline__ void do_step(u64 *sm, const PassParams &p, const Tables &tb, const TileCtx &tc, const int f,
                                        const int lbits, const bool din, const bool dout, const u64 *__restrict__ src,
                                        u64 *__restrict__ dst) {
    constexpr int RAD = 1 << B;
    constexpr int G = kElemsPerThread >> B;
    const int lw = LW >= 0 ? LW : (int)p.log_w;
    const u32 nthreads = blockDim.x, tid = threadIdx.x;
    const u32 wmask = (1u << lw) - 1;
    const u32 es = p.estride;
    // compile-time tile geometry (LW >= 0) is only dispatched when every in-column word offset fits 32 bits
    // (launch_pass checks): offsets then cost one IMAD.WIDE on the FMA pipe instead of 64-bit ALU chains
    using idx_t = typename std::conditional<(LW >= 0), u32, u64>::type;
#pragma unroll 1
    for (int gi = 0; gi < G; gi++) {
        const u32 g = gi * nthreads + tid;
        const u32 i0 = ((g >> f) << (f + B)) | (g & ((1u << f) - 1));
        const u32 c = i0 & wmask, rpos0 = i0 >> lw;
        u64 x[RAD];
        if (FIRST && din) {
            // rows rpos0 + (K << (f - lw)), lane c: 16 coalesced global loads (2 x 128 B per warp each)
            const u64 e0 = tc.in_base + (u64)rpos0 * p.in_rs + (u64)c * p.in_cs;
            const idx_t stj = (idx_t)(p.in_rs << (f - lw));
            const u64 *sp = src + e0 * es;
            const idx_t stw = stj * (idx_t)es;
            if (p.has_pre && tc.pre_tab) {
                const u64 *tp = tc.pre_tab + e0;
                u64 tw[RAD];
                static_for<0, RAD>([&](auto K) {
                    x[K] = sp[(idx_t)K * stw];
                    tw[K] = __ldg(tp + (idx_t)K * stj);
                });
                static_for<0, RAD>([&](auto K) { x[K] = mul(x[K], tw[K]); });
            } else {
                static_for<0, RAD>([&](auto K) { x[K] = sp[(idx_t)K * stw]; });
            }
        } else {
            static_for<0, RAD>([&](auto K) { x[K] = sm[padi(i0 + ((u32)K << f))]; });
        }

        if (FIRST && p.has_pre && !tc.pre_tab) {
            // no full table: x[k] *= q^(in index), in index = A + k * (in_rs << (f - lw)), as a progression
            u64 A = tc.in_base + (u64)rpos0 * p.in_rs + (u64)c * p.in_cs;
            u64 t = tw_lookup(tc.sc_lo, tc.sc_hi, p.hi_len, A);
            static_for<0, RAD>([&](auto K) {
                x[K] = mul(x[K], t);
                if constexpr (decltype(K)::value + 1 < RAD) t = mul(t, tc.pre_step);
            });
        }

        dft_regs<B, INV>(x);

        u32 iR0 = 0;
        if (!LAST) {
            // inner twiddle omega_{R_m}^(kappa * rlow), R_m = 2^(lbits+B)
            const u32 rlow = rpos0 & ((1u << lbits) - 1);
            const int sh = 12 - lbits - B;
            static_for<1, RAD>([&](auto KAP) {
                constexpr int q = brev_c(decltype(KAP)::value, B);
                x[q] = mul(x[q], __ldg(tb.t4096 + (((u32)KAP * rlow) << sh)));
            });
            x[0] = canon(x[0]);
        } else {
            // output index of this pass's digit contributed by the earlier fields
            if (B1 > 0) {
                u32 v1 = rpos0 >> (LOGR - B1);
                iR0 = p.bitrev_digit ? brev_rt(v1, B1) : v1;
            }
            if (B2 > 0) {
                u32 v2 = (rpos0 >> (LOGR - B1 - B2)) & ((1u << B2) - 1);
                iR0 |= (p.bitrev_digit ? brev_rt(v2, B2) : v2) << B1;
            }
            constexpr int SH = B1 + B2;  // kappa of this field enters i_R shifted by SH
            bool scaled = false;
            if (tc.sm2) {
                // inter-pass twiddle / inverse post-scale from the prefetched tile: row = output index
                static_for<0, RAD>([&](auto KAP) {
                    constexpr int q = brev_c(decltype(KAP)::value, B);
                    const u32 row = iR0 + ((u32)KAP << SH);
                    x[q] = mul(x[q], tc.sm2[padi((row << lw) + c)]);
                });
                scaled = true;
            } else if (p.has_outer) {
                const u64 lower = tc.low_base + (u64)c * p.low_cs;
                const u64 A = ((u64)iR0 * lower * p.outer_mult) & p.n_mask;
                const u64 Bs = ((lower << SH) * p.outer_mult) & p.n_mask;
                u64 t = tw_lookup(tb.tw_lo, tb.tw_hi, p.hi_len, A);
                const u64 st = tw_lookup(tb.tw_lo, tb.tw_hi, p.hi_len, Bs);
                static_for<0, RAD>([&](auto KAP) {
                    constexpr int q = brev_c(decltype(KAP)::value, B);
                    x[q] = mul(x[q], t);
                    if constexpr (decltype(KAP)::value + 1 < RAD) t = mul(t, st);
                });
                scaled = true;
            } else if (p.has_post) {
                const u64 A = tc.out_base + (u64)c * p.out_cs + (u64)iR0 * p.out_rs;
                u64 t = tw_lookup(tc.sc_lo, tc.sc_hi, p.hi_len, A);
                static_for<0, RAD>([&](auto KAP) {
                    constexpr int q = brev_c(decltype(KAP)::value, B);
                    x[q] = mul(x[q], t);
                    if constexpr (decltype(KAP)::value + 1 < RAD) t = mul(t, p.post_step);
                });
                scaled = true;
            }
            if (!scaled) {
                static_for<0, RAD>([&](auto K) { x[K] = canon(x[K]); });
            }
        }
        if (LAST && dout) {
            // straight to global: natural digit -> output row i_R; bit-reversed digit -> row = position
            const idx_t ors = (idx_t)p.out_rs * (idx_t)es;
            if (p.bitrev_digit) {
                const u64 off = (tc.out_base + (u64)c * p.out_cs + (u64)rpos0 * p.out_rs) * es;
                u64 *dp = dst + off;
                static_for<0, RAD>([&](auto Q) { dp[(idx_t)Q * ors] = x[Q]; });
                if (tc.dst2) {
                    u64 *dp2 = tc.dst2 + off;
                    static_for<0, RAD>([&](auto Q) { dp2[(idx_t)Q * ors] = x[Q]; });
                }
            } else {
                constexpr int SH = B1 + B2;
                u64 *dp = dst + (tc.out_base + (u64)c * p.out_cs + (u64)iR0 * p.out_rs) * es;
                static_for<0, RAD>([&](auto KAP) { dp[(idx_t)((u32)KAP << SH) * ors] = x[brev_c(decltype(KAP)::value, B)]; });
            }
        } else if (p.bitrev_digit) {
            // bit-reversed digit: register index q -> field value q
            static_for<0, RAD>([&](auto Q) { sm[padi(i0 + ((u32)Q << f))] = x[Q]; });
        } else {
            // natural digit: output kappa -> field value kappa
            static_for<0, RAD>([&](auto KAP) { sm[padi(i0 + ((u32)KAP << f))] = x[brev_c(decltype(KAP)::value, B)]; });
        }
    }
    if (!(LAST && dout)) __syncthreads();
}

template <int LOGR>
struct Steps {
    static constexpr int N = LOGR <= 4 ? 1 : (LOGR <= 8 ? 2 : 3);
    static constexpr int A = N == 1 ? LOGR : (N == 2 ? (LOGR + 1) / 2 : (LOGR + 2) / 3);
    static constexpr int Bb = N == 1 ? 0 : (N == 2 ? LOGR - A : (LOGR - A + 1) / 2);
    static constexpr int C = N == 3 ? LOGR - A - Bb : 0;
};

// SC: LDE scatter (destination per coset block from a pointer table + optional second copy); a separate instantiation
// so that the ordinary passes keep their single-destination store path
template <int LOGR, int LW, bool INV, bool SC = false>
__global__ void __launch_bounds__(256, 3) ntt_pass_kernel(const PassParams p, const Tables tb, const u64 *__restrict__ in,
                                                          u64 *__restrict__ out) {
    extern __shared__ u64 sm[];
    using S = Steps<LOGR>;
    const int lw = LW >= 0 ? LW : (int)p.log_w;
    const u32 R = 1u << LOGR, W = 1u << lw, T = R << lw;
    const u32 nthreads = blockDim.x, tid = threadIdx.x;

    // ---- batch decode
    // linear block id = tile * nbatch + batch: the batch (column / coset / lane) varies fastest, so the
    // CTAs that share a twiddle-table tile run together and the tables are served from L2
    // grid = (batch, tiles lo, tiles hi): blocks are dispatched x-fastest
    u32 b = blockIdx.x, lane = 0;
    if (p.lanes == 3) { lane = b % 3; b /= 3; }
    const u32 cos = b & (p.ncos - 1);
    const u32 col = b >> p.log_ncos;
    const u64 *src = in + (u64)col * p.in_col_stride + (u64)cos * p.in_cos_stride + lane;
    u64 *dst = (SC ? p.out_cos_ptr[cos] : out + (u64)cos * p.out_cos_stride) + (u64)col * p.out_col_stride + lane;

    // ---- tile decode
    TileCtx tc;
    tc.in_base = tc.out_base = tc.low_base = 0;
    {
        u32 t = blockIdx.y + blockIdx.z * gridDim.y;
        for (u32 d = 0; d < p.ndims; d++) {
            const u32 idx = t & (p.dims[d].ext - 1);
            t >>= p.dims[d].log_ext;
            tc.in_base += (u64)idx * p.dims[d].in_str;
            tc.out_base += (u64)idx * p.dims[d].out_str;
            tc.low_base += (u64)idx * p.dims[d].low_str;
        }
    }
    tc.sc_lo = tb.sc_lo ? tb.sc_lo + (u64)cos * 4096 : nullptr;
    tc.sc_hi = tb.sc_hi ? tb.sc_hi + (u64)cos * p.hi_len : nullptr;
    tc.pre_step = (p.has_pre && tb.pre_step) ? tb.pre_step[cos] : 0;
    tc.pre_tab = p.pre_tab ? p.pre_tab + (u64)cos * p.pre_cos_stride : nullptr;
    tc.dst2 = nullptr;
    if constexpr (SC) {
        if (p.out_dup_ptr) {
            u64 *b2 = p.out_dup_ptr[cos];
            if (b2) tc.dst2 = b2 + (u64)col * p.dup_col_stride + lane;
        }
    }

    // ---- prefetch the last step's multiplier tile (inter-pass twiddles, or the inverse post-scale) into
    //      the second shared buffer with cp.async: it lands while the sub-NTT runs
    tc.sm2 = nullptr;
    {
        const u64 *ltab = nullptr;
        u64 lrs = 0, lcs = 0;
        if (p.has_outer && p.outer_tab) {
            ltab = p.outer_tab + tc.low_base; lrs = p.outer_S; lcs = p.low_cs;
        } else if (p.has_post && p.post_tab) {
            ltab = p.post_tab + tc.out_base; lrs = p.out_rs; lcs = p.out_cs;
        }
        if (ltab) {
            using idx_t = typename std::conditional<(LW >= 0), u32, u64>::type;
            u64 *sm2 = sm + (T + (T >> 4) + 1);
            tc.sm2 = sm2;
            const idx_t lrs_i = (idx_t)lrs, lcs_i = (idx_t)lcs;
#pragma unroll
            for (int k = 0; k < kElemsPerThread; k++) {
                const u32 i = k * nthreads + tid;
                const u32 c = i & (W - 1), r = i >> lw;
                cp_async8(sm2 + padi(i), ltab + ((idx_t)r * lrs_i + (idx_t)c * lcs_i));
            }
            cp_async_commit();
        }
    }

    // lane-contiguous tiles (strided passes) skip the shared-memory staging on the way in / out
    const bool din = !p.in_r_fast, dout = !p.out_r_fast;
    const u32 es = p.estride;
    if (!din) {
        // ---- global -> shared, coalesced along the transform index; T = 16 * nthreads
        const bool pre = p.has_pre && tc.pre_tab;
        constexpr int CH = 8;   // loads in flight per thread and batch
#pragma unroll 1
        for (int k0 = 0; k0 < kElemsPerThread; k0 += CH) {
            u64 v[CH], tw[CH];
            using idx_t = typename std::conditional<(LW >= 0), u32, u64>::type;
            const u64 *sp = src + tc.in_base * es;
            const u64 *tp = pre ? tc.pre_tab + tc.in_base : nullptr;
#pragma unroll
            for (int k = 0; k < CH; k++) {
                const u32 i = (k0 + k) * nthreads + tid;
                const u32 r = i & (R - 1), c = i >> LOGR;
                const idx_t e = (idx_t)r * (idx_t)p.in_rs + (idx_t)c * (idx_t)p.in_cs;
                v[k] = sp[e * (idx_t)es];
                if (pre) tw[k] = __ldg(tp + e);
            }
#pragma unroll
            for (int k = 0; k < CH; k++) {
                const u32 i = (k0 + k) * nthreads + tid;
                const u32 r = i & (R - 1), c = i >> LOGR;
                sm[padi((r << lw) + c)] = pre ? mul(v[k], tw[k]) : v[k];
            }
        }
        __syncthreads();
    }

    // ---- CTA-level sub-NTT (the prefetched multiplier tile must be complete and visible to all
    //      threads before the last step)
    auto tile_ready = [&]() {
        if (tc.sm2) {
            cp_async_wait_all();
            __syncthreads();
        }
    };
    if constexpr (S::N == 1) {
        tile_ready();
        do_step<S::A, INV, true, true, 0, 0, LOGR, LW>(sm, p, tb, tc, lw, 0, din, dout, src, dst);
    } else if constexpr (S::N == 2) {
        do_step<S::A, INV, true, false, 0, 0, LOGR, LW>(sm, p, tb, tc, lw + LOGR - S::A, LOGR - S::A, din, dout, src, dst);
        tile_ready();
        do_step<S::Bb, INV, false, true, S::A, 0, LOGR, LW>(sm, p, tb, tc, lw, 0, din, dout, src, dst);
    } else {
        do_step<S::A, INV, true, false, 0, 0, LOGR, LW>(sm, p, tb, tc, lw + LOGR - S::A, LOGR - S::A, din, dout, src, dst);
        do_step<S::Bb, INV, false, false, S::A, 0, LOGR, LW>(sm, p, tb, tc, lw + S::C, S::C, din, dout, src, dst);
        tile_ready();
        do_step<S::C, INV, false, true, S::A, S::Bb, LOGR, LW>(sm, p, tb, tc, lw, 0, din, dout, src, dst);
    }
    if (dout) return;

    // ---- shared -> global.  rho = output row (natural digit: i_R, stored at the digit-reversed
    // position; bit-reversed digit: the position itself).
    auto pos_of = [&](u32 rho) -> u32 {
        if (p.bitrev_digit) return rho;
        if (S::N == 1) return rho;
        if (S::N == 2) return ((rho & ((1u << S::A) - 1)) << (LOGR - S::A)) | (rho >> S::A);
        u32 k1 = rho & ((1u << S::A) - 1), k2 = (rho >> S::A) & ((1u << S::Bb) - 1), k3 = rho >> (S::A + S::Bb);
        return (k1 << (LOGR - S::A)) | (k2 << S::C) | k3;
    };
    {
        using idx_t = typename std::conditional<(LW >= 0), u32, u64>::type;
        u64 *dp = dst + tc.out_base * es;
        u64 *dp2 = (SC && tc.dst2) ? tc.dst2 + tc.out_base * es : nullptr;
#pragma unroll 4
        for (int k = 0; k < kElemsPerThread; k++) {
            const u32 i = k * nthreads + tid;
            const u32 rho = i & (R - 1), c = i >> LOGR;
            const idx_t o = ((idx_t)rho * (idx_t)p.out_rs + (idx_t)c * (idx_t)p.out_cs) * (idx_t)es;
            const u64 v = sm[padi((pos_of(rho) << lw) + c)];
            dp[o] = v;
            if (SC && dp2) dp2[o] = v;
        }
    }
}

template <int LOGR, int LW>
static void launch_t(const PassParams &p, const Tables &t, bool inverse, const u64 *in, u64 *out, unsigned ntiles,
                     unsigned nbatch, cudaStream_t stream) {
    const unsigned T = 1u << (LOGR + p.log_w);
    const unsigned threads = T / kElemsPerThread;
    const bool two = (p.has_outer && p.outer_tab) || (p.has_post && p.post_tab);
    const size_t smem = (size_t)(T + (T >> 4) + 1) * sizeof(u64) * (two ? 2 : 1);
    // per instantiation and per device: allow > 48 KiB of dynamic shared memory
    static bool attr_set[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !attr_set[dev]) {
        cudaFuncSetAttribute(ntt_pass_kernel<LOGR, LW, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024);
        cudaFuncSetAttribute(ntt_pass_kernel<LOGR, LW, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024);
        if (dev >= 0 && dev < 64) attr_set[dev] = true;
    }
    const unsigned ty = ntiles < 32768u ? ntiles : 32768u;   // ntiles is a power of two
    dim3 grid(nbatch, ty, ntiles / ty);
    if (inverse) {
        ntt_pass_kernel<LOGR, LW, true><<<grid, threads, smem, stream>>>(p, t, in, out);
    } else if (p.out_cos_ptr) {
        static bool attr_sc[64] = {false};
        if (dev < 0 || dev >= 64 || !attr_sc[dev]) {
            cudaFuncSetAttribute(ntt_pass_kernel<LOGR, LW, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024);
            if (dev >= 0 && dev < 64) attr_sc[dev] = true;
        }
        ntt_pass_kernel<LOGR, LW, false, true><<<grid, threads, smem, stream>>>(p, t, in, out);
    } else {
        ntt_pass_kernel<LOGR, LW, false><<<grid, threads, smem, stream>>>(p, t, in, out);
    }
}

static bool g_wide_index = false;
void wide_index_configure(int enabled) { g_wide_index = enabled != 0; }

void launch_pass(const PassParams &p, const Tables &t, bool inverse, const u64 *in, u64 *out, unsigned ntiles,
                 unsigned nbatch, cudaStream_t stream) {
    // the shapes large transforms are made of get log2(W) fixed at compile time
    // ... provided every word offset inside a column (and inside the twiddle / scale tables) fits in 32 bits
    const bool small = !g_wide_index && ((p.n_mask + 1) * (u64)p.estride) <= (1ull << 31);
    if (!small) goto generic;
    if (p.log_r == 8 && p.log_w == 4) return launch_t<8, 4>(p, t, inverse, in, out, ntiles, nbatch, stream);
    if (p.log_r == 7 && p.log_w == 5) return launch_t<7, 5>(p, t, inverse, in, out, ntiles, nbatch, stream);
    if (p.log_r == 6 && p.log_w == 6) return launch_t<6, 6>(p, t, inverse, in, out, ntiles, nbatch, stream);
generic:
    switch (p.log_r) {
#define MS_CASE(L) case L: launch_t<L, -1>(p, t, inverse, in, out, ntiles, nbatch, stream); break;
        MS_CASE(1) MS_CASE(2) MS_CASE(3) MS_CASE(4) MS_CASE(5) MS_CASE(6)
        MS_CASE(7) MS_CASE(8) MS_CASE(9) MS_CASE(10) MS_CASE(11) MS_CASE(12)
#undef MS_CASE
        default: break;
    }
}

__global__ void build_pow_table_kernel(u64 *dst, u64 count, const u64 *lo, const u64 *hi, u32 hi_len) {
    const u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    if (i < count) dst[i] = tw_lookup(lo, hi, hi_len, i);
}
__global__ void build_outer_table_kernel(u64 *dst, u64 count, u64 S, u64 mult, u64 n_mask, const u64 *lo, const u64 *hi,
                                         u32 hi_len) {
    const u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    if (i >= count) return;
    const u64 iR = i / S, lower = i % S;
    dst[i] = tw_lookup(lo, hi, hi_len, (iR * lower * mult) & n_mask);
}
void build_pow_table(u64 *dst, u64 count, const u64 *lo, const u64 *hi, u32 hi_len, cudaStream_t stream) {
    build_pow_table_kernel<<<(unsigned)((count + 255) / 256), 256, 0, stream>>>(dst, count, lo, hi, hi_len);
}
void build_outer_table(u64 *dst, u64 R, u64 S, u64 mult, u64 n_mask, const u64 *lo, const u64 *hi, u32 hi_len,
                       cudaStream_t stream) {
    const u64 count = R * S;
    build_outer_table_kernel<<<(unsigned)((count + 255) / 256), 256, 0, stream>>>(dst, count, S, mult, n_mask, lo, hi,
                                                                                    hi_len);
}

void steps_of(int log_r, int out[3], int *nsteps) {
    int n = log_r <= 4 ? 1 : (log_r <= 8 ? 2 : 3);
    int a = n == 1 ? log_r : (n == 2 ? (log_r + 1) / 2 : (log_r + 2) / 3);
    int b = n == 1 ? 0 : (n == 2 ? log_r - a : (log_r - a + 1) / 2);
    int c = n == 3 ? log_r - a - b : 0;
    out[0] = a; out[1] = b; out[2] = c;
    *nsteps = n;
}

std::vector<int> choose_digits(unsigned log_n) {
    std::vector<int> d;
    if (log_n <= (unsigned)kTileLog) {
        d.push_back((int)log_n);
        return d;
    }
    unsigned m = (log_n + 7) / 8;
    unsigned base = log_n / m, rem = log_n % m;
    for (unsigned i = 0; i < m; i++) d.push_back((int)(base + (i < rem ? 1 : 0)));
    return d;
}

// ------------------------------------------------------------------------------------------
// Definition-based kernel: out[i] = sum_j in[j] * (offset * g^i)^j  (forward), or its inverse
// (in[j] evaluated at g^-i, scaled by n^-1 * offset^-i).  O(n) per thread.
__global__ void ntt_naive_kernel(const u64 *__restrict__ in, u64 in_stride_words, u64 *__restrict__ out,
                                 u64 out_stride_words, unsigned log_n, unsigned estride, unsigned lanes, bool inverse,
                                 u64 root, u64 offset) {
    const u64 n = 1ull << log_n;
    const u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned lane = blockIdx.y % lanes, col = blockIdx.y / lanes;
    const u64 *src = in + (u64)col * in_stride_words + lane;
    u64 *dst = out + (u64)col * out_stride_words + lane;
    u64 acc = 0;
    if (!inverse) {
        u64 x = mul(offset, pow(root, i));
        for (u64 j = n; j-- > 0;) acc = add(mul(acc, x), src[j * estride]);
    } else {
        u64 x = pow(root, i);  // `root` is already the inverse root for inverse plans
        for (u64 j = n; j-- > 0;) acc = add(mul(acc, x), src[j * estride]);
        acc = mul(acc, mul(inv(to_mont(n)), pow(inv(offset), i)));
    }
    dst[i * estride] = acc;
}

void launch_naive(const u64 *in, u64 in_stride_words, u64 *out, u64 out_stride_words, unsigned log_n, unsigned estride,
                  unsigned lanes, unsigned ncols, bool inverse, u64 root_mont, u64 offset_mont, cudaStream_t stream) {
    const u64 n = 1ull << log_n;
    unsigned threads = n < 128 ? (unsigned)n : 128;
    dim3 grid((unsigned)((n + threads - 1) / threads), ncols * lanes);
    ntt_naive_kernel<<<grid, threads, 0, stream>>>(in, in_stride_words, out, out_stride_words, log_n, estride, lanes,
                                                   inverse, root_mont, offset_mont);
}

}  // namespace msntt
