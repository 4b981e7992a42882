// dft.cuh — in-register radix-2^B (B <= 4) DFT networks over Goldilocks shared by the NTT passes
// (ntt.cu) and the FRI fold (fri.cu).  Twiddles of these levels are 16th roots of unity, i.e.
// compile-time constants (arkworks' omega_16 = 2^156 mod p, so they are +-powers of two in
// Montgomery form).
#pragma once
#include "field.cuh"

namespace msntt {
using namespace gl;

// omega_16^k, k = 0..7, Montgomery form; forward and inverse.
template <bool INV>
__host__ __device__ __forceinline__ constexpr u64 w16(int k) {
    constexpr u64 F[8] = {0x00000000FFFFFFFFULL, 0x0000000010000000ULL, 0xFEFFFFFF01000001ULL, 0xFFEFFFFF00000001ULL,
                          0xFFFFFFFEFFFF0001ULL, 0x00000FFFFFFFF000ULL, 0x0000010000000000ULL, 0x0000000000000010ULL};
    constexpr u64 I[8] = {0x00000000FFFFFFFFULL, 0xFFFFFFFEFFFFFFF1ULL, 0xFFFFFEFF00000001ULL, 0xFFFFEFFF00001001ULL,
                          0x0000000000010000ULL, 0x0010000000000000ULL, 0x00FFFFFFFF000000ULL, 0xFFFFFFFEF0000001ULL};
    return INV ? I[k] : F[k];
}

// The same constants as signed powers of two: Montgomery word of omega_16^k = (neg ? p - 2^m : 2^m).  A butterfly then
// needs no multiplication: t = mul_pow2<m>(v) (a 128-bit shift + the Montgomery reduction) and, for a negative constant,
// the sum and the difference swap places.
struct W16Shift {
    int m;
    bool neg;
};
template <bool INV>
__host__ __device__ constexpr W16Shift w16_shift(int k) {
    constexpr W16Shift F[8] = {{0, false}, {28, false}, {88, true}, {52, true}, {16, true}, {76, false}, {40, false}, {4, false}};
    constexpr W16Shift I[8] = {{0, false}, {4, true}, {40, true}, {76, true}, {16, false}, {52, false}, {88, false}, {28, true}};
    return INV ? I[k] : F[k];
}
__host__ __device__ constexpr u64 pow2_mod_p(int m) {   // 2^m mod p, m < 96
    return m < 64 ? (1ULL << m) : ((1ULL << (m - 32)) - (1ULL << (m - 64)));   // 2^64 = 2^32 - 1
}
template <bool INV, int K>
__host__ __device__ constexpr bool w16_shift_ok() {
    constexpr W16Shift s = w16_shift<INV>(K);
    constexpr u64 v = pow2_mod_p(s.m);
    return (s.neg ? P - v : v) == w16<INV>(K);
}
static_assert(w16_shift_ok<false, 1>() && w16_shift_ok<false, 2>() && w16_shift_ok<false, 3>() && w16_shift_ok<false, 4>() &&
              w16_shift_ok<false, 5>() && w16_shift_ok<false, 6>() && w16_shift_ok<false, 7>(), "forward 16th roots");
static_assert(w16_shift_ok<true, 1>() && w16_shift_ok<true, 2>() && w16_shift_ok<true, 3>() && w16_shift_ok<true, 4>() &&
              w16_shift_ok<true, 5>() && w16_shift_ok<true, 6>() && w16_shift_ok<true, 7>(), "inverse 16th roots");

// compile-time loop: f(IC<I>) for I in [0, N)
template <int V>
struct IC {
    static constexpr int value = V;
    __host__ __device__ constexpr operator int() const { return V; }
};
template <int I, int N, typename F>
__device__ __forceinline__ void static_for(F &&f) {
    if constexpr (I < N) {
        f(IC<I>{});
        static_for<I + 1, N>(f);
    }
}
__host__ __device__ constexpr int brev_c(int k, int bits) {
    int r = 0;
    for (int b = 0; b < bits; b++) r |= ((k >> b) & 1) << (bits - 1 - b);
    return r;
}

// In-register 2^B-point DFT.  Input x[k] natural, canonical.  Output index kappa ends up in
// register brev<B>(kappa), lazy (any u64).  DIT network laid over naturally stored inputs:
// level s pairs registers `span = 2^(B-s)` apart; the twiddle omega_{2^s}^j has j = the
// bit-reversal of the register-index bits above the span bit.  t = w*b is canonical after the
// Montgomery reduction, so a +- t needs a single repair (lazy add/sub).
template <int B, bool INV, int S, int A>
struct Bfly {
    static __device__ __forceinline__ void run(u64 (&x)[1 << B]) {
        constexpr int span = 1 << (B - S);
        if constexpr ((A & span) == 0) {
            constexpr int j = brev_c(A >> (B - S + 1), S - 1);
            const u64 u = x[A], v = x[A + span];
            if constexpr (j == 0) {
                if constexpr (S == 1) {  // both operands canonical
                    x[A] = add_lc(u, v);
                    x[A + span] = sub_lc(u, v);
                } else {
                    x[A] = add_ll(u, v);
                    x[A + span] = sub_ll(u, v);
                }
            } else {
#ifdef MS_DFT_CONST_MUL      // A/B: the constants through the generic multiplication
                constexpr u64 w = w16<INV>(j * (16 >> S));
                const u64 t = mul(v, w);
                x[A] = add_lc(u, t);
                x[A + span] = sub_lc(u, t);
#else
                constexpr W16Shift sh = w16_shift<INV>(j * (16 >> S));
                const u64 t = mul_pow2<sh.m>(v);
                if constexpr (sh.neg) {          // u + (-t), u - (-t)
                    x[A] = sub_lc(u, t);
                    x[A + span] = add_lc(u, t);
                } else {
                    x[A] = add_lc(u, t);
                    x[A + span] = sub_lc(u, t);
                }
#endif
            }
        }
        if constexpr (A + 1 < (1 << B))
            Bfly<B, INV, S, A + 1>::run(x);
        else if constexpr (S < B)
            Bfly<B, INV, S + 1, 0>::run(x);
    }
};
#ifndef MS_DFT_REPAIR_EACH
// The same network on the redundant 96-bit form (field.cuh::L96): no repair between butterflies, one reduction per
// output.  The Montgomery word of a twiddle is +-2^m, and a Montgomery product by it multiplies the value by
// +-2^(m - 64) = +-2^K (2^96 = -1): K = m - 64 for m >= 64, and K = m + 32 with the sign flipped for m < 64.
//
// Bound, with b_s the bound on |value| entering level s (inputs are u64, so b_1 = 2^64, non-negative):
//   level 1:   sums and differences of two inputs: |.| < 2^65
//   level s>1: a twiddled operand W has |W| < 2^65 + b_s / 2 (l96_mul_pow2), so |u +- W| < b_s + 2^65 + b_s / 2:
//              b_3 < 2^67, b_4 < 2^68, outputs of level 4 in (-2^69, 2^69).
// Register 0 also carries kBias = 2^7 p (= 0 mod p, < 2^71).  In this network register 0's contents only ever reach the
// untwiddled side of a butterfly, so every output carries exactly + kBias: outputs lie in (2^70, 2^72), non-negative and
// below 2^95, as l96_reduce needs.
constexpr u64 kBiasLo = P << 7;                 // 2^7 p = 2^71 - 2^39 + 2^7 as 96 bits
constexpr u32 kBiasHi = (u32)(P >> 57);
static_assert(kBiasHi == 127 && kBiasLo == 0xFFFFFF8000000080ULL, "2^7 p");
template <int B, bool INV, int S, int A>
struct BflyL {
    static __host__ __device__ __forceinline__ void run(L96 (&x)[1 << B]) {
        constexpr int span = 1 << (B - S);
        if constexpr ((A & span) == 0) {
            constexpr int j = brev_c(A >> (B - S + 1), S - 1);
            const L96 u = x[A], v = x[A + span];
            if constexpr (j == 0) {
                x[A] = l96_add(u, v);
                x[A + span] = l96_sub(u, v);
            } else {
                constexpr W16Shift sh = w16_shift<INV>(j * (16 >> S));
                constexpr int K = sh.m >= 64 ? sh.m - 64 : sh.m + 32;
                constexpr bool neg = sh.neg != (sh.m < 64);
                const L96 t = l96_mul_pow2<K>(v);
                x[A] = neg ? l96_sub(u, t) : l96_add(u, t);
                x[A + span] = neg ? l96_add(u, t) : l96_sub(u, t);
            }
        }
        if constexpr (A + 1 < (1 << B))
            BflyL<B, INV, S, A + 1>::run(x);
        else if constexpr (S < B)
            BflyL<B, INV, S + 1, 0>::run(x);
    }
};
#endif

// x[k]: any u64 in; output index kappa in register brev<B>(kappa), any u64 (a Montgomery product with a canonical
// factor, or canon, makes it canonical)
template <int B, bool INV>
__host__ __device__ __forceinline__ void dft_regs(u64 (&x)[1 << B]) {
#ifdef MS_DFT_REPAIR_EACH
    Bfly<B, INV, 1, 0>::run(x);
#else
    L96 y[1 << B];
    for (int i = 0; i < (1 << B); i++) y[i] = l96(x[i]);
    y[0] = l96_add(y[0], L96{(u32)kBiasLo, (u32)(kBiasLo >> 32), kBiasHi});
    BflyL<B, INV, 1, 0>::run(y);
    for (int i = 0; i < (1 << B); i++) x[i] = l96_reduce(y[i]);
#endif
}

}  // namespace msntt
