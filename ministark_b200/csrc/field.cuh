// field.cuh — Goldilocks Fp (p = 2^64 - 2^32 + 1) and Fq3 = Fp[X]/(X^3 - 2) device arithmetic.
//
// Memory representation is the reference's: every 64-bit word is the canonical (< p)
// Montgomery residue x * 2^64 mod p (gpu/src/metal/felt_u64.h.metal:118,127; the Rust
// side builds constants as raw Montgomery BigInts, gpu/src/fields.rs:82).  These
// routines are the sm_90a counterpart of felt_u64.h.metal:147-177 (Fp) and :205-236
// (Fq3), re-derived rather than transcribed:
//
//   * mont_mul: 64x64->128 product (4 IMAD.WIDE) followed by the Goldilocks-special
//     Montgomery reduction  t = hi - (a - (a >> 32) - e),  a = lo + (lo << 32) (carry e),
//     which needs no second multiplication because -p^{-1} = -(2^32 + 1) mod 2^64.
//     The result is canonical whenever one operand is canonical; the other operand may
//     be ANY u64 ("lazy" value), which the NTT butterflies exploit.
//   * lazy add/sub: values in [0, 2^64) representing themselves mod p.  2^64 = eps
//     (mod p) with eps = 2^32 - 1, so a carry out of 64 bits is repaired by adding eps
//     and a borrow by subtracting eps.
//
// Integer modular arithmetic only: tensor cores are not applicable (DESIGN.md §3).
#pragma once
#ifndef __CUDACC_RTC__
#include <cstdint>
#endif

namespace gl {

typedef unsigned long long u64;
typedef unsigned int u32;

constexpr u64 P = 0xFFFFFFFF00000001ULL;
constexpr u64 EPS = 0xFFFFFFFFULL;        // 2^64 mod p  == Montgomery form of 1
constexpr u64 ONE = EPS;
constexpr u64 R2 = 0xFFFFFFFE00000001ULL; // 2^128 mod p
constexpr u64 TWO = 0x1FFFFFFFEULL;       // Montgomery form of 2 (Fq3 non-residue)

#if defined(__CUDACC__)
#define GL_DEV __device__ __forceinline__
#define GL_HD __host__ __device__ __forceinline__
#else
#define GL_DEV inline
#define GL_HD inline
#endif

// ---- canonical <-> canonical ------------------------------------------------------
#if defined(__CUDACC__) && (defined(MS_CANON_MAD) || defined(MS_ADD_MAD))
// eps = 2^32 - 1 as a run-time operand: with an immediate ptxas strength-reduces  c * eps + s  back into an ALU carry chain;
// from constant memory it stays one IMAD.WIDE on the FMA pipe
static __constant__ u32 kEpsOperand = 0xFFFFFFFFu;
#endif
#if defined(__CUDA_ARCH__) && defined(MS_CANON_MAD)
// c = carry of x + eps = (x >= p); x - p = x + c * eps (mod 2^64): the conditional subtraction as ONE multiply-add on
// the FMA pipe instead of a 64-bit compare + subtract + select on the ALU pipe
__device__ __forceinline__ u64 canon(u64 x) {
    u64 r;
    asm("{\n\t.reg .u32 x0, x1, t0, t1, c;\n\tmov.b64 {x0, x1}, %1;\n\tadd.cc.u32 t0, x0, 0xffffffff;\n\taddc.cc.u32 t1, x1, 0;\n\t"
        "addc.u32 c, 0, 0;\n\tmad.wide.u32 %0, c, %2, %1;\n\t}"
        : "=l"(r) : "l"(x), "r"(kEpsOperand));
    return r;
}
#else
// x >= p  <=>  high word all ones and low word non-zero; then x - p = (0 : low - 1): two compares, one decrement, one select
GL_HD u64 canon(u64 x) {
    u32 x0 = (u32)x, x1 = (u32)(x >> 32);
    const bool c = (x1 == 0xFFFFFFFFu) && (x0 != 0);
    x0 -= c ? 1u : 0u;
    x1 = c ? 0u : x1;
    return ((u64)x1 << 32) | x0;
}
#endif

GL_HD u64 add(u64 a, u64 b) {  // a, b < p
    u64 s = a + b;
    u64 t = s + EPS;           // s - p (mod 2^64)
    return (s < a || t < s) ? t : s;
}
GL_HD u64 sub(u64 a, u64 b) {  // a, b < p
    u64 d = a - b;
    return a < b ? d - EPS : d;  // + p
}
GL_HD u64 neg(u64 a) { return a ? P - a : 0; }

// ---- lazy arithmetic (any u64 in, any u64 out; value preserved mod p) ---------------
// lc: second operand canonical (< p)  -> a single repair suffices.
// ll: both operands arbitrary u64     -> up to two repairs.
// Device versions are carry-chain PTX (5 / 5 / 9 / 8 SASS instructions instead of the 8 / 8 / 12 /
// 12 the compiler makes of the portable forms below, which the host keeps).
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ u64 pack64(u32 lo, u32 hi) { u64 r; asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "r"(lo), "r"(hi)); return r; }
__device__ __forceinline__ void unpack64(u64 v, u32 &lo, u32 &hi) { asm("mov.b64 {%0,%1}, %2;" : "=r"(lo), "=r"(hi) : "l"(v)); }
// s = a + t; on carry add eps = 2^32 - 1, i.e. low -= c, high += c - borrow
#if defined(MS_ADD_MAD)
// the repair s += c * eps as a multiply-add (FMA pipe): 3 ALU + 1 IMAD.WIDE instead of 6 ALU instructions
__device__ __forceinline__ u64 add_lc(u64 a, u64 t) {
    u32 a0, a1, t0, t1;
    u64 r;
    unpack64(a, a0, a1); unpack64(t, t0, t1);
    asm("{\n\t.reg .u32 s0, s1, c;\n\t.reg .u64 s;\n\tadd.cc.u32 s0, %1, %3;\n\taddc.cc.u32 s1, %2, %4;\n\taddc.u32 c, 0, 0;\n\t"
        "mov.b64 s, {s0, s1};\n\tmad.wide.u32 %0, c, %5, s;\n\t}"
        : "=l"(r) : "r"(a0), "r"(a1), "r"(t0), "r"(t1), "r"(kEpsOperand));
    return r;
}
#else
__device__ __forceinline__ u64 add_lc(u64 a, u64 t) {
    u32 a0, a1, t0, t1, s0, s1;
    unpack64(a, a0, a1); unpack64(t, t0, t1);
    asm("{\n\t.reg .u32 c;\n\tadd.cc.u32 %0, %2, %4;\n\taddc.cc.u32 %1, %3, %5;\n\taddc.u32 c, 0, 0;\n\t"
        "sub.cc.u32 %0, %0, c;\n\tsubc.u32 %1, %1, 0;\n\tadd.u32 %1, %1, c;\n\t}"
        : "=r"(s0), "=r"(s1) : "r"(a0), "r"(a1), "r"(t0), "r"(t1));
    return pack64(s0, s1);
}
#endif
// d = a - t; on borrow subtract eps (m = 0xffffffff is eps as a low word)
__device__ __forceinline__ u64 sub_lc(u64 a, u64 t) {
    u32 a0, a1, t0, t1, s0, s1;
    unpack64(a, a0, a1); unpack64(t, t0, t1);
    asm("{\n\t.reg .u32 m;\n\tsub.cc.u32 %0, %2, %4;\n\tsubc.cc.u32 %1, %3, %5;\n\tsubc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 %0, %0, m;\n\tsubc.u32 %1, %1, 0;\n\t}"
        : "=r"(s0), "=r"(s1) : "r"(a0), "r"(a1), "r"(t0), "r"(t1));
    return pack64(s0, s1);
}
// Both repairs are exact 64-bit additions of eps = (0 : 0xffffffff) gated by the previous carry (m = -carry), so the
// carry of each repair is the true carry — including a + t == 2^64 exactly, where the first sum is 0 (an earlier
// version repaired with "low -= c, high -= borrow, high += c" and took the carry of the last add, which is spurious
// in exactly that case: found by the brainfuck MemValInv column, whose words 2^63 + 2^63 sum to 2^64).
// (PTX carry flags follow the hardware: after add.cc CF is the carry, after sub.cc it is NOT borrow.)
__device__ __forceinline__ u64 add_ll(u64 a, u64 t) {
    u32 a0, a1, t0, t1, s0, s1;
    unpack64(a, a0, a1); unpack64(t, t0, t1);
    asm("{\n\t.reg .u32 c, m;\n\tadd.cc.u32 %0, %2, %4;\n\taddc.cc.u32 %1, %3, %5;\n\taddc.u32 c, 0, 0;\n\tsub.u32 m, 0, c;\n\t"
        "add.cc.u32 %0, %0, m;\n\taddc.cc.u32 %1, %1, 0;\n\taddc.u32 c, 0, 0;\n\tsub.u32 m, 0, c;\n\t"
        "add.cc.u32 %0, %0, m;\n\taddc.u32 %1, %1, 0;\n\t}"
        : "=r"(s0), "=r"(s1) : "r"(a0), "r"(a1), "r"(t0), "r"(t1));
    return pack64(s0, s1);
}
__device__ __forceinline__ u64 sub_ll(u64 a, u64 t) {
    u32 a0, a1, t0, t1, s0, s1;
    unpack64(a, a0, a1); unpack64(t, t0, t1);
    asm("{\n\t.reg .u32 m;\n\tsub.cc.u32 %0, %2, %4;\n\tsubc.cc.u32 %1, %3, %5;\n\tsubc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 %0, %0, m;\n\tsubc.cc.u32 %1, %1, 0;\n\tsubc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 %0, %0, m;\n\tsubc.u32 %1, %1, 0;\n\t}"
        : "=r"(s0), "=r"(s1) : "r"(a0), "r"(a1), "r"(t0), "r"(t1));
    return pack64(s0, s1);
}
#else
inline u64 add_lc(u64 a, u64 t) {
    u64 s = a + t;
    return s < a ? s + EPS : s;
}
inline u64 sub_lc(u64 a, u64 t) {
    u64 d = a - t;
    return a < t ? d - EPS : d;
}
inline u64 add_ll(u64 a, u64 b) {
    u64 s = a + b;
    if (s < a) { u64 s2 = s + EPS; s = s2 < s ? s2 + EPS : s2; }
    return s;
}
inline u64 sub_ll(u64 a, u64 b) {
    u64 d = a - b;
    if (a < b) { u64 d2 = d - EPS; d = d < EPS ? d2 - EPS : d2; }
    return d;
}
#endif

// ---- redundant 96-bit form (the in-register DFT networks of dft.cuh) ----------------------
// A value is the signed 96-bit integer w0 + w1 * 2^32 + (s32)w2 * 2^64, congruent to the field element mod p.  Sums and
// differences are exact 3-limb carry chains with no repair; the networks keep |value| < 2^95 (bounds in dft.cuh) and
// reduce once per output.
struct L96 {
    u32 w0, w1, w2;
};
GL_HD L96 l96(u64 x) { return L96{(u32)x, (u32)(x >> 32), 0u}; }
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ L96 l96_add(L96 a, L96 b) {
    L96 r;
    asm("add.cc.u32 %0, %3, %6;\n\taddc.cc.u32 %1, %4, %7;\n\taddc.u32 %2, %5, %8;"
        : "=r"(r.w0), "=r"(r.w1), "=r"(r.w2) : "r"(a.w0), "r"(a.w1), "r"(a.w2), "r"(b.w0), "r"(b.w1), "r"(b.w2));
    return r;
}
__device__ __forceinline__ L96 l96_sub(L96 a, L96 b) {
    L96 r;
    asm("sub.cc.u32 %0, %3, %6;\n\tsubc.cc.u32 %1, %4, %7;\n\tsubc.u32 %2, %5, %8;"
        : "=r"(r.w0), "=r"(r.w1), "=r"(r.w2) : "r"(a.w0), "r"(a.w1), "r"(a.w2), "r"(b.w0), "r"(b.w1), "r"(b.w2));
    return r;
}
#else
inline L96 l96_add(L96 a, L96 b) {
    const u64 s0 = (u64)a.w0 + b.w0, s1 = (u64)a.w1 + b.w1 + (s0 >> 32);
    return L96{(u32)s0, (u32)s1, a.w2 + b.w2 + (u32)(s1 >> 32)};
}
inline L96 l96_sub(L96 a, L96 b) {
    const u64 d0 = (u64)a.w0 - b.w0, d1 = (u64)a.w1 - b.w1 - (d0 >> 63);
    return L96{(u32)d0, (u32)d1, a.w2 - b.w2 - (u32)(d1 >> 63)};
}
#endif
// v * 2^K (mod p), K in [0, 96).  v * 2^r (r = K % 32) is the four limbs y0..y3 (y3 signed); placed q = K / 32 limbs up
// they form Lo + Hi * 2^96 with Lo in [0, 2^96), and 2^96 = -1 gives Lo - Hi.  Lo's top limb t is folded with
// 2^64 = 2^32 - 1, so Lo becomes (lo0 + lo1 2^32) + t 2^32 - t, in (-2^32, 2^65).  For |v| < 2^b: |Hi| <= 2^(b + K - 96)
// <= 2^(b - 1), so the result W has |W| < 2^65 + 2^(b - 1).
template <int K>
GL_HD L96 l96_mul_pow2(L96 v) {
    static_assert(K > 0 && K < 96, "shift out of range");
    constexpr int q = K / 32, r = K % 32;
    u32 y0, y1, y2, y3;
    if constexpr (r == 0) {
        y0 = v.w0, y1 = v.w1, y2 = v.w2, y3 = (u32)((int)v.w2 >> 31);
    } else {
        y0 = v.w0 << r;
        y1 = (v.w1 << r) | (v.w0 >> (32 - r));
        y2 = (v.w2 << r) | (v.w1 >> (32 - r));
        y3 = (u32)((int)v.w2 >> (32 - r));
    }
    if constexpr (q == 0) {           // Lo = (y0, y1, t = y2), Hi = y3
        const u32 s = (u32)((int)y3 >> 31);
        return l96_sub(l96_sub(l96_add(L96{y0, y1, 0u}, L96{0u, y2, 0u}), L96{y2, 0u, 0u}), L96{y3, s, s});
    } else if constexpr (q == 1) {    // Lo = (0, y0, t = y1), Hi = y2 + y3 2^32
        const u32 s = (u32)((int)y3 >> 31);
        return l96_sub(l96_sub(L96{0u, y0, 0u}, L96{y1, 0u, 0u}), l96_sub(L96{y2, y3, s}, L96{0u, y1, 0u}));
    } else {                          // Lo = (0, 0, t = y0), Hi = y1 + y2 2^32 + y3 2^64
        return l96_sub(l96_sub(L96{0u, y0, 0u}, L96{y0, 0u, 0u}), L96{y1, y2, y3});
    }
}
// any u64 congruent to v, for 0 <= v < 2^72: v = lo + c 2^64 = lo + c (2^32 - 1), and c (2^32 - 1) < 2^40 < p is
// canonical, so one lazy addition finishes it
GL_HD u64 l96_reduce(L96 v) {
    return add_lc(((u64)v.w1 << 32) | v.w0, (u64)v.w2 * 0xFFFFFFFFull);
}

// ---- Montgomery multiplication ---------------------------------------------------------
// returns a*b*2^-64 mod p, canonical, provided a*b < p * 2^64 (i.e. one operand < p).
GL_HD u64 mont_reduce(u64 hi, u64 lo) {
#if defined(__CUDA_ARCH__)
    // A1 = lo1 + lo0 (carry e); b = (A1:lo0) - (A1 + e)  [A1 + e never wraps]; r = hi - b (+p on borrow)
    u32 r0, r1, r2, r3, q0, q1;
    unpack64(lo, r0, r1); unpack64(hi, r2, r3);
    asm("{\n\t.reg .u32 A1, e, B0, B1, m;\n\t"
        "add.cc.u32 A1, %3, %2;\n\taddc.u32 e, 0, 0;\n\tadd.u32 e, e, A1;\n\t"
        "sub.cc.u32 B0, %2, e;\n\tsubc.u32 B1, A1, 0;\n\t"
        "sub.cc.u32 %0, %4, B0;\n\tsubc.cc.u32 %1, %5, B1;\n\tsubc.u32 m, 0, 0;\n\t"
        "sub.cc.u32 %0, %0, m;\n\tsubc.u32 %1, %1, 0;\n\t}"
        : "=&r"(q0), "=&r"(q1) : "r"(r0), "r"(r1), "r"(r2), "r"(r3));
    return pack64(q0, q1);
#else
    u64 a = lo + (lo << 32);
    u64 e = a < lo;                    // carry out of the 64-bit add
    u64 b = a - (a >> 32) - e;         // never underflows: a >= (a>>32) + e
    u64 r = hi - b;
    return hi < b ? r - EPS : r;       // + p
#endif
}
GL_HD u64 mul(u64 a, u64 b) {
#if defined(__CUDA_ARCH__)
    return mont_reduce(__umul64hi(a, b), a * b);
#else
    unsigned __int128 x = (unsigned __int128)a * b;
    return mont_reduce((u64)(x >> 64), (u64)x);
#endif
}
// x * W * 2^-64 mod p for a twiddle whose Montgomery word W is the power of two 2^M (the 16th roots of unity all are,
// up to sign: dft.cuh) — the 128-bit product is a shift, so no multiplication instruction is spent; same canonical
// result as mul(x, 2^M mod p).  x may be any u64.
template <int M>
GL_HD u64 mul_pow2(u64 x) {
    static_assert(M > 0 && M < 96, "shift out of range");
    if constexpr (M < 64) {
        return mont_reduce(x >> (64 - M), x << M);       // x * 2^M < p * 2^64: canonical
    } else {
        // 2^M * 2^-64 = 2^k, k = M - 64 < 32:  x * 2^k = lo + hi * 2^64 = lo + hi * eps  (hi < 2^k, so hi * eps < p)
        constexpr int k = M - 64;
        const u64 lo = x << k, hi = x >> (64 - k);
        return canon(add_lc(lo, (hi << 32) - hi));
    }
}
GL_HD u64 sqr(u64 a) { return mul(a, a); }
GL_HD u64 to_mont(u64 x_canon) { return mul(x_canon, R2); }
GL_HD u64 from_mont(u64 w) { return mul(w, 1); }

GL_HD u64 pow(u64 a, u64 e) {
    u64 r = ONE;
    while (e) {
        if (e & 1) r = mul(r, a);
        a = sqr(a);
        e >>= 1;
    }
    return r;
}
// a^(p-2) = a^(2^64 - 2^32 - 1); exponent bits MSB first: 31 ones, one zero, 32 ones.
// Built from a^(2^k - 1) blocks, ~73 multiplications (the reference uses a chain of
// similar length, felt_u64.h.metal:97-109).
GL_HD u64 inv(u64 a) {
    u64 x1 = a;
    u64 x2 = mul(sqr(x1), x1);                 // 2^2-1
    u64 x3 = mul(sqr(x2), x1);                 // 2^3-1
    u64 x6 = x3; for (int i = 0; i < 3; i++) x6 = sqr(x6); x6 = mul(x6, x3);
    u64 x12 = x6; for (int i = 0; i < 6; i++) x12 = sqr(x12); x12 = mul(x12, x6);
    u64 x24 = x12; for (int i = 0; i < 12; i++) x24 = sqr(x24); x24 = mul(x24, x12);
    u64 x30 = x24; for (int i = 0; i < 6; i++) x30 = sqr(x30); x30 = mul(x30, x6);
    u64 x31 = mul(sqr(x30), x1);
    u64 x32 = mul(sqr(x31), x1);
    u64 r = x31;                                // top 31 ones
    for (int i = 0; i < 33; i++) r = sqr(r);    // the zero bit + 32 more positions
    return mul(r, x32);                         // low 32 ones
}

// ---- Fq3 ---------------------------------------------------------------------------------
struct Fq3 {
    u64 c0, c1, c2;
};
GL_HD Fq3 fq3(u64 a) { return Fq3{a, 0, 0}; }
GL_HD Fq3 add(Fq3 a, Fq3 b) { return Fq3{add(a.c0, b.c0), add(a.c1, b.c1), add(a.c2, b.c2)}; }
GL_HD Fq3 sub(Fq3 a, Fq3 b) { return Fq3{sub(a.c0, b.c0), sub(a.c1, b.c1), sub(a.c2, b.c2)}; }
GL_HD Fq3 neg(Fq3 a) { return Fq3{neg(a.c0), neg(a.c1), neg(a.c2)}; }
GL_HD Fq3 mul(Fq3 a, u64 b) { return Fq3{mul(a.c0, b), mul(a.c1, b), mul(a.c2, b)}; }
// (a0 + a1 X + a2 X^2)(b0 + b1 X + b2 X^2) mod X^3 - 2, 6 base multiplications
// (Karatsuba-style cross terms; same field element as felt_u64.h.metal:205-231).
GL_HD Fq3 mul(Fq3 a, Fq3 b) {
    u64 v0 = mul(a.c0, b.c0), v1 = mul(a.c1, b.c1), v2 = mul(a.c2, b.c2);
    u64 x12 = sub(sub(mul(add(a.c1, a.c2), add(b.c1, b.c2)), v1), v2);  // a1b2 + a2b1
    u64 x01 = sub(sub(mul(add(a.c0, a.c1), add(b.c0, b.c1)), v0), v1);  // a0b1 + a1b0
    u64 x02 = sub(sub(mul(add(a.c0, a.c2), add(b.c0, b.c2)), v0), v2);  // a0b2 + a2b0
    return Fq3{add(v0, add(x12, x12)), add(x01, add(v2, v2)), add(x02, v1)};
}
GL_HD Fq3 sqr(Fq3 a) { return mul(a, a); }
GL_HD Fq3 pow(Fq3 a, u64 e) {
    Fq3 r = fq3(ONE);
    while (e) {
        if (e & 1) r = mul(r, a);
        a = sqr(a);
        e >>= 1;
    }
    return r;
}
// inverse through the norm to Fp (the reference leaves Fq3::inverse unimplemented,
// felt_u64.h.metal:267-270; eval_cpu.rs uses ark-ff's CubicExtField::inverse).
GL_HD Fq3 inv(Fq3 a) {
    u64 s0 = sub(sqr(a.c0), mul(TWO, mul(a.c1, a.c2)));
    u64 s1 = sub(mul(TWO, sqr(a.c2)), mul(a.c0, a.c1));
    u64 s2 = sub(sqr(a.c1), mul(a.c0, a.c2));
    u64 nrm = add(mul(a.c0, s0), mul(TWO, add(mul(a.c2, s1), mul(a.c1, s2))));
    u64 ni = inv(nrm);
    return Fq3{mul(s0, ni), mul(s1, ni), mul(s2, ni)};
}

}  // namespace gl
