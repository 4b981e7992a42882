"""CPU-only: the in-register DFT networks of csrc/dft.cuh on the redundant 96-bit form (field.cuh::L96), compiled for the
host behind a few CUDA stand-ins and compared with the field definition of the DFT — on random words, on every edge word
in every position, and on random tuples of edge words — plus the limb primitives over all pairs of edge words."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ministark_b200", "csrc")
P = 2**64 - 2**32 + 1
R = 2**64
EPS = 2**32 - 1

# the edge words of test_lazy_primitives_all_edge_pairs: 0, 1, p - 1, eps, 2^63, 2^64 - 1 and their neighbours, words
# whose pairwise sums are exactly 2^64
EDGES = sorted({0, 1, 2, P - 2, P - 1, P, P + 1, EPS - 1, EPS, EPS + 1, 2**63 - 1, 2**63, 2**63 + 1, 2**64 - 2, 2**64 - 1,
                2**32, 2**32 + 1, 2**64 - 2**32, 2**64 - 2**32 - 1, 2**62, 3 * 2**62, 2**64 - EPS, 2**64 - EPS - 1,
                2**64 - P + 1, 2**64 - P, 2**31, 2**64 - 2**31, 0x5555555555555555, 0xAAAAAAAAAAAAAAAB, 12345,
                2**64 - 12345, 0xFFFFFFFF00000000, 0x00000000FFFFFFFE, 0x0000000100000001, 0xFFFFFFFEFFFFFFFF,
                2**48, 2**64 - 2**48, 7})

SRC = r"""
#define __host__
#define __device__
#define __forceinline__ inline
#include "dft.cuh"
using namespace gl;
template <int B, bool INV> static void run(u64 *x, long n) {
    for (long i = 0; i < n; i++) {
        u64 v[1 << B];
        for (int k = 0; k < (1 << B); k++) v[k] = x[i * (1 << B) + k];
        msntt::dft_regs<B, INV>(v);
        for (int k = 0; k < (1 << B); k++) x[i * (1 << B) + k] = v[k];
    }
}
extern "C" void dft(int b, int inv, u64 *x, long n) {
    switch (2 * b + inv) {
    case 2: run<1, false>(x, n); break; case 3: run<1, true>(x, n); break;
    case 4: run<2, false>(x, n); break; case 5: run<2, true>(x, n); break;
    case 6: run<3, false>(x, n); break; case 7: run<3, true>(x, n); break;
    case 8: run<4, false>(x, n); break; case 9: run<4, true>(x, n); break;
    }
}
static void put(const L96 &v, u32 *o) { o[0] = v.w0; o[1] = v.w1; o[2] = v.w2; }
template <int K> static void shl_k(const u32 *a, u32 *o, long n) {
    for (long i = 0; i < n; i++) put(l96_mul_pow2<K>(L96{a[3 * i], a[3 * i + 1], a[3 * i + 2]}), o + 3 * i);
}
template <int K> static void shl_dispatch(int k, const u32 *a, u32 *o, long n) {
    if constexpr (K < 96) { if (k == K) shl_k<K>(a, o, n); else shl_dispatch<K + 1>(k, a, o, n); }
}
extern "C" void limb_ops(const u32 *a, const u32 *b, u32 *sum, u32 *dif, long n) {
    for (long i = 0; i < n; i++) {
        const L96 x{a[3 * i], a[3 * i + 1], a[3 * i + 2]}, y{b[3 * i], b[3 * i + 1], b[3 * i + 2]};
        put(l96_add(x, y), sum + 3 * i);
        put(l96_sub(x, y), dif + 3 * i);
    }
}
extern "C" void mul_pow2(int k, const u32 *a, u32 *o, long n) { shl_dispatch<1>(k, a, o, n); }
extern "C" void reduce(const u32 *a, u64 *o, long n) {
    for (long i = 0; i < n; i++) o[i] = l96_reduce(L96{a[3 * i], a[3 * i + 1], a[3 * i + 2]});
}
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("dft_limbs")
    src, so = tmp / "dft.cpp", tmp / "dft.so"
    src.write_text(SRC)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", "-I", CSRC, "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.dft.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_long]
    L.limb_ops.argtypes = [C.c_void_p] * 4 + [C.c_long]
    L.mul_pow2.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_long]
    L.reduce.argtypes = [C.c_void_p, C.c_void_p, C.c_long]
    return L


def _omega(b, inv):
    """the 2^b-th root of unity of the networks: arkworks' omega_16 = 2^156 (as a field element), or its inverse"""
    w16 = pow(2, 156, P)
    w = pow(w16, 16 >> b, P)
    return pow(w, P - 2, P) if inv else w


def _brev(k, bits):
    return int(format(k, f"0{bits}b")[::-1], 2) if bits else 0


def _want(rows, b, inv):
    """output kappa in register brev(kappa): sum_k x_k omega^(k kappa), canonical (Montgomery words are linear)"""
    n = 1 << b
    w = _omega(b, inv)
    tw = [pow(w, e, P) for e in range(n)]
    out = []
    for row in rows:
        xs = [int(v) % P for v in row]
        o = [0] * n
        for kap in range(n):
            o[_brev(kap, b)] = sum(xs[k] * tw[(k * kap) % n] for k in range(n)) % P
        out.append(o)
    return np.array(out, dtype=np.uint64)


def _run(lib, rows, b, inv):
    x = np.ascontiguousarray(np.array(rows, dtype=np.uint64).reshape(-1))
    lib.dft(b, int(inv), x.ctypes.data, x.size >> b)
    return x.reshape(-1, 1 << b)


def _check(lib, rows, b, inv):
    got = _run(lib, rows, b, inv)
    assert np.array_equal(np.array([[int(v) % P for v in r] for r in got], dtype=np.uint64), _want(rows, b, inv))


@pytest.mark.parametrize("b", [1, 2, 3, 4])
@pytest.mark.parametrize("inv", [False, True])
def test_networks_random_and_edge_positions(lib, b, inv):
    n = 1 << b
    rng = random.Random(1000 * b + inv)
    rows = [[rng.randrange(P) for _ in range(n)] for _ in range(300)]          # canonical
    rows += [[rng.randrange(R) for _ in range(n)] for _ in range(300)]         # any u64
    for e in EDGES:
        for pos in range(n):
            for bg in (0, P - 1, 2**64 - 1, 2**63):
                row = [bg] * n
                row[pos] = e
                rows.append(row)
    _check(lib, rows, b, inv)


@pytest.mark.parametrize("inv", [False, True])
def test_networks_random_edge_tuples(lib, inv):
    """200 000 seeded 16-tuples of edge words through the radix-16 network, every output checked mod p: the expected
    outputs are sums of per-(edge word, position) contributions, exact in Python integers"""
    b, n = 4, 16
    rng = np.random.default_rng(7 + inv)
    edges = np.array(EDGES, dtype=np.uint64)
    idx = rng.integers(0, len(EDGES), size=(200_000, n))
    rows = edges[idx]
    got = _run(lib, rows, b, inv)
    w = _omega(b, inv)
    contrib = np.zeros((len(EDGES), n, n), dtype=object)
    for ei, e in enumerate(EDGES):
        for k in range(n):
            for kap in range(n):
                contrib[ei, k, _brev(kap, b)] = e % P * pow(w, k * kap, P) % P
    for r in range(0, len(rows), 50_000):
        blk = idx[r:r + 50_000]
        acc = np.zeros((len(blk), n), dtype=object)
        for k in range(n):
            acc += contrib[blk[:, k], k, :]
        acc %= P
        g = got[r:r + 50_000].astype(object) % P
        assert (acc == g).all()


def _l96(v):
    v %= 2**96
    return [v & 0xFFFFFFFF, (v >> 32) & 0xFFFFFFFF, v >> 64]


def _val(limbs):
    v = int(limbs[0]) | int(limbs[1]) << 32 | int(limbs[2]) << 64
    return v - 2**96 if v >> 95 else v


def test_limb_primitives_edge_pairs(lib):
    """3-limb add/sub, the shift-by-2^K fold for every K and the final reduction, over all pairs of edge words lifted
    into the signed 96-bit ranges the networks produce"""
    vals = []
    for e in EDGES:
        for hi in (0, 1, -1, 2, -2, 7, -8, 31, -32):
            vals.append(e + hi * R)
    a_v = [x for x in vals for _ in vals]
    b_v = [y for _ in vals for y in vals]
    a = np.array([_l96(v) for v in a_v], dtype=np.uint32)
    b = np.array([_l96(v) for v in b_v], dtype=np.uint32)
    s, d = np.zeros_like(a), np.zeros_like(a)
    lib.limb_ops(a.ctypes.data, b.ctypes.data, s.ctypes.data, d.ctypes.data, len(a))
    assert all(_val(s[i]) == a_v[i] + b_v[i] for i in range(len(a)))
    assert all(_val(d[i]) == a_v[i] - b_v[i] for i in range(len(a)))
    src = np.array([_l96(v) for v in vals], dtype=np.uint32)
    for k in range(1, 96):
        o = np.zeros_like(src)
        lib.mul_pow2(k, src.ctypes.data, o.ctypes.data, len(src))
        for v, lim in zip(vals, o):
            w = _val(lim)
            assert (w - v * pow(2, k, P)) % P == 0
            assert abs(w) < 2**65 + 2**max(abs(v).bit_length() - 1, 0)
    # reduction: every value in [2^70, 2^72) the networks hand over, edge-structured
    red_in = [((1 << 70) + e + hi * R) for e in EDGES for hi in range(0, 3 * 2**6, 7)] + [2**72 - 1, 2**70]
    r_src = np.array([_l96(v) for v in red_in], dtype=np.uint32)
    out = np.zeros(len(red_in), dtype=np.uint64)
    lib.reduce(r_src.ctypes.data, out.ctypes.data, len(red_in))
    assert all((int(o) - v) % P == 0 for o, v in zip(out, red_in))
