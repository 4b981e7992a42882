"""CPU-only: pin the C oracle (oracle/gl_oracle.c) against (a) the constants the
reference carries, (b) the independent big-int spec oracle/pyspec.py incl. the
O(n^2) DFT definition, (c) hashlib.  There are no reference golden vectors for
this path (SURVEY.md §8c, "parity unpinned")."""
import hashlib
import random

import numpy as np
import pytest

from oracle import pyspec as S

P = S.P


def test_reference_constants(orc):
    # gpu/src/metal/felt_u64.h.metal:118,127 ; gpu/src/fields.rs:82
    assert orc.lib().orc_fp_one() == 4294967295 == S.ONE_MONT
    assert S.R2_MONT == 18446744065119617025
    assert orc.lib().orc_fp_from_canonical(2) == 8589934590
    # gpu/src/fields.rs:85-90 QUADRATIC_NONRESIDUE_TO_T
    assert orc.lib().orc_fp_from_canonical(16140901060737761281) == 2305843009213693952
    # 7 generates F_p^*, two-adic root (SURVEY.md §8c)
    assert S.TWO_ADIC_ROOT == 1753635133440165772
    assert orc.root_of_unity(20) == S.to_mont(3511170319078647661)
    assert orc.generator() == S.to_mont(7)
    for k in range(0, 33):
        w = S.from_mont(orc.root_of_unity(k))
        assert pow(w, 1 << k, P) == 1 and (k == 0 or pow(w, 1 << (k - 1), P) == P - 1)


def test_bit_reverse_golden(orc):
    # gpu/src/utils.rs:233-236
    v = np.arange(16, dtype=np.uint64)
    got = orc.bit_reverse(v, 1, 4)
    assert got.tolist() == [0, 8, 4, 12, 2, 10, 6, 14, 1, 9, 5, 13, 3, 11, 7, 15]
    assert [S.bit_reverse_index(16, i) for i in range(16)] == got.tolist()


def test_field_ops_vs_bigint(orc):
    rng = random.Random(1)
    edge = [0, 1, 2, P - 1, P - 2, 2**32, 2**32 - 1, 2**32 + 1, 2**63, 2**64 - 2**32, 0xFFFFFFFF, 0xFFFFFFFF00000000]
    vals = edge + [rng.randrange(P) for _ in range(200)]
    L = orc.lib()
    for a in vals:
        am = S.to_mont(a)
        assert L.orc_fp_from_canonical(a) == am and L.orc_fp_to_canonical(am) == a
        for b in vals[:24]:
            bm = S.to_mont(b)
            assert L.orc_fp_mul1(am, bm) == S.to_mont(a * b)
            assert L.orc_fp_add1(am, bm) == S.to_mont(a + b)
            assert L.orc_fp_sub1(am, bm) == S.to_mont(a - b)
        if a:
            assert L.orc_fp_inv1(am) == S.to_mont(pow(a, -1, P))
        assert L.orc_fp_pow1(am, 12345) == S.to_mont(pow(a, 12345, P))


def test_fq3_vs_bigint(orc):
    rng = random.Random(2)
    for _ in range(50):
        a = tuple(rng.randrange(P) for _ in range(3))
        b = tuple(rng.randrange(P) for _ in range(3))
        am = np.array([S.to_mont(x) for x in a], dtype=np.uint64)
        bm = np.array([S.to_mont(x) for x in b], dtype=np.uint64)
        out = np.empty(3, dtype=np.uint64)
        orc.lib().orc_fq3_mul1(orc._p(am), orc._p(bm), orc._p(out))
        assert tuple(S.from_mont(int(x)) for x in out) == S.fq3_mul(a, b)
        orc.lib().orc_fq3_inv1(orc._p(am), orc._p(out))
        inv = tuple(S.from_mont(int(x)) for x in out)
        assert S.fq3_mul(a, inv) == (1, 0, 0)
        assert inv == S.fq3_inv(a)
        orc.lib().orc_fq3_pow1(orc._p(am), 77, orc._p(out))
        assert tuple(S.from_mont(int(x)) for x in out) == S.fq3_pow(a, 77)


@pytest.mark.parametrize("log_n", [0, 1, 2, 3, 5, 8])
@pytest.mark.parametrize("offset", [1, 7, 1234567891011])
def test_ntt_vs_definition(orc, log_n, offset):
    n = 1 << log_n
    rng = random.Random(log_n * 7 + offset % 97)
    coeffs = [rng.randrange(P) for _ in range(n)]
    want = S.dft_naive(coeffs, log_n, offset)
    assert S.ntt(coeffs, log_n, offset) == want
    assert S.intt(want, log_n, offset) == coeffs
    m = orc.to_mont(np.array([coeffs], dtype=np.uint64))
    got = orc.from_mont(orc.ntt(m, 1, log_n, S.to_mont(offset)))
    assert got[0].tolist() == want
    back = orc.from_mont(orc.ntt(orc.to_mont(np.array([want], dtype=np.uint64)), 1, log_n, S.to_mont(offset), inverse=True))
    assert back[0].tolist() == coeffs


def test_ntt_fq3_lanes_and_multicolumn(orc):
    log_n, n = 6, 64
    rng = random.Random(5)
    cols = [[tuple(rng.randrange(P) for _ in range(3)) for _ in range(n)] for _ in range(3)]
    mat = orc.to_mont(np.array([[x for el in col for x in el] for col in cols], dtype=np.uint64))
    got = orc.from_mont(orc.ntt(mat, 3, log_n, S.to_mont(7)))
    for c, col in enumerate(cols):
        for lane in range(3):
            want = S.ntt([el[lane] for el in col], log_n, 7)
            assert got[c][lane::3].tolist() == want


@pytest.mark.parametrize("log_blowup", [0, 1, 2, 3, 4])
def test_lde_vs_spec(orc, log_blowup):
    log_n, n = 5, 32
    rng = random.Random(11 + log_blowup)
    coeffs = [rng.randrange(P) for _ in range(n)]
    m = orc.to_mont(np.array([coeffs, coeffs[::-1]], dtype=np.uint64))
    for bitrev in (False, True):
        got = orc.from_mont(orc.lde(m, 1, log_n, log_blowup, S.to_mont(7), bitrev=bitrev))
        assert got[0].tolist() == S.lde(coeffs, log_n, log_blowup, 7, bitrev)
        assert got[1].tolist() == S.lde(coeffs[::-1], log_n, log_blowup, 7, bitrev)


def test_lde_prefix_property(orc):
    # src/prover.rs:86-91: the first ce_domain_size entries of a bit-reversed LDE,
    # bit-reversed back, are the evaluations over the smaller coset offset*<g_ce>.
    log_n, log_b, log_ce = 4, 3, 1
    rng = random.Random(3)
    coeffs = [rng.randrange(P) for _ in range(1 << log_n)]
    full = S.lde(coeffs, log_n, log_b, 7, True)
    ce = 1 << (log_n + log_ce)
    assert S.bit_reverse(full[:ce]) == S.ntt(coeffs, log_n + log_ce, 7)


def test_sha256_vs_hashlib(orc):
    rng = random.Random(9)
    for ln in [0, 1, 3, 55, 56, 57, 63, 64, 65, 119, 120, 128, 136, 216, 256, 384, 1000]:
        msg = bytes(rng.randrange(256) for _ in range(ln))
        assert orc.sha256(msg) == hashlib.sha256(msg).digest()


@pytest.mark.parametrize("lanes,ncols", [(1, 1), (1, 17), (3, 9), (1, 32), (3, 16)])
def test_hash_rows_and_merkle(orc, lanes, ncols):
    nrows = 16
    mat = orc.rand_matrix(ncols, nrows, lanes, seed=77)
    canon = orc.from_mont(mat)
    got = orc.hash_rows(mat, lanes)
    leaves = []
    for i in range(nrows):
        if lanes == 1:
            row = [int(canon[c][i]) for c in range(ncols)]
        else:
            row = [tuple(int(x) for x in canon[c][3 * i:3 * i + 3]) for c in range(ncols)]
        leaves.append(S.hash_row(row, lanes))
        assert got[i].tobytes() == leaves[-1]
    nodes = orc.merkle_nodes(got)
    want = S.merkle_nodes(leaves)
    assert [nodes[k].tobytes() for k in range(nrows)] == want
    assert nodes[0].tobytes() == bytes(32)


def test_merkle_two_leaves(orc):
    leaves = np.frombuffer(hashlib.sha256(b"a").digest() + hashlib.sha256(b"b").digest(), dtype=np.uint8).reshape(2, 32)
    nodes = orc.merkle_nodes(leaves)
    assert nodes[1].tobytes() == hashlib.sha256(leaves.tobytes()).digest()


@pytest.mark.parametrize("lanes", [1, 3])
@pytest.mark.parametrize("log_ff", [1, 2, 3, 4])
def test_fri_drp_equals_per_coset_definition(orc, lanes, log_ff):
    log_n = 6
    n = 1 << log_n
    rng = random.Random(100 + lanes + log_ff)
    if lanes == 1:
        ev = [rng.randrange(P) for _ in range(n)]
        alpha = rng.randrange(P)
        flat = ev
        aflat = [alpha]
    else:
        ev = [tuple(rng.randrange(P) for _ in range(3)) for _ in range(n)]
        alpha = tuple(rng.randrange(P) for _ in range(3))
        flat = [x for e in ev for x in e]
        aflat = list(alpha)
    want = S.fri_apply_drp(ev, log_n, log_ff, alpha, lanes)
    assert want == S.fri_fold_definition(ev, log_n, log_ff, alpha, lanes)
    got = orc.from_mont(orc.fri_apply_drp(orc.to_mont(np.array(flat, dtype=np.uint64)), lanes, log_n, log_ff,
                                          orc.to_mont(np.array(aflat, dtype=np.uint64))))
    wflat = want if lanes == 1 else [x for e in want for x in e]
    assert got.tolist() == wflat


def test_pointwise_and_sum_columns(orc):
    n = 64
    a = orc.rand_matrix(1, n, 3, seed=1)[0]
    b = orc.rand_matrix(1, n, 1, seed=2)[0]
    ac, bc = orc.from_mont(a), orc.from_mont(b)
    got = orc.from_mont(orc.pointwise("mul", a, 3, b, 1, shift=5))
    for i in range(n):
        want = S.fq3_mul(tuple(int(x) for x in ac[3 * i:3 * i + 3]), (int(bc[(i + 5) % n]), 0, 0))
        assert tuple(int(x) for x in got[3 * i:3 * i + 3]) == want
    got = orc.from_mont(orc.pointwise("inv", b, 1))
    assert all(int(got[i]) * int(bc[i]) % P == 1 for i in range(n))
    got = orc.from_mont(orc.pointwise("exp", a, 3, exponent=5))
    assert tuple(int(x) for x in got[:3]) == S.fq3_pow(tuple(int(x) for x in ac[:3]), 5)
    m = orc.rand_matrix(5, n, 1, seed=3)
    s = orc.from_mont(orc.sum_columns(m, 1))
    mc = orc.from_mont(m)
    assert s.tolist() == [sum(int(mc[c][i]) for c in range(5)) % P for i in range(n)]


def test_deep_helpers(orc):
    n = 32
    rng = random.Random(4)
    coeffs = [tuple(rng.randrange(P) for _ in range(3)) for _ in range(n)]
    zs = [tuple(rng.randrange(P) for _ in range(3)) for _ in range(2)]
    cs = [tuple(rng.randrange(P) for _ in range(3)) for _ in range(2)]
    flat = lambda v: orc.to_mont(np.array([x for e in v for x in e], dtype=np.uint64))
    got = orc.from_mont(orc.divide_out_points(flat(coeffs), flat(zs), flat(cs)))
    want = S.divide_out_points(coeffs, zs, cs)
    assert got.tolist() == [x for e in want for x in e]
    h = orc.from_mont(orc.horner(flat(coeffs), 3, flat(zs[:1])))
    assert tuple(int(x) for x in h) == S.horner(coeffs, zs[0], 3)
    base = [rng.randrange(P) for _ in range(n)]
    h = orc.from_mont(orc.horner(orc.to_mont(np.array(base, dtype=np.uint64)), 1, flat(zs[:1])))
    assert tuple(int(x) for x in h) == S.horner(base, zs[0], 1)


def test_pow_grind_vs_hashlib(orc):
    # PublicCoin::verify_proof_of_work (src/random.rs:129-132): leading zero bits of SHA-256(seed || nonce_be)
    seed = hashlib.sha256(b"pow").digest()
    for bits in (0, 1, 5, 11):
        nonce = orc.pow_grind(seed, bits)
        def lz(n):
            d = hashlib.sha256(seed + n.to_bytes(8, "big")).digest()
            return len(bin(int.from_bytes(d, "big"))) - 2 if False else 256 - int.from_bytes(d, "big").bit_length()
        assert nonce >= 1 and lz(nonce) >= bits
        assert all(lz(k) < bits for k in range(1, nonce))


def test_pow_grind_past_the_first_device_launch(orc):
    # the serial search behind the 24-bit cases of tests/test_gpu_commit_stages_fri.py::test_pow_grind_smallest_nonce,
    # whose answers lie in the first, second and third 2^24-nonce launch of the device grind (about 16 s on one core)
    for tag, nonce in ((b"g0", 10056532), (b"g2", 28919286), (b"g5", 41922605), (b"g3", 45695959)):
        assert orc.pow_grind(hashlib.sha256(tag).digest(), 24) == nonce, tag


def test_scan_affine_oracle_vs_definition(orc):
    # x_0 = init, x_(i+1) = x_i * a_i + b_i in big-int Python
    n = 37
    a = orc.rand_matrix(1, n, 3, seed=5)[0]
    b = orc.rand_matrix(1, n, 1, seed=6)[0]
    init = orc.rand_matrix(1, 1, 3, seed=7)[0]
    x = tuple(S.from_mont(int(w)) for w in init)
    want_ex, want_in = [], []
    for i in range(n):
        want_ex.append(x)
        ai = tuple(S.from_mont(int(w)) for w in a[3 * i:3 * i + 3])
        x = S.fq3_add(S.fq3_mul(x, ai), (S.from_mont(int(b[i])), 0, 0))
        want_in.append(x)
    canon = lambda arr: [tuple(S.from_mont(int(w)) for w in arr[3 * i:3 * i + 3]) for i in range(n)]
    assert canon(orc.scan_affine(3, n, init, a=a, fa=3, b=b, fb=1, inclusive=False)) == want_ex
    assert canon(orc.scan_affine(3, n, init, a=a, fa=3, b=b, fb=1, inclusive=True)) == want_in


def test_work_split_does_not_change_results(orc):
    """the oracle's two ways of using the threads (whole columns per thread / every butterfly level across the threads) and
    the parallel bit reverse (from 2^17 elements, gpu/src/utils.rs:48-78) give the same words, whatever the thread count"""
    import hashlib
    import os
    import subprocess
    import sys
    code = r'''
import hashlib, numpy as np
from oracle import oracle as orc
h = hashlib.sha256()
for lanes, ncols in ((1, 3), (3, 2)):
    m = orc.rand_matrix(ncols, 1 << 15, lanes, seed=ncols)
    p = orc.ntt(m, lanes, 15, inverse=True)
    assert np.array_equal(orc.ntt(p, lanes, 15), m)
    h.update(p.tobytes())
    h.update(orc.lde(p, lanes, 15, 2, orc.generator(), True).tobytes())       # 2^17 points: the parallel bit reverse
    h.update(orc.lde(p, lanes, 15, 1, orc.generator(), False).tobytes())      # the zero-padded DIF branch
print(h.hexdigest())
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    got = set()
    for env in ({"ORACLE_COLUMN_PARALLEL": "1"}, {"ORACLE_COLUMN_PARALLEL": "0"}, {"OMP_NUM_THREADS": "1"}, {"OMP_NUM_THREADS": "5"}):
        out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, cwd=root)
        assert out.returncode == 0, out.stderr
        got.add(out.stdout.strip())
    assert len(got) == 1
