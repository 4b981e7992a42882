"""Rescue-Prime over Goldilocks, restated with Python integers for the tests of examples/rescue.

Independent of ministark_b200/examples/rescue.py: the parameters follow the reference's recipe
(examples/rescue/rescue.rs:100-214) with the Gauss-Jordan step of Algorithm 4 of eprint 2020/1143 as published (the
reference assigns pivot * m[r][j] where the elimination subtracts it).  Values are canonical integers."""
import hashlib

P = 2**64 - 2**32 + 1
M, CAPACITY, ROUNDS, SECURITY = 12, 4, 7, 128


def alphas():
    """Algorithm 6: the least alpha >= 3 coprime to p - 1, and its inverse mod p - 1"""
    a = 3
    while True:
        g, x = _egcd(a, P - 1)
        if g == 1:
            return a, x % (P - 1)
        a += 1


def _egcd(a, b):
    x0, x1, r0, r1 = 1, 0, a, b
    while r1:
        q = r0 // r1
        r0, r1 = r1, r0 - q * r1
        x0, x1 = x1, x0 - q * x1
    return r0, x0


def round_constants():
    """2 m N values: SHAKE-256 of the seed, 9 bytes per constant read little-endian, reduced mod p"""
    seed = f"Rescue-XLIX({P},{M},{CAPACITY},{SECURITY})".encode()
    count = 2 * M * ROUNDS
    stream = hashlib.shake_256(seed).digest(9 * count)
    return [int.from_bytes(stream[9 * i:9 * i + 9], "little") % P for i in range(count)]


def rref(rows):
    """reduced row echelon form over Fp (Gauss-Jordan)"""
    m = [list(r) for r in rows]
    nr, nc = len(m), len(m[0])
    lead = 0
    for r in range(nr):
        if lead >= nc:
            break
        i = r
        while m[i][lead] == 0:
            i += 1
            if i == nr:
                i, lead = r, lead + 1
                if lead == nc:
                    return m
        m[i], m[r] = m[r], m[i]
        inv = pow(m[r][lead], P - 2, P)
        m[r] = [v * inv % P for v in m[r]]
        for i in range(nr):
            if i != r and m[i][lead]:
                f = m[i][lead]
                m[i] = [(a - f * b) % P for a, b in zip(m[i], m[r])]
        lead += 1
    return m


def mds():
    """the transpose of the right half of rref(G), G[i][j] = 7^(i j), i < m, j < 2m"""
    g = [[pow(7, i * j, P) for j in range(2 * M)] for i in range(M)]
    e = rref(g)
    return [[e[j][M + i] for j in range(M)] for i in range(M)]


ALPHA, ALPHA_INV = alphas()
RC = round_constants()
MDS = mds()


def permute(state):
    s = list(state)
    for r in range(ROUNDS):
        s = [pow(v, ALPHA, P) for v in s]
        s = [(sum(MDS[i][j] * s[j] for j in range(M)) + RC[2 * M * r + i]) % P for i in range(M)]
        s = [pow(v, ALPHA_INV, P) for v in s]
        s = [(sum(MDS[i][j] * s[j] for j in range(M)) + RC[2 * M * r + M + i]) % P for i in range(M)]
    return s


def round_states(state):
    """the 8 states of one permutation as the trace holds them: before rounds 0..6, then the output"""
    s = list(state)
    out = []
    for r in range(ROUNDS):
        out.append(s)
        s = [pow(v, ALPHA, P) for v in s]
        s = [(sum(MDS[i][j] * s[j] for j in range(M)) + RC[2 * M * r + i]) % P for i in range(M)]
        s = [pow(v, ALPHA_INV, P) for v in s]
        s = [(sum(MDS[i][j] * s[j] for j in range(M)) + RC[2 * M * r + M + i]) % P for i in range(M)]
    out.append(s)
    return out


def chain_trace(seed, K, L):
    """(rows, digests): the n = 8 K L rows of 12 canonical words and the K four-word digests.  Chain k starts from
    (s_0, s_1, s_2, s_3, w_K^k, 0, ..., 0) with w_K the generator of the order-K subgroup, and applies the permutation L
    times; row 8 (L k + j) + r holds permutation j's state before round r, and its output at r = 7."""
    two_adic_root = pow(7, (P - 1) >> 32, P)
    w = pow(two_adic_root, (1 << 32) // K, P)
    rows, digests = [], []
    for k in range(K):
        s = [v % P for v in seed] + [pow(w, k, P)] + [0] * (M - 5)
        for _ in range(L):
            block = round_states(s)
            rows += block
            s = block[-1]
        digests.append(s[:4])
    return rows, digests
