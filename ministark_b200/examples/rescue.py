"""examples/rescue: K chains of the Rescue-Prime permutation, and preimages of K Rescue-Prime hashes, over Goldilocks,
Fq = Fq3, with the traces built on the GPU.

The permutation is Rescue-Prime with the parameters of the published Rp64_256 instance: state width m = 12, capacity 4
(the last four words), N = 7 rounds, 128-bit security level, alpha = 7 and alpha^-1 = 10540996611094048183 (the inverse
of 7 mod p - 1).  The parameters follow the reference's recipe (examples/rescue/rescue.rs:100-214):
  * 2 m N = 168 round constants from SHAKE-256 of "Rescue-XLIX(18446744069414584321,12,4,128)", 9 bytes per constant
    read little-endian and reduced mod p;
  * the MDS matrix is the transpose of the right half of the reduced row echelon form of G[i][j] = 7^(i j), 12 x 24.
    It is built by Algorithm 4 of eprint 2020/1143 as written: the reference's Gauss-Jordan step (rescue.rs:256-262)
    assigns pivot * m[r][j] where the elimination subtracts it, and its matrix is not the published one.
A round is S-box (x^7), MDS, the first twelve constants, inverse S-box (x^(1/7)), MDS, the second twelve constants; the
MDS matrix acts on the state as a column vector.  The reference's example is an unfinished stub over the 252-bit field,
so there is no reference output to compare with: oracle/rescue_oracle.py restates all of this independently.

The claim (RescueChainsClaim): chain k = 0..K-1 starts from (s_0, s_1, s_2, s_3, w_K^k, 0, ..., 0), w_K =
domain_generator(log2 K), and applies the permutation L times; K and L are powers of two.  The public inputs are s, K, L
and the K digests, digest_k being the first four words of chain k's final state.  The tag w_K^k keeps the chains apart: it
is X at the chain's first row, so its boundary constraint needs no counter column.

Trace layout, n = 8 K L rows:

    base columns       0..11: S_0..S_11, the state.  Chain k holds rows [8 L k, 8 L (k + 1)); row 8 j + r of a chain
                       holds permutation j's state before round r for r < 7, and its output at r = 7.
    extension column   12: R, an inclusive running evaluation over the challenge gamma (Fq3): R_i = R_(i-1) mul_i + add_i
                       with mul = 1 + e (gamma^4 - 1), add = e (S_0 + gamma S_1 + gamma^2 S_2 + gamma^3 S_3), e the
                       periodic selector of the chain-end rows 8 L (k + 1) - 1.  Declared (AirConfig.extension_columns),
                       so the prover builds it on the device.

Constraints, in this order (ROUND, LINK, START, and the three on R):
    ROUND  0..11   MDS s^7 + c1_r = (MDS^-1 (t - c2_r))^7, s this row, t the next, on every row with r != 7: c1_r and
                   MDS^-1 c2_r are degree-7 polynomials in y = x^(n / 8), which is w_8^r on the rows of round r, and
                   the zerofier y - w_8^7 of the r = 7 rows is divided out of x^n - 1
    LINK  12..23   t = s on the r = 7 rows but the K chain ends {g^(8 L (k + 1) - 1)}, whose zerofier (g x)^K - 1 is
                   multiplied in
    START 24..35   (S_w - s_w) / (x^K - 1) for w < 4 (s_w = Hint(1 + w)), (S_4 - X) / (x^K - 1), S_w / (x^K - 1) for w > 4
    36             R = 0 on the first row (never a chain end)
    37             R_(i+1) = R_i where row i + 1 is not a chain end, the last row excepted: zerofier
                   (x^n - 1) / (((g^2 x)^K - 1) (x - g^(n - 1)))
    38             R_(i+1) = R_i gamma^4 + S_0 + gamma S_1 + gamma^2 S_2 + gamma^3 S_3 at row i + 1 where row i + 1 is a
                   chain end: zerofier (g^2 x)^K - 1
    39             R = Hint(0) on the last row: the Horner evaluation at gamma of the 4 K digest words, which gen_hints
                   computes from the public digests.  A prover that changed a digest would need a gamma at which two
                   different degree-(4K - 1) polynomials agree: probability at most 4K / |Fq3| by Schwartz-Zippel.

The constraints use no periodic column: every row pattern is a zerofier or a polynomial in a power of x, which any
verifier (and oracle/stark_oracle.py) evaluates at the out-of-domain point.  By the reference's degree rule
(constraints.rs:404-455, air.py's `degree`) the round constraints have degree 7 (n - 1) + n / 8 - n over a trace of
degree n - 1, which rounds up to a ce blow-up of 8; every other constraint has blow-up 1.  OPTIONS uses an LDE blow-up of 8: 40 queries
of 3 bits plus 8 bits of grinding give 128 bits, which is also the cap of Proof.security_level_bits; the field term,
192 - log2(8 n), stays above it up to n = 2^61.

The hash (hash(words)) is the reference's Rescue::finish (rescue.rs:49-97) over this permutation with rate 8 (words
0..7), capacity 4 and a 4-word digest: pad with one 1 and then zeros to B = floor(length / 8) + 1 blocks, start from the
all-zero state, add each block into words 0..7 and permute, and squeeze words 0..3.

The hash claim (RescueHashClaim(length, digests)): I know K = len(digests) messages of `length` words each, and message
k hashes to digests[k].  K is a power of two; L is the smallest power of two >= B, and n = 8 K L.  The public inputs are
K, the length and the 4 K digest words.  The proof shows knowledge of the preimages; it is not zero-knowledge (the
reference's proofs are not either), so it does not hide them.

Its trace, n = 8 K L rows (gen_hash_trace):

    base columns       0..11: S_0..S_11, laid out as in the chains trace.  Message k holds rows [8 L k, 8 L (k + 1));
                       row 8 j + r holds permutation j's state before round r (block j added) and its output at r = 7.
                       Permutations B..L-1 absorb zero blocks: they satisfy every constraint and leave the digest alone.
    base column        12: M, the absorbed words: row 8 L k + 8 j + i holds word i of padded block j of message k for
                       j < B, and 0 for j >= B.
    extension column   13: R as in the chains trace, its selector on the digest rows 8 L k + 8 B - 1 instead of the chain
                       ends (the same rows when B = L).

Constraints, in this order (hash_air_config(K, length).groups(n) gives their index ranges):
    ROUND  12      as in the chains AIR
    LINK   12      on the chains AIR's rows (the r = 7 rows but the chain ends): t_w = s_w + M(1 + w) for w < 8, t_w =
                   s_w for w >= 8, M(o) the absorbed word o rows below.  None when L = 1: every r = 7 row is then a chain
                   end, chain_ends / last_rounds is a constant and the quotient would be a plain polynomial
    START  12      over x^K - 1: S_w = M(w) for w < 8 and S_w = 0 for w >= 8 (the zero state plus block 0)
    PAD    8 - t   t = length - 8 (B - 1): for each padded position p = length .. 8 B - 1, M = [p = length] over
                   (g^(-p) x)^K - 1
    R      4       as in the chains AIR, with the digest rows in place of the chain ends: (g^2 x)^K - 1 becomes
                   (g^(2 - 8 B) x)^K - 1
48 - t constraints in all, 36 - t when L = 1; the ce blow-up stays 8 and OPTIONS is reused.  The constraints read M at
row offsets 0 through 8.
"""
import hashlib
import operator

import numpy as np

from .. import expr as E
from ..air import AirConfig, ProofOptions, RunningColumn, domain_generator
from ..prover import Stark, Trace

P = E.P
_R = 2**64
_RINV = pow(_R, -1, P)
WIDTH, CAPACITY, ROUNDS, SECURITY_BITS = 12, 4, 7, 128
ALPHA = 7
ALPHA_INV = pow(ALPHA, -1, P - 1)                       # 10540996611094048183
DIGEST = 4                                              # words of a chain's digest: the first four of its final state
RATE = 8                                                # the hash absorbs into words 0..7; words 8..11 are the capacity
OPTIONS = ProofOptions(40, 8, 8, 8, 64)
SECURITY_LEVEL = 128
ROUND = range(0, 12)                                    # constraint indices, see the module docstring
LINK = range(12, 24)
START = range(24, 36)


def _round_constants():
    seed = f"Rescue-XLIX({P},{WIDTH},{CAPACITY},{SECURITY_BITS})".encode()
    count = 2 * WIDTH * ROUNDS
    stream = hashlib.shake_256(seed).digest(9 * count)
    return [int.from_bytes(stream[9 * i:9 * (i + 1)], "little") % P for i in range(count)]


def _echelon(m):
    """reduced row echelon form over Fp by Gauss-Jordan elimination (Algorithm 4 of eprint 2020/1143)"""
    m = [list(r) for r in m]
    rows, cols = len(m), len(m[0])
    lead = 0
    for r in range(rows):
        while lead < cols and all(m[i][lead] == 0 for i in range(r, rows)):
            lead += 1
        if lead == cols:
            break
        i = next(i for i in range(r, rows) if m[i][lead])
        m[r], m[i] = m[i], m[r]
        inv = pow(m[r][lead], -1, P)
        m[r] = [v * inv % P for v in m[r]]
        for i in range(rows):
            if i != r and m[i][lead]:
                f = m[i][lead]
                m[i] = [(a - f * b) % P for a, b in zip(m[i], m[r])]
        lead += 1
    return m


def _mds():
    gen = [[pow(7, i * j, P) for j in range(2 * WIDTH)] for i in range(WIDTH)]
    ech = _echelon(gen)
    return [[ech[j][WIDTH + i] for j in range(WIDTH)] for i in range(WIDTH)]


def _inverse(m):
    k = len(m)
    aug = _echelon([list(row) + [int(i == j) for j in range(k)] for i, row in enumerate(m)])
    assert all(aug[i][i] == 1 for i in range(k)), "singular matrix"
    return [row[k:] for row in aug]


RC = _round_constants()
MDS = _mds()
MDS_INV = _inverse(MDS)


def _mat_vec(m, v):
    return [sum(a * b for a, b in zip(row, v)) % P for row in m]


def round_states(state):
    """the eight states of one permutation as the trace holds them: before rounds 0..6, then the output"""
    s = [int(v) % P for v in state]
    out = []
    for r in range(ROUNDS):
        out.append(s)
        u = _mat_vec(MDS, [pow(v, ALPHA, P) for v in s])
        u = [(a + c) % P for a, c in zip(u, RC[2 * WIDTH * r:2 * WIDTH * r + WIDTH])]
        v = _mat_vec(MDS, [pow(a, ALPHA_INV, P) for a in u])
        s = [(a + c) % P for a, c in zip(v, RC[2 * WIDTH * r + WIDTH:2 * WIDTH * (r + 1)])]
    out.append(s)
    return out


def permute(state):
    """the Rescue-Prime permutation of a 12-word state (canonical integers)"""
    return round_states(state)[-1]


def _check_shape(seed, K, L):
    if len(seed) != DIGEST or any(not 0 <= int(v) < P for v in seed):
        raise ValueError("the seed is four canonical field elements")
    for name, v in (("K", K), ("L", L)):
        if v < 1 or v & (v - 1):
            raise ValueError(f"{name} = {v} is not a power of two")
    if (8 * K * L).bit_length() - 1 > 32:
        raise ValueError(f"8 K L = {8 * K * L} rows: the trace domain has at most 2^32 points")


def gen_trace(seed, K, L, device=None):
    """(Trace, digests) of the K chains of L permutations from `seed` (four canonical words); digests: K tuples of four
    canonical words.  device=None: computed on the host with Python integers (small K L only: about 0.2 ms per
    permutation).  device: built on that device by ms_rescue_chains and handed over as a resident (12, n) tensor, the
    digests read back from its chain-end rows."""
    seed = [int(v) for v in seed]
    _check_shape(seed, K, L)
    n = 8 * K * L
    if device is None:
        w = domain_generator(K.bit_length() - 1)
        cols = np.empty((WIDTH, n), dtype=np.uint64)
        digests = []
        for k in range(K):
            s = seed + [pow(w, k, P)] + [0] * (WIDTH - DIGEST - 1)
            for j in range(L):
                block = round_states(s)
                row = 8 * (L * k + j)
                cols[:, row:row + 8] = np.array([[v * _R % P for v in st] for st in block], dtype=np.uint64).T
                s = block[-1]
            digests.append(tuple(s[:DIGEST]))
        return Trace(cols), digests
    import torch
    dev = _torch_device(device)
    out = torch.empty((WIDTH, n), dtype=torch.int64, device=dev)
    ctx = _context(dev)
    if out.is_cuda:                     # the context's stream may not be torch's: torch's work on this memory is done
        torch.cuda.current_stream(dev).synchronize()
    ctx.rescue_chains(seed, K, L, out)
    ctx.sync()                          # complete before the prover reads it on its own stream
    ends = out[:DIGEST, 8 * L - 1::8 * L].cpu().numpy().view(np.uint64)
    digests = [tuple(int(w) * _RINV % P for w in ends[:, k]) for k in range(K)]
    return Trace(out), digests


# ---------------------------------------------------------------------------------------------------- the hash
def hash(words):
    """the Rescue-Prime hash of a message of canonical words (the reference's Rescue::finish, rescue.rs:49-97, with
    width 12, rate 8, capacity 4): pad with one 1 and then zeros to a multiple of the rate, start from the all-zero
    state, add each 8-word block into words 0..7 and permute, and squeeze the first four words.  Returns a 4-tuple."""
    words = [int(v) for v in words]
    if any(not 0 <= v < P for v in words):
        raise ValueError("message words must be canonical field elements (0 <= word < p)")
    padded = _padded(words, _blocks(len(words)))
    s = [0] * WIDTH
    for j in range(0, len(padded), RATE):
        s = permute([(a + b) % P for a, b in zip(s[:RATE], padded[j:j + RATE])] + s[RATE:])
    return tuple(s[:DIGEST])


def _blocks(length):
    """B, the number of rate blocks of a padded message of `length` words: the padding always appends the 1"""
    return length // RATE + 1


def _padded(words, num_blocks):
    """the message, its 1 and zeros up to num_blocks rate blocks"""
    return list(words) + [1] + [0] * (RATE * num_blocks - len(words) - 1)


def _hash_shape(K, length):
    """(B, L) for K messages of `length` words: B rate blocks each, L the smallest power of two >= B permutations per
    chain; ValueError unless K is a power of two, length >= 0 and 8 K L <= 2^32"""
    if K < 1 or K & (K - 1):
        raise ValueError(f"K = {K} messages is not a power of two")
    if length < 0:
        raise ValueError(f"length = {length} is negative")
    B = _blocks(length)
    L = 1 << (B - 1).bit_length()
    if (8 * K * L).bit_length() - 1 > 32:
        raise ValueError(f"8 K L = {8 * K * L} rows: the trace domain has at most 2^32 points")
    return B, L


def _messages(messages):
    """(K, length) C-contiguous uint64 array of canonical words, or ValueError"""
    if isinstance(messages, np.ndarray):
        if messages.ndim != 2 or messages.dtype != np.uint64:
            raise ValueError("messages: a (K, length) uint64 array")
        arr = np.ascontiguousarray(messages)
    else:
        rows = [[int(v) for v in m] for m in messages]
        if len({len(r) for r in rows}) > 1:
            raise ValueError("every message of a claim has the same length")
        try:
            arr = np.array(rows, dtype=np.uint64).reshape(len(rows), len(rows[0]) if rows else 0)
        except OverflowError:
            raise ValueError("message words must be canonical field elements (0 <= word < p)") from None
    if (arr >= np.uint64(P)).any():
        raise ValueError("message words must be canonical field elements (0 <= word < p)")
    return arr


def gen_hash_trace(messages, device=None):
    """(Trace, digests) of RescueHashClaim for K messages of one length: `messages` is K equal-length sequences or a
    (K, length) uint64 array of canonical words, K a power of two; digests: K tuples of four canonical words.
    device=None: computed on the host with Python integers (small shapes only).  device: built on that device by
    ms_rescue_hash and handed over as a resident (13, n) tensor, the digests read back from the digest rows."""
    msgs = _messages(messages)
    K, length = msgs.shape
    B, L = _hash_shape(K, length)
    n = 8 * K * L
    if device is None:
        cols = np.zeros((WIDTH + 1, n), dtype=np.uint64)
        digests = []
        for k in range(K):
            padded = _padded([int(v) for v in msgs[k]], L)        # the filler blocks are zero
            base = 8 * L * k
            s = [0] * WIDTH
            for j in range(L):
                s = [(a + b) % P for a, b in zip(s[:RATE], padded[RATE * j:RATE * (j + 1)])] + s[RATE:]
                block = round_states(s)
                cols[:WIDTH, base + 8 * j:base + 8 * j + 8] = np.array([[v * _R % P for v in st] for st in block],
                                                                        dtype=np.uint64).T
                s = block[-1]
                if j == B - 1:
                    digests.append(tuple(s[:DIGEST]))
            cols[WIDTH, base:base + 8 * L] = [v * _R % P for v in padded]
        return Trace(cols), digests
    import torch
    dev = _torch_device(device)
    out = torch.empty((WIDTH + 1, n), dtype=torch.int64, device=dev)
    ctx = _context(dev)
    if out.is_cuda:                     # the context's stream may not be torch's: torch's work on this memory is done
        torch.cuda.current_stream(dev).synchronize()
    ctx.rescue_hash(msgs, K, length, out)
    ctx.sync()                          # complete before the prover reads it on its own stream
    rows = _from_mont(out[:DIGEST, 8 * B - 1::8 * L].cpu().numpy().view(np.uint64))
    return Trace(out), [tuple(r) for r in rows.T.tolist()]


def _from_mont(w):
    """canonical values of a uint64 array of Montgomery words, vectorised: w 2^-64 = -w 2^32 (mod p), since 2^96 = -1.
    With w = h 2^32 + l: w 2^32 = h 2^64 + l 2^32 = (h + l) 2^32 - h, so the value is h - (h + l) 2^32."""
    p, eps = np.uint64(P), np.uint64(2**32 - 1)                    # eps = 2^64 mod p
    h, lo = w >> np.uint64(32), w & eps
    s = h + lo                                                      # < 2^33
    t = ((s & eps) << np.uint64(32)) + (s >> np.uint64(32)) * eps  # = s 2^32 (mod p), below 2^64 < 2 p
    t = np.where(t >= p, t - p, t)
    return np.where(h >= t, h - t, p - (t - h))


_CONTEXTS = {}


def _torch_device(device):
    import torch
    dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def _context(dev):
    """one context per device for building traces, queued on torch's current stream"""
    import torch
    from .. import Context
    key = (dev.type, dev.index)
    if key not in _CONTEXTS:
        _CONTEXTS[key] = Context(dev.index or 0)
    ctx = _CONTEXTS[key]
    if dev.type == "cuda":
        ctx.set_stream(torch.cuda.current_stream(dev).cuda_stream)
    return ctx


# ---------------------------------------------------------------------------------------------------------- the AIR
def _interpolate(values):
    """coefficients of the polynomial p of degree < I with p(w_I^j) = values[j] (I = len(values), a power of two): the
    Periodic form of a column of period I"""
    size = len(values)
    w_inv = pow(domain_generator(size.bit_length() - 1), -1, P)
    scale = pow(size, -1, P)
    return [scale * sum(v * pow(w_inv, j * k % size, P) for j, v in enumerate(values)) % P for k in range(size)]


def _selector(position, interval):
    """Periodic column of period `interval` that is 1 at rows = position (mod interval) and 0 elsewhere: the coefficients
    (1 / I) w_I^(-position k) in closed form"""
    w_inv = pow(domain_generator(interval.bit_length() - 1), -1, P)
    step = pow(w_inv, position, P)
    c, coeffs = pow(interval, -1, P), []
    for _ in range(interval):
        coeffs.append(c)
        c = c * step % P
    return E.Periodic(coeffs, interval)


def _round_coefficients():
    """c1_r[w] and (MDS^-1 c2_r)[w] as polynomials in y = x^(n / 8), which is w_8^r on the rows of round r: per word,
    the 8 coefficients of the interpolant of (value in round 0, ..., value in round 6, 0)"""
    c1 = [[RC[2 * WIDTH * r + w] for r in range(ROUNDS)] + [0] for w in range(WIDTH)]
    d = [_mat_vec(MDS_INV, RC[2 * WIDTH * r + WIDTH:2 * WIDTH * (r + 1)]) for r in range(ROUNDS)]
    d = [[d[r][w] for r in range(ROUNDS)] + [0] for w in range(WIDTH)]
    return [_interpolate(v) for v in c1], [_interpolate(v) for v in d]


C1_COEFFS, D_COEFFS = _round_coefficients()


def _linear(terms):
    acc = None
    for t in terms:
        acc = t if acc is None else acc + t
    return acc


def _round_constraints(n):
    """ROUND: MDS s^7 + c1_r = (MDS^-1 (t - c2_r))^7 for every word, s this row and t the next, on every row with r != 7
    (both AIRs: the permutation sits at rows 8 j .. 8 j + 7 of every chain)"""
    x, T, one = E.X(), E.Trace, E.Constant(1)
    all_rows = x ** n - one
    last_rounds = x ** (n // 8) - E.Constant(pow(domain_generator(3), 7, P))          # zero on the r = 7 rows
    y = [one, x ** (n // 8)]                                                             # w_8^r on round r's rows
    for _ in range(6):
        y.append(y[-1] * y[1])
    c1 = [_linear(E.Constant(c) * y[k] for k, c in enumerate(C1_COEFFS[w])) for w in range(WIDTH)]
    d = [_linear(E.Constant(c) * y[k] for k, c in enumerate(D_COEFFS[w])) for w in range(WIDTH)]
    s7 = [T(j, 0) ** ALPHA for j in range(WIDTH)]
    on_rounds = last_rounds / all_rows
    rounds = []
    for w in range(WIDTH):
        fwd = _linear(E.Constant(MDS[w][j]) * s7[j] for j in range(WIDTH)) + c1[w]
        back = _linear(E.Constant(MDS_INV[w][j]) * T(j, 1) for j in range(WIDTH)) - d[w]
        rounds.append((fwd - back ** ALPHA) * on_rounds)
    return rounds


def _digest_constraints(n, K, position, R):
    """the four constraints on the running column R (both AIRs), K chains of n / K rows whose digest sits at row
    `position` of the chain (0 <= position < n / K, never 0): R = 0 on the first row; R_(i+1) = R_i where row i + 1 is
    not a digest row, the last row excepted; R_(i+1) = R_i gamma^4 + S_0 + gamma S_1 + gamma^2 S_2 + gamma^3 S_3 where
    it is; R = Hint(0) on the last row"""
    g = domain_generator(n.bit_length() - 1)
    x, T, one = E.X(), E.Trace, E.Constant(1)
    all_rows = x ** n - one
    gamma = E.Challenge(0)
    gpow = [one, gamma, gamma * gamma, gamma * gamma * gamma]
    g4 = gpow[2] * gpow[2]
    # zero on the rows i with i + 1 = position (mod n / K); the shift is reduced mod n / K, which leaves its K-th power
    # unchanged and makes it g^2 for a digest on the chain's last row
    before_digests = (E.Constant(pow(g, (1 - position) % (n // K), P)) * x) ** K - one
    last = E.Constant(pow(g, n - 1, P))
    lin_next = _linear(gpow[w] * T(w, 1) for w in range(DIGEST))
    hold = (T(R, 1) - T(R, 0)) * before_digests * (x - last) / all_rows
    absorb = (T(R, 1) - T(R, 0) * g4 - lin_next) / before_digests
    return [T(R, 0) / (x - one), hold, absorb, (T(R, 0) - E.Hint(0)) / (x - last)]


def _digest_column(position, interval):
    """R, the inclusive running evaluation over gamma of the digests at rows = position (mod interval)"""
    gamma = E.Challenge(0)
    e = _selector(position, interval)
    lin = _linear(E.Trace(w, 0) * (gamma ** w) if w else E.Trace(0, 0) for w in range(DIGEST))
    return RunningColumn(init=0, mul=E.Constant(1) + e * (gamma ** 4 - E.Constant(1)), add=e * lin, inclusive=True)


class RescueAirConfig(AirConfig):
    """The AIR of RescueChainsClaim for CHAINS = K chains (air_config(K)); L is trace_len / (8 K)."""
    NUM_BASE_COLUMNS = WIDTH
    NUM_EXTENSION_COLUMNS = 1
    FQ_IS_FP = False
    CHAINS = None

    @classmethod
    def _shape(cls, trace_len):
        K = cls.CHAINS
        if K is None:
            raise ValueError("use air_config(K): the AIR depends on the number of chains")
        if trace_len % (8 * K) or trace_len < 8 * K:
            raise ValueError(f"a trace of {trace_len} rows does not hold {K} chains of 8-row permutations")
        return K, trace_len // (8 * K)

    @classmethod
    def constraints(cls, trace_len):
        K, L = cls._shape(trace_len)
        n = trace_len
        g = domain_generator(n.bit_length() - 1)
        x, T, one = E.X(), E.Trace, E.Constant(1)
        last_rounds = x ** (n // 8) - E.Constant(pow(domain_generator(3), 7, P))      # zero on the r = 7 rows
        chain_ends = (E.Constant(g) * x) ** K - one                                     # zero on rows 8 L (k + 1) - 1
        chain_starts = x ** K - one                                                     # zero on rows 8 L k
        link = [(T(w, 1) - T(w, 0)) * chain_ends / last_rounds for w in range(WIDTH)]
        start = ([(T(w, 0) - E.Hint(1 + w)) / chain_starts for w in range(DIGEST)] + [(T(DIGEST, 0) - x) / chain_starts]
                 + [T(w, 0) / chain_starts for w in range(DIGEST + 1, WIDTH)])
        return _round_constraints(n) + link + start + _digest_constraints(n, K, 8 * L - 1, WIDTH)

    @classmethod
    def extension_columns(cls, trace_len):
        _, L = cls._shape(trace_len)
        return [_digest_column(8 * L - 1, 8 * L)]

    @classmethod
    def gen_hints(cls, trace_len, claim, challenges):
        """[the Horner evaluation at gamma of the digest words, s_0, s_1, s_2, s_3]"""
        if claim.K != cls.CHAINS or trace_len != 8 * claim.K * claim.L:
            raise ValueError(f"a trace of {trace_len} rows is not {claim.K} chains of {claim.L} permutations")
        return [digest_evaluation(claim.digests, challenges[0])] + list(claim.seed)


def digest_evaluation(digests, gamma):
    """R's value on the last row: acc <- acc gamma^4 + d_0 + gamma d_1 + gamma^2 d_2 + gamma^3 d_3 over the chains in
    order, from acc = 0 (gamma: a 3-tuple).  Any tuple width W works the same way, acc <- acc gamma^W + sum_w gamma^w
    d_w, as long as every tuple has W words (examples/merkle binds 5-word tuples)."""
    # that is sum_j a_j gamma^j with a_(W (K - 1 - k) + w) = word w of tuple k, evaluated in blocks of `block`
    # coefficients: inside a block a dot product of base-field words with gamma^0 .. gamma^(block - 1), one component at
    # a time; across blocks Horner steps by gamma^block (about 25 times faster than one Fq3 product per word)
    gamma = E._q(gamma)
    a = [int(w) % P for dg in reversed(digests) for w in dg]
    block = max(1, min(1024, len(a)))
    powers = [(1, 0, 0)]
    for _ in range(block - 1):
        powers.append(E.q_mul(powers[-1], gamma))
    step = E.q_mul(powers[-1], gamma)
    components = list(zip(*powers))
    acc = (0, 0, 0)
    for start in range((len(a) - 1) // block * block, -1, -block):
        chunk = a[start:start + block]
        acc = E.q_add(E.q_mul(acc, step), tuple(sum(map(operator.mul, chunk, c)) % P for c in components))
    return acc


_CONFIGS = {}


def air_config(K):
    """the AIR class for K chains (one class per K, so that provers cache one compiled AIR per shape)"""
    if K not in _CONFIGS:
        _CONFIGS[K] = type(f"RescueAirConfigK{K}", (RescueAirConfig,), {"CHAINS": K})
    return _CONFIGS[K]


class RescueChainsClaim(Stark):
    """K chains of L Rescue-Prime permutations from `seed` end in `digests` (K four-word tuples, canonical integers)"""

    def __init__(self, seed, K, L, digests):
        seed = [int(v) for v in seed]
        _check_shape(seed, K, L)
        digests = [tuple(int(w) for w in d) for d in digests]
        if len(digests) != K or any(len(d) != DIGEST or not all(0 <= w < P for w in d) for d in digests):
            raise ValueError(f"expected {K} digests of {DIGEST} canonical words")
        self.seed, self.K, self.L, self.digests = seed, int(K), int(L), digests
        self.AirConfig = air_config(self.K)

    def get_public_inputs(self):
        return self

    def public_inputs_bytes(self, claim):
        """the seed words, K and L as u64, then the 4 K digest words; every value 8 bytes little-endian"""
        words = list(claim.seed) + [claim.K, claim.L] + [w for d in claim.digests for w in d]
        return b"".join(int(w).to_bytes(8, "little") for w in words)


# ------------------------------------------------------------------------------------------ the hash claim and its AIR
M = WIDTH                                               # base column of the absorbed words
HASH_R = WIDTH + 1                                      # the running column of the hash AIR


class RescueHashAirConfig(AirConfig):
    """The AIR of RescueHashClaim for MESSAGES = K messages of LENGTH words (hash_air_config(K, length)); the trace has
    exactly 8 K L rows."""
    NUM_BASE_COLUMNS = WIDTH + 1
    NUM_EXTENSION_COLUMNS = 1
    FQ_IS_FP = False
    MESSAGES = None
    LENGTH = None

    @classmethod
    def _shape(cls, trace_len):
        K, length = cls.MESSAGES, cls.LENGTH
        if K is None:
            raise ValueError("use hash_air_config(K, length): the AIR depends on the number and length of the messages")
        B, L = _hash_shape(K, length)
        if trace_len != 8 * K * L:
            raise ValueError(f"a trace of {trace_len} rows is not {K} messages of {length} words ({8 * K * L} rows)")
        return K, B, L

    @classmethod
    def groups(cls, trace_len):
        """{name: range of constraint indices} for ROUND, LINK, START, PAD and R; LINK is empty when L = 1"""
        _, B, L = cls._shape(trace_len)
        sizes = [("ROUND", WIDTH), ("LINK", WIDTH if L > 1 else 0), ("START", WIDTH), ("PAD", RATE * B - cls.LENGTH),
                 ("R", 4)]
        out, at = {}, 0
        for name, size in sizes:
            out[name] = range(at, at + size)
            at += size
        return out

    @classmethod
    def constraints(cls, trace_len):
        K, B, L = cls._shape(trace_len)
        n, length = trace_len, cls.LENGTH
        g = domain_generator(n.bit_length() - 1)
        x, T, one = E.X(), E.Trace, E.Constant(1)
        last_rounds = x ** (n // 8) - E.Constant(pow(domain_generator(3), 7, P))      # zero on the r = 7 rows
        chain_ends = (E.Constant(g) * x) ** K - one                                     # zero on rows 8 L (k + 1) - 1
        chain_starts = x ** K - one                                                     # zero on rows 8 L k
        # with L = 1 every r = 7 row is a chain end: chain_ends / last_rounds is a constant and there is nothing to link
        link = [] if L == 1 else [
            ((T(w, 1) - T(w, 0) - T(M, 1 + w)) if w < RATE else (T(w, 1) - T(w, 0))) * chain_ends / last_rounds
            for w in range(WIDTH)]
        start = [((T(w, 0) - T(M, w)) if w < RATE else T(w, 0)) / chain_starts for w in range(WIDTH)]
        pad = [((T(M, 0) - one) if p == length else T(M, 0)) / ((E.Constant(pow(g, n - p, P)) * x) ** K - one)
               for p in range(length, RATE * B)]
        return _round_constraints(n) + link + start + pad + _digest_constraints(n, K, 8 * B - 1, HASH_R)

    @classmethod
    def extension_columns(cls, trace_len):
        _, B, L = cls._shape(trace_len)
        return [_digest_column(8 * B - 1, 8 * L)]

    @classmethod
    def gen_hints(cls, trace_len, claim, challenges):
        """[the Horner evaluation at gamma of the digest words]"""
        if (claim.K, claim.length) != (cls.MESSAGES, cls.LENGTH):
            raise ValueError(f"the claim is {claim.K} messages of {claim.length} words, the AIR "
                             f"{cls.MESSAGES} of {cls.LENGTH}")
        cls._shape(trace_len)
        return [digest_evaluation(claim.digests, challenges[0])]


_HASH_CONFIGS = {}


def hash_air_config(K, length):
    """the AIR class for K messages of `length` words (one class per shape, so that provers cache one compiled AIR per
    shape)"""
    key = (int(K), int(length))
    if key not in _HASH_CONFIGS:
        _hash_shape(*key)
        _HASH_CONFIGS[key] = type(f"RescueHashAirConfigK{key[0]}Len{key[1]}", (RescueHashAirConfig,),
                                  {"MESSAGES": key[0], "LENGTH": key[1]})
    return _HASH_CONFIGS[key]


class RescueHashClaim(Stark):
    """I know K = len(digests) messages of `length` words each, and message k hashes to digests[k] (hash(): four
    canonical words).  K is a power of two; the witness is the trace of gen_hash_trace.

    The proof shows knowledge of the preimages; it does not hide them.  It is not zero-knowledge (the reference's proofs
    are not either): its queries open trace rows, message words included, and its out-of-domain evaluations depend on
    them."""

    def __init__(self, length, digests):
        digests = [tuple(int(w) for w in d) for d in digests]
        K = len(digests)
        _hash_shape(K, int(length))
        if any(len(d) != DIGEST or not all(0 <= w < P for w in d) for d in digests):
            raise ValueError(f"expected {K} digests of {DIGEST} canonical words")
        self.length, self.K, self.digests = int(length), K, digests
        self.AirConfig = hash_air_config(K, self.length)

    def get_public_inputs(self):
        return self

    def public_inputs_bytes(self, claim):
        """K, then the length, then the 4 K digest words; every value 8 bytes little-endian"""
        return np.array([claim.K, claim.length] + [w for d in claim.digests for w in d], dtype="<u8").tobytes()
