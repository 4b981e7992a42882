"""examples/wots: K Winternitz one-time signatures over Rescue-Prime, proved valid in one proof, over Goldilocks,
Fq = Fq3, with the signatures and the chain trace built on the GPU.

The scheme.  WOTS+ with the parameters XMSS and SPHINCS+ use at 256 bits: w = 16, l1 = 64 message digits, l2 = 3
checksum digits, l = 67 chains.  `permute` is examples/rescue's permutation (state words 0..11, capacity words 8..11),
and every word is a canonical Goldilocks element.
  * Message digits.  The signed message m is four canonical words (rescue.hash(words) turns a longer message into four
    words first).  For w = 0..3 and t = 0..15, d_(16 w + t) = (m_w >> 4 t) & 15.  The checksum is
    c = sum_(j<64) (15 - d_j) <= 960, and d_(64 + t) = (c >> 4 t) & 15 for t = 0..2.
  * Key.  A key has a secret sigma (4 words) and a public seed rho = (rho_0, rho_1).  The capacity words separate the
    three uses of the permutation by word 8, and carry (i, rho_0, rho_1) in words 9..11:
      - secret of chain i: sk_i = words 0..3 of permute(sigma || 0^4 || 16, i, rho_0, rho_1);
      - chain step s = 0..14: F_(i,s)(x) = words 0..3 of permute(x || 0^4 || 1 + s, i, rho_0, rho_1);
      - fold: acc_0 = 0^4, acc_(i+1) = words 0..3 of permute(end_i || acc_i || 0, i, rho_0, rho_1), where
        end_i = F_(i,14) o ... o F_(i,0)(sk_i).
    The public key is pk = (rho_0, rho_1, root_0..3), six words, with root = acc_67.
  * Sign.  sig_i = F_(i,d_i - 1) o ... o F_(i,0)(sk_i), 67 x 4 words.
  * Verify.  end_i = F_(i,14) o ... o F_(i,d_i)(sig_i), then fold, then compare the result with root.
A key must sign only once: a second signature under the same key reveals chain values that let anyone sign other
messages, and the claim does not track key reuse.  The proof is not zero-knowledge: the signatures are opened like any
witness.

The claim (SignaturesClaim(public_keys, messages)): for every k = 0..K-1 the prover holds a valid signature of
messages[k] under public_keys[k].  K is any count >= 1.  Its public inputs are K, then per signature the six key words
and the four message words.

Trace layout.  Block b of 128 rows is chain i = b mod 67 of signature k = b div 67; there are B = 2^ceil(log2 67 K)
blocks and n = 128 B rows (so K <= 500,812), and blocks 67 K .. B - 1 are padding: digit 0, start value 0, i = rho = 0
and LAST = 1, so every padding block is the same block, whose fold starts from 0^4 and ends in the constant pad_root().
A block is 16 slots of 8 rows: slot s < 15 is chain step s, slot 15 the fold.  Row 8 s + r of a block holds the slot's
permutation state before round r for r < 7, and its output at r = 7, as in every Rescue trace.  Slot s < 15 permutes
(x_s || 0^4 || 1 + s, i, rho_0, rho_1) with x_0 the signature element and x_(s+1) = F_(i,s)(x_s) for s >= d (the step
is applied) or x_s (it is skipped); slot 15 permutes (x_15 || acc || 0, i, rho_0, rho_1), acc the previous block's fold
output, or 0^4 after a block with LAST = 1 and at block 0.

    base columns       0..11: S, the state
    base column        12: ACT, on chain slot s: 1 iff step s is applied (s >= d); 0 on the fold slot
    base column        13: CNT, the digit count-down max(d - s, 0) on slot s; 0 on the fold slot
    base column        14: LAST, 1 on every row of the last chain block (i = 66) of each signature and of every padding
                       block
    extension column   15: R, an inclusive running evaluation over gamma (Fq3) of one 9-word tuple per block, bound at
                       its first row: (d, LAST, i, rho_0, rho_1, LAST root_0..3), root the fold output 127 rows on.
                       Padding tuples are (0, 1, 0, 0, 0, pad_root()).  Declared, so the prover builds it on the device.

Constraints, in this order (air_config(K).groups(n) gives their index ranges).  z = x^B is w_16^s on the first rows of
slot s ("slot inputs", zerofier x^(n / 8) - 1), and the chain slots are those with z != w_16^15:
    ROUND  12   rescue's round constraints, unchanged
    CAP     8   on slot inputs: S_8 = t(z), t the degree-15 interpolant of (1, 2, ..., 15, 0); on chain-slot inputs
                S_4..S_7 = 0, and S_9..S_11 equal to those of the next slot's input
    LINK    4   on chain-slot inputs, read at offsets 0, 7 and 8: S_w(8) = ACT S_w(7) + (1 - ACT) S_w(0) for w < 4
    ACT     2   on chain-slot inputs ACT (ACT - 1) = 0; on slots 0..13 ACT (1 - ACT(8)) = 0 (monotone)
    CNT     2   on chain-slot inputs CNT(8) = CNT - 1 + ACT; on slot inputs CNT f(z) = 0, f the interpolant of the
                fold slot's selector.  Monotone ACT and a count from d down to 0 make ACT_s = [s >= d] exactly: the right
                number of steps at the wrong slots would apply other tweaks and prove another statement
    ACC     9   on block ends but the last, the next fold input S_(4+w)(121) = (1 - LAST) S_w(0) for w < 4; the fold
                input of block 0 S_(4+w)(120) = 0; LAST constant within a block
    R       4   R = lin on the first row; R_(i+1) = R_i where row i + 1 is not a block start, the last row excepted;
                R_(i+1) = R_i gamma^9 + lin(i + 1) where it is; R = Hint(0) on the last row, the Horner evaluation of the
                B public tuples (rescue.digest_evaluation), which the verifier computes from the keys and messages
A padding block ends with LAST = 1 rather than carrying its fold into the next one, so the padding costs no sequential
work: 67 K blocks padded to B would otherwise need B - 67 K folds one after another (up to about 67 K of them).
41 constraints in all.  Every constraint divides by one of examples/merkle's paths zerofiers (every row, the slot
inputs, the r = 7 rows, the block ends, the first and the last row).  ROUND sets the ce blow-up at 8, and rescue.OPTIONS
is reused.
"""
import functools

import numpy as np

from .. import expr as E
from ..air import AirConfig, RunningColumn, domain_generator
from ..prover import Stark, Trace
from .merkle import _zerofiers
from .rescue import (DIGEST, OPTIONS, P, SECURITY_LEVEL, WIDTH, _context, _interpolate, _linear, _round_constraints,
                     _selector, _torch_device, digest_evaluation, permute, round_states)

__all__ = ["OPTIONS", "SECURITY_LEVEL", "SignaturesClaim", "air_config", "digits", "gen_trace", "public_key", "sign",
           "sign_batch", "verify"]

_R = 2**64
DIGITS, MSG_DIGITS, CHAINS = 16, 64, 67           # w, l1, l = l1 + l2
STEPS = DIGITS - 1                                # chain steps 0..14
SECRET_TWEAK = 16                                 # word 8 of the chain-secret derivation; 1 + s for step s, 0 for the fold
SEED, PK = 2, 6                                   # words of a public seed and of a public key
BLOCK = 128                                       # rows per chain: 16 slots of 8
ACT, CNT, LAST, R_COL = WIDTH, WIDTH + 1, WIDTH + 2, WIDTH + 3
NUM_BASE = WIDTH + 3
TUPLE = 9                                         # words bound per block
MAX_KEYS = (1 << 25) // CHAINS                    # 500,812: n = 128 B <= 2^32


# --------------------------------------------------------------------------------------------------------- the scheme
def _words(words, count, what):
    t = tuple(int(w) for w in words)
    if len(t) != count or not all(0 <= w < P for w in t):
        raise ValueError(f"{what} is not {count} canonical field elements")
    return t


def digits(message):
    """the 67 base-16 digits of a four-word message: its 64 nibbles, least significant first within each word, then the
    three nibbles of the checksum sum_(j<64) (15 - d_j)"""
    m = _words(message, DIGEST, "a message")
    d = [(m[w] >> 4 * t) & 15 for w in range(DIGEST) for t in range(16)]
    c = sum(15 - v for v in d)
    return d + [(c >> 4 * t) & 15 for t in range(CHAINS - MSG_DIGITS)]


def _tweaked(x, tail, tweak, i, seed):
    """words 0..3 of permute(x || tail || tweak, i, rho_0, rho_1)"""
    return tuple(permute(list(x) + list(tail) + [tweak, i, seed[0], seed[1]])[:DIGEST])


def _steps(x, i, seed, start, stop):
    """F_(i,stop-1) o ... o F_(i,start)(x)"""
    for s in range(start, stop):
        x = _tweaked(x, (0,) * DIGEST, 1 + s, i, seed)
    return x


def _root(ends, seed):
    acc = (0,) * DIGEST
    for i, end in enumerate(ends):
        acc = _tweaked(end, acc, 0, i, seed)
    return acc


def _key_chains(secret, seed, dig=None):
    """(signature, ends) of one key: the chain values after d_i steps (none without digits) and after 15"""
    sig, ends = [], []
    for i in range(CHAINS):
        x = _tweaked(secret, (0,) * DIGEST, SECRET_TWEAK, i, seed)
        for s in range(STEPS):
            if dig is not None and s == dig[i]:
                sig.append(x)
            x = _steps(x, i, seed, s, s + 1)
        if dig is not None and dig[i] == STEPS:
            sig.append(x)
        ends.append(x)
    return sig, ends


def public_key(secret, seed):
    """(rho_0, rho_1, root_0..3) of the key with secret `secret` (four words) and public seed `seed` (two words)"""
    secret, seed = _words(secret, DIGEST, "the secret"), _words(seed, SEED, "the seed")
    return seed + _root(_key_chains(secret, seed)[1], seed)


def sign(secret, seed, message):
    """the signature of a four-word message: 67 four-word chain values"""
    secret, seed = _words(secret, DIGEST, "the secret"), _words(seed, SEED, "the seed")
    return _key_chains(secret, seed, digits(message))[0]


def _signature(signature):
    sig = [_words(x, DIGEST, "a signature element") for x in signature]
    if len(sig) != CHAINS:
        raise ValueError(f"a signature has {CHAINS} elements, not {len(sig)}")
    return sig


def _ends(pk, message, signature):
    seed, d = pk[:SEED], digits(message)
    return [_steps(x, i, seed, d[i], STEPS) for i, x in enumerate(_signature(signature))]


def verify(public_key, message, signature):
    """True iff `signature` (67 four-word elements) signs `message` (four words) under `public_key` (six words)"""
    pk = _words(public_key, PK, "a public key")
    return _root(_ends(pk, message, signature), pk[:SEED]) == pk[SEED:]


# ------------------------------------------------------------------------------------------------ batches and the trace
def _table(rows, width, what):
    """a (K, width) C-contiguous uint64 array of canonical words from rows (a sequence, an array or a tensor)"""
    if hasattr(rows, "data_ptr"):
        rows = rows.cpu().numpy().view(np.uint64)
    try:
        arr = np.ascontiguousarray(np.array([[int(w) for w in r] for r in rows], dtype=np.uint64).reshape(-1, width))
    except (OverflowError, ValueError):
        raise ValueError(f"{what}: rows of {width} canonical words") from None
    if arr.shape[0] != len(rows) or (arr >= np.uint64(P)).any():
        raise ValueError(f"{what}: rows of {width} canonical words")
    return arr


def _count(K):
    if not 1 <= K <= MAX_KEYS:
        raise ValueError(f"K = {K} signatures is outside 1..{MAX_KEYS}")
    return K


def _blocks(K):
    """B = 2^ceil(log2 67 K), the trace's chain blocks"""
    _count(K)
    return 1 << (CHAINS * K - 1).bit_length()


def _device_call(fn, *args):
    from .. import MsError
    try:
        fn(*args)
    except MsError as e:
        raise ValueError(str(e).split(": ", 1)[-1]) from None


def sign_batch(secrets, seeds, messages, device=None):
    """(signatures, public_keys) of K keys: key k has secret secrets[k] (four words) and seed seeds[k] (two words) and
    signs messages[k] (four words).  device=None: on the host with Python integers (small K only: about 1,200
    permutations per key); signatures is K lists of 67 four-tuples and public_keys K six-tuples.  device: ms_rescue_wots_sign
    on that device; signatures is a (K, 67, 4) and public_keys a (K, 6) int64 tensor of canonical words there."""
    sec, sd, msg = _table(secrets, DIGEST, "secrets"), _table(seeds, SEED, "seeds"), _table(messages, DIGEST, "messages")
    K = _count(len(sec))
    if len(sd) != K or len(msg) != K:
        raise ValueError(f"{K} secrets, {len(sd)} seeds and {len(msg)} messages")
    if device is None:
        sigs, pks = [], []
        for k in range(K):
            seed = tuple(int(w) for w in sd[k])
            sig, ends = _key_chains(tuple(int(w) for w in sec[k]), seed, digits(msg[k]))
            sigs.append(sig)
            pks.append(seed + _root(ends, seed))
        return sigs, pks
    import torch
    dev = _torch_device(device)
    sigs = torch.empty((K, CHAINS, DIGEST), dtype=torch.int64, device=dev)
    pks = torch.empty((K, PK), dtype=torch.int64, device=dev)
    ctx = _context(dev)
    if sigs.is_cuda:                    # the context's stream may not be torch's: torch's work on this memory is done
        torch.cuda.current_stream(dev).synchronize()
    _device_call(ctx.rescue_wots_sign, sec, sd, msg, K, sigs, pks)
    ctx.sync()
    return sigs, pks


def _block_rows(x, d, i, seed, acc):
    """(the 16 permutations' round states of one block, the fold output): chain steps from x with digit d, then the
    fold with acc"""
    blocks = []
    for s in range(STEPS):
        st = round_states(list(x) + [0] * DIGEST + [1 + s, i, seed[0], seed[1]])
        blocks.append(st)
        if s >= d:
            x = tuple(st[-1][:DIGEST])
    st = round_states(list(x) + list(acc) + [0, i, seed[0], seed[1]])
    blocks.append(st)
    return blocks, tuple(st[-1][:DIGEST])


def gen_trace(public_keys, messages, signatures, device=None):
    """the Trace of SignaturesClaim(public_keys, messages) from signatures[k] (67 four-word elements each).  A signature
    that does not verify raises ValueError naming the first such k.  device=None: computed on the host with Python
    integers (small K only: 16 permutations per chain block).  device: built on that device by ms_rescue_wots_trace
    and handed over as a resident (15, n) tensor (the signatures may be a (K, 67, 4) int64 tensor there)."""
    pks, msg = _table(public_keys, PK, "public keys"), _table(messages, DIGEST, "messages")
    K = _count(len(pks))
    if len(msg) != K or len(signatures) != K:
        raise ValueError(f"{K} public keys, {len(msg)} messages and {len(signatures)} signatures")
    B = _blocks(K)
    n = BLOCK * B
    if device is None:
        cols = np.zeros((NUM_BASE, n), dtype=np.uint64)
        acc = (0,) * DIGEST
        for b in range(B):
            k, i = divmod(b, CHAINS)
            if k < K:
                if i == 0:
                    pk, dig = tuple(int(w) for w in pks[k]), digits(msg[k])
                    sig = _signature(signatures[k].tolist() if hasattr(signatures[k], "tolist") else signatures[k])
                x, d, seed, last = sig[i], dig[i], pk[:SEED], int(i == CHAINS - 1)
            else:
                x, d, i, seed, last = (0,) * DIGEST, 0, 0, (0, 0), 1
            states, out = _block_rows(x, d, i, seed, acc)
            rows = slice(BLOCK * b, BLOCK * (b + 1))
            cols[:WIDTH, rows] = np.array([[w * _R % P for w in st] for perm in states for st in perm], dtype=np.uint64).T
            cols[ACT, rows] = np.repeat([_R % P * (s >= d) for s in range(STEPS)] + [0], 8).astype(np.uint64)
            cols[CNT, rows] = np.repeat([max(d - s, 0) * _R % P for s in range(STEPS)] + [0], 8).astype(np.uint64)
            cols[LAST, rows] = last * _R % P
            if last and k < K and out != pk[SEED:]:
                raise ValueError(f"signature {k} does not verify: its root differs from its public key")
            acc = (0,) * DIGEST if last else out
        return Trace(cols)
    import torch
    dev = _torch_device(device)
    if isinstance(signatures, torch.Tensor):
        sigs = signatures.to(dev).contiguous()
        if sigs.dtype != torch.int64 or tuple(sigs.shape) != (K, CHAINS, DIGEST):
            raise ValueError(f"signatures: a ({K}, {CHAINS}, {DIGEST}) int64 tensor")
    else:
        sigs = _table([x for s in signatures for x in _flat(s)], DIGEST, "signatures")
        if len(sigs) != K * CHAINS:
            raise ValueError(f"signatures: {K} signatures of {CHAINS} elements")
    out = torch.empty((NUM_BASE, n), dtype=torch.int64, device=dev)
    ctx = _context(dev)
    if out.is_cuda:                     # the context's stream may not be torch's: torch's work on this memory is done
        torch.cuda.current_stream(dev).synchronize()
    _device_call(ctx.rescue_wots_trace, pks, msg, sigs, K, out)
    ctx.sync()                          # complete before the prover reads it on its own stream
    return Trace(out)


def _flat(signature):
    rows = signature.tolist() if hasattr(signature, "tolist") else list(signature)
    if len(rows) != CHAINS:
        raise ValueError(f"a signature has {CHAINS} elements, not {len(rows)}")
    return rows


# ----------------------------------------------------------------------------------------------------------- the AIR
W16 = domain_generator(4)
TWEAK_COEFFS = _interpolate([1 + s for s in range(STEPS)] + [0])          # S_8 on slot s's input, as a polynomial in z
FOLD_COEFFS = _interpolate([0] * STEPS + [1])                            # the fold slot's selector


def _lin(offset):
    """CNT + gamma LAST + gamma^2 S_9 + gamma^3 S_10 + gamma^4 S_11 + sum_w gamma^(5 + w) LAST S_w(127) at row offset
    `offset`: the tuple a block start binds"""
    T, gamma = E.Trace, E.Challenge(0)
    last = T(LAST, offset)
    words = [T(CNT, offset), last] + [T(w, offset) for w in range(9, WIDTH)] \
        + [last * T(w, offset + BLOCK - 1) for w in range(DIGEST)]
    return _linear(words[w] * (gamma ** w) if w else words[0] for w in range(TUPLE))


class WotsAirConfig(AirConfig):
    """The AIR of SignaturesClaim for SIGNATURES = K signatures (air_config(K)); the trace has exactly 128 B rows."""
    NUM_BASE_COLUMNS = NUM_BASE
    NUM_EXTENSION_COLUMNS = 1
    FQ_IS_FP = False
    SIGNATURES = None

    @classmethod
    def _shape(cls, trace_len):
        K = cls.SIGNATURES
        if K is None:
            raise ValueError("use air_config(K): the AIR depends on the number of signatures")
        B = _blocks(K)
        if trace_len != BLOCK * B:
            raise ValueError(f"a trace of {trace_len} rows is not {K} signatures ({BLOCK * B} rows)")
        return K, B

    @classmethod
    def groups(cls, trace_len):
        """{name: range of constraint indices} for ROUND, CAP, LINK, ACT, CNT, ACC and R"""
        cls._shape(trace_len)
        out, at = {}, 0
        for name, size in [("ROUND", WIDTH), ("CAP", 8), ("LINK", DIGEST), ("ACT", 2), ("CNT", 2), ("ACC", 9),
                           ("R", 4)]:
            out[name] = range(at, at + size)
            at += size
        return out

    @classmethod
    def constraints(cls, trace_len):
        K, B = cls._shape(trace_len)
        n = trace_len
        x, T, one = E.X(), E.Trace, E.Constant(1)
        all_rows, slot_inputs, _, block_ends = _zerofiers(n, B)
        last = E.Constant(pow(domain_generator(n.bit_length() - 1), n - 1, P))
        z = [one, x ** B]                                                         # w_16^s on slot s's input
        for _ in range(14):
            z.append(z[-1] * z[1])
        tweak = _linear(E.Constant(c) * z[k] for k, c in enumerate(TWEAK_COEFFS))
        fold = _linear(E.Constant(c) * z[k] for k, c in enumerate(FOLD_COEFFS))
        chain = z[1] - E.Constant(pow(W16, 15, P))                                # zero on the fold slot's input
        a = T(ACT, 0)
        cap = ([(T(8, 0) - tweak) / slot_inputs] + [T(w, 0) * chain / slot_inputs for w in range(DIGEST, 8)]
               + [(T(w, 8) - T(w, 0)) * chain / slot_inputs for w in range(9, WIDTH)])
        link = [(T(w, 8) - a * T(w, 7) - (one - a) * T(w, 0)) * chain / slot_inputs for w in range(DIGEST)]
        act = [a * (a - one) * chain / slot_inputs,
               a * (one - T(ACT, 8)) * (z[1] - E.Constant(pow(W16, 14, P))) * chain / slot_inputs]
        cnt = [(T(CNT, 8) - T(CNT, 0) + one - a) * chain / slot_inputs, T(CNT, 0) * fold / slot_inputs]
        keep = one - T(LAST, 0)
        acc = ([(T(DIGEST + w, 121) - keep * T(w, 0)) * (x - last) / block_ends for w in range(DIGEST)]
               + [T(DIGEST + w, 120) / (x - one) for w in range(DIGEST)]
               + [(T(LAST, 1) - T(LAST, 0)) * block_ends / all_rows])
        g9 = E.Challenge(0) ** TUPLE
        r = [(T(R_COL, 0) - _lin(0)) / (x - one),
             (T(R_COL, 1) - T(R_COL, 0)) * block_ends / all_rows,
             (T(R_COL, 1) - T(R_COL, 0) * g9 - _lin(1)) * (x - last) / block_ends,
             (T(R_COL, 0) - E.Hint(0)) / (x - last)]
        return _round_constraints(n) + cap + link + act + cnt + acc + r

    @classmethod
    def extension_columns(cls, trace_len):
        cls._shape(trace_len)
        e = _selector(0, BLOCK)
        return [RunningColumn(init=0, mul=E.Constant(1) + e * (E.Challenge(0) ** TUPLE - E.Constant(1)), add=e * _lin(0),
                              inclusive=True)]

    @classmethod
    def gen_hints(cls, trace_len, claim, challenges):
        """[the Horner evaluation at gamma of the B block tuples]"""
        if claim.K != cls.SIGNATURES:
            raise ValueError(f"the claim is {claim.K} signatures, the AIR {cls.SIGNATURES}")
        _, B = cls._shape(trace_len)
        return [digest_evaluation(block_tuples(claim.public_keys, claim.messages, B), challenges[0])]


@functools.lru_cache(maxsize=None)
def pad_root():
    """the fold output of every padding block: chain 0 under the zero seed, all 15 steps from 0^4, folded onto 0^4"""
    seed = (0,) * SEED
    return _root([_steps((0,) * DIGEST, 0, seed, 0, STEPS)], seed)


def block_tuples(public_keys, messages, B):
    """the B tuples R binds: (d_i, LAST, i, rho_0, rho_1, LAST root_0..3) for chain i of each signature, then
    (0, 1, 0, 0, 0, pad_root()) for each padding block"""
    out = []
    for pk, m in zip(public_keys, messages):
        for i, d in enumerate(digits(m)):
            last = i == CHAINS - 1
            out.append((d, int(last), i) + tuple(pk[:SEED]) + (tuple(pk[SEED:]) if last else (0,) * DIGEST))
    return out + [(0, 1, 0, 0, 0) + pad_root()] * (B - len(out))


_CONFIGS = {}


def air_config(K):
    """the AIR class for K signatures (one class per K, so that provers cache one compiled AIR per shape)"""
    K = int(K)
    if K not in _CONFIGS:
        _blocks(K)
        _CONFIGS[K] = type(f"WotsAirConfigK{K}", (WotsAirConfig,), {"SIGNATURES": K})
    return _CONFIGS[K]


class SignaturesClaim(Stark):
    """For every k = 0..K-1 the prover holds a valid signature of messages[k] (four canonical words) under
    public_keys[k] (six canonical words: the seed, then the root).  K is any count >= 1; the witness is the trace of
    gen_trace.

    The proof is not zero-knowledge: its queries open trace rows, so signature elements and chain values are revealed,
    and its out-of-domain evaluations depend on them.  Nor does the claim track key reuse: a key must sign only once."""

    def __init__(self, public_keys, messages):
        self.public_keys = [_words(pk, PK, "a public key") for pk in public_keys]
        self.messages = [_words(m, DIGEST, "a message") for m in messages]
        self.K = _count(len(self.public_keys))
        if len(self.messages) != self.K:
            raise ValueError(f"{self.K} public keys and {len(self.messages)} messages")
        self.AirConfig = air_config(self.K)

    def get_public_inputs(self):
        return self

    def public_inputs_bytes(self, claim):
        """K, then per signature its six public-key words and its four message words; every value 8 bytes
        little-endian"""
        words = [claim.K]
        for pk, m in zip(claim.public_keys, claim.messages):
            words += list(pk) + list(m)
        return np.array(words, dtype="<u8").tobytes()
