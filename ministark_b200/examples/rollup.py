"""examples/rollup: K balance transfers that take one public Rescue-Prime account root to another, over Goldilocks,
Fq = Fq3, with the balances resolved and the trace built on the GPU.

The statement (TransfersClaim(depth, old_root, new_root, transfers)).  An account is a leaf of the depth-D Rescue-Prime
Merkle tree of examples/merkle (the same merge and heap): its four words are (balance, nonce, owner_0, owner_1), leaf i
is account i, and an all-zero leaf is an empty account.  `transfers` is K triples (sender, receiver, amount), K a power
of two, both accounts < 2^D and amount < 2^32; sender == receiver is allowed.  Starting from the tree whose root is
old_root, transfer k = 0..K-1, in order, first sets the sender's balance to balance - amount and its nonce to nonce + 1,
then sets the receiver's balance to balance + amount; both steps keep the owner words.  The result is the tree whose
root is new_root.  A transfer is valid only if the balance each of its two steps writes is a field element in
[0, 2^32): whenever the old balances are below 2^32 this is integer arithmetic, so a sender cannot overdraw and a
receiver cannot overflow.  Balances, nonces and owners are witness; nonces are field elements and are not
range-checked; transfers are not authorised (no signatures: the claim is what a sequencer proves about the batch it
applied).

The trace, n = 32 K L rows (L the smallest power of two >= D, n >= 256): transfer k is write 2 k (the sender step,
delta = -amount, nonce increment 1) then write 2 k + 1 (the receiver step, delta = +amount, increment 0), and columns
0..14 are examples/merkle's updates trace of these 2 K writes: write w's old path at rows 16 L w, its new path at
16 L w + 8 L.  Then

    base column        15: DELTA, write w's delta on row 16 L w (its old path's first row), 0 elsewhere
    base column        16: NINC, write w's nonce increment on that row, 0 elsewhere
    base columns   17..20: B0..B3, the four 8-bit limbs of write w's new balance on that row, 0 elsewhere
    base column        21: M, the multiplicities of the range lookup (filled by the prover)
    base column        22: TBL, 0, 1, ..., 255, then 255 repeated
    extension column   23: R, an inclusive running evaluation over gamma of the 2 K tuples (IDX, DELTA, NINC) at the old
                       paths' first rows: mul = 1 + e (gamma^3 - 1), add = e lin, e the selector of rows 16 L w
    extension column   24: S, the range lookup's running sum (declared by the package)

Constraints, in this order (rollup_air_config(K, depth).groups(n) gives their index ranges):
    ROUND .. CHAIN  the updates AIR's over 2 K writes, unchanged (its R is replaced by the one below)
    BAL     1   new balance = old balance + DELTA
    NONCE   1   new nonce = old nonce + NINC
    KEEP    2   the owner words are kept
    LIMB    1   B0 + 2^8 B1 + 2^16 B2 + 2^24 B3 = new balance
                These four groups sit on the path ends with SIDE = 1 (factor SIDE over the path ends' zerofier) and read
                the old leaf at offset 1 and the new leaf at offset 1 + 8 L, so write w's new path end checks write
                w + 1, and the last row (write 2 K - 1's) wraps around to write 0: every write once, no new zerofier.
    TBL     3   TBL = 0 on the first row; (TBL' - TBL) (TBL' - TBL - 1) = 0 on every row but the last; TBL = 255 on the
                last row.  With n >= 256 the table then holds every value 0..255.
    R       4   R = lin on the first row; R_(i+1) = R_i where row i + 1 is not a path start, the last row excepted;
                R_(i+1) = R_i (1 + (1 - SIDE') (gamma^3 - 1)) + (1 - SIDE') lin(i + 1) where it is; R = Hint(0) on the
                last row, the Horner evaluation of the 2 K public tuples
    LOOKUP  3   the declared Lookup(table=(TBL,), values=((B0,), (B1,), (B2,), (B3,)), multiplicity=M, running_sum=S),
                no selectors (rows without a write look up 0); its constraints are the package's, appended last
Every constraint divides by one of the paths AIR's zerofiers (the evaluator's batched inverses of more would not fit
its registers).  ROUND sets the ce blow-up at 8, and rescue.OPTIONS is reused.  The proof is not zero-knowledge."""
import numpy as np

from .. import expr as E
from ..air import AirConfig, Lookup, RunningColumn, domain_generator
from ..prover import Stark, Trace
from . import merkle
from .merkle import BIT, IDX, SIDE, _check_words, _path_shape, _zerofiers
from .rescue import DIGEST, OPTIONS, P, SECURITY_LEVEL, WIDTH, _context, _selector, _torch_device, digest_evaluation

__all__ = ["OPTIONS", "SECURITY_LEVEL", "TransfersClaim", "apply", "leaf", "rollup_air_config"]

_R = 2**64
DELTA, NINC, B0, M_COL, TBL = WIDTH + 3, WIDTH + 4, WIDTH + 5, WIDTH + 9, WIDTH + 10     # base columns 15, 16, 17, 21, 22
R_COL, S_COL = WIDTH + 11, WIDTH + 12                                                  # extension columns 23, 24
NUM_BASE = WIDTH + 11
TUPLE = 3                                               # words bound per write: the account, the delta, the increment
AMOUNT_BOUND = BALANCE_BOUND = 1 << 32


def leaf(balance, nonce=0, owner=(0, 0)):
    """the four words of an account: (balance, nonce, owner_0, owner_1)"""
    return _check_words((balance, nonce) + tuple(owner), "an account")


def _shape(K, depth):
    """L; ValueError unless K is a power of two, 1 <= depth <= 32 and 256 <= 32 K L <= 2^32"""
    L = _path_shape(4 * K, depth)
    if 32 * K * L < 256:
        raise ValueError(f"32 K L = {32 * K * L} rows: the byte table needs at least 256 (K L >= 8)")
    return L


def _check_transfers(transfers, depth):
    """K (sender, receiver, amount) triples of ints, or ValueError"""
    if hasattr(transfers, "data_ptr"):
        transfers = transfers.cpu().numpy().view(np.uint64)
    out = []
    for k, t in enumerate(transfers):
        t = tuple(int(v) for v in t)
        if len(t) != 3:
            raise ValueError(f"transfer {k} is not a (sender, receiver, amount) triple")
        for side, a in zip(("sender", "receiver"), t[:2]):
            if not 0 <= a < 1 << depth:
                raise ValueError(f"{side} {a} of transfer {k} is not below 2^{depth}")
        if not 0 <= t[2] < AMOUNT_BOUND:
            raise ValueError(f"amount {t[2]} of transfer {k} is not below 2^32")
        out.append(t)
    return out


def _writes(transfers):
    """[(account, delta, nonce increment)]: write 2 k and 2 k + 1 of transfer k, delta a field element"""
    out = []
    for s, r, a in transfers:
        out += [(s, (P - a) % P, 1), (r, a, 0)]
    return out


# --------------------------------------------------------------------------------------------------------- the trace
def apply(nodes, depth, transfers, device=None):
    """(Trace, new_nodes, roots) of TransfersClaim: transfers[k] = (sender, receiver, amount) applied to the accounts of
    the depth-D heap `nodes`, k = 0..K-1 in order (K a power of two).  new_nodes is the heap after every transfer, roots
    the K + 1 roots, roots[0] that of `nodes` and roots[k + 1] that after transfer k.  The caller's heap is never
    modified.  An invalid transfer (a balance written outside [0, 2^32)) raises ValueError naming the first one, its step
    and the account.
    device=None: computed on the host with Python integers from a heap of merkle.tree(..., device=None) (small shapes
    only); new_nodes is a list like it.  device: ms_rescue_rollup on that device, applied to a copy of the heap made
    there (the heap in device or host memory); the trace is a resident (23, n) tensor and new_nodes a (2^(D + 1), 4)
    int64 tensor on that device."""
    txs = _check_transfers(transfers, depth)
    K = len(txs)
    L = _shape(K, depth)
    n = 32 * K * L
    if device is None:
        heap = [tuple(int(w) for w in v) for v in nodes]
        if len(heap) != 2 << depth:
            raise ValueError(f"a heap of {len(heap)} nodes is not a tree of depth {depth}")
        writes = _writes(txs)
        accounts, new_leaves, balances = {}, [], []
        for w, (a, delta, ninc) in enumerate(writes):
            bal, nonce, o0, o1 = accounts.get(a, heap[(1 << depth) + a])
            bal = (bal + delta) % P
            if bal >= BALANCE_BOUND:
                raise ValueError(f"the {'receiver' if w & 1 else 'sender'} step of transfer {w // 2} leaves account {a} "
                                 f"with balance {bal}, not below 2^32")
            accounts[a] = (bal, (nonce + ninc) % P, o0, o1)
            new_leaves.append(accounts[a])
            balances.append(bal)
        trace, heap, roots = merkle.update(heap, depth, [a for a, _, _ in writes], new_leaves)
        cols = np.zeros((NUM_BASE, n), dtype=np.uint64)
        cols[:SIDE + 1] = trace.base_columns()
        for w, ((_, delta, ninc), bal) in enumerate(zip(writes, balances)):
            row = 16 * L * w
            cols[DELTA, row] = delta * _R % P
            cols[NINC, row] = ninc * _R % P
            for q in range(4):
                cols[B0 + q, row] = (bal >> 8 * q & 255) * _R % P
        cols[TBL] = np.array([min(i, 255) * _R % P for i in range(n)], dtype=np.uint64)
        return Trace(cols), heap, roots[::2]
    import torch
    from .. import MsError
    dev = _torch_device(device)
    if isinstance(nodes, torch.Tensor):
        heap = nodes.to(dev, copy=True)
    else:
        heap = torch.from_numpy(np.array(nodes, dtype=np.uint64).view(np.int64)).to(dev)
    if heap.dtype != torch.int64 or tuple(heap.shape) != (2 << depth, DIGEST):
        raise ValueError(f"nodes: a ({2 << depth}, 4) heap of canonical words")
    heap = heap.contiguous()
    out = torch.empty((NUM_BASE, n), dtype=torch.int64, device=dev)
    roots = torch.empty((K + 1, DIGEST), dtype=torch.int64, device=dev)
    ctx = _context(dev)
    if out.is_cuda:                     # the context's stream may not be torch's: torch's work on this memory is done
        torch.cuda.current_stream(dev).synchronize()
    try:
        ctx.rescue_rollup(heap, depth, np.array(txs, dtype=np.uint64).reshape(K, 3), K, out, roots)
    except MsError as e:
        raise ValueError(str(e).split("ms_rescue_rollup: ", 1)[-1]) from None
    ctx.sync()                          # complete before the prover reads it on its own stream
    return Trace(out), heap, [tuple(int(w) for w in r) for r in roots.cpu().numpy().view(np.uint64)]


# ----------------------------------------------------------------------------------------------------------- the AIR
def _lin(offset):
    """IDX + gamma DELTA + gamma^2 NINC at row offset `offset`: the tuple an old path's first row binds"""
    T, gamma = E.Trace, E.Challenge(0)
    return T(IDX, offset) + gamma * T(DELTA, offset) + gamma * gamma * T(NINC, offset)


class RollupAirConfig(AirConfig):
    """The AIR of TransfersClaim for TRANSFERS = K transfers over a tree of DEPTH = D levels (rollup_air_config(K,
    depth)); the trace has exactly 32 K L rows."""
    NUM_BASE_COLUMNS = NUM_BASE
    NUM_EXTENSION_COLUMNS = 2
    FQ_IS_FP = False
    TRANSFERS = None
    DEPTH = None

    @classmethod
    def _shape(cls, trace_len):
        K, depth = cls.TRANSFERS, cls.DEPTH
        if K is None:
            raise ValueError("use rollup_air_config(K, depth): the AIR depends on the number of transfers and the depth")
        L = _shape(K, depth)
        if trace_len != 32 * K * L:
            raise ValueError(f"a trace of {trace_len} rows is not {K} transfers of depth {depth} ({32 * K * L} rows)")
        return K, depth, L

    @classmethod
    def groups(cls, trace_len):
        """{name: range of constraint indices} for the updates AIR's ROUND, CAP, LINK, SIDE, SIB, BIT, IDX, ROOT and
        CHAIN, then BAL, NONCE, KEEP, LIMB, TBL, R and the package's LOOKUP; LINK is empty when L = 1"""
        K, depth, L = cls._shape(trace_len)
        out = {name: r for name, r in merkle.updates_air_config(2 * K, depth).groups(trace_len).items() if name != "R"}
        at = out["CHAIN"].stop
        for name, size in [("BAL", 1), ("NONCE", 1), ("KEEP", 2), ("LIMB", 1), ("TBL", 3), ("R", 4), ("LOOKUP", 3)]:
            out[name] = range(at, at + size)
            at += size
        return out

    @classmethod
    def constraints(cls, trace_len):
        K, depth, L = cls._shape(trace_len)
        n = trace_len
        x, T, one = E.X(), E.Trace, E.Constant(1)
        all_rows, _, _, path_ends = _zerofiers(n, 4 * K)
        last = E.Constant(pow(domain_generator(n.bit_length() - 1), n - 1, P))
        updates = merkle.updates_air_config(2 * K, depth).constraints(n)[:-4]           # without its R

        def word(w, offset):                            # leaf word w of the path starting `offset` rows on
            b = T(BIT, offset)
            return (one - b) * T(w, offset) + b * T(w + DIGEST, offset)

        # on the new paths' ends (SIDE = 1): the next write's old leaf 1 row on, its new leaf 1 + 8 L rows on
        on = T(SIDE, 0) / path_ends
        old, new = (lambda w: word(w, 1)), (lambda w: word(w, 1 + 8 * L))
        limbs = T(B0, 1) + E.Constant(1 << 8) * T(B0 + 1, 1) + E.Constant(1 << 16) * T(B0 + 2, 1) \
            + E.Constant(1 << 24) * T(B0 + 3, 1)
        leaves = [(new(0) - old(0) - T(DELTA, 1)) * on, (new(1) - old(1) - T(NINC, 1)) * on,
                  (new(2) - old(2)) * on, (new(3) - old(3)) * on, (limbs - new(0)) * on]
        step = T(TBL, 1) - T(TBL, 0)
        tbl = [T(TBL, 0) / (x - one), step * (step - one) * (x - last) / all_rows,
               (T(TBL, 0) - E.Constant(255)) / (x - last)]
        # R: a write's tuple is bound where its old path starts, the row after a path end with SIDE = 0 there
        g3, os = E.Challenge(0) ** TUPLE, one - T(SIDE, 1)
        r = [(T(R_COL, 0) - _lin(0)) / (x - one),
             (T(R_COL, 1) - T(R_COL, 0)) * path_ends / all_rows,
             (T(R_COL, 1) - T(R_COL, 0) * (one + os * (g3 - one)) - os * _lin(1)) * (x - last) / path_ends,
             (T(R_COL, 0) - E.Hint(0)) / (x - last)]
        return updates + leaves + tbl + r

    @classmethod
    def extension_columns(cls, trace_len):
        _, _, L = cls._shape(trace_len)
        e = _selector(0, 16 * L)
        return [RunningColumn(init=0, mul=E.Constant(1) + e * (E.Challenge(0) ** TUPLE - E.Constant(1)), add=e * _lin(0),
                              inclusive=True), None]

    @classmethod
    def lookups(cls, trace_len):
        cls._shape(trace_len)
        T = E.Trace
        return [Lookup(table=(T(TBL, 0),), values=tuple((T(B0 + q, 0),) for q in range(4)), multiplicity=M_COL,
                       running_sum=S_COL)]

    @classmethod
    def gen_hints(cls, trace_len, claim, challenges):
        """[the Horner evaluation at gamma of the 2 K (account, delta, nonce increment) write tuples, the old root's four
        words, the new root's four words]"""
        if (claim.K, claim.depth) != (cls.TRANSFERS, cls.DEPTH):
            raise ValueError(f"the claim is {claim.K} transfers of depth {claim.depth}, the AIR {cls.TRANSFERS} of depth "
                             f"{cls.DEPTH}")
        cls._shape(trace_len)
        return [digest_evaluation(_writes(claim.transfers), challenges[0])] + list(claim.old_root) + list(claim.new_root)


_CONFIGS = {}


def rollup_air_config(K, depth):
    """the AIR class for K transfers over a tree of `depth` levels (one class per shape, so that provers cache one
    compiled AIR per shape)"""
    key = (int(K), int(depth))
    if key not in _CONFIGS:
        _shape(*key)
        _CONFIGS[key] = type(f"RollupAirConfigK{key[0]}D{key[1]}", (RollupAirConfig,),
                             {"TRANSFERS": key[0], "DEPTH": key[1]})
    return _CONFIGS[key]


class TransfersClaim(Stark):
    """Starting from the depth-D Rescue-Prime account tree whose root is `old_root`, applying transfers[k] = (sender,
    receiver, amount) for k = 0..K-1 in order, each a valid transfer, gives the tree whose root is `new_root`.  K is a
    power of two; the witness is the trace of apply().

    The proof is not zero-knowledge: its queries open trace rows, so balances, nonces, owners, siblings and
    intermediate roots are revealed, and its out-of-domain evaluations depend on them."""

    def __init__(self, depth, old_root, new_root, transfers):
        self.depth = int(depth)
        if not 1 <= self.depth <= merkle.MAX_DEPTH:
            raise ValueError(f"depth {self.depth} is outside 1..{merkle.MAX_DEPTH}")
        self.transfers = _check_transfers(transfers, self.depth)
        self.K = len(self.transfers)
        _shape(self.K, self.depth)
        self.old_root = _check_words(old_root, "the old root")
        self.new_root = _check_words(new_root, "the new root")
        self.AirConfig = rollup_air_config(self.K, self.depth)

    def get_public_inputs(self):
        return self

    def public_inputs_bytes(self, claim):
        """D, K, the old root's four words, the new root's four words, then per transfer its sender, receiver and
        amount; every value 8 bytes little-endian"""
        words = [claim.depth, claim.K] + list(claim.old_root) + list(claim.new_root)
        for t in claim.transfers:
            words += list(t)
        return np.array(words, dtype="<u8").tobytes()
