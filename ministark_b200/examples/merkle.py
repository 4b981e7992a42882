"""examples/merkle: K authentication paths in one Rescue-Prime Merkle tree, proved against its public root, over
Goldilocks, Fq = Fq3, with the tree and the path trace built on the GPU.

The statement (MerklePathsClaim(depth, root, leaves, indices)): for k = 0..K-1, leaf `leaves[k]` (four canonical words)
sits at position `indices[k]` of the depth-D Rescue-Prime Merkle tree whose root is `root`.  K is a power of two,
1 <= D <= 32 and 0 <= indices[k] < 2^D (an index may repeat); L is the smallest power of two >= D and n = 8 K L <= 2^32.
One short proof stands for K authentication paths.

The tree.  merge(a, b) = words 0..3 of rescue.permute(a || b || 0, 0, 0, 0): the sponge's fixed-length 2-to-1
compression, one permutation with the capacity starting at zero and no padding.  It is deliberately not
rescue.hash(a + b), which pads the 8 words to two rate blocks and would take two permutations per level.  The tree is a
heap: node 1 is the root, node 2^D + i is leaf i, node v = merge(node 2 v, node 2 v + 1).

Trace layout, n = 8 K L rows (gen_trace); path k holds rows [8 L k, 8 L (k + 1)), its permutation j = 0..L-1 rows
8 (L k + j) + r, laid out as in the chains trace of examples/rescue:

    base columns       0..11: S, the state: before round r for r < 7, the output at r = 7.  Permutation j takes
                       (cur, sib_j, 0^4) when b_j = 0 and (sib_j, cur, 0^4) when b_j = 1, with b_j = bit j of the index,
                       sib_j = node ((2^D + index) >> j) ^ 1 and cur the leaf (j = 0) or words 0..3 of permutation
                       j - 1's output.  The filler permutations j >= D take b_j = 0 and sib = 0.  The root is words 0..3
                       of row 8 (L k + D) - 1.
    base column        12: BIT, b_j on the eight rows of permutation j.
    base column        13: IDX, index >> j on the rows of permutation j; the path's first row holds the whole index.
    extension column   14: R, an inclusive running evaluation over gamma (Fq3) of the 5-tuples (leaf_0..3, IDX) at each
                       path's first row, leaf word w = (1 - BIT) S_w + BIT S_(w + 4) there: mul = 1 + e (gamma^5 - 1),
                       add = e lin, e the selector of rows 8 L k.  Declared, so the prover builds it on the device.

Constraints, in this order (air_config(K, depth).groups(n) gives their index ranges):
    ROUND  12   rescue's round constraints, unchanged
    CAP     4   S_w = 0 for w = 8..11 on the r = 0 rows: over x^(n / 8) - 1
    LINK    4   on the r = 7 rows but the path ends, b' = BIT on the next row: (1 - b') (t_w - s_w) + b' (t_(w+4) - s_w)
                = 0 for w < 4, s this row and t the next; the other half of t is the sibling and is free
    BIT     2   BIT (BIT - 1) = 0 on every row; BIT constant across the rows of a permutation (r != 7)
    IDX     3   IDX constant across the rows of a permutation; IDX = 2 IDX' + BIT on the r = 7 rows but the path ends;
                IDX = BIT on the path ends.  Together: IDX at row 8 L k = sum_(j<L) b_j 2^j exactly (< 2^32 < p), so the
                public bound indices[k] < 2^D forces the filler bits to zero
    ROOT    4   S_w = Hint(1 + w) on rows 8 L k + 8 D - 1: over ((g^(n - 8 D + 1)) x)^K - 1
    R       4   R = lin on the first row; R_(i+1) = R_i where row i + 1 is not a path start, the last row excepted;
                R_(i+1) = R_i gamma^5 + lin(i + 1) where it is; R = Hint(0) on the last row, the Horner evaluation of the
                K public 5-tuples (rescue.digest_evaluation)
33 constraints in all; at L = 1 (D = 1) every r = 7 row is a path end, so LINK and the IDX step are dropped and 28
remain.  ROUND sets the ce blow-up at 8, and rescue.OPTIONS is reused.

Ordered writes (MerkleUpdatesClaim(depth, old_root, new_root, indices, new_leaves)): starting from the depth-D tree whose
root is old_root, replacing leaf indices[k] with new_leaves[k] for k = 0..K-1, one write after another, gives the tree
whose root is new_root.  Indices may repeat, and a later write to the same leaf overwrites an earlier one.  The old
leaves are witness.  Write k is proved by two paths with the same siblings and index bits: the old path from the leaf
it replaces ends in root_k, the new path from new_leaves[k] in root_(k + 1); by collision resistance of merge,
root_(k + 1) is then the root of tree_k with that one leaf replaced.  update() builds the trace, n = 16 K L rows: the
paths trace of 2 K paths, path 2 k write k's old path and path 2 k + 1 its new path (8 L rows later), with

    base columns       0..13: S, BIT and IDX as in the paths trace; the siblings are those of tree_k
    base column        14: SIDE, 0 on the old path's rows and 1 on the new path's
    extension column   15: R, the running evaluation of the paths trace over the 5-tuples (new leaf, IDX) at the new
                       paths' first rows (rows 8 L (2 k + 1)); declared with the selector of those rows

The two paths of a write sit one above the other rather than side by side: 24 state columns would need 24 ROUND
constraints, more live values than the evaluator's registers hold.  Every constraint below is divided by one of the
paths AIR's zerofiers, for the same reason.  Constraints, in this order (updates_air_config(K, depth).groups(n)):
    ROUND  12   rescue's round constraints
    CAP     4   as in the paths AIR
    LINK    4   as in the paths AIR, over 2 K paths (dropped when L = 1)
    SIDE    3   SIDE = 0 on the first row, constant within a path, SIDE' = 1 - SIDE at the path ends but the last row
    SIB     5   on the old paths' r = 0 rows (factor 1 - SIDE), the new path 8 L rows on takes the same sibling half,
                (1 - BIT) (S_(w+4) - S'_(w+4)) + BIT (S_w - S'_w) = 0 for w < 4, S' = S 8 L rows on, and the same BIT
    BIT     2   as in the paths AIR
    IDX     3   as in the paths AIR over 2 K paths (2 when L = 1)
    ROOT    8   S_w = Hint(1 + w) on row 8 D - 1 (write 0's old root), S_w = Hint(5 + w) on row n - 1 - 8 (L - D) (write
                K - 1's new root), read 8 D - 1 rows after the first and 8 (L - D) rows before the last
    CHAIN   4   on the new paths' root rows but write K - 1's (factor SIDE over the 2 K roots' zerofier), S_w 8 L rows on
                = S_w: write k + 1 starts from the root write k ends in (dropped when K = 1)
    R       4   R = 0 on the first row; R_(i+1) = R_i where row i + 1 is not a path start, the last row excepted;
                R_(i+1) = R_i (1 + SIDE' (gamma^5 - 1)) + SIDE' lin(i + 1) where it is; R = Hint(0) on the last row
49 constraints in all at L > 1 and K > 1.  ROUND sets the ce blow-up at 8, and rescue.OPTIONS is reused.
"""
import numpy as np

from .. import expr as E
from ..air import AirConfig, RunningColumn, domain_generator
from ..prover import Stark, Trace
from .rescue import (DIGEST, OPTIONS, P, SECURITY_LEVEL, WIDTH, _context, _linear, _round_constraints, _selector,
                     _torch_device, digest_evaluation, permute, round_states)

__all__ = ["MerklePathsClaim", "MerkleUpdatesClaim", "OPTIONS", "SECURITY_LEVEL", "air_config", "gen_trace", "merge",
           "path", "root", "tree", "update", "updates_air_config"]

_R = 2**64
BIT, IDX, R_COL = WIDTH, WIDTH + 1, WIDTH + 2         # base columns 12, 13 and the running column 14
TUPLE = DIGEST + 1                                    # words bound per path: the leaf and the index
MAX_DEPTH = 32


def merge(a, b):
    """words 0..3 of the permutation of (a, b, 0, 0, 0, 0): the parent of children a and b (canonical 4-tuples)"""
    return tuple(permute(list(a) + list(b) + [0] * DIGEST)[:DIGEST])


def _path_shape(K, depth):
    """L, the smallest power of two >= depth; ValueError unless K is a power of two, 1 <= depth <= 32 and 8 K L <= 2^32"""
    if K < 1 or K & (K - 1):
        raise ValueError(f"K = {K} paths is not a power of two")
    if not 1 <= depth <= MAX_DEPTH:
        raise ValueError(f"depth {depth} is outside 1..{MAX_DEPTH}")
    L = 1 << (depth - 1).bit_length()
    if (8 * K * L).bit_length() - 1 > 32:
        raise ValueError(f"8 K L = {8 * K * L} rows: the trace domain has at most 2^32 points")
    return L


def _check_indices(indices, depth):
    idx = [int(i) for i in indices]
    for k, i in enumerate(idx):
        if not 0 <= i < 1 << depth:
            raise ValueError(f"index {i} of path {k} is not in 0..2^{depth} - 1")
    return idx


def _check_words(words, what):
    t = tuple(int(w) for w in words)
    if len(t) != DIGEST or not all(0 <= w < P for w in t):
        raise ValueError(f"{what} is not {DIGEST} canonical field elements")
    return t


# ---------------------------------------------------------------------------------------------------------- the tree
def tree(leaves, device=None):
    """the heap of the tree over `leaves` (2^D leaves of four canonical words: a sequence of 4-tuples, or a (2^D, 4)
    uint64 array or int64 tensor).  device=None: on the host with Python integers (small D only, about 0.2 ms per node),
    a list of 2^(D + 1) 4-tuples, entry 0 unused (zeros).  device: built on that device by ms_rescue_merkle_tree, a
    resident (2^(D + 1), 4) int64 tensor of canonical words, row 0 zeros."""
    if device is None:
        leaves = [_check_words(leaf, "a leaf") for leaf in leaves]
        depth = _depth_of(len(leaves))
        nodes = [(0,) * DIGEST] * (1 << depth) + leaves
        for v in range((1 << depth) - 1, 0, -1):
            nodes[v] = merge(nodes[2 * v], nodes[2 * v + 1])
        return nodes
    import torch
    dev = _torch_device(device)
    if isinstance(leaves, torch.Tensor):
        src = leaves.to(dev).contiguous()
        if src.dtype != torch.int64 or src.dim() != 2 or src.shape[1] != DIGEST:
            raise ValueError("leaves: a (2^D, 4) int64 tensor")
        if ((src < 0) & (src >= P - 2**64)).any():        # int64 words p .. 2^64 - 1
            raise ValueError("leaf words must be canonical field elements (0 <= word < p)")
    else:
        arr = _leaf_array(leaves)
        src = torch.from_numpy(arr.view(np.int64)).to(dev)
    depth = _depth_of(src.shape[0])
    nodes = torch.empty((2 << depth, DIGEST), dtype=torch.int64, device=dev)
    ctx = _context(dev)
    if nodes.is_cuda:                   # the context's stream may not be torch's: torch's work on this memory is done
        torch.cuda.current_stream(dev).synchronize()
    ctx.rescue_merkle_tree(src, depth, nodes)
    ctx.sync()
    return nodes


def _depth_of(count):
    if count < 2 or count & (count - 1) or count.bit_length() - 1 > MAX_DEPTH:
        raise ValueError(f"{count} leaves: a tree of depth 1..{MAX_DEPTH} has 2^D leaves")
    return count.bit_length() - 1


def _leaf_array(leaves):
    """(2^D, 4) C-contiguous uint64 array of canonical words, or ValueError"""
    if isinstance(leaves, np.ndarray):
        if leaves.ndim != 2 or leaves.shape[1] != DIGEST or leaves.dtype != np.uint64:
            raise ValueError("leaves: a (2^D, 4) uint64 array")
        arr = np.ascontiguousarray(leaves)
    else:
        try:
            arr = np.array([[int(w) for w in leaf] for leaf in leaves], dtype=np.uint64).reshape(-1, DIGEST)
        except (OverflowError, ValueError):
            raise ValueError("leaves: 2^D leaves of four canonical words") from None
    if (arr >= np.uint64(P)).any():
        raise ValueError("leaf words must be canonical field elements (0 <= word < p)")
    return arr


def _node(nodes, v):
    if isinstance(nodes, list):
        return tuple(nodes[v])
    return tuple(int(w) for w in np.asarray(_host_rows(nodes, [v]))[0])


def _host_rows(nodes, rows):
    """rows of a heap as a (len(rows), 4) uint64 array (the heap a list, an array or a tensor)"""
    if isinstance(nodes, list):
        return np.array([nodes[v] for v in rows], dtype=np.uint64).reshape(-1, DIGEST)
    if isinstance(nodes, np.ndarray):
        return nodes[np.asarray(rows, dtype=np.int64)].astype(np.uint64)
    import torch
    sel = torch.as_tensor(np.asarray(rows, dtype=np.int64), device=nodes.device)
    return nodes.index_select(0, sel).cpu().numpy().view(np.uint64)


def root(nodes):
    """the root (node 1) of a heap, four canonical words"""
    return _node(nodes, 1)


def path(nodes, depth, index):
    """the D siblings of leaf `index` from the bottom up: node ((2^D + index) >> j) ^ 1 for j = 0..D-1"""
    index = _check_indices([index], depth)[0]
    return [tuple(int(w) for w in r) for r in _host_rows(nodes, [((1 << depth) + index >> j) ^ 1 for j in range(depth)])]


# --------------------------------------------------------------------------------------------------------- the trace
def gen_trace(nodes, depth, indices, device=None):
    """(Trace, leaves) of MerklePathsClaim for the K = len(indices) paths through the heap `nodes` of depth D; leaves:
    the K leaves at those positions, 4-tuples of canonical words.  device=None: computed on the host with Python
    integers from a heap of tree(..., device=None) (small shapes only).  device: built on that device by
    ms_rescue_merkle_paths from a heap in device or host memory, and handed over as a resident (14, n) tensor."""
    idx = _check_indices(indices, depth)
    K = len(idx)
    L = _path_shape(K, depth)
    n = 8 * K * L
    leaves = [tuple(int(w) for w in r) for r in _host_rows(nodes, [(1 << depth) + i for i in idx])]
    if device is None:
        cols = np.zeros((WIDTH + 2, n), dtype=np.uint64)
        for k, i in enumerate(idx):
            cur, v = list(leaves[k]), (1 << depth) + i
            for j in range(L):
                bit = (i >> j) & 1 if j < depth else 0
                sib = list(_node(nodes, (v >> j) ^ 1)) if j < depth else [0] * DIGEST
                block = round_states((sib + cur if bit else cur + sib) + [0] * DIGEST)
                row = 8 * (L * k + j)
                cols[:WIDTH, row:row + 8] = np.array([[w * _R % P for w in st] for st in block], dtype=np.uint64).T
                cols[BIT, row:row + 8] = bit * _R % P
                cols[IDX, row:row + 8] = (i >> j) * _R % P
                cur = block[-1][:DIGEST]
        return Trace(cols), leaves
    import torch
    dev = _torch_device(device)
    out = torch.empty((WIDTH + 2, n), dtype=torch.int64, device=dev)
    ctx = _context(dev)
    if out.is_cuda:                     # the context's stream may not be torch's: torch's work on this memory is done
        torch.cuda.current_stream(dev).synchronize()
    heap = np.array(nodes, dtype=np.uint64) if isinstance(nodes, list) else nodes
    ctx.rescue_merkle_paths(heap, depth, np.array(idx, dtype=np.uint64), K, out)
    ctx.sync()                          # complete before the prover reads it on its own stream
    return Trace(out), leaves


# ----------------------------------------------------------------------------------------------------------- the AIR
def _lin(offset, first=0, bit=BIT, idx=IDX):
    """sum_(w<4) gamma^w ((1 - BIT) S_w + BIT S_(w+4)) + gamma^4 IDX at row offset `offset`, S the state in base columns
    first..first+11: the tuple a path start binds"""
    T, gamma, one = E.Trace, E.Challenge(0), E.Constant(1)
    b = T(bit, offset)
    words = [(one - b) * T(first + w, offset) + b * T(first + w + DIGEST, offset) for w in range(DIGEST)] + [T(idx, offset)]
    return _linear(words[w] * (gamma ** w) if w else words[0] for w in range(TUPLE))


def _zerofiers(n, K):
    """(every row, the r = 0 rows, the r = 7 rows, the path ends 8 L (k + 1) - 1) of K paths over n rows"""
    g = domain_generator(n.bit_length() - 1)
    x, one = E.X(), E.Constant(1)
    return (x ** n - one, x ** (n // 8) - one, x ** (n // 8) - E.Constant(pow(domain_generator(3), 7, P)),
            (E.Constant(g) * x) ** K - one)


def _cap(n, first=0):
    """CAP: the capacity words of the state in base columns first..first+11 are zero on the r = 0 rows"""
    _, first_rounds, _, _ = _zerofiers(n, 1)
    return [E.Trace(first + w, 0) / first_rounds for w in range(2 * DIGEST, WIDTH)]


def _link(n, K, first=0, bit=BIT):
    """LINK: on the r = 7 rows but the path ends, words 0..3 of the output (state in base columns first..first+11) are
    the half of the next row's state that BIT there selects"""
    _, _, last_rounds, path_ends = _zerofiers(n, K)
    T, one = E.Trace, E.Constant(1)
    nb = T(bit, 1)
    return [((one - nb) * (T(first + w, 1) - T(first + w, 0)) + nb * (T(first + w + DIGEST, 1) - T(first + w, 0)))
            * path_ends / last_rounds for w in range(DIGEST)]


def _bit_idx(n, K, L, bit=BIT, idx=IDX):
    """(BIT, IDX): BIT boolean and constant across a permutation; IDX constant across a permutation, IDX = 2 IDX' + BIT
    on the r = 7 rows but the path ends (L > 1), IDX = BIT on the path ends"""
    all_rows, _, last_rounds, path_ends = _zerofiers(n, K)
    T, one = E.Trace, E.Constant(1)
    within = last_rounds / all_rows                                                 # every row but r = 7
    bits = [T(bit, 0) * (T(bit, 0) - one) / all_rows, (T(bit, 1) - T(bit, 0)) * within]
    idxs = [(T(idx, 1) - T(idx, 0)) * within]
    if L > 1:
        idxs.append((T(idx, 0) - E.Constant(2) * T(idx, 1) - T(bit, 0)) * path_ends / last_rounds)
    idxs.append((T(idx, 0) - T(bit, 0)) / path_ends)
    return bits, idxs


def _running(n, K, col, lin):
    """R in base-or-extension column `col`: R = lin on the first row; R_(i+1) = R_i where row i + 1 is not a path start,
    the last row excepted; R_(i+1) = R_i gamma^5 + lin(i + 1) where it is; R = Hint(0) on the last row"""
    all_rows, _, _, path_ends = _zerofiers(n, K)
    x, T, one = E.X(), E.Trace, E.Constant(1)
    last = E.Constant(pow(domain_generator(n.bit_length() - 1), n - 1, P))
    g5 = E.Challenge(0) ** TUPLE
    return [(T(col, 0) - lin(0)) / (x - one),
            (T(col, 1) - T(col, 0)) * path_ends / all_rows,
            (T(col, 1) - T(col, 0) * g5 - lin(1)) * (x - last) / path_ends,
            (T(col, 0) - E.Hint(0)) / (x - last)]


def _running_column(L, lin):
    """the declared R: mul = 1 + e (gamma^5 - 1), add = e lin, e the selector of the path starts 8 L k"""
    e = _selector(0, 8 * L)
    return RunningColumn(init=0, mul=E.Constant(1) + e * (E.Challenge(0) ** TUPLE - E.Constant(1)), add=e * lin(0),
                         inclusive=True)


class MerkleAirConfig(AirConfig):
    """The AIR of MerklePathsClaim for PATHS = K paths in a tree of DEPTH = D levels (air_config(K, depth)); the trace
    has exactly 8 K L rows."""
    NUM_BASE_COLUMNS = WIDTH + 2
    NUM_EXTENSION_COLUMNS = 1
    FQ_IS_FP = False
    PATHS = None
    DEPTH = None

    @classmethod
    def _shape(cls, trace_len):
        K, depth = cls.PATHS, cls.DEPTH
        if K is None:
            raise ValueError("use air_config(K, depth): the AIR depends on the number of paths and the depth")
        L = _path_shape(K, depth)
        if trace_len != 8 * K * L:
            raise ValueError(f"a trace of {trace_len} rows is not {K} paths of depth {depth} ({8 * K * L} rows)")
        return K, depth, L

    @classmethod
    def groups(cls, trace_len):
        """{name: range of constraint indices} for ROUND, CAP, LINK, BIT, IDX, ROOT and R; LINK is empty when L = 1"""
        _, _, L = cls._shape(trace_len)
        sizes = [("ROUND", WIDTH), ("CAP", DIGEST), ("LINK", DIGEST if L > 1 else 0), ("BIT", 2),
                 ("IDX", 3 if L > 1 else 2), ("ROOT", DIGEST), ("R", 4)]
        out, at = {}, 0
        for name, size in sizes:
            out[name] = range(at, at + size)
            at += size
        return out

    @classmethod
    def constraints(cls, trace_len):
        K, depth, L = cls._shape(trace_len)
        n = trace_len
        g = domain_generator(n.bit_length() - 1)
        x, T, one = E.X(), E.Trace, E.Constant(1)
        # with L = 1 every r = 7 row is a path end: path_ends / last_rounds is a constant and there is nothing to link
        link = [] if L == 1 else _link(n, K)
        bit, idx = _bit_idx(n, K, L)
        at_root = (E.Constant(pow(g, n - 8 * depth + 1, P)) * x) ** K - one           # zero on rows 8 L k + 8 D - 1
        roots = [(T(w, 0) - E.Hint(1 + w)) / at_root for w in range(DIGEST)]
        # R: a path start is row 8 L k; the rows before one are the path ends
        return _round_constraints(n) + _cap(n) + link + bit + idx + roots + _running(n, K, R_COL, _lin)

    @classmethod
    def extension_columns(cls, trace_len):
        _, _, L = cls._shape(trace_len)
        return [_running_column(L, _lin)]

    @classmethod
    def gen_hints(cls, trace_len, claim, challenges):
        """[the Horner evaluation at gamma of the K (leaf, index) tuples, root_0, root_1, root_2, root_3]"""
        if (claim.K, claim.depth) != (cls.PATHS, cls.DEPTH):
            raise ValueError(f"the claim is {claim.K} paths of depth {claim.depth}, the AIR {cls.PATHS} of depth "
                             f"{cls.DEPTH}")
        cls._shape(trace_len)
        tuples = [tuple(leaf) + (i,) for leaf, i in zip(claim.leaves, claim.indices)]
        return [digest_evaluation(tuples, challenges[0])] + list(claim.root)


_CONFIGS = {}


def air_config(K, depth):
    """the AIR class for K paths in a tree of `depth` levels (one class per shape, so that provers cache one compiled AIR
    per shape)"""
    key = (int(K), int(depth))
    if key not in _CONFIGS:
        _path_shape(*key)
        _CONFIGS[key] = type(f"MerkleAirConfigK{key[0]}D{key[1]}", (MerkleAirConfig,), {"PATHS": key[0], "DEPTH": key[1]})
    return _CONFIGS[key]


class MerklePathsClaim(Stark):
    """For k = 0..K-1, leaves[k] (four canonical words) sits at position indices[k] of the depth-D Rescue-Prime Merkle
    tree whose root is `root`.  K is a power of two; the witness is the trace of gen_trace.

    The proof is not zero-knowledge (the reference's proofs are not either): its queries open trace rows, so leaves,
    siblings and index bits are revealed, and its out-of-domain evaluations depend on them."""

    def __init__(self, depth, root, leaves, indices):
        self.depth = int(depth)
        self.leaves = [_check_words(leaf, "a leaf") for leaf in leaves]
        self.K = len(self.leaves)
        _path_shape(self.K, self.depth)
        if len(indices) != self.K:
            raise ValueError(f"{len(indices)} indices for {self.K} leaves")
        self.indices = _check_indices(indices, self.depth)
        self.root = _check_words(root, "the root")
        self.AirConfig = air_config(self.K, self.depth)

    def get_public_inputs(self):
        return self

    def public_inputs_bytes(self, claim):
        """D, K, the four root words, then per path its four leaf words and its index; every value 8 bytes
        little-endian"""
        words = [claim.depth, claim.K] + list(claim.root)
        for leaf, i in zip(claim.leaves, claim.indices):
            words += list(leaf) + [i]
        return np.array(words, dtype="<u8").tobytes()


# ------------------------------------------------------------------------------------------------ ordered leaf writes
def _new_leaves(new_leaves, K):
    """K new leaves as 4-tuples of canonical words (a sequence of 4-tuples, a (K, 4) uint64 array or int64 tensor)"""
    if hasattr(new_leaves, "data_ptr"):
        new_leaves = new_leaves.cpu().numpy().view(np.uint64)
    rows = [tuple(int(w) for w in r) for r in _leaf_array(new_leaves)] if len(new_leaves) else []
    if len(rows) != K:
        raise ValueError(f"{len(rows)} new leaves for {K} indices")
    return rows


def update(nodes, depth, indices, new_leaves, device=None):
    """(Trace, new_nodes, roots) of MerkleUpdatesClaim: write k replaces leaf indices[k] of the depth-D heap `nodes`
    with new_leaves[k], for k = 0..K-1 in this order (K = len(indices), a power of two; a later write to the same leaf
    overwrites an earlier one).  new_nodes is the heap after every write; roots the K + 1 roots, roots[0] that of
    `nodes` and roots[k + 1] that after write k.  The caller's heap is never modified.
    device=None: computed on the host with Python integers from a heap of tree(..., device=None) (small shapes only);
    new_nodes is a list like it.  device: ms_rescue_merkle_updates on that device, applied to a copy of the heap made
    there (the heap in device or host memory); the trace is a resident (15, n) tensor and new_nodes a (2^(D + 1), 4)
    int64 tensor on that device."""
    idx = _check_indices(indices, depth)
    K = len(idx)
    L = _path_shape(2 * K, depth)
    new = _new_leaves(new_leaves, K)
    n = 16 * K * L
    if device is None:
        heap = [tuple(int(w) for w in v) for v in nodes]
        if len(heap) != 2 << depth:
            raise ValueError(f"a heap of {len(heap)} nodes is not a tree of depth {depth}")
        cols = np.zeros((WIDTH + 3, n), dtype=np.uint64)
        roots = [heap[1]]
        for k, i in enumerate(idx):
            v = (1 << depth) + i
            cur = [list(heap[v]), list(new[k])]                     # the old and the new path's current node
            for j in range(L):
                bit = (i >> j) & 1 if j < depth else 0
                sib = list(heap[(v >> j) ^ 1]) if j < depth else [0] * DIGEST
                if j < depth:
                    heap[v >> j] = tuple(cur[1])
                for side in range(2):                               # path 2 k + side
                    block = round_states((sib + cur[side] if bit else cur[side] + sib) + [0] * DIGEST)
                    row = 8 * (L * (2 * k + side) + j)
                    cols[:WIDTH, row:row + 8] = np.array([[w * _R % P for w in st] for st in block], dtype=np.uint64).T
                    cols[BIT, row:row + 8] = bit * _R % P
                    cols[IDX, row:row + 8] = (i >> j) * _R % P
                    cols[SIDE, row:row + 8] = side * _R % P
                    cur[side] = block[-1][:DIGEST]
                if j == depth - 1:
                    heap[1] = tuple(cur[1])
                    roots.append(heap[1])
        return Trace(cols), heap, roots
    import torch
    dev = _torch_device(device)
    if isinstance(nodes, torch.Tensor):
        heap = nodes.to(dev, copy=True)
    else:
        heap = torch.from_numpy(np.array(nodes, dtype=np.uint64).view(np.int64)).to(dev)
    if heap.dtype != torch.int64 or tuple(heap.shape) != (2 << depth, DIGEST):
        raise ValueError(f"nodes: a ({2 << depth}, 4) heap of canonical words")
    heap = heap.contiguous()
    out = torch.empty((WIDTH + 3, n), dtype=torch.int64, device=dev)
    roots = torch.empty((K + 1, DIGEST), dtype=torch.int64, device=dev)
    ctx = _context(dev)
    if out.is_cuda:                     # the context's stream may not be torch's: torch's work on this memory is done
        torch.cuda.current_stream(dev).synchronize()
    ctx.rescue_merkle_updates(heap, depth, np.array(idx, dtype=np.uint64), np.array(new, dtype=np.uint64).reshape(K, 4),
                              K, out, roots)
    ctx.sync()                          # complete before the prover reads it on its own stream
    return Trace(out), heap, [tuple(int(w) for w in r) for r in roots.cpu().numpy().view(np.uint64)]


SIDE, U_R = WIDTH + 2, WIDTH + 3        # the updates trace's base column 14 and its running column 15


class MerkleUpdatesAirConfig(AirConfig):
    """The AIR of MerkleUpdatesClaim for WRITES = K writes into a tree of DEPTH = D levels (updates_air_config(K,
    depth)); the trace has exactly 16 K L rows."""
    NUM_BASE_COLUMNS = WIDTH + 3
    NUM_EXTENSION_COLUMNS = 1
    FQ_IS_FP = False
    WRITES = None
    DEPTH = None

    @classmethod
    def _shape(cls, trace_len):
        K, depth = cls.WRITES, cls.DEPTH
        if K is None:
            raise ValueError("use updates_air_config(K, depth): the AIR depends on the number of writes and the depth")
        L = _path_shape(2 * K, depth)
        if trace_len != 16 * K * L:
            raise ValueError(f"a trace of {trace_len} rows is not {K} writes of depth {depth} ({16 * K * L} rows)")
        return K, depth, L

    @classmethod
    def groups(cls, trace_len):
        """{name: range of constraint indices} for ROUND, CAP, LINK, SIDE, SIB, BIT, IDX, ROOT, CHAIN and R; LINK is
        empty when L = 1 and CHAIN when K = 1"""
        K, _, L = cls._shape(trace_len)
        sizes = [("ROUND", WIDTH), ("CAP", DIGEST), ("LINK", DIGEST if L > 1 else 0), ("SIDE", 3), ("SIB", DIGEST + 1),
                 ("BIT", 2), ("IDX", 3 if L > 1 else 2), ("ROOT", 2 * DIGEST), ("CHAIN", DIGEST if K > 1 else 0),
                 ("R", 4)]
        out, at = {}, 0
        for name, size in sizes:
            out[name] = range(at, at + size)
            at += size
        return out

    @classmethod
    def constraints(cls, trace_len):
        K, depth, L = cls._shape(trace_len)
        n = trace_len
        g = domain_generator(n.bit_length() - 1)
        x, T, one = E.X(), E.Trace, E.Constant(1)
        all_rows, first_rounds, _, path_ends = _zerofiers(n, 2 * K)
        last = E.Constant(pow(g, n - 1, P))
        # path 2 k (write k's old path) and path 2 k + 1 (its new path), 8 L rows apart: the paths AIR's constraints on
        # 2 K paths, with LINK dropped at L = 1 as there.  Every zerofier below is one of the paths AIR's: the
        # evaluator's batched inverses of more would not fit its registers
        link = [] if L == 1 else _link(n, 2 * K)
        side, old = T(SIDE, 0), one - T(SIDE, 0)
        sides = [side / (x - one), (T(SIDE, 1) - side) * path_ends / all_rows,
                 (T(SIDE, 1) + side - one) * (x - last) / path_ends]
        b = T(BIT, 0)
        sib = [((one - b) * (T(w + DIGEST, 0) - T(w + DIGEST, 8 * L)) + b * (T(w, 0) - T(w, 8 * L))) * old / first_rounds
               for w in range(DIGEST)] + [(b - T(BIT, 8 * L)) * old / first_rounds]
        bit, idx = _bit_idx(n, 2 * K, L)
        # the old root of write 0 (row 8 D - 1) and the new root of write K - 1 (row n - 1 - 8 (L - D)), read from the
        # first and the last row
        roots = ([(T(w, 8 * depth - 1) - E.Hint(1 + w)) / (x - one) for w in range(DIGEST)]
                 + [(T(w, 8 * (depth - L)) - E.Hint(1 + DIGEST + w)) / (x - last) for w in range(DIGEST)])
        # on the new paths' roots (rows 8 L (2 k + 1) + 8 D - 1) but write K - 1's: the next write's old root, 8 L on
        at_root = (E.Constant(pow(g, n - 8 * depth + 1, P)) * x) ** (2 * K) - one       # zero on rows 8 L t + 8 D - 1
        last_write = x - E.Constant(pow(g, n - 8 * L + 8 * depth - 1, P))
        chain = [] if K == 1 else [(T(w, 8 * L) - T(w, 0)) * side * last_write / at_root for w in range(DIGEST)]
        # R: the (new leaf, IDX) tuple is bound where a new path starts, the row after a path end with SIDE = 1 there
        g5, ns = E.Challenge(0) ** TUPLE, T(SIDE, 1)
        r = [T(U_R, 0) / (x - one),
             (T(U_R, 1) - T(U_R, 0)) * path_ends / all_rows,
             (T(U_R, 1) - T(U_R, 0) * (one + ns * (g5 - one)) - ns * _lin(1)) * (x - last) / path_ends,
             (T(U_R, 0) - E.Hint(0)) / (x - last)]
        return _round_constraints(n) + _cap(n) + link + sides + sib + bit + idx + roots + chain + r

    @classmethod
    def extension_columns(cls, trace_len):
        _, _, L = cls._shape(trace_len)
        e = _selector(8 * L, 16 * L)
        return [RunningColumn(init=0, mul=E.Constant(1) + e * (E.Challenge(0) ** TUPLE - E.Constant(1)), add=e * _lin(0),
                              inclusive=True)]

    @classmethod
    def gen_hints(cls, trace_len, claim, challenges):
        """[the Horner evaluation at gamma of the K (new leaf, index) tuples, the old root's four words, the new
        root's four words]"""
        if (claim.K, claim.depth) != (cls.WRITES, cls.DEPTH):
            raise ValueError(f"the claim is {claim.K} writes of depth {claim.depth}, the AIR {cls.WRITES} of depth "
                             f"{cls.DEPTH}")
        cls._shape(trace_len)
        tuples = [tuple(leaf) + (i,) for leaf, i in zip(claim.new_leaves, claim.indices)]
        return [digest_evaluation(tuples, challenges[0])] + list(claim.old_root) + list(claim.new_root)


_UPDATE_CONFIGS = {}


def updates_air_config(K, depth):
    """the AIR class for K writes into a tree of `depth` levels (one class per shape, so that provers cache one compiled
    AIR per shape)"""
    key = (int(K), int(depth))
    if key not in _UPDATE_CONFIGS:
        _path_shape(2 * key[0], key[1])
        _UPDATE_CONFIGS[key] = type(f"MerkleUpdatesAirConfigK{key[0]}D{key[1]}", (MerkleUpdatesAirConfig,),
                                    {"WRITES": key[0], "DEPTH": key[1]})
    return _UPDATE_CONFIGS[key]


class MerkleUpdatesClaim(Stark):
    """Starting from the depth-D Rescue-Prime Merkle tree whose root is `old_root`, replacing leaf indices[k] with
    new_leaves[k] (four canonical words) for k = 0..K-1, one write after another, gives the tree whose root is
    `new_root`.  K is a power of two and an index may repeat (order matters then); the old leaves are witness, not
    public input.  The witness is the trace of update().

    The proof is not zero-knowledge: its queries open trace rows, so old leaves, siblings, intermediate roots and index
    bits are revealed, and its out-of-domain evaluations depend on them."""

    def __init__(self, depth, old_root, new_root, indices, new_leaves):
        self.depth = int(depth)
        self.new_leaves = [_check_words(leaf, "a new leaf") for leaf in new_leaves]
        self.K = len(self.new_leaves)
        _path_shape(2 * self.K, self.depth)
        if len(indices) != self.K:
            raise ValueError(f"{len(indices)} indices for {self.K} new leaves")
        self.indices = _check_indices(indices, self.depth)
        self.old_root = _check_words(old_root, "the old root")
        self.new_root = _check_words(new_root, "the new root")
        self.AirConfig = updates_air_config(self.K, self.depth)

    def get_public_inputs(self):
        return self

    def public_inputs_bytes(self, claim):
        """D, K, the old root's four words, the new root's four words, then per write its four new-leaf words and its
        index; every value 8 bytes little-endian"""
        words = [claim.depth, claim.K] + list(claim.old_root) + list(claim.new_root)
        for leaf, i in zip(claim.new_leaves, claim.indices):
            words += list(leaf) + [i]
        return np.array(words, dtype="<u8").tobytes()
