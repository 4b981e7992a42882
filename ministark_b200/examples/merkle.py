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
"""
import numpy as np

from .. import expr as E
from ..air import AirConfig, RunningColumn, domain_generator
from ..prover import Stark, Trace
from .rescue import (DIGEST, OPTIONS, P, SECURITY_LEVEL, WIDTH, _context, _linear, _round_constraints, _selector,
                     _torch_device, digest_evaluation, permute, round_states)

__all__ = ["MerklePathsClaim", "OPTIONS", "SECURITY_LEVEL", "air_config", "gen_trace", "merge", "path", "root", "tree"]

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
def _lin(offset):
    """sum_(w<4) gamma^w ((1 - BIT) S_w + BIT S_(w+4)) + gamma^4 IDX at row offset `offset`: the tuple a path start binds"""
    T, gamma, one = E.Trace, E.Challenge(0), E.Constant(1)
    b = T(BIT, offset)
    words = [(one - b) * T(w, offset) + b * T(w + DIGEST, offset) for w in range(DIGEST)] + [T(IDX, offset)]
    return _linear(words[w] * (gamma ** w) if w else words[0] for w in range(TUPLE))


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
        all_rows = x ** n - one
        first_rounds = x ** (n // 8) - one                                              # zero on the r = 0 rows
        last_rounds = x ** (n // 8) - E.Constant(pow(domain_generator(3), 7, P))      # zero on the r = 7 rows
        path_ends = (E.Constant(g) * x) ** K - one                                      # zero on rows 8 L (k + 1) - 1
        last = E.Constant(pow(g, n - 1, P))
        cap = [T(w, 0) / first_rounds for w in range(2 * DIGEST, WIDTH)]
        # with L = 1 every r = 7 row is a path end: path_ends / last_rounds is a constant and there is nothing to link
        nb = T(BIT, 1)
        link = [] if L == 1 else [
            ((one - nb) * (T(w, 1) - T(w, 0)) + nb * (T(w + DIGEST, 1) - T(w, 0))) * path_ends / last_rounds
            for w in range(DIGEST)]
        within = last_rounds / all_rows                                                 # every row but r = 7
        bit = [T(BIT, 0) * (T(BIT, 0) - one) / all_rows, (T(BIT, 1) - T(BIT, 0)) * within]
        idx = [(T(IDX, 1) - T(IDX, 0)) * within]
        if L > 1:
            idx.append((T(IDX, 0) - E.Constant(2) * T(IDX, 1) - T(BIT, 0)) * path_ends / last_rounds)
        idx.append((T(IDX, 0) - T(BIT, 0)) / path_ends)
        at_root = (E.Constant(pow(g, n - 8 * depth + 1, P)) * x) ** K - one           # zero on rows 8 L k + 8 D - 1
        roots = [(T(w, 0) - E.Hint(1 + w)) / at_root for w in range(DIGEST)]
        # R: a path start is row 8 L k; the rows before one are the path ends
        gamma = E.Challenge(0)
        g5 = gamma ** TUPLE
        r = [(T(R_COL, 0) - _lin(0)) / (x - one),
             (T(R_COL, 1) - T(R_COL, 0)) * path_ends / all_rows,
             (T(R_COL, 1) - T(R_COL, 0) * g5 - _lin(1)) * (x - last) / path_ends,
             (T(R_COL, 0) - E.Hint(0)) / (x - last)]
        return _round_constraints(n) + cap + link + bit + idx + roots + r

    @classmethod
    def extension_columns(cls, trace_len):
        _, _, L = cls._shape(trace_len)
        e = _selector(0, 8 * L)
        return [RunningColumn(init=0, mul=E.Constant(1) + e * (E.Challenge(0) ** TUPLE - E.Constant(1)), add=e * _lin(0),
                              inclusive=True)]

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
