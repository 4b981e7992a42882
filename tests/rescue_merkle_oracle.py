"""The Rescue-Prime Merkle tree and the trace of examples/merkle's authentication-path claim, restated with Python
integers for the tests.  TEST INFRASTRUCTURE ONLY.

Independent of ministark_b200/examples/merkle.py: it builds on the restated permutation of oracle/rescue_oracle.py.  A
parent is words 0..3 of the permutation of (left child, right child, 0, 0, 0, 0); the heap has the root at node 1 and
leaf i at node 2^D + i.  Values are canonical integers."""
from oracle import rescue_oracle as RO

P = RO.P
W = 4                                   # words per node


def compress(a, b):
    return RO.permute(list(a) + list(b) + [0] * (RO.M - 2 * W))[:W]


def heap(leaves):
    """[None, node 1, ..., node 2^(D + 1) - 1] over the 2^D leaves"""
    count = len(leaves)
    assert count >= 2 and count & (count - 1) == 0
    nodes = [None] * count + [list(leaf) for leaf in leaves]
    for v in range(count - 1, 0, -1):
        nodes[v] = compress(nodes[2 * v], nodes[2 * v + 1])
    return nodes


def path_rows(nodes, depth, index):
    """the 8 L rows of one path, 14 canonical words each (S_0..S_11, BIT, IDX), L the smallest power of two >= depth"""
    L = 1
    while L < depth:
        L *= 2
    v = (1 << depth) + index
    cur, rows = list(nodes[v]), []
    for j in range(L):
        if j < depth:
            b, sib = (index >> j) & 1, list(nodes[(v >> j) ^ 1])
        else:
            b, sib = 0, [0] * W
        state = (sib + cur if b else cur + sib) + [0] * (RO.M - 2 * W)
        states = RO.round_states(state)
        rows += [st + [b, index >> j] for st in states]
        cur = states[-1][:W]
    return rows


def paths_trace(nodes, depth, indices):
    """(rows, leaves, roots): the n = 8 K L trace rows, the K leaves and the root each path ends in (row 8 (L k + D) - 1)"""
    rows, leaves, roots = [], [], []
    for i in indices:
        block = path_rows(nodes, depth, i)
        roots.append(block[8 * depth - 1][:W])
        leaves.append(list(nodes[(1 << depth) + i]))
        rows += block
    return rows, leaves, roots
