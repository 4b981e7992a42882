"""The trace of examples/merkle's ordered-write claim (MerkleUpdatesClaim), restated with Python integers for the tests.
TEST INFRASTRUCTURE ONLY.

Independent of ministark_b200/examples/merkle.py: it builds on tests/rescue_merkle_oracle.py.  Each write is applied
to a copy of the heap in turn: its old path is the restated authentication path of the leaf it replaces in the tree as
it stands, its new path the same with the new leaf, and the nodes on the path take the new path's values.  Values are
canonical integers."""
import rescue_merkle_oracle as MO

W = MO.W


def updates_trace(nodes, depth, indices, new_leaves):
    """(rows, roots, heap): the n = 16 K L trace rows (S_0..S_11, BIT, IDX, SIDE; write k's old path, then its new
    path), the
    K + 1 roots (before the first write and after each) and the heap after every write ([None, node 1, ...], as MO.heap gives it)"""
    heap = [None] + [list(v) for v in nodes[1:]]
    roots, rows = [list(heap[1])], []
    for i, leaf in zip(indices, new_leaves):
        old = MO.path_rows(heap, depth, i)
        v = (1 << depth) + i
        heap[v] = list(leaf)
        for j in range(1, depth + 1):                   # the path's nodes as the new leaf makes them
            p = v >> j
            heap[p] = MO.compress(heap[2 * p], heap[2 * p + 1])
        new = MO.path_rows(heap, depth, i)              # the siblings are off the path: the write left them as they were
        assert new[8 * depth - 1][:W] == heap[1]
        rows += [r + [0] for r in old] + [r + [1] for r in new]
        roots.append(list(heap[1]))
    return rows, roots, heap
