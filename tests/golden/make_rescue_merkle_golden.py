"""Generates tests/golden/rescue_merkle_d16_k1024.json: the Rescue-Prime Merkle tree of depth 16 and the trace of
examples/merkle's claim for K = 2^10 paths through it (L = 16, 2^17 rows) as the restatement
(tests/rescue_merkle_oracle.py) writes them — TEST INFRASTRUCTURE, run offline (well under a minute on eight cores):

    python tests/golden/make_rescue_merkle_golden.py

The leaves are leaves(depth, seed) and the indices indices(K, depth, seed): SHAKE-256 of a fixed string and the seed,
read as little-endian 64-bit words, masked to 63 bits for the leaves (so every word is canonical) and to D bits for the
indices.  The file holds the shape, the seed, the root, the SHA-256 of the heap (2^(D + 1) x 4 canonical words, row 0
zeros, little-endian), the SHA-256 of the (14, n) column-major matrix of Montgomery words and the first indices.
tests/test_gpu_rescue_merkle.py checks the device tree and trace against it."""
import hashlib
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
DEPTH, K, SEED = 16, 1 << 10, 1
P = 2**64 - 2**32 + 1
CHUNK = 64                          # paths (and, for the tree, subtrees) per worker task


def _words(tag, seed, count):
    stream = hashlib.shake_256(b"ministark_b200 examples/merkle " + tag + b" %d" % seed).digest(8 * count)
    return np.frombuffer(stream, dtype="<u8").astype(np.uint64)


def leaves(depth, seed):
    """(2^depth, 4) uint64 array of canonical words, the same for every caller"""
    return (_words(b"leaves", seed, 4 << depth) & np.uint64(2**63 - 1)).reshape(1 << depth, 4)


def indices(K, depth, seed):
    """K uint64 indices below 2^depth"""
    return _words(b"indices", seed, K) & np.uint64((1 << depth) - 1)


def heap_sha256(nodes):
    return hashlib.sha256(np.ascontiguousarray(nodes, dtype="<u8").tobytes()).hexdigest()


def _subtree(args):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import rescue_merkle_oracle as MO
    return MO.heap([[int(w) for w in leaf] for leaf in args])


def _paths(args):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import rescue_merkle_oracle as MO
    nodes, depth, idx = args
    rows, _, _ = MO.paths_trace(nodes, depth, idx)
    return np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T


def oracle_heap(lv, pool):
    """the heap over the leaves: 2^s subtrees in parallel, then the levels above them"""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import rescue_merkle_oracle as MO
    count = len(lv)
    sub = min(count // 2, 1 << 10)                  # leaves per subtree
    parts = pool.map(_subtree, [lv[i:i + sub] for i in range(0, count, sub)])
    nodes = [None] * (2 * count)
    for p, part in enumerate(parts):                # subtree p's node u (depth of u within it: bit_length - 1)
        for u in range(1, 2 * sub):
            level = u.bit_length() - 1
            nodes[(((count // sub) + p) << level) + u - (1 << level)] = part[u]
    for v in range(count // sub - 1, 0, -1):
        nodes[v] = MO.compress(nodes[2 * v], nodes[2 * v + 1])
    return nodes


def record(depth, K, seed):
    lv, idx = leaves(depth, seed), [int(i) for i in indices(K, depth, seed)]
    with Pool() as pool:
        nodes = oracle_heap(lv, pool)
        cols = pool.map(_paths, [(nodes, depth, idx[i:i + CHUNK]) for i in range(0, K, CHUNK)])
    trace = np.ascontiguousarray(np.concatenate(cols, axis=1))
    heap = np.array([[0] * 4] + nodes[1:], dtype=np.uint64)
    return {"depth": depth, "K": K, "seed": seed, "root": [int(w) for w in nodes[1]], "heap_sha256": heap_sha256(heap),
            "trace_sha256": hashlib.sha256(trace.tobytes()).hexdigest(), "first_indices": idx[:8]}


if __name__ == "__main__":
    gold = record(DEPTH, K, SEED)
    with open(os.path.join(HERE, "rescue_merkle_d16_k1024.json"), "w") as f:
        json.dump(gold, f)
        f.write("\n")
