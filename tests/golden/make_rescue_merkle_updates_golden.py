"""Generates tests/golden/rescue_merkle_updates_d16_k1024.json: K = 2^10 ordered leaf writes into the Rescue-Prime
Merkle tree of depth 16, as the restatement (tests/rescue_merkle_updates_oracle.py) applies them: the trace of
examples/merkle's write claim (L = 16, 2^18 rows), the roots and the final heap — TEST INFRASTRUCTURE, run offline
(about two minutes; the writes are applied one after another):

    python tests/golden/make_rescue_merkle_updates_golden.py

The tree's leaves are leaves(depth, seed) of make_rescue_merkle_golden.py; the new leaves are leaves drawn the same way
from a "new leaves" tag, and the indices indices(K, depth, seed) from an "update indices" tag (SHAKE-256 of a fixed
string and the seed, little-endian 64-bit words, masked to 63 bits for leaf words and to D bits for indices).  A random
stream of 2^10 indices below 2^16 rarely repeats an index or writes a sibling pair, so writes() forces both: write 7
repeats write 3's index, write 12 writes the sibling of write 11's leaf and write 13 that leaf again.  The file holds
the shape, the seed, the old and the new root, the SHA-256 of the final heap (2^(D + 1) x 4 canonical words, row 0
zeros, little-endian), the SHA-256 of the (15, n) column-major matrix of Montgomery words and the first roots.
tests/test_gpu_rescue_merkle_updates.py checks the device against it."""
import hashlib
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_rescue_merkle_golden import _words, heap_sha256, leaves, oracle_heap  # noqa: E402

DEPTH, K, SEED = 16, 1 << 10, 1
P = 2**64 - 2**32 + 1


def writes(K, depth, seed):
    """(indices, new leaves): K uint64 indices below 2^depth with a forced repeat and sibling pair, and a (K, 4) uint64
    array of canonical words"""
    idx = _words(b"update indices", seed, K) & np.uint64((1 << depth) - 1)
    if K >= 16:
        idx[7] = idx[3]
        idx[12] = idx[11] ^ np.uint64(1)
        idx[13] = idx[11]
    new = (_words(b"new leaves", seed, 4 * K) & np.uint64(2**63 - 1)).reshape(K, 4)
    return idx, new


def record(depth, K, seed):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import rescue_merkle_updates_oracle as UO
    lv = leaves(depth, seed)
    idx, new = writes(K, depth, seed)
    with Pool() as pool:
        nodes = oracle_heap(lv, pool)
    rows, roots, heap = UO.updates_trace(nodes, depth, [int(i) for i in idx], [[int(w) for w in r] for r in new])
    trace = np.ascontiguousarray(np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T)
    final = np.array([[0] * 4] + heap[1:], dtype=np.uint64)
    return {"depth": depth, "K": K, "seed": seed, "old_root": roots[0], "new_root": roots[-1],
            "heap_sha256": heap_sha256(final), "trace_sha256": hashlib.sha256(trace.tobytes()).hexdigest(),
            "first_roots": roots[:4]}


if __name__ == "__main__":
    gold = record(DEPTH, K, SEED)
    with open(os.path.join(HERE, "rescue_merkle_updates_d16_k1024.json"), "w") as f:
        json.dump(gold, f)
        f.write("\n")
