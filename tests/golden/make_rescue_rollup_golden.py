"""Generates tests/golden/rescue_rollup_d16_k512.json: K = 2^9 balance transfers over the accounts of a depth-16
Rescue-Prime Merkle tree, as the restatement (tests/rescue_rollup_oracle.py) applies them: the trace of examples/rollup's
transfer claim (L = 16, 2^18 rows), the roots and the final heap — TEST INFRASTRUCTURE, run offline (about two minutes;
the writes are applied one after another):

    python tests/golden/make_rescue_rollup_golden.py

accounts(depth, seed) gives every account a balance below 2^31, a nonce below 2^16 and two 63-bit owner words, except
account 0, whose balance is 2^32 - 1, and every 64th account, which is empty (all zero).  transfers(nodes, depth, K,
seed) draws senders and receivers among accounts 1..2^D - 1 and amounts that keep every balance in [0, 2^32), and
forces: a self-transfer (transfer 5), a zero amount (9), one account touched by transfers 20..27 (sender of the first
four, receiver of the last four), a sender left at exactly 0 (30) and a receiver brought to exactly 2^32 - 1 by
account 0 (31).  Randomness is SHAKE-256 of a fixed string and the seed (make_rescue_merkle_golden._words).  The file
holds the shape, the seed, the old and the new root, the SHA-256 of the final heap (2^(D + 1) x 4 canonical words, row
0 zeros, little-endian), the SHA-256 of the (23, n) column-major matrix of Montgomery words and the first roots.
tests/test_gpu_rescue_rollup.py checks the device against it."""
import hashlib
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_rescue_merkle_golden import _words, heap_sha256, oracle_heap  # noqa: E402

DEPTH, K, SEED = 16, 1 << 9, 1
P = 2**64 - 2**32 + 1
TOP = 2**32 - 1


def accounts(depth, seed):
    """(2^depth, 4) uint64 leaves (balance, nonce, owner_0, owner_1)"""
    w = _words(b"rollup accounts", seed, 4 << depth).reshape(1 << depth, 4)
    lv = np.stack([w[:, 0] & np.uint64(2**31 - 1), w[:, 1] & np.uint64(2**16 - 1), w[:, 2] & np.uint64(2**63 - 1),
                   w[:, 3] & np.uint64(2**63 - 1)], axis=1)
    lv[::64] = 0
    lv[0] = (TOP, 0, 1, 2)
    return lv


def transfers(lv, depth, K, seed):
    """K (sender, receiver, amount) triples, valid when applied in order to the accounts lv"""
    r = [int(v) for v in _words(b"rollup transfers", seed, 3 * K)]
    bal = {}
    get = lambda a: bal.get(a, int(lv[a][0]))
    touched = 1 + r[0] % ((1 << depth) - 1)
    out = []
    for k in range(K):
        s, d = 1 + r[3 * k] % ((1 << depth) - 1), 1 + r[3 * k + 1] % ((1 << depth) - 1)
        if k == 5:
            d = s
        if 20 <= k < 24:
            s = touched
        elif 24 <= k < 28:
            d = touched
        if k == 31:
            s = 0
        bs, br = get(s), get(d)
        amount = r[3 * k + 2] % (bs + 1)
        if s != d:
            amount = min(amount, TOP - br)
        if k == 9:
            amount = 0
        elif k == 30:
            amount = bs
            assert s != d and br + bs <= TOP
        elif k == 31:
            amount = TOP - br
        bal[s] = bs - amount
        bal[d] = get(d) + amount
        out.append((s, d, amount))
    return out


def record(depth, K, seed):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import rescue_rollup_oracle as RO
    lv = accounts(depth, seed)
    with Pool() as pool:
        nodes = oracle_heap(lv, pool)
    txs = transfers(lv, depth, K, seed)
    rows, roots, heap = RO.rollup_trace(nodes, depth, txs)
    trace = np.ascontiguousarray(np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T)
    final = np.array([[0] * 4] + heap[1:], dtype=np.uint64)
    return {"depth": depth, "K": K, "seed": seed, "old_root": roots[0], "new_root": roots[-1],
            "heap_sha256": heap_sha256(final), "trace_sha256": hashlib.sha256(trace.tobytes()).hexdigest(),
            "first_roots": roots[:4]}


if __name__ == "__main__":
    gold = record(DEPTH, K, SEED)
    with open(os.path.join(HERE, "rescue_rollup_d16_k512.json"), "w") as f:
        json.dump(gold, f)
        f.write("\n")
