"""Generates tests/golden/rescue_wots_k7.json: K = 7 Winternitz one-time signatures over Rescue-Prime, as the restatement
(tests/rescue_wots_oracle.py) signs them, and the trace of examples/wots's claim over them (469 chain blocks and 43
padding blocks, 2^16 rows) — TEST INFRASTRUCTURE, run offline (a few minutes):

    python tests/golden/make_rescue_wots_golden.py

keys(seed) gives every key a secret of four 63-bit words and a seed of two, except keys 3 and 4, which share one seed.
messages(seed) forces: the all-zero message (key 0: every digit 0, checksum digits (0, 12, 3)), a message of words
p - 1 (key 1: half its digits 15, so those chains take no step), and a message whose checksum's middle digit is 0 (key
2).  Randomness is SHAKE-256 of a fixed string and the seed (make_rescue_merkle_golden._words).  The file holds K, the
seed, the public keys, the SHA-256 of the signatures (K x 67 x 4 canonical words, little-endian), of the public keys
(K x 6) and of the (15, n) column-major matrix of Montgomery words.  tests/test_gpu_rescue_wots.py checks the device
against it."""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
from make_rescue_merkle_golden import _words  # noqa: E402

K, SEED = 7, 1
P = 2**64 - 2**32 + 1
MASK = np.uint64(2**63 - 1)


def keys(K, seed):
    """((K, 4) secrets, (K, 2) seeds) as uint64 arrays of canonical words"""
    secrets = (_words(b"wots secrets", seed, 4 * K) & MASK).reshape(K, 4)
    seeds = (_words(b"wots seeds", seed, 2 * K) & MASK).reshape(K, 2)
    if K > 4:
        seeds[4] = seeds[3]
    return secrets, seeds


def _checksum_digits(m):
    d = [(int(m[w]) >> 4 * t) & 15 for w in range(4) for t in range(16)]
    c = sum(15 - v for v in d)
    return [(c >> 4 * t) & 15 for t in range(3)]


def messages(K, seed):
    """(K, 4) uint64 array of canonical words"""
    msgs = (_words(b"wots messages", seed, 4 * K) & MASK).reshape(K, 4)
    msgs[0] = 0
    if K > 1:
        msgs[1] = P - 1
    if K > 2:
        # the first of a run of candidates whose checksum's middle digit is 0 (about one in 16 is)
        msgs[2] = next(m for j in range(1000) for m in [_words(b"wots checksum", 1000 * seed + j, 4) & MASK]
                       if _checksum_digits(m)[1] == 0)
    return msgs


def sha(words):
    return hashlib.sha256(np.ascontiguousarray(np.array(words, dtype=np.uint64)).astype("<u8").tobytes()).hexdigest()


def record(K, seed):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import rescue_wots_oracle as WO
    secrets, seeds = keys(K, seed)
    msgs = messages(K, seed)
    pks = [WO.keygen([int(w) for w in secrets[k]], [int(w) for w in seeds[k]])[0] for k in range(K)]
    sigs = [WO.sign([int(w) for w in secrets[k]], [int(w) for w in seeds[k]], [int(w) for w in msgs[k]])
            for k in range(K)]
    rows, roots = WO.wots_trace(pks, [[int(w) for w in m] for m in msgs], sigs)
    assert roots == [pk[2:] for pk in pks]
    trace = np.ascontiguousarray(np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T)
    return {"K": K, "seed": seed, "public_keys": pks, "signatures_sha256": sha(sigs), "public_keys_sha256": sha(pks),
            "trace_sha256": hashlib.sha256(trace.tobytes()).hexdigest()}


if __name__ == "__main__":
    gold = record(K, SEED)
    with open(os.path.join(HERE, "rescue_wots_k7.json"), "w") as f:
        json.dump(gold, f)
        f.write("\n")
