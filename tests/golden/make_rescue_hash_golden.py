"""Generates tests/golden/rescue_hash_k65536_len60.json: the trace of examples/rescue's hash claim for K = 2^16 messages
of 60 words (B = L = 8 permutations each, 2^22 rows) as the restated sponge (tests/rescue_hash_oracle.py) writes it —
TEST INFRASTRUCTURE, run offline (a few minutes on eight cores, about 1 GB of memory):

    python tests/golden/make_rescue_hash_golden.py

The messages are messages(K, length): SHAKE-256 of a fixed string, read as little-endian 64-bit words masked to 63
bits, so every word is canonical.  The file holds K, the length, the SHA-256 of the (13, 2^22) column-major matrix of
Montgomery words, the SHA-256 of the K x 4 digest words (canonical, little-endian, message by message) and the first 8
digests.  tests/test_gpu_rescue_hash.py checks the device trace against it."""
import hashlib
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
K, LENGTH = 1 << 16, 60
P = 2**64 - 2**32 + 1
CHUNK = 512                         # messages per worker task


def messages(K, length):
    """(K, length) uint64 array of canonical words, the same for every caller"""
    stream = hashlib.shake_256(b"ministark_b200 examples/rescue hash messages").digest(8 * K * length)
    return (np.frombuffer(stream, dtype="<u8") & np.uint64(2**63 - 1)).astype(np.uint64).reshape(K, length)


def digests_sha256(digests):
    return hashlib.sha256(np.array(digests, dtype="<u8").tobytes()).hexdigest()


def _chunk(msgs):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import rescue_hash_oracle as HO
    rows, digests = HO.hash_trace([[int(w) for w in m] for m in msgs])
    cols = np.array([[v * 2**64 % P for v in r] for r in rows], dtype=np.uint64).T
    return cols, digests


def record(msgs):
    K, length = msgs.shape
    parts = [msgs[i:i + CHUNK] for i in range(0, K, CHUNK)]
    with Pool() as pool:
        done = pool.map(_chunk, parts)
    trace = np.ascontiguousarray(np.concatenate([c for c, _ in done], axis=1))
    digests = [d for _, ds in done for d in ds]
    return {"K": K, "length": length, "trace_sha256": hashlib.sha256(trace.tobytes()).hexdigest(),
            "digests_sha256": digests_sha256(digests), "first_digests": digests[:8]}


if __name__ == "__main__":
    gold = record(messages(K, LENGTH))
    with open(os.path.join(HERE, "rescue_hash_k65536_len60.json"), "w") as f:
        json.dump(gold, f)
        f.write("\n")
