"""column generators shared by tests/test_gpu_ntt.py and tests/test_gpu_ntt_paths.py: random words seasoned with the
values that break lazy / modular arithmetic, and the structured columns a real execution trace has"""
import numpy as np

import ministark_b200 as ms


def edge_column(n, lanes, rng):
    """random words seasoned with the values that break lazy/modular arithmetic"""
    P = ms.P
    edge = np.array([0, 1, P - 1, P - 2, 2**32 - 1, 2**32, 2**32 + 1, 0xFFFFFFFF00000000, 2**63, P - 2**32], dtype=np.uint64)
    v = rng.integers(0, P, size=n * lanes, dtype=np.uint64)
    k = min(len(edge), v.size)
    v[rng.choice(v.size, size=k, replace=False)] = edge[:k]
    return v


def structured_columns(n, rng):
    """columns a real execution trace has: constants, 0/1 flags, counters, a handful of repeated values such as the
    Montgomery words of 1/2 = 2^63 and 1/4 = 2^62 (their pairwise sums hit 2^64 exactly), runs, alternations"""
    R, P = 2**64, ms.P
    mont = lambda v: np.array([int(x) * R % P for x in v], dtype=np.uint64)
    inv = [0] + [pow(v, -1, P) for v in range(1, 9)]
    cols = [
        np.zeros(n, dtype=np.uint64), np.full(n, ms.ONE, dtype=np.uint64), np.full(n, 2**63, dtype=np.uint64), np.full(n, P - 1, dtype=np.uint64),
        mont(np.arange(n) % 2), mont(np.arange(n)), mont([inv[int(k)] for k in rng.integers(0, 5, size=n)]),
        mont([inv[(i // 3) % 9] for i in range(n)]), np.where(np.arange(n) % 2 == 0, np.uint64(2**63), np.uint64(2**62)),
        np.where(np.arange(n) < n // 2, np.uint64(2**63), np.uint64(0)), mont([P - 1 - (i % 4) for i in range(n)]),
        np.where(rng.integers(0, 2, size=n) == 0, np.uint64(2**63), np.uint64(P - 2**63)),
    ]
    return np.stack(cols)
