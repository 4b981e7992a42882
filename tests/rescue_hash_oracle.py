"""The Rescue-Prime sponge over Goldilocks and the trace of examples/rescue's hash claim, restated with Python integers
for the tests.  TEST INFRASTRUCTURE ONLY.

Independent of ministark_b200/examples/rescue.py: it builds on the restated permutation of oracle/rescue_oracle.py and
follows the reference's Rescue::finish (examples/rescue/rescue.rs:49-97) with rate 8, capacity 4 and 4 digest words.
Values are canonical integers."""
from oracle import rescue_oracle as RO

P = RO.P
RATE, DIGEST = 8, 4


def pad(words):
    """the message, then one 1, then zeros up to a multiple of the rate"""
    out = list(words) + [1]
    while len(out) % RATE:
        out.append(0)
    return out


def sponge_hash(words):
    """four canonical words: absorb the padded message block by block into the zero state, squeeze the first four"""
    assert all(0 <= w < P for w in words)
    state = [0] * RO.M
    padded = pad(words)
    for b in range(len(padded) // RATE):
        for i in range(RATE):
            state[i] = (state[i] + padded[RATE * b + i]) % P
        state = RO.permute(state)
    return state[:DIGEST]


def hash_trace(messages):
    """(rows, digests): the n = 8 K L rows of 13 canonical words (the state S_0..S_11, then the absorbed word M) and the
    K four-word digests.  Message k holds rows [8 L k, 8 L (k + 1)); B is the number of padded blocks and L the smallest
    power of two >= B, permutations B..L-1 absorbing zero blocks.  Row 8 (L k + j) + r holds permutation j's state
    before round r (block j added) and its output at r = 7; M at row 8 (L k + j) + i is word i of block j."""
    length = len(messages[0])
    assert all(len(m) == length for m in messages)
    B = length // RATE + 1
    L = 1
    while L < B:
        L *= 2
    rows, digests = [], []
    for m in messages:
        blocks = pad(m) + [0] * (RATE * (L - B))
        state = [0] * RO.M
        for j in range(L):
            block = blocks[RATE * j:RATE * (j + 1)]
            state = [(s + b) % P for s, b in zip(state, block + [0] * (RO.M - RATE))]
            states = RO.round_states(state)
            rows += [st + [block[r]] for r, st in enumerate(states)]
            state = states[-1]
            if j == B - 1:
                digests.append(state[:DIGEST])
    return rows, digests
