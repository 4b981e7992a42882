"""Winternitz one-time signatures over Rescue-Prime and the trace of examples/wots's claim (SignaturesClaim), restated
with Python integers for the tests.  TEST INFRASTRUCTURE ONLY.

Independent of ministark_b200/examples/wots.py: it builds on the restated permutation of oracle/rescue_oracle.py.  A
chain step, the chain secret and the fold are one permutation each, told apart by capacity word 8 (1 + s, 16, 0) and
carrying (i, rho_0, rho_1) in words 9..11.  block_rows takes the step pattern and the tweaks as arguments, so that the
tests can build traces that break one rule at a time.  Values are canonical integers."""
from oracle import rescue_oracle as RO

P = RO.P
CHAINS, STEPS = 67, 15


def digits(m):
    d = [(m[w] >> 4 * t) & 15 for w in range(4) for t in range(16)]
    c = sum(15 - v for v in d)
    return d + [(c >> 4 * t) & 15 for t in range(3)]


def _h(x, tail, tweak, i, rho):
    return RO.permute(list(x) + list(tail) + [tweak, i] + list(rho))[:4]


def keygen(secret, rho):
    """(public key, the 67 chain secrets)"""
    sks = [_h(secret, [0] * 4, 16, i, rho) for i in range(CHAINS)]
    acc = [0] * 4
    for i, x in enumerate(sks):
        for s in range(STEPS):
            x = _h(x, [0] * 4, 1 + s, i, rho)
        acc = _h(x, acc, 0, i, rho)
    return list(rho) + acc, sks


def sign(secret, rho, m):
    _, sks = keygen(secret, rho)
    out = []
    for i, (x, d) in enumerate(zip(sks, digits(m))):
        for s in range(d):
            x = _h(x, [0] * 4, 1 + s, i, rho)
        out.append(x)
    return out


def block_rows(x, acts, cnts, i, rho, acc, last, tweaks=None, rhos=None):
    """(the 128 rows of one block, 15 canonical words each: S_0..S_11, ACT, CNT, LAST; the fold output).  Slot s < 15
    permutes (x || 0^4 || tweaks[s], i, rhos[s]) and moves x to its output where acts[s] = 1; slot 15 permutes
    (x || acc || 0, i, rhos[15]).  By default tweaks[s] = 1 + s and rhos[s] = rho."""
    tweaks = tweaks or [1 + s for s in range(STEPS)]
    rhos = rhos or [rho] * 16
    rows = []
    for s in range(16):
        state = list(x) + (list(acc) if s == STEPS else [0] * 4) + [tweaks[s] if s < STEPS else 0, i] + list(rhos[s])
        act, cnt = (acts[s], cnts[s]) if s < STEPS else (0, 0)
        states = RO.round_states(state)
        rows += [st + [act, cnt, last] for st in states]
        if s < STEPS and act:
            x = states[-1][:4]
    return rows, rows[-1][:4]


def wots_trace(public_keys, messages, signatures):
    """(rows, roots): the n = 128 B trace rows of K signatures and the root each signature's folds reach.  Padding
    blocks have digit 0, start value 0, i = rho = 0 and LAST = 1, so each folds onto 0^4 alone"""
    K = len(public_keys)
    B = 1
    while B < CHAINS * K:
        B *= 2
    rows, roots, acc = [], [], [0] * 4
    for b in range(B):
        k, i = divmod(b, CHAINS)
        if k < K:
            d, x, rho, last = digits(messages[k])[i], signatures[k][i], public_keys[k][:2], int(i == CHAINS - 1)
        else:
            d, x, i, rho, last = 0, [0] * 4, 0, [0, 0], 1
        acts = [int(s >= d) for s in range(STEPS)]
        cnts = [max(d - s, 0) for s in range(STEPS)]
        block, out = block_rows(x, acts, cnts, i, rho, acc, last)
        rows += block
        if last and k < K:
            roots.append(out)
        acc = [0] * 4 if last else out
    return rows, roots
