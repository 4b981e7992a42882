"""The trace of examples/rollup's transfer claim (TransfersClaim), restated with Python integers for the tests.
TEST INFRASTRUCTURE ONLY.

Independent of ministark_b200/examples/rollup.py: it builds on tests/rescue_merkle_updates_oracle.py.  The transfers are
applied one after another to the accounts, each as its sender write and then its receiver write; the restated updates
trace of those 2 K writes gives columns 0..14, and the balance, lookup and table columns follow from the writes.
Values are canonical integers."""
import rescue_merkle_updates_oracle as UO

P = 2**64 - 2**32 + 1


class InvalidTransfer(ValueError):
    """the first write whose new balance is not below 2^32: transfer k, side 'sender' or 'receiver', the account, the
    balance"""
    def __init__(self, k, side, account, balance):
        super().__init__(f"the {side} step of transfer {k} leaves account {account} with balance {balance}, not below 2^32")
        self.k, self.side, self.account, self.balance = k, side, account, balance


def rollup_trace(nodes, depth, transfers):
    """(rows, roots, heap): the n = 32 K L trace rows (S_0..S_11, BIT, IDX, SIDE, DELTA, NINC, B0..B3, M = 0, TBL), the
    K + 1 roots (before the first transfer and after each) and the heap after every transfer ([None, node 1, ...]).
    Raises InvalidTransfer for the first write that leaves a balance outside [0, 2^32)."""
    leaf_of = {}
    idx, new, extra = [], [], []
    for k, (s, r, a) in enumerate(transfers):
        for side, acc, delta, ninc in (("sender", s, -a % P, 1), ("receiver", r, a, 0)):
            bal, nonce, o0, o1 = leaf_of.get(acc, nodes[(1 << depth) + acc])
            bal = (bal + delta) % P
            if bal >= 2**32:
                raise InvalidTransfer(k, side, acc, bal)
            leaf_of[acc] = [bal, (nonce + ninc) % P, o0, o1]
            idx.append(acc)
            new.append(list(leaf_of[acc]))
            extra.append([delta, ninc] + [bal >> 8 * q & 255 for q in range(4)])
    rows, roots, heap = UO.updates_trace(nodes, depth, idx, new)
    per_write = len(rows) // len(idx)                  # 16 L
    rows = [r + (extra[i // per_write] if i % per_write == 0 else [0] * 6) + [0, min(i, 255)]
            for i, r in enumerate(rows)]
    return rows, roots[::2], heap
