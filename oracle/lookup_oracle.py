"""lookup_oracle.py — CPU oracle for the multiplicity columns of LogUp lookups declared by an AIR.  TEST INFRASTRUCTURE ONLY.

A lookup (ministark_b200/air.py, Lookup) is restated here from its definition, independently of the product's compiler
and kernels: every table word, value word and selector is evaluated as a whole column by eval_oracle.evaluate on the trace
domain (offset 1, so X = g_n^i and Trace(c, off) = column[(i + off) mod n]) and turned into canonical integers; the table
becomes a Python dict from tuple to its lowest row; then every (row, value tuple) with selector 1 adds 1 at that row, or
counts as missing, and a selector other than 0 or 1 counts as bad.

Expressions are in the tuple exchange format of eval_oracle; Expr objects and field values are accepted too.
"""
import numpy as np

from . import eval_oracle
from . import oracle as orc
from . import pyspec as S
from .extension_oracle import _tuple

_RINV = pow(2**64, -1, S.P)


def _column(e, log_n, base_cols):
    words = eval_oracle.evaluate(_tuple(e), log_n, orc.ONE, base_cols, fq_lanes=1)
    return [int(w) * _RINV % S.P for w in np.asarray(words, dtype=np.uint64)[:1 << log_n]]


def multiplicities(table, values, selectors, base_cols):
    """table: W expressions; values: Q tuples of W expressions; selectors: None or Q expressions; base_cols: (nbase, n)
    Montgomery words.  Returns (m, missing, bad): m the n Montgomery words of the multiplicity column, missing[q] =
    (count, lowest row or None) of the rows whose tuple q is not in the table, bad = (count, lowest row or None) of the
    (row, tuple) pairs whose selector is neither 0 nor 1."""
    base_cols = np.ascontiguousarray(base_cols, dtype=np.uint64)
    n = base_cols.shape[1]
    log_n = n.bit_length() - 1
    tcols = [_column(e, log_n, base_cols) for e in table]
    first = {}
    for j in range(n):
        first.setdefault(tuple(c[j] for c in tcols), j)
    counts = [0] * n
    missing, bad_rows = [], []
    for q, v in enumerate(values):
        vcols = [_column(e, log_n, base_cols) for e in v]
        sel = [1] * n if selectors is None else _column(selectors[q], log_n, base_cols)
        miss = []
        for i in range(n):
            if sel[i] == 0:
                continue
            if sel[i] != 1:
                bad_rows.append(i)
                continue
            j = first.get(tuple(c[i] for c in vcols))
            if j is None:
                miss.append(i)
            else:
                counts[j] += 1
        missing.append((len(miss), min(miss) if miss else None))
    m = np.array([S.to_mont(c) for c in counts], dtype=np.uint64)
    return m, missing, (len(bad_rows), min(bad_rows) if bad_rows else None)


def fill(config, base_cols):
    """a copy of base_cols with every multiplicity column of config's lookups filled, in declaration order"""
    base = np.array(base_cols, dtype=np.uint64, copy=True)
    n = base.shape[1]
    for lk in config.lookups(n):
        m, missing, bad = multiplicities(lk.table, lk.values, lk.selectors, base)
        assert not any(c for c, _ in missing) and not bad[0], (missing, bad)
        base[lk.multiplicity] = m
    return base
