"""permutation_oracle.py — CPU oracle for the target columns of sorted-copy permutations declared by an AIR.  TEST
INFRASTRUCTURE ONLY.

A permutation (ministark_b200/air.py, Permutation) is restated here from its definition, independently of the product's
compiler and kernels: every source word is evaluated as a whole column by eval_oracle.evaluate on the trace domain
(offset 1, so X = g_n^i and Trace(c, off) = column[(i + off) mod n]) and turned into canonical integers; the rows' tuples
are ordered by Python's stable `sorted`, and target column k holds word k of the sorted tuples.

Expressions are in the tuple exchange format of eval_oracle; Expr objects and field values are accepted too.
"""
import numpy as np

from . import pyspec as S
from .lookup_oracle import _column


def targets(source, base_cols):
    """source: W expressions; base_cols: (nbase, n) Montgomery words.  Returns the (W, n) Montgomery words of the target
    columns."""
    base_cols = np.ascontiguousarray(base_cols, dtype=np.uint64)
    n = base_cols.shape[1]
    cols = [_column(e, n.bit_length() - 1, base_cols) for e in source]
    rows = sorted(zip(*cols))
    return np.array([[S.to_mont(t[k]) for t in rows] for k in range(len(source))], dtype=np.uint64).reshape(len(source), n)


def fill(config, base_cols):
    """a copy of base_cols with every permutation's target columns filled, in declaration order"""
    base = np.array(base_cols, dtype=np.uint64, copy=True)
    for pm in config.permutations(base.shape[1]):
        base[list(pm.target)] = targets(pm.source, base)
    return base
