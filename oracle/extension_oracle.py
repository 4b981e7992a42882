"""extension_oracle.py — CPU oracle for extension columns declared by an AIR.  TEST INFRASTRUCTURE ONLY.

A declared column (ministark_b200/air.py, RunningColumn) is the recurrence  x_0 = init, x_(i+1) = x_i * mul(i) + add(i)
over the trace domain; row i holds x_i, or x_(i+1) when inclusive.  Restated here from that definition, independently of
the product's compiler and kernels: mul and add are evaluated as whole columns by eval_oracle.evaluate on the trace domain
(offset 1, so X = g_n^i and Trace(c, off) = column[(i + off) mod n]; a zero denominator inverts to 0, as the C oracle's
inversion does), init likewise on a one-point domain, and the recurrence runs in the C oracle's serial scan.

Expressions are in the tuple exchange format of eval_oracle; field values (ints, or 3-tuples for Fq3) are accepted too.
"""
import numpy as np

from . import eval_oracle
from . import oracle as orc
from . import pyspec as S


def _tuple(v):
    if hasattr(v, "to_tuple"):
        return v.to_tuple()
    if isinstance(v, tuple) and v and isinstance(v[0], str):
        return v
    if isinstance(v, (tuple, list)):
        return ('const', tuple(int(c) % S.P for c in v), True)
    return ('const', (int(v) % S.P, 0, 0), False)


def columns(decl, base_cols, lanes, challenges=(), hints=()):
    """decl: [(init, mul, add, inclusive)]; base_cols: (nbase, n) Montgomery words.  Returns (K, n * lanes) Montgomery
    words."""
    base_cols = np.ascontiguousarray(base_cols, dtype=np.uint64)
    n = base_cols.shape[1]
    log_n = n.bit_length() - 1
    out = []
    for init, mul, add, inclusive in decl:
        x0 = eval_oracle.evaluate(_tuple(init), 0, orc.ONE, None, fq_lanes=lanes, challenges=challenges, hints=hints)
        init3 = np.zeros(3, dtype=np.uint64)
        init3[:lanes] = x0[:lanes]
        a = eval_oracle.evaluate(_tuple(mul), log_n, orc.ONE, base_cols, fq_lanes=lanes, challenges=challenges, hints=hints)
        b = eval_oracle.evaluate(_tuple(add), log_n, orc.ONE, base_cols, fq_lanes=lanes, challenges=challenges, hints=hints)
        out.append(orc.scan_affine(lanes, n, init3, a=a, fa=lanes, b=b, fb=lanes, inclusive=inclusive))
    return np.stack(out)


def builder(config, base_cols, public_inputs=None):
    """the ext_builder stark_oracle.cpu_prove takes for an AIR that declares its extension columns: challenges -> the
    columns, with the hints gen_hints makes from them"""
    n = np.asarray(base_cols).shape[1]
    lanes = 1 if config.FQ_IS_FP else 3

    def build(challenges):
        hints = config.gen_hints(n, public_inputs, challenges)
        decl = [(c.init, c.mul, c.add, c.inclusive) for c in config.extension_columns(n)]
        return columns(decl, base_cols, lanes, challenges, hints)

    return build
