"""check_oracle.py — CPU oracle for the constraint check.  TEST INFRASTRUCTURE ONLY.

Restates Constraint::check (src/constraints.rs:168-249) and the loop of the reference's unfinished
default_validate_constraints (src/debug.rs:10-128, left there as a comment) as a memoised tree walk over
Expr.to_tuple() forms (the exchange format of eval_oracle.py), vectorised over the rows of the trace domain with the C
oracle's pointwise field ops and a numpy None mask per node:
    neg, pow       None stays None
    add            None if either operand is None
    mul            Some * Some; Some(x) * None and None * Some(x): Some(0) if x = 0, else None; None * None: None
    div            Some(a) / Some(b): 0/0 = Some(0), a/0 = None, else a / b;
                   Some(x) / None and None / Some(x): Some(0) if x = 0, else None; None / None: None
A constraint holds at a row when its value is Some.  Leaves: x = g_n^row (the trace domain, no offset),
Trace(col, off) = column[(row + off) rem_euclid n], challenges and hints as given, periodic columns evaluated at
y = x^(n / interval_size).  It is independent of expr.compile_check_program and of csrc/check.cu.
"""
import numpy as np

from . import eval_oracle as EO
from . import oracle as orc
from . import pyspec as S


def _lift(v):
    return (v, 0, 0) if isinstance(v, int) else tuple(v)


def _mont(v, lanes):
    return np.array([S.to_mont(int(c)) for c in _lift(v)[:lanes]], dtype=np.uint64)


def _zero(arr, lanes):
    return ~arr.reshape(-1, lanes).any(axis=1)


def check(constraints, log_n, base_cols, ext_cols=None, fq_lanes=1, challenges=(), hints=()):
    """constraints: Expr.to_tuple() forms; base_cols (nbase, n) and ext_cols (next, n * fq_lanes): natural-order
    Montgomery words.  Returns [(first_row or None, count)] per constraint."""
    n = 1 << log_n
    nbase = 0 if base_cols is None else base_cols.shape[0]
    xs = EO.x_lde(log_n, orc.ONE)
    memo = {}
    some = np.zeros(n, dtype=bool)

    def full(v, lanes):
        return orc.pointwise_const("fill", None, 1, _mont(v, lanes), lanes, n=n, dfield=lanes)

    def walk(e):
        if id(e) in memo:
            return memo[id(e)]
        k = e[0]
        if k == "x":
            r = (xs, 1, some)
        elif k == "const":
            lanes = fq_lanes if e[2] else 1
            r = (full(e[1], lanes), lanes, some)
        elif k in ("chal", "hint"):
            r = (full((challenges if k == "chal" else hints)[e[1]], fq_lanes), fq_lanes, some)
        elif k == "trace":
            col, off = e[1], e[2]
            src, lanes = (base_cols[col], 1) if col < nbase else (ext_cols[col - nbase], fq_lanes)
            r = (np.roll(src.reshape(n, lanes), -(off % n), axis=0).reshape(-1).copy(), lanes, some)
        elif k == "periodic":
            coeffs, interval = e[1], e[2]
            lanes = fq_lanes if any(isinstance(c, tuple) for c in coeffs) else 1
            g = S.root_of_unity(log_n)
            vals = []
            for i in range(interval):
                y = pow(g, i * (n // interval), S.P)
                acc = [0, 0, 0]
                for c in reversed([_lift(c) for c in coeffs]):
                    acc = [(acc[w] * y + c[w]) % S.P for w in range(3)]
                vals.append([S.to_mont(acc[w]) for w in range(lanes)])
            tab = np.array(vals, dtype=np.uint64).reshape(interval, lanes)
            r = (np.tile(tab, (n // interval, 1)).reshape(-1).copy(), lanes, some)
        elif k == "neg":
            a = walk(e[1])
            r = (orc.pointwise("neg", a[0], a[1]), a[1], a[2])
        elif k == "pow":
            a = walk(e[1])
            r = (orc.pointwise("exp", a[0], a[1], exponent=e[2]), a[1], a[2])
        elif k == "add":
            a, b = walk(e[1]), walk(e[2])
            lanes = max(a[1], b[1])
            r = (orc.pointwise("add", a[0], a[1], b[0], b[1], dfield=lanes), lanes, a[2] | b[2])
        elif k in ("mul", "div"):
            a, b = walk(e[1]), walk(e[2])
            lanes = max(a[1], b[1])
            rhs, rl = (b[0], b[1]) if k == "mul" else (orc.pointwise("inv", b[0], b[1]), b[1])
            val = orc.pointwise("mul", a[0], a[1], rhs, rl, dfield=lanes)
            za, zb, na, nb = _zero(a[0], a[1]), _zero(b[0], b[1]), a[2], b[2]
            one_none = na ^ nb
            none = (na & nb) | (one_none & ~np.where(na, zb, za))
            if k == "div":
                none |= ~na & ~nb & zb & ~za                    # a / 0
            val.reshape(n, lanes)[one_none & ~none] = 0         # Some(0) from a zero times / over None
            r = (val, lanes, none)
        else:
            raise ValueError(k)
        memo[id(e)] = r
        return r

    out = []
    for c in constraints:
        none = walk(c)[2]
        cnt = int(none.sum())
        out.append((int(np.argmax(none)) if cnt else None, cnt))
    return out


def leaf_values(constraint, row, log_n, base_cols, ext_cols=None, fq_lanes=1, challenges=(), hints=()):
    """what the reference's comment prints for a failing row: "x", every Trace(col, offset), Challenge(i) and Hint(i)
    leaf of the constraint with its value (canonical integers; 3-tuples for Fq3), sorted by label, deduplicated"""
    n = 1 << log_n
    nbase = 0 if base_cols is None else base_cols.shape[0]

    def canon(words):
        v = tuple(S.from_mont(int(w)) for w in words)
        return v[0] if len(v) == 1 else v

    def field_value(v):
        return _lift(v) if fq_lanes == 3 else _lift(v)[0]

    vals = {"x": pow(S.root_of_unity(log_n), row, S.P)}
    stack, seen = [constraint], set()
    while stack:
        e = stack.pop()
        if id(e) in seen:
            continue
        seen.add(id(e))
        if e[0] == "trace":
            col, off = e[1], e[2]
            pos = (row + off) % n
            if col < nbase:
                vals[f"Trace(col={col:0>3}, offset={off:0>3})"] = canon(base_cols[col][pos:pos + 1])
            else:
                vals[f"Trace(col={col:0>3}, offset={off:0>3})"] = canon(ext_cols[col - nbase][pos * fq_lanes:(pos + 1) * fq_lanes])
        elif e[0] == "chal":
            vals[f"Challenge({e[1]})"] = field_value(challenges[e[1]])
        elif e[0] == "hint":
            vals[f"Hint({e[1]})"] = field_value(hints[e[1]])
        else:
            stack.extend(a for a in e[1:] if isinstance(a, tuple) and a and isinstance(a[0], str))
    return sorted(vals.items())
