"""helpers shared by tests/test_expr_compiler.py and tests/test_cpp_host.py: a big-integer interpreter of the evaluator's
instruction set (csrc/eval.cu) and a direct recursive evaluation of an expression DAG; and the edge-operand programs shared
by tests/test_gpu_eval_edges.py and tests/test_eval_jit_source.py"""
import random
import sys

import numpy as np

from ministark_b200 import expr as E
from oracle import pyspec as S

P = E.P
R = 2**64
RINV = pow(R, -1, P)


def run_program(prog, x, cols, col_is_q, row, m):
    """big-int interpreter of the 4-word instructions; returns the stored Fq element (3-tuple of canonical ints)"""
    regs = {}
    out = None
    for op_w, d, a, b in prog.code.tolist():
        op, qa, qb = op_w & 0xFF, (op_w >> 8) & 1, (op_w >> 9) & 1
        if op == E.OP_X:
            regs[d] = (x, 0, 0)
        elif op == E.OP_CONST:
            regs[d] = tuple(int(w) * RINV % P for w in prog.consts[a])
        elif op == E.OP_TRACE:
            v = cols[a][(row + b) % m]
            assert bool(qa) == bool(col_is_q[a])
            regs[d] = tuple(v) if qa else (v, 0, 0)
        elif op == E.OP_NEG:
            regs[d] = E.q_neg(regs[a])
        elif op == E.OP_ADD:
            regs[d] = E.q_add(regs[a], regs[b])
        elif op == E.OP_SUB:
            regs[d] = E.q_add(regs[a], E.q_neg(regs[b]))
        elif op == E.OP_PERIODIC:
            v = cols[a][row % (1 << b)]          # the table rides in the column list after the trace columns
            regs[d] = tuple(v) if qa else (v, 0, 0)
        elif op == E.OP_MUL:
            regs[d] = E.q_mul(regs[a], regs[b])
        elif op == E.OP_INV:
            regs[d] = E.q_inv(regs[a]) if any(regs[a]) else (0, 0, 0)
        elif op == E.OP_POW:
            regs[d] = E.q_pow(regs[a], b)
        elif op == E.OP_STORE:
            out = regs[a]
        else:
            raise AssertionError(op)
        assert d < E.MAX_REGS
    return out


def periodic_value(coeffs, interval, x, n):
    """P(x^(n / interval)) by Horner, the verifier's formula (src/verifier.rs:221-230)"""
    y = pow(x, n // interval, P)
    acc = (0, 0, 0)
    for c in reversed(coeffs):
        c = c if isinstance(c, tuple) else (c, 0, 0)
        acc = E.q_add(E.q_mul(acc, (y, 0, 0)), c)
    return acc


def direct(expr, x, cols, row, m, challenges=(), hints=(), ccoefs=(), lde_step=1):
    memo = {}

    def ev(e):
        if id(e) in memo:
            return memo[id(e)]
        k, a = e.kind, e.args
        if k == "x":
            v = (x, 0, 0)
        elif k == "const":
            v = tuple(a[0])
        elif k == "chal":
            v = E._q(challenges[a[0]])
        elif k == "hint":
            v = E._q(hints[a[0]])
        elif k == "ccoef":
            v = E._q(ccoefs[a[0]])
        elif k == "trace":
            t = cols[a[0]][(row + lde_step * a[1]) % m]
            v = tuple(t) if isinstance(t, tuple) else (t, 0, 0)
        elif k == "periodic":
            v = periodic_value(a[0], a[1], x, m // lde_step)
        elif k == "neg":
            v = E.q_neg(ev(a[0]))
        elif k == "add":
            v = E.q_add(ev(a[0]), ev(a[1]))
        elif k == "mul":
            v = E.q_mul(ev(a[0]), ev(a[1]))
        elif k == "div":
            den = ev(a[1])
            v = E.q_mul(ev(a[0]), E.q_inv(den) if any(den) else (0, 0, 0))
        elif k == "pow":
            v = E.q_pow(ev(a[0]), a[1])
        else:
            raise AssertionError(k)
        memo[id(e)] = v
        return v

    import sys
    sys.setrecursionlimit(20000)
    return ev(expr)


def random_columns(rng, nbase, next_, m):
    cols = [[rng.randrange(P) for _ in range(m)] for _ in range(nbase)]
    cols += [[tuple(rng.randrange(P) for _ in range(3)) for _ in range(m)] for _ in range(next_)]
    return cols, [False] * nbase + [True] * next_


# ---- every opcode of the evaluator on edge operands (tests/test_gpu_eval_edges.py on the device, tests/test_eval_jit_source.py
# for the host branches of the specialised kernel's source).  Values are Montgomery words; the reference is pyspec's
# big-integer arithmetic on the canonical values, independent of field.cuh and of the C oracle.
EPS = 2**32 - 1                      # 2^64 mod p: the Montgomery word of 1
EDGE_LOG_M = 11
POW_EXPONENTS = (0, 1, 2, 3, 7, 2**16 + 1, 2**32 - 1)


def edge_words(rng):
    """Fp operands where the carry chains of add / sub / neg and of the Montgomery reduction turn over"""
    words = [0, 1, 2, EPS, P - 1, P - 2, EPS - 1, EPS + 1, 2**32 + 1, 2**62, 2**63 - 1, 2**63, 2**63 + 1, P - 2**32,
             0xFFFFFFFE_FFFFFFFF, 2 * R % P, (P - 1) * R % P, pow(2, -1, P) * R % P]     # the last three: 2, -1, 1/2 (= 2^63)
    words = list(dict.fromkeys(words))
    words += [rng.randrange(P) for _ in range(24 - len(words))]
    return words


def edge_fq3(rng):
    """Fq3 operands: zero, one, two and three non-zero components drawn from the Fp edge words, and random elements"""
    pool = [(0, 0, 0)]
    for k in range(3):
        pool += [tuple(w if j == k else 0 for j in range(3)) for w in (1, EPS, P - 1, 2**63)]
    for k in range(3):
        for u, v in ((EPS, P - 1), (2**63, 2**32), (P - 2, 0xFFFFFFFE_FFFFFFFF)):
            it = iter((u, v))
            pool.append(tuple(0 if j == k else next(it) for j in range(3)))
    pool += [(P - 1, P - 1, P - 1), (EPS, EPS, EPS), (2**63, 2**63, 2**63), (1, P - 1, 2**32), (P - EPS, 2, 2**63 + 1),
             (2**62, P - 2**32, EPS - 1)]
    pool += [tuple(rng.randrange(P) for _ in range(3)) for _ in range(40 - len(pool))]
    return pool


def edge_columns(fq, seed=5):
    """(columns, col_is_q): columns are lists of 2^EDGE_LOG_M Montgomery 3-tuples.  Columns 2k, 2k + 1 (k = 2 ta + tb) hold
    every pair of the operand pools of types ta, tb (0: Fp, 1: Fq) in their first points and random elements after;
    columns 8 + t cycle through the pool of type t, columns 10 + t through its non-zero elements.  With fq == 1 (Fq = Fp)
    the Fq pool is the Fp pool."""
    rng = random.Random(seed)
    m = 1 << EDGE_LOG_M
    fp = [(w, 0, 0) for w in edge_words(rng)]
    pools = [fp, edge_fq3(rng) if fq == 3 else fp]
    rand = [lambda: (rng.randrange(P), 0, 0), lambda: tuple(rng.randrange(P) for _ in range(3)) if fq == 3 else (rng.randrange(P), 0, 0)]
    cols, isq = [], []
    for ta in (0, 1):
        for tb in (0, 1):
            pa, pb = pools[ta], pools[tb]
            n = len(pa) * len(pb)
            assert n <= m
            cols.append([pa[i // len(pb)] for i in range(n)] + [rand[ta]() for _ in range(m - n)])
            cols.append([pb[i % len(pb)] for i in range(n)] + [rand[tb]() for _ in range(m - n)])
            isq += [ta, tb]
    for t in (0, 1):
        cols.append([pools[t][i % len(pools[t])] for i in range(m)])
        isq.append(t)
    for t in (0, 1):
        nz = [v for v in pools[t] if any(v)]
        cols.append([nz[i % len(nz)] for i in range(m)])
        isq.append(t)
    return cols, isq


def _fast_pow(a, e):
    return (pow(a[0], e, P), 0, 0) if not a[1] and not a[2] else S.fq3_pow(a, e)


def _fast_inv(a):
    return (pow(a[0], P - 2, P), 0, 0) if not a[1] and not a[2] else S.fq3_inv(a)


def edge_programs():
    """[(name, Program, operand columns, reference)]: raw programs, so that every operand-field combination is emitted
    whether or not compile_program would emit it.  reference(a, b) maps canonical 3-tuples to the canonical result."""
    fname = ("Fp", "Fq")
    out = []

    def prog(name, body, ncols_used, res_q, ref):
        code = body + [[E.OP_STORE | (res_q << 8), 0, 2 if len(body) > 1 else 0, 0]]
        out.append((name, E.Program(np.array(code, dtype=np.uint32), np.zeros((1, 3), dtype=np.uint64), 3, bool(res_q)), ncols_used, ref))

    binary = ((E.OP_ADD, "ADD", S.fq3_add), (E.OP_SUB, "SUB", S.fq3_sub), (E.OP_MUL, "MUL", S.fq3_mul))
    for op, opname, ref in binary:
        for ta in (0, 1):
            for tb in (0, 1):
                k = 2 * ta + tb
                body = [[E.OP_TRACE | (ta << 8), 0, 2 * k, 0], [E.OP_TRACE | (tb << 8), 1, 2 * k + 1, 0],
                        [op | (ta << 8) | (tb << 9), 2, 0, 1]]
                prog(f"{opname}({fname[ta]},{fname[tb]})", body, (2 * k, 2 * k + 1), ta | tb, lambda a, b, f=ref: f(a, b))
    for t in (0, 1):
        load = [E.OP_TRACE | (t << 8), 0, 8 + t, 0]
        prog(f"NEG({fname[t]})", [load, [E.OP_NEG | (t << 8), 2, 0, 0]], (8 + t,), t, lambda a, b: S.fq3_sub((0, 0, 0), a))
        for e in POW_EXPONENTS:
            prog(f"POW({fname[t]}, {e})", [load, [E.OP_POW | (t << 8), 2, 0, e]], (8 + t,), t, lambda a, b, e=e: _fast_pow(a, e))
        prog(f"INV({fname[t]})", [[E.OP_TRACE | (t << 8), 0, 10 + t, 0], [E.OP_INV | (t << 8), 2, 0, 0]], (10 + t,), t,
             lambda a, b: _fast_inv(a))
    prog("STORE(Fp)", [[E.OP_TRACE, 0, 8, 0]], (8,), 0, lambda a, b: a)
    return out


def edge_reference(cols, used, ref, fq):
    """the program's output words (M x fq Montgomery words, natural order) and a describer of the operands at a point"""
    m = len(cols[0])
    words = []
    for i in range(m):
        ops = [tuple(w * RINV % P for w in cols[c][i]) for c in used] + [None]
        words += [w * R % P for w in ref(ops[0], ops[1])[:fq]]

    def operands(i):
        return ", ".join("(" + ", ".join(f"{w:#x}" for w in cols[c][i][:fq]) + ")" for c in used)
    return np.array(words, dtype=np.uint64), operands


def column_words(col, is_q, fq):
    """a column of Montgomery 3-tuples as the evaluator reads it: one word per point, or fq words for an Fq column"""
    lanes = fq if is_q else 1
    return np.array([v[w] for v in col for w in range(lanes)], dtype=np.uint64)


