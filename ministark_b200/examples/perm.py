"""A permutation-argument AIR with Fq = Fq3: base-field data columns, two extension-field running products
built from a verifier challenge, and one degree-4 constraint that forces ce_blowup = 4.

The shape is the reference's `evaluate_permutation_constraint` (tests/constraint.rs:220-284: original / shuffled
columns, running products  p_(i+1) = p_i * (alpha - v_i)) promoted to a full AIR the way examples/brainfuck uses
it (extension columns in Fq3 built after the base-trace commitment, src/prover.rs:56-72).  It exists to drive the
prover through every Fq3 path: extension-trace LDE + commitment, mixed Fp/Fq3 constraint evaluation, a 4-column
Fq3 composition trace, Fq3 DEEP and Fq3 FRI.

    base columns       0: a      1: b = a shuffled      2: c = a^4
    extension columns  3: op (running product over a)   4: sp (running product over b)

PermAirConfig leaves the extension columns to the trace's host callback (gen_trace); PermDeclaredAirConfig has the same
constraints and declares the two running products instead (AirConfig.extension_columns), so that the prover builds them
on the device from a base-only trace (gen_trace(..., extension=False)).
"""
import random

import numpy as np

from .. import expr as E
from ..air import AirConfig, RunningColumn, domain_generator
from ..prover import Stark, Trace

P = E.P
_R = 2**64


class PermAirConfig(AirConfig):
    NUM_BASE_COLUMNS = 3
    NUM_EXTENSION_COLUMNS = 2
    FQ_IS_FP = False

    @staticmethod
    def constraints(trace_len):
        g = domain_generator(trace_len.bit_length() - 1)
        x, T = E.X(), E.Trace
        one = E.Constant(1)
        first, last = E.Constant(1), E.Constant(pow(g, trace_len - 1, P))
        alpha = E.Challenge(0)
        a, b, c, op, sp = 0, 1, 2, 3, 4
        all_rows = x ** trace_len - one
        but_last = (x - last) / all_rows
        return [
            (T(op, 0) - one) / (x - first),
            (T(sp, 0) - one) / (x - first),
            (T(op, 0) * (alpha - T(a, 0)) - T(op, 1)) * but_last,
            (T(sp, 0) * (alpha - T(b, 0)) - T(sp, 1)) * but_last,
            (T(op, 0) * (alpha - T(a, 0)) - T(sp, 0) * (alpha - T(b, 0))) / (x - last),
            (T(c, 0) - T(a, 0) ** 4) / all_rows,
        ]


class PermDeclaredAirConfig(PermAirConfig):
    """PermAirConfig with its extension columns declared: op_0 = sp_0 = 1, op_(i+1) = op_i * (alpha - a_i),
    sp_(i+1) = sp_i * (alpha - b_i) — what gen_trace's callback computes, row by row on the host"""

    @staticmethod
    def extension_columns(trace_len):
        alpha, a, b = E.Challenge(0), E.Trace(0, 0), E.Trace(1, 0)
        return [RunningColumn(init=1, mul=alpha - a), RunningColumn(init=1, mul=alpha - b)]


def gen_trace(n, seed=1, extension=True):
    """the perm trace of n rows; extension=False: base columns only (for PermDeclaredAirConfig)"""
    rng = random.Random(seed)
    a = [rng.randrange(P) for _ in range(n)]
    b = list(a)
    rng.shuffle(b)
    c = [pow(v, 4, P) for v in a]
    base = np.array([[v * _R % P for v in col] for col in (a, b, c)], dtype=np.uint64)

    def build_extension(challenges):
        alpha = tuple(challenges[0])
        cols = []
        for src in (a, b):
            acc, out = (1, 0, 0), []
            for v in src:
                out.extend(acc)
                acc = E.q_mul(acc, ((alpha[0] - v) % P, alpha[1], alpha[2]))
            cols.append([w * _R % P for w in out])
        return np.array(cols, dtype=np.uint64)

    return Trace(base, build_extension if extension else None)


class PermClaim(Stark):
    AirConfig = PermAirConfig

    def get_public_inputs(self):
        return []


class PermDeclaredClaim(PermClaim):
    AirConfig = PermDeclaredAirConfig
