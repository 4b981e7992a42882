"""A LogUp range check with Fq = Fq3: every value of column v lies in the table column t = 0, 1, ..., n - 1.

The argument is the logarithmic-derivative lookup (LogUp): with a verifier challenge alpha and the multiplicity m_i of
t_i among the values,
    sum_i m_i / (alpha - t_i)  =  sum_i 1 / (alpha - v_i)
holds (as rational functions of alpha) exactly when every v_i is a table entry.  The extension column s is the running
sum of the difference, declared in the AIR (AirConfig.extension_columns) and built by the prover on the device:

    base columns       0: v (values)   1: t (table)   2: m (multiplicity of t_i in v)
    extension column   3: s,  s_0 = 0,  s_(i+1) = s_i + m_i / (alpha - t_i) - 1 / (alpha - v_i)

Constraints: t_0 = 0 and t_(i+1) = t_i + 1; s_0 = 0; the transition with its denominators cleared,
(s_(i+1) - s_i)(alpha - t_i)(alpha - v_i) = m_i (alpha - v_i) - (alpha - t_i), on every row but the last; and at the last
row the whole sum is zero, s_(n-1)(alpha - t)(alpha - v) + m (alpha - v) - (alpha - t) = 0.  The declaration adds no
constraint of its own: these are what make a proof of this AIR a proof of the range check.
"""
import numpy as np

from .. import expr as E
from ..air import AirConfig, RunningColumn, domain_generator
from ..prover import Stark, Trace

P = E.P
_R = 2**64
V, T, M, S = 0, 1, 2, 3


class LookupAirConfig(AirConfig):
    NUM_BASE_COLUMNS = 3
    NUM_EXTENSION_COLUMNS = 1
    FQ_IS_FP = False

    @staticmethod
    def constraints(trace_len):
        g = domain_generator(trace_len.bit_length() - 1)
        x, tr = E.X(), E.Trace
        one = E.Constant(1)
        first, last = E.Constant(1), E.Constant(pow(g, trace_len - 1, P))
        alpha = E.Challenge(0)
        all_rows = x ** trace_len - one
        but_last = (x - last) / all_rows
        dt, dv = alpha - tr(T, 0), alpha - tr(V, 0)
        step = tr(M, 0) * dv - dt                        # (m / (alpha - t) - 1 / (alpha - v)) * dt * dv
        return [
            tr(T, 0) / (x - first),
            (tr(T, 1) - tr(T, 0) - one) * but_last,
            tr(S, 0) / (x - first),
            ((tr(S, 1) - tr(S, 0)) * dt * dv - step) * but_last,
            (tr(S, 0) * dt * dv + step) / (x - last),
        ]

    @staticmethod
    def extension_columns(trace_len):
        alpha = E.Challenge(0)
        return [RunningColumn(init=0, add=E.Trace(M, 0) / (alpha - E.Trace(T, 0)) - E.Constant(1) / (alpha - E.Trace(V, 0)))]


def gen_trace(n, seed=1):
    """n random values in [0, n), the table 0..n-1 and the multiplicities; base columns only (s is declared)"""
    v = np.random.default_rng(seed).integers(0, n, size=n, dtype=np.uint64)
    m = np.bincount(v.astype(np.int64), minlength=n).astype(np.uint64)
    # Montgomery form of a value below 2^32: x * (2^64 mod p) = x * (2^32 - 1), which stays below p
    base = np.stack([v, np.arange(n, dtype=np.uint64), m]) * np.uint64(_R % P)
    return Trace(base)


class LookupClaim(Stark):
    AirConfig = LookupAirConfig

    def get_public_inputs(self):
        return []
