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
from ..air import AirConfig, Lookup, RunningColumn, domain_generator
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


# ---- the same range check declared as one Lookup: the package writes the last three constraints, declares s and fills m
class DeclaredLookupAirConfig(AirConfig):
    """LookupAirConfig's range check with its lookup declared (air.Lookup): the AIR's own constraints are the two on t; the
    three LogUp constraints, the running sum s and the multiplicities m are the package's.  Its proofs are byte for byte
    those of LookupAirConfig."""
    NUM_BASE_COLUMNS = 3
    NUM_EXTENSION_COLUMNS = 1
    FQ_IS_FP = False

    @staticmethod
    def constraints(trace_len):
        return LookupAirConfig.constraints(trace_len)[:2]

    @staticmethod
    def lookups(trace_len):
        return [Lookup(table=(E.Trace(T, 0),), values=((E.Trace(V, 0),),), multiplicity=M, running_sum=S)]


class DeclaredLookupClaim(Stark):
    AirConfig = DeclaredLookupAirConfig

    def get_public_inputs(self):
        return []

    @staticmethod
    def gen_trace(n, seed=1, multiplicities=False):
        """gen_trace's columns with m left zero for the prover to fill (or, with multiplicities=True, counted on the host)"""
        trace = gen_trace(n, seed)
        if not multiplicities:
            trace.base_columns()[M] = 0
        return trace


# ---- a two-word table, two value tuples and a selector: (a, a^2) on every row and (b, b^2) where f is 1
TS, US, AS, BS, CS, DS, FS, MS, SS = range(9)


class SquareLookupAirConfig(AirConfig):
    """Squares by lookup: the table is (t, u) with t = 0, 1, ..., n - 1 and u = t^2 (constrained below); every row looks
    up (a, c), and (b, d) where the boolean column f is 1.  The lookup is the only constraint on a, b, c and d, so a proof
    shows c = a^2 and, where f = 1, d = b^2 with a, b < n.  Many rows look up the same table entry, so the multiplicities
    run well above 1.

        base columns       0: t  1: u  2: a  3: b  4: c  5: d  6: f  7: m (multiplicity, filled by the prover)
        extension column   8: s (the lookup's running sum, declared by the package)"""
    NUM_BASE_COLUMNS = 8
    NUM_EXTENSION_COLUMNS = 1
    FQ_IS_FP = False

    @staticmethod
    def constraints(trace_len):
        g = domain_generator(trace_len.bit_length() - 1)
        x, tr = E.X(), E.Trace
        one = E.Constant(1)
        last = E.Constant(pow(g, trace_len - 1, P))
        all_rows = x ** trace_len - one
        return [
            tr(TS, 0) / (x - one),
            (tr(TS, 1) - tr(TS, 0) - one) * ((x - last) / all_rows),
            (tr(US, 0) - tr(TS, 0) * tr(TS, 0)) / all_rows,
            tr(FS, 0) * (one - tr(FS, 0)) / all_rows,
        ]

    @staticmethod
    def lookups(trace_len):
        tr = E.Trace
        return [Lookup(table=(tr(TS, 0), tr(US, 0)), values=((tr(AS, 0), tr(CS, 0)), (tr(BS, 0), tr(DS, 0))),
                       multiplicity=MS, running_sum=SS, selectors=(E.Constant(1), tr(FS, 0)))]


def _square_columns(n, seed):
    """canonical columns t, u, a, b, c, d, f and m = 0 as int64 (n <= 2^31, so every value is below 2^62)"""
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.int64)
    a, b = rng.integers(0, n, size=n, dtype=np.int64), rng.integers(0, n, size=n, dtype=np.int64)
    f = rng.integers(0, 2, size=n, dtype=np.int64)
    d = np.where(f == 1, b * b, rng.integers(0, 1 << 62, size=n, dtype=np.int64))      # anything where f = 0
    return np.stack([t, t * t, a, b, a * a, d, f, np.zeros(n, dtype=np.int64)])


def _to_mont(x):
    """x * 2^64 mod p for canonical uint64 words below 2^62: with x = h 2^32 + l and 2^64 = 2^32 - 1 (mod p), that is
    l 2^32 - h - l"""
    h, l = x >> np.uint64(32), x & np.uint64(0xFFFFFFFF)
    v, s = l << np.uint64(32), h + l
    return np.where(v >= s, v - s, v + (np.uint64(P) - s))


class SquareLookupClaim(Stark):
    AirConfig = SquareLookupAirConfig

    def get_public_inputs(self):
        return []

    @staticmethod
    def gen_trace(n, seed=1, device=None):
        """random a, b < n, f and the values the lookup needs, m left zero.  device: the columns are built on that CUDA
        device (torch, then ms_pointwise_const into Montgomery form) and handed over as a device tensor; no host trace."""
        assert n & (n - 1) == 0 and n <= 1 << 31
        if device is None:
            return Trace(_to_mont(_square_columns(n, seed).astype(np.uint64)))
        import torch
        from .. import FP, Context
        device = torch.device(device)
        g = torch.Generator(device=device).manual_seed(seed)
        t = torch.arange(n, dtype=torch.int64, device=device)
        a = torch.randint(0, n, (n,), generator=g, dtype=torch.int64, device=device)
        b = torch.randint(0, n, (n,), generator=g, dtype=torch.int64, device=device)
        f = torch.randint(0, 2, (n,), generator=g, dtype=torch.int64, device=device)
        junk = torch.randint(0, 1 << 62, (n,), generator=g, dtype=torch.int64, device=device)
        cols = torch.stack([t, t * t, a, b, a * a, torch.where(f == 1, b * b, junk), f, torch.zeros_like(t)]).contiguous()
        # canonical -> Montgomery: the Montgomery product with 2^128 mod p is x * 2^64 mod p
        ctx = Context(device.index or 0, stream=torch.cuda.current_stream(device).cuda_stream)
        ctx.pointwise_const("mul", cols, FP, cols, FP, [pow(_R, 2, P)], FP, cols.numel())
        torch.cuda.current_stream(device).synchronize()     # the prover reads the tensor on its own stream
        return Trace(cols)
