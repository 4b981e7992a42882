"""A read/write memory log with Fq = Fq3: every read returns the value last written to its address, and the reads return
the public values, in order.

The log lists the accesses in execution order.  A sorted copy of the same accesses, ordered by (address, clock), is tied
to the log by a permutation argument; on the sorted table, consecutive rows of one address are consecutive accesses to
it, so "a read returns the last value written" becomes a constraint between neighbouring rows:

    base columns       0: clk  1: addr  2: val  3: w (1 write, 0 read)          the log, clk = 0, 1, ..., n - 1
                       4: s_addr  5: s_clk  6: s_val  7: s_w                   the log sorted by (addr, clk, val, w)
                       8: nl (1 on every row but the last)  9: m (multiplicities of the clock lookup)
    extension columns  10: e (running evaluation of the read values)  11: s (the lookup's running sum)
                       12: z (the permutation's running product)

With delta = s_addr' - s_addr:
  * the log: clk_0 = 0, clk' = clk + 1, w boolean;
  * the sorted table: s_addr_0 = 0, s_w_0 = 1, delta (delta - 1) = 0 (addresses are contiguous), delta (1 - s_w') = 0 (the
    first access to an address is a write), (1 - delta)(1 - s_w')(s_val' - s_val) = 0 (a read returns the last value);
  * nl is 1 on every row but the last, where it is 0;
  * clock order within an address: a lookup of (1 - delta)(s_clk' - s_clk - 1) into the table clk = 0..n-1, behind the
    selector nl (the wrap from the last row to the first is not a step);
  * the reads: e is the inclusive running evaluation e_(i+1) = e_i (1 + (1 - w_i)(gamma - 1)) + (1 - w_i) val_i over the
    log, so its last row is the Horner evaluation at gamma of the read values, which must equal Hint(0), computed by
    gen_hints from the public values;
  * the permutation: z_0 = 1, z_(i+1) = z_i (alpha - c(log_i)) / (alpha - c(sorted_i)) with
    c(t) = t_0 + beta t_1 + beta^2 t_2 + beta^3 t_3, and z ending at 1.

Two AIRs state this.  MemoryAirConfig writes every constraint and extension column out by hand, and its trace carries
the sorted table and the multiplicities, computed on the host with numpy.  MemoryDeclaredAirConfig declares the lookup
(air.Lookup) and the permutation (air.Permutation): the package generates their constraints and columns, and the prover
fills the sorted table and the multiplicities on the device.  Both prove to the same bytes.

The sorted order is constrained by the AIR itself (the address constraints and the clock lookup); the permutation argument
only proves that the sorted table holds the log's accesses.  The proof is not zero-knowledge: the log is not hidden.
"""
import numpy as np

from .. import expr as E
from ..air import AirConfig, Lookup, Permutation, RunningColumn, domain_generator
from ..prover import Stark, Trace
from .lookup import _to_mont
from .rescue import digest_evaluation

P = E.P
_R = 2**64
CLK, ADDR, VAL, WR, S_ADDR, S_CLK, S_VAL, S_W, NL, M = range(10)
EV, SUM, PROD = 10, 11, 12
LOG, SORTED = (ADDR, CLK, VAL, WR), (S_ADDR, S_CLK, S_VAL, S_W)      # the permutation's tuple: (addr, clk, val, w)


def _clock_step():
    """the lookup's value: (1 - delta)(s_clk' - s_clk - 1), 0 where the address changes"""
    T, one = E.Trace, E.Constant(1)
    delta = T(S_ADDR, 1) - T(S_ADDR, 0)
    return (one - delta) * (T(S_CLK, 1) - T(S_CLK, 0) - one)


def _memory_constraints(trace_len):
    """the constraints on the log, the sorted table, nl and e (both AIRs)"""
    g = domain_generator(trace_len.bit_length() - 1)
    x, T, one = E.X(), E.Trace, E.Constant(1)
    first, last = E.Constant(1), E.Constant(pow(g, trace_len - 1, P))
    all_rows = x ** trace_len - one
    but_last = (x - last) / all_rows
    gamma = E.Challenge(0)
    delta = T(S_ADDR, 1) - T(S_ADDR, 0)
    read, read1 = one - T(WR, 0), one - T(WR, 1)
    return [
        T(CLK, 0) / (x - first),
        (T(CLK, 1) - T(CLK, 0) - one) * but_last,
        T(WR, 0) * (one - T(WR, 0)) / all_rows,
        T(S_ADDR, 0) / (x - first),
        (T(S_W, 0) - one) / (x - first),
        delta * (delta - one) * but_last,
        delta * (one - T(S_W, 1)) * but_last,
        (one - delta) * (one - T(S_W, 1)) * (T(S_VAL, 1) - T(S_VAL, 0)) * but_last,
        (T(NL, 0) - one) * but_last,
        T(NL, 0) / (x - last),
        (T(EV, 0) - read * T(VAL, 0)) / (x - first),
        (T(EV, 1) - T(EV, 0) * (one + read1 * (gamma - one)) - read1 * T(VAL, 1)) * but_last,
        (T(EV, 0) - E.Hint(0)) / (x - last),
    ]


def _read_column():
    gamma, read = E.Challenge(0), E.Constant(1) - E.Trace(WR, 0)
    return RunningColumn(init=0, mul=E.Constant(1) + read * (gamma - E.Constant(1)), add=read * E.Trace(VAL, 0),
                         inclusive=True)


def read_evaluation(reads, gamma):
    """e's last row: acc <- acc gamma + r over the read values in order, from acc = 0 (gamma: a 3-tuple)"""
    return digest_evaluation([(r,) for r in reads], gamma)


class _MemoryConfig(AirConfig):
    NUM_BASE_COLUMNS = 10
    NUM_EXTENSION_COLUMNS = 3
    FQ_IS_FP = False

    @staticmethod
    def gen_hints(trace_len, claim, challenges):
        return [read_evaluation(claim.reads, challenges[0])]


class MemoryAirConfig(_MemoryConfig):
    """The memory AIR with every constraint written out: its own, then the clock lookup's three (alpha_L =
    Challenge(1)), then the permutation's three (alpha = Challenge(2), beta = Challenge(3))."""

    @staticmethod
    def _denominators():
        T = E.Trace
        alpha_l, alpha, beta = E.Challenge(1), E.Challenge(2), E.Challenge(3)
        b2 = beta * beta
        b3 = b2 * beta

        def c(cols):
            return T(cols[0], 0) + beta * T(cols[1], 0) + b2 * T(cols[2], 0) + b3 * T(cols[3], 0)
        return alpha_l - T(CLK, 0), alpha_l - _clock_step(), alpha - c(LOG), alpha - c(SORTED)

    @staticmethod
    def constraints(trace_len):
        g = domain_generator(trace_len.bit_length() - 1)
        x, T, one = E.X(), E.Trace, E.Constant(1)
        first, last = E.Constant(1), E.Constant(pow(g, trace_len - 1, P))
        but_last = (x - last) / (x ** trace_len - one)
        d_table, d_value, d_log, d_sorted = MemoryAirConfig._denominators()
        s, s1, z, z1 = T(SUM, 0), T(SUM, 1), T(PROD, 0), T(PROD, 1)
        num = T(M, 0) * d_value - T(NL, 0) * d_table         # (m / d_table - nl / d_value) d_table d_value
        return _memory_constraints(trace_len) + [
            s / (x - first),
            ((s1 - s) * d_table * d_value - num) * but_last,
            (s * d_table * d_value + num) / (x - last),
            (z - one) / (x - first),
            (z1 * d_sorted - z * d_log) * but_last,
            (z * d_log - d_sorted) / (x - last),
        ]

    @staticmethod
    def extension_columns(trace_len):
        d_table, d_value, d_log, d_sorted = MemoryAirConfig._denominators()
        return [_read_column(),
                RunningColumn(init=0, add=E.Trace(M, 0) / d_table - E.Trace(NL, 0) / d_value),
                RunningColumn(init=1, mul=d_log / d_sorted)]


class MemoryDeclaredAirConfig(_MemoryConfig):
    """MemoryAirConfig with its clock lookup and its permutation declared: its own constraints are the thirteen on the
    log, the sorted table, nl and e; the package generates the rest and fills s_addr, s_clk, s_val, s_w and m."""

    @staticmethod
    def constraints(trace_len):
        return _memory_constraints(trace_len)

    @staticmethod
    def extension_columns(trace_len):
        return [_read_column(), None, None]

    @staticmethod
    def lookups(trace_len):
        return [Lookup(table=(E.Trace(CLK, 0),), values=((_clock_step(),),), multiplicity=M, running_sum=SUM,
                       selectors=(E.Trace(NL, 0),))]

    @staticmethod
    def permutations(trace_len):
        return [Permutation(source=tuple(E.Trace(c, 0) for c in LOG), target=SORTED, running_product=PROD)]


def _log_columns(n, A, seed):
    """canonical clk, addr, val, w of a log that first writes addresses 0..A-1 in order, then reads or writes random
    addresses (int64; values below 2^62)"""
    rng = np.random.default_rng(seed)
    addr = np.concatenate([np.arange(A, dtype=np.int64), rng.integers(0, A, size=n - A, dtype=np.int64)])
    w = np.concatenate([np.ones(A, dtype=np.int64), rng.integers(0, 2, size=n - A, dtype=np.int64)])
    written = rng.integers(0, 1 << 62, size=n, dtype=np.int64)
    order = np.argsort(addr, kind="stable")                 # by (addr, clk): every run starts with a write
    last_write = np.maximum.accumulate(np.where(w[order] == 1, np.arange(n), 0))
    val = np.empty(n, dtype=np.int64)
    val[order] = written[order][last_write]
    return np.arange(n, dtype=np.int64), addr, val, w


def _check_shape(n, A):
    if n & (n - 1) or n < 4 or not 1 <= A <= n:
        raise ValueError(f"a log of n = {n} rows over A = {A} addresses: n must be a power of two >= 4, 1 <= A <= n")


def _host_columns(n, A, seed, filled):
    """the ten canonical base columns (int64) of gen_trace's host log; filled: with the sorted table and m computed with
    numpy"""
    clk, addr, val, w = _log_columns(n, A, seed)
    cols = np.zeros((10, n), dtype=np.int64)
    cols[CLK], cols[ADDR], cols[VAL], cols[WR] = clk, addr, val, w
    cols[NL, :n - 1] = 1
    if filled:
        order = np.lexsort([cols[c] for c in reversed(LOG)])        # lexsort's last key is the primary one; stable
        cols[list(SORTED)] = cols[list(LOG)][:, order]
        same = cols[S_ADDR, 1:] == cols[S_ADDR, :-1]
        step = np.where(same, cols[S_CLK, 1:] - cols[S_CLK, :-1] - 1, 0)      # rows 0..n-2, where nl = 1
        cols[M] = np.bincount(step, minlength=n)
    return cols


def gen_trace(n, A, seed=1, device=None):
    """(Trace, reads): the log of n accesses to A addresses (a first pass writes each address once, then seeded random
    reads and writes), nl, and the sorted table and m left zero for the prover to fill (MemoryDeclaredAirConfig); reads:
    the values the reads return, in order.  device: the columns are built on that CUDA device with torch and handed over
    as a device tensor."""
    _check_shape(n, A)
    if device is None:
        cols = _host_columns(n, A, seed, False)
        return Trace(_to_mont(cols.astype(np.uint64))), cols[VAL][cols[WR] == 0].tolist()
    import torch
    from .. import FP, Context
    device = torch.device(device)
    g = torch.Generator(device=device).manual_seed(seed)
    i64 = dict(dtype=torch.int64, device=device)
    clk = torch.arange(n, **i64)
    addr = torch.cat([torch.arange(A, **i64), torch.randint(0, A, (n - A,), generator=g, **i64)])
    w = torch.cat([torch.ones(A, **i64), torch.randint(0, 2, (n - A,), generator=g, **i64)])
    written = torch.randint(0, 1 << 62, (n,), generator=g, **i64)
    order = torch.argsort(addr, stable=True)
    last_write = torch.cummax(torch.where(w[order] == 1, clk, 0), 0).values
    val = torch.empty_like(written)
    val[order] = written[order][last_write]
    cols = torch.zeros((10, n), **i64)
    cols[CLK], cols[ADDR], cols[VAL], cols[WR] = clk, addr, val, w
    cols[NL, :n - 1] = 1
    reads = val[w == 0].cpu().tolist()
    ctx = Context(device.index or 0, stream=torch.cuda.current_stream(device).cuda_stream)
    ctx.pointwise_const("mul", cols, FP, cols, FP, [pow(_R, 2, P)], FP, cols.numel())   # -> Montgomery words
    torch.cuda.current_stream(device).synchronize()     # the prover reads the tensor on its own stream
    return Trace(cols), reads


class MemoryClaim(Stark):
    """the reads of a memory log return `reads` (canonical integers), in order; the hand-written AIR"""
    AirConfig = MemoryAirConfig

    def __init__(self, reads):
        self.reads = [int(r) for r in reads]
        if not all(0 <= r < P for r in self.reads):
            raise ValueError("read values must be canonical field elements")

    def get_public_inputs(self):
        return self

    def public_inputs_bytes(self, claim):
        """the number of reads as u64, then the read values; every value 8 bytes little-endian"""
        return np.array([len(claim.reads)] + claim.reads, dtype="<u8").tobytes()

    @staticmethod
    def gen_trace(n, A, seed=1):
        """(Trace, reads): gen_trace's host log with the sorted table and m computed on the host with numpy"""
        _check_shape(n, A)
        cols = _host_columns(n, A, seed, True)
        return Trace(_to_mont(cols.astype(np.uint64))), cols[VAL][cols[WR] == 0].tolist()


class MemoryDeclaredClaim(MemoryClaim):
    """the same claim over MemoryDeclaredAirConfig: the prover fills the sorted table and m"""
    AirConfig = MemoryDeclaredAirConfig

    @staticmethod
    def gen_trace(n, A, seed=1, device=None):
        return gen_trace(n, A, seed, device)
