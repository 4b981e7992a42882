"""GPU parity of the NTT paths the small-size tests never reach, word for word against the CPU oracle.

A plan (csrc/api_ntt.cu, ntt_get_plan) builds full device tables for the inter-pass twiddles, the coset pre-scale and
the inverse post-scale when they fit and their cudaMalloc succeeds.  Without one, the pass kernel (csrc/ntt.cu, do_step)
computes those factors as geometric progressions from the two-level tables.  At the sizes of tests/test_gpu_ntt.py every
table is built, so these progressions, the split tile grid (more than 32768 tiles, first at 2^28 points) and the
64-bit-offset pass instantiations (columns of more than 2^31 words) are compared with the oracle only here:

* "ntt_table_words" caps the full tables of a context's plans: 0 drops them all; 2^log_n - 1 drops those of the first
  pass, the pre-scale and the post-scale and keeps the later passes' twiddles, the mix the prover's 2^28-point
  composition interpolation runs with;
* "ntt_wide_index" forces the 64-bit-offset instantiations at any size;
* the large cases run 2^22..2^28-point transforms with the default plans, resident on the device.

Each oracle result is computed once and every path is compared with it; a forward result also checks the inverse
through the round trip."""
import contextlib

import numpy as np
import pytest
import torch

import ministark_b200 as ms
from tests_helpers_ntt import edge_column, structured_columns

pytestmark = pytest.mark.gpu

GiB = 1 << 30
FIELDS = pytest.mark.parametrize("field", [ms.FP, ms.FQ3], ids=["fp", "fq3"])
DEFAULT = {}
NO_TABLES = {"table_words": 0}


@pytest.fixture(scope="module")
def ctx():
    c = ms.Context(0)
    yield c
    c.close()


@pytest.fixture
def release(ctx):
    """after a large case: frees the context's plans and scratch and torch's cached blocks (the GPU is shared)"""
    yield
    ctx.set_option("drop_plans", 1)
    ctx.set_option("drop_scratch", 1)
    torch.cuda.empty_cache()


@contextlib.contextmanager
def paths(ctx, table_words=-1, wide=0, tma=1):
    """runs the block with these switches; the defaults are restored whatever happens.  Setting "ntt_table_words" drops
    the context's cached plans, so the next transform builds its plan under the limit."""
    try:
        ctx.set_option("ntt_table_words", table_words)
        ctx.set_option("ntt_wide_index", wide)
        ctx.set_option("ntt_tma", tma)
        yield
    finally:
        ctx.set_option("ntt_table_words", -1)
        ctx.set_option("ntt_wide_index", 0)
        ctx.set_option("ntt_tma", 1)


def digits(log_n):
    """msntt::choose_digits: one pass per digit"""
    if log_n <= 12:
        return [log_n]
    m = (log_n + 7) // 8
    base, rem = divmod(log_n, m)
    return [base + (i < rem) for i in range(m)]


def columns(field, log_n, ncols, seed):
    """edge-seasoned random columns, then (up to 2^17 points) structured ones: Fp columns as they are, Fq3 columns with
    three structured columns as their lanes"""
    rng = np.random.default_rng(seed)
    n = 1 << log_n
    cols = [edge_column(n, field, rng) for _ in range(min(ncols, 2))]
    if len(cols) < ncols:
        s = structured_columns(n, rng)
        if field == ms.FQ3:
            s = [np.stack([s[i], s[(i + 5) % 12], s[(i + 8) % 12]], axis=1).reshape(-1) for i in range(12)]
        cols += list(s)
    return np.ascontiguousarray(np.stack(cols[:ncols]))


def dev(a):
    d = torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()
    torch.cuda.synchronize()        # the context's stream does not wait for torch's
    return d


def ntt(ctx, d, field, log_n, inverse, offset):
    ctx.ntt_batch(d, field, log_n, d.shape[0], inverse=inverse, offset=offset)
    ctx.sync()


def lde(ctx, coeffs, field, log_n, log_b):
    out = torch.empty((coeffs.shape[0], (field << log_n) << log_b), dtype=torch.int64, device="cuda")
    ctx.lde_batch(coeffs, out, field, log_n, log_b, coeffs.shape[0], offset=ms.GENERATOR, bitrev=True)
    ctx.sync()
    return out


def assert_words(got, want, field, what, block_rows=None):
    """bit-for-bit equality of (ncols, rows * field) words; `got` may be a device tensor, copied back in slices so that a
    2^28-point Fq3 column needs no second host copy.  A mismatch names the number of differing words and the first ones
    by column, row, lane and (for a bit-reversed LDE) coset block."""
    ncols, width = want.shape
    step = 1 << 25
    nbad, first = 0, []
    for c in range(ncols):
        for w0 in range(0, width, step):
            w = want[c, w0:w0 + step]
            g = got[c, w0:w0 + step]
            if isinstance(g, torch.Tensor):
                g = g.cpu().numpy().view(np.uint64)
            bad = np.flatnonzero(g != w)
            nbad += bad.size
            for i in bad[:max(0, 6 - len(first))]:
                row, lane = divmod(w0 + int(i), field)
                where = f"col {c} row {row}"
                if block_rows:
                    where += f" (block {row // block_rows} row {row % block_rows})"
                if field > 1:
                    where += f" lane {lane}"
                first.append(f"{where}: {int(g[i]):#x} != {int(w[i]):#x}")
    assert nbad == 0, f"{what}: {nbad} of {want.size} words differ; " + "; ".join(first)


def _host_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def need(device_bytes, host_bytes):
    """skips, naming the bytes, when the shared GPU or the host cannot hold a large case (never allocates to find out)"""
    free, _ = torch.cuda.mem_get_info()
    if free < device_bytes:
        pytest.skip(f"needs {device_bytes / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB free")
    avail = _host_available()
    if avail < host_bytes:
        pytest.skip(f"needs {host_bytes / GiB:.1f} GiB of available host memory, {avail / GiB:.1f} GiB available")


# ---- (a) no full tables at all, small sizes: one digit (the pre-scale progression reads shared memory), two, three ----
@FIELDS
@pytest.mark.parametrize("log_n", [4, 8, 12, 13, 16, 17, 20])
@pytest.mark.parametrize("coset", [False, True], ids=["plain", "coset"])
def test_tableless_natural_order(ctx, orc, field, log_n, coset):
    offset = orc.generator() if coset else orc.ONE
    cols = columns(field, log_n, 2 if log_n > 17 else 6, seed=10 * log_n + field + coset)
    want = orc.ntt(cols, field, log_n, offset)
    for cfg in (DEFAULT, NO_TABLES):
        with paths(ctx, **cfg):
            d = dev(cols)
            ntt(ctx, d, field, log_n, False, offset)
            assert_words(d, want, field, f"forward {cfg}")
            ntt(ctx, d, field, log_n, True, offset)
            assert_words(d, cols, field, f"inverse {cfg}")


@FIELDS
@pytest.mark.parametrize("log_n", [12, 16, 20])
def test_tableless_bitrev_lde(ctx, orc, field, log_n):
    """up to 16 coset blocks: the pre-scale progression of every block starts from its own pre_step"""
    coeffs = columns(field, log_n, 1 if log_n > 17 else 4, seed=20 * log_n + field)
    d = dev(coeffs)
    for log_b in (0, 1, 3, 4):
        want = orc.lde(coeffs, field, log_n, log_b, orc.generator(), bitrev=True)
        for cfg in (DEFAULT, NO_TABLES):
            with paths(ctx, **cfg):
                assert_words(lde(ctx, d, field, log_n, log_b), want, field, f"x{1 << log_b} {cfg}", 1 << log_n)


@pytest.mark.parametrize("world", [2, 4])
def test_tableless_lde_scatter(ctx, orc, world):
    """ms_lde_batch_scatter (a shape of test_lde_scatter_into_row_slabs) without tables: every coset block lands in the
    slab that owns its rows, plus the local copy of block 0"""
    log_n, log_b, ncols, field = 16, 2, 4, ms.FP
    nb, n, N = 1 << log_b, 1 << log_n, 1 << (log_n + log_b)
    rows_per, per_rank = N // world, nb // world
    total_cols, lo = ncols + 3, 2
    coeffs = columns(field, log_n, ncols, seed=world)
    want = orc.lde(coeffs, field, log_n, log_b, orc.generator(), True)
    with paths(ctx, **NO_TABLES):
        d_coeffs = dev(coeffs)
        work = torch.zeros((ncols, N * field), dtype=torch.int64, device="cuda")
        slabs = [torch.zeros((total_cols, rows_per * field), dtype=torch.int64, device="cuda") for _ in range(world)]
        torch.cuda.synchronize()
        blocks = [slabs[q // per_rank].data_ptr() + (lo * rows_per + (q % per_rank) * n) * field * 8 for q in range(nb)]
        dups = [work.data_ptr() if q == 0 else 0 for q in range(nb)]
        ctx.lde_batch_scatter(d_coeffs, work, field, log_n, log_b, ncols, blocks, rows_per, dups, N)
        ctx.sync()
    for j in range(world):
        got = slabs[j].cpu().numpy().view(np.uint64)
        assert_words(got[lo:lo + ncols], want[:, j * rows_per * field:(j + 1) * rows_per * field], field, f"slab {j}")
        assert not got[:lo].any() and not got[lo + ncols:].any()
    assert_words(work.cpu().numpy().view(np.uint64)[:, :n * field], want[:, :n * field], field, "local copy of block 0")


@FIELDS
def test_tableless_gpufft_host_columns(ctx, orc, field):
    """GpuFft / GpuIfft plans made under the limit, on staged host columns (ms_ntt_execute)"""
    log_n = 17
    cols = columns(field, log_n, 3, seed=30 + field)
    want = orc.ntt(cols, field, log_n, orc.generator())
    with paths(ctx, **NO_TABLES):
        got = [c.copy() for c in cols]
        fft = ms.GpuFft(ms.Domain(log_n, orc.generator()), field, ctx)
        for g in got:
            fft.encode(g)
        fft.execute()
        assert_words(np.stack(got), want, field, "GpuFft")
        ifft = ms.GpuIfft(ms.Domain(log_n, orc.generator()), field, ctx)
        for g in got:
            ifft.encode(g)
        ifft.execute()
        assert_words(np.stack(got), cols, field, "GpuIfft")


# ---- (c) the limit really removes the tables: with it, a new plan launches one kernel per pass and no table builder ----
def test_table_limit_removes_the_tables(ctx, orc):
    log_n, n = 20, 1 << 20
    m = len(digits(log_n))
    d = dev(orc.rand_matrix(1, n, 1, seed=9))
    out = torch.empty((1, n << 3), dtype=torch.int64, device="cuda")
    calls = {
        "forward coset": lambda: ctx.ntt_batch(d, ms.FP, log_n, offset=ms.GENERATOR),
        "inverse coset": lambda: ctx.ntt_batch(d, ms.FP, log_n, inverse=True, offset=ms.GENERATOR),
        "lde x8": lambda: ctx.lde_batch(d, out, ms.FP, log_n, 3),
    }
    # table builders per plan: the twiddles of the m - 1 strided passes, then the pre-scale table (one builder per coset
    # block) or the post-scale table; the mixed limit drops pass 0's twiddles and the scale tables
    builders = {
        "default": {"forward coset": (m - 1) + 1, "inverse coset": (m - 1) + 1, "lde x8": (m - 1) + 8},
        "no tables": {k: 0 for k in calls},
        "mixed": {k: m - 2 for k in calls},
    }
    for name, cfg in (("default", DEFAULT), ("no tables", NO_TABLES), ("mixed", {"table_words": n - 1})):
        for call, fn in calls.items():
            with paths(ctx, **cfg):
                before = ctx.launches
                fn()
                ctx.sync()
                assert ctx.launches - before == m + builders[name][call], (name, call)


# ---- (b) mixed tables, the production shape, and (d) the 64-bit-offset instantiations -----------------------------------
@FIELDS
@pytest.mark.parametrize("log_n", [16, 20, 24], ids=lambda v: f"2p{v}")
def test_mixed_tables_and_wide_index(ctx, orc, release, field, log_n):
    """one oracle forward coset transform and one x8 LDE; the x4 LDE is the first half of the x8 one (block q < 4 of both
    holds the coset offset * g_8^bitrev3(q) = offset * g_4^bitrev2(q)).  The 64-bit-offset runs use the tile kernel, which
    the TMA pipeline would otherwise pre-empt for the Fp 256 x 16 passes."""
    n = 1 << log_n
    cols = columns(field, log_n, 2 if log_n <= 16 else 1, seed=40 * log_n + field)
    g = orc.generator()
    want = orc.ntt(cols, field, log_n, g)
    want_lde = orc.lde(cols, field, log_n, 3, g, bitrev=True)
    cases = [("mixed tables, TMA", dict(table_words=n - 1, tma=1), 3),
             ("mixed tables, tile kernel", dict(table_words=n - 1, tma=0), 3),
             ("64-bit offsets", dict(wide=1, tma=0), 2),
             ("64-bit offsets, no tables", dict(wide=1, tma=0, table_words=0), 2)]
    for name, cfg, log_b in cases:
        with paths(ctx, **cfg):
            d = dev(cols)
            ntt(ctx, d, field, log_n, False, g)
            assert_words(d, want, field, f"{name}: forward coset")
            ntt(ctx, d, field, log_n, True, g)
            assert_words(d, cols, field, f"{name}: inverse coset")
            got = lde(ctx, d, field, log_n, log_b)
            assert_words(got, want_lde[:, :(field << log_n) << log_b], field, f"{name}: lde x{1 << log_b}", n)
            del d, got


# ---- (e) large sizes, default plans -------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [22, 23, 25, 26, 27, 28], ids=lambda v: f"2p{v}")
def test_large_fp_forward_coset(ctx, orc, release, log_n):
    """2^28 points: 65536 tiles per pass, the first split grid (grid.z = 2)"""
    n = 1 << log_n
    words = n * 8
    need(3 * words + GiB, 2 * words + GiB)      # data, natural-order scratch, pre-scale table / input, oracle result
    col = edge_column(n, 1, np.random.default_rng(log_n)).reshape(1, n)
    want = orc.ntt(col, 1, log_n, orc.generator())
    d = dev(col)
    ntt(ctx, d, ms.FP, log_n, False, ms.GENERATOR)
    assert_words(d, want, 1, f"2^{log_n} forward coset")
    del want
    ntt(ctx, d, ms.FP, log_n, True, ms.GENERATOR)
    assert_words(d, col, 1, f"2^{log_n} inverse coset")


@pytest.mark.parametrize("log_n", [27, 28], ids=lambda v: f"2p{v}")
def test_large_fq3_inverse_coset(ctx, orc, release, log_n):
    """the composition polynomial's interpolation of a 2^(log_n - 4)-row brainfuck proof, call for call: digits [7,7,7,7]
    at 2^28, no twiddle table for pass 0, no post-scale table"""
    n = 1 << log_n
    words = n * 3 * 8
    need(2 * words + GiB, 2 * words + GiB)      # data and natural-order scratch / input and oracle result
    col = edge_column(n, 3, np.random.default_rng(log_n)).reshape(1, 3 * n)
    want = orc.ntt(col, 3, log_n, orc.generator(), inverse=True)
    d = dev(col)
    ntt(ctx, d, ms.FQ3, log_n, True, ms.GENERATOR)
    assert_words(d, want, 3, f"2^{log_n} Fq3 inverse coset")
    del want
    ntt(ctx, d, ms.FQ3, log_n, False, ms.GENERATOR)
    assert_words(d, col, 3, f"2^{log_n} Fq3 forward coset")


def test_large_fp_lde_2p24_x16(ctx, orc, release):
    """ncos * N = 2^28 words: exactly the largest pre-scale table a plan builds; then the same call with no tables"""
    log_n, log_b = 24, 4
    n = 1 << log_n
    out_words = (n << log_b) * 8
    need(2 * out_words + GiB, out_words + GiB)   # output and pre-scale table / oracle result
    coeffs = edge_column(n, 1, np.random.default_rng(7)).reshape(1, n)
    want = orc.lde(coeffs, 1, log_n, log_b, orc.generator(), bitrev=True)
    d = dev(coeffs)
    for cfg in (DEFAULT, NO_TABLES):
        with paths(ctx, **cfg):
            assert_words(lde(ctx, d, ms.FP, log_n, log_b), want, 1, f"2^24 x16 {cfg}", n)
