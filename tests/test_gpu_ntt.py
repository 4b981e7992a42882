"""GPU parity: NTT / iNTT / LDE through the C ABI vs the CPU oracle — bit exact.

Mirrors the reference's differential pattern (gpu/tests/shaders.rs:16-117: random polynomial,
GPU transform, assert_eq element-wise against ark-poly) with the oracle in arkworks' place, and
widens it: every size 2^0..2^21 (the reference tests 2048, 4096, 65536), plain and coset,
Fp and Fq3, host pointers (staged) and resident device pointers, batched columns."""
import numpy as np
import pytest

import ministark_b200 as ms
from tests_helpers_ntt import edge_column, structured_columns

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    return ms.Context(0)


@pytest.mark.parametrize("log_n", list(range(0, 19)))
@pytest.mark.parametrize("coset", [False, True])
def test_fft_ifft_fp_all_sizes(ctx, orc, log_n, coset):
    rng = np.random.default_rng(log_n * 2 + coset)
    n = 1 << log_n
    offset = orc.generator() if coset else orc.ONE
    col = edge_column(n, 1, rng)
    # GpuFft::encode / execute on a host slice (gpu/tests/shaders.rs:17-40)
    got = col.copy()
    fft = ms.GpuFft(ms.Domain(log_n, offset), ms.FP, ctx)
    fft.encode(got)
    fft.execute()
    want = orc.ntt(col.reshape(1, -1), 1, log_n, offset)[0]
    assert np.array_equal(got, want)
    # GpuIfft (gpu/tests/shaders.rs:94-117)
    ifft = ms.GpuIfft(ms.Domain(log_n, offset), ms.FP, ctx)
    back = got.copy()
    ifft.encode(back)
    ifft.execute()
    assert np.array_equal(back, col)
    assert np.array_equal(orc.ntt(want.reshape(1, -1), 1, log_n, offset, inverse=True)[0], col)


@pytest.mark.parametrize("log_n", [1, 4, 7, 11, 12, 13, 16])
@pytest.mark.parametrize("coset", [False, True])
def test_fft_fq3(ctx, orc, log_n, coset):
    # gpu/tests/shaders.rs:43-66: Fq3 coefficients, Fp twiddles
    rng = np.random.default_rng(100 + log_n)
    offset = orc.generator() if coset else orc.ONE
    col = edge_column(1 << log_n, 3, rng)
    got = col.copy()
    fft = ms.GpuFft(ms.Domain(log_n, offset), ms.FQ3, ctx)
    fft.encode(got)
    fft.execute()
    want = orc.ntt(col.reshape(1, -1), 3, log_n, offset)[0]
    assert np.array_equal(got, want)
    ifft = ms.GpuIfft(ms.Domain(log_n, offset), ms.FQ3, ctx)
    ifft.encode(got)
    ifft.execute()
    assert np.array_equal(got, col)


@pytest.mark.parametrize("log_n,ncols", [(5, 7), (11, 17), (12, 9), (14, 5), (17, 3)])
def test_matrix_interpolate_multi_column(ctx, orc, log_n, ncols):
    # Matrix::interpolate encodes every column into one batch (src/matrix.rs:101-116)
    trace = orc.rand_matrix(ncols, 1 << log_n, 1, seed=log_n)
    m = ms.Matrix(trace, ms.FP, ctx)
    polys = m.interpolate(ms.Domain(log_n))
    assert np.array_equal(polys.cols, orc.ntt(trace, 1, log_n, inverse=True))
    # and many encodes on one plan, mixed lengths are rejected like the reference's assert_eq!
    fft = ms.GpuFft(ms.Domain(log_n), ms.FP, ctx)
    with pytest.raises(ms.MsError):
        fft.encode(np.zeros(3, dtype=np.uint64))


@pytest.mark.parametrize("log_n,log_b", [(0, 3), (2, 2), (3, 4), (4, 1), (5, 3), (9, 2), (11, 4), (12, 3), (13, 3), (16, 2), (17, 3)])
@pytest.mark.parametrize("bitrev", [True, False])
def test_lde_fp(ctx, orc, log_n, log_b, bitrev):
    # Matrix::(bit_reversed_)evaluate over the LDE coset offset = Fp::GENERATOR (src/matrix.rs:237-251)
    ncols = 3
    coeffs = orc.rand_matrix(ncols, 1 << log_n, 1, seed=7 * log_n + log_b)
    m = ms.Matrix(coeffs, ms.FP, ctx)
    dom = ms.Domain(log_n + log_b, ms.GENERATOR)
    got = (m.bit_reversed_evaluate(dom) if bitrev else m.evaluate(dom)).cols
    want = orc.lde(coeffs, 1, log_n, log_b, orc.generator(), bitrev=bitrev)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("log_n,log_b,ncols", [(10, 4, 17), (10, 4, 3), (10, 3, 17), (8, 4, 5), (6, 4, 9), (10, 4, 1), (9, 4, 17),
                                                 (11, 4, 17), (12, 4, 17), (7, 5, 33), (10, 2, 26), (13, 4, 17)])
def test_lde_and_interpolate_many_columns_small_sizes(ctx, orc, log_n, log_b, ncols):
    # shapes the full prover produces (e.g. brainfuck: 17 base columns, n = 2^10, blow-up 16)
    trace = orc.rand_matrix(ncols, 1 << log_n, 1, seed=31 * log_n + ncols)
    m = ms.Matrix(trace, ms.FP, ctx)
    polys = m.interpolate(ms.Domain(log_n))
    want_polys = orc.ntt(trace, 1, log_n, inverse=True)
    assert np.array_equal(polys.cols, want_polys)
    got = polys.bit_reversed_evaluate(ms.Domain(log_n + log_b, ms.GENERATOR)).cols
    assert np.array_equal(got, orc.lde(want_polys, 1, log_n, log_b, orc.generator(), bitrev=True))


@pytest.mark.parametrize("log_n,log_b", [(4, 2), (11, 4), (13, 3)])
def test_lde_fq3(ctx, orc, log_n, log_b):
    coeffs = orc.rand_matrix(2, 1 << log_n, 3, seed=log_n)
    m = ms.Matrix(coeffs, ms.FQ3, ctx)
    got = m.bit_reversed_evaluate(ms.Domain(log_n + log_b, ms.GENERATOR)).cols
    assert np.array_equal(got, orc.lde(coeffs, 3, log_n, log_b, orc.generator(), bitrev=True))


def test_resident_device_pointers_and_strides(ctx, orc):
    torch = pytest.importorskip("torch")
    log_n, ncols, stride = 14, 4, (1 << 14) + 64   # padded column stride
    host = np.zeros((ncols, stride), dtype=np.uint64)
    trace = orc.rand_matrix(ncols, 1 << log_n, 1, seed=5)
    host[:, : 1 << log_n] = trace
    dev = torch.from_numpy(host.view(np.int64)).cuda()
    ctx.ntt_batch(dev, ms.FP, log_n, ncols, col_stride=stride, inverse=True)
    ctx.sync()
    got = dev.cpu().numpy().view(np.uint64)
    assert np.array_equal(got[:, : 1 << log_n], orc.ntt(trace, 1, log_n, inverse=True))
    assert not got[:, 1 << log_n:].any()      # padding untouched
    # resident LDE: coefficients -> evaluations, both on device
    out = torch.empty((ncols, 1 << (log_n + 2)), dtype=torch.int64, device="cuda")
    ctx.lde_batch(dev, out, ms.FP, log_n, 2, ncols, in_stride=stride)
    ctx.sync()
    want = orc.lde(orc.ntt(trace, 1, log_n, inverse=True), 1, log_n, 2, orc.generator(), bitrev=True)
    assert np.array_equal(out.cpu().numpy().view(np.uint64), want)


@pytest.mark.parametrize("log_n", [20])
def test_config1_roundtrip_2p20(ctx, orc, log_n):
    # BASELINE config 1: 2^20-point forward+inverse NTT, single column, bit-exact round trip
    col = orc.rand_matrix(1, 1 << log_n, 1, seed=1000)[0]
    for offset in (orc.ONE, orc.generator()):
        got = col.copy()
        ctx.ntt_batch(got, ms.FP, log_n, 1, offset=offset)
        assert np.array_equal(got, orc.ntt(col.reshape(1, -1), 1, log_n, offset)[0])
        ctx.ntt_batch(got, ms.FP, log_n, 1, inverse=True, offset=offset)
        assert np.array_equal(got, col)


def test_large_sizes_by_properties(ctx, orc):
    """2^24 (BASELINE config 3 column length): size-independent properties on device —
    round trip, linearity, and the LDE prefix property used by prover.rs:86-91."""
    torch = pytest.importorskip("torch")
    log_n = 24
    n = 1 << log_n
    a = torch.empty(n, dtype=torch.int64, device="cuda")
    b = torch.empty(n, dtype=torch.int64, device="cuda")
    ctx.fill_random(a, n, 1)
    ctx.fill_random(b, n, 2)
    s = torch.empty_like(a)
    ctx.pointwise("add", s, ms.FP, a, ms.FP, b, ms.FP, n=n)
    a0 = a.clone()
    for t in (a, b, s):
        ctx.ntt_batch(t, ms.FP, log_n, offset=ms.GENERATOR)
    s2 = torch.empty_like(a)
    ctx.pointwise("add", s2, ms.FP, a, ms.FP, b, ms.FP, n=n)
    ctx.sync()
    assert torch.equal(s, s2)                                  # NTT(a+b) == NTT(a)+NTT(b)
    ctx.ntt_batch(a, ms.FP, log_n, inverse=True, offset=ms.GENERATOR)
    ctx.sync()
    assert torch.equal(a, a0)                                  # iNTT(NTT(a)) == a
    # spot-check 64 evaluations against Horner on the host via the oracle's field ops
    coeffs = a0.cpu().numpy().view(np.uint64)
    ctx.ntt_batch(a, ms.FP, log_n, offset=ms.GENERATOR)
    ctx.sync()
    ev = a.cpu().numpy().view(np.uint64)
    g = orc.root_of_unity(log_n)
    for i in (1, n // 2 + 3, 9999999):
        x = orc.fp_mul(orc.generator(), orc.fp_pow(g, i))
        pt = np.array([x, 0, 0], dtype=np.uint64)
        assert int(orc.horner(coeffs, 1, pt)[0]) == int(ev[i])


# ---- edge arithmetic: the lazy primitives and structured (non-random) columns ---------------------------------------
_EDGE = [0, 1, 2, 3, 2**31, 2**32 - 2, 2**32 - 1, 2**32, 2**32 + 1, 2**33 - 2, 2**33 - 1, 2**33, 2**62, 2**63 - 1, 2**63, 2**63 + 1,
         2**63 + 2**31, 2**64 - 2**33, 2**64 - 2**32 - 1, ms.P - 2, ms.P - 1, ms.P, ms.P + 1, ms.P + 2**32 - 2, 2**64 - 2**32 + 2**31,
         2**64 - 2**31, 2**64 - 2, 2**64 - 1, 0xFFFFFFFF00000000, 0x00000000FFFFFFFF, 0x8000000080000000, 0x7FFFFFFFFFFFFFFF,
         0xFFFFFFFEFFFFFFFF, 0xFFFFFFFF7FFFFFFF, 0x0000000100000000, 0x00000001FFFFFFFF, 0xAAAAAAAAAAAAAAAA, 0x5555555555555555]


def test_lazy_primitives_all_edge_pairs(ctx):
    """add_lc / sub_lc / add_ll / sub_ll / mul of csrc/field.cuh on every pair of edge words (incl. a + b == 2^64 exactly,
    a == b, operands >= p) plus random pairs, against big-integer arithmetic mod p"""
    import ctypes as C
    rng = np.random.default_rng(1)
    a = np.array([x for x in _EDGE for _ in _EDGE] + list(rng.integers(0, 2**64, size=4096, dtype=np.uint64)), dtype=np.uint64)
    b = np.array([y for _ in _EDGE for y in _EDGE] + list(rng.integers(0, 2**64, size=4096, dtype=np.uint64)), dtype=np.uint64)
    # pairs that sum to exactly 2^64 and pairs that differ by exactly eps / p
    extra = [(x, (2**64 - x) % 2**64) for x in _EDGE if x] + [(x, (x + 2**32 - 1) % 2**64) for x in _EDGE] + [(x, (x + ms.P) % 2**64) for x in _EDGE]
    a = np.concatenate([a, np.array([e[0] for e in extra], dtype=np.uint64)])
    b = np.concatenate([b, np.array([e[1] for e in extra], dtype=np.uint64)])
    n = a.size
    out = np.empty(5 * n, dtype=np.uint64)
    ctx._ck(ctx.lib.ms_debug_lazy_ops(ctx.h, a.ctypes.data, b.ctypes.data, n, out.ctypes.data))
    out = out.reshape(5, n)
    P, RINV = ms.P, pow(2**64, -1, ms.P)
    for i in range(n):
        x, y = int(a[i]), int(b[i])
        yc = y - P if y >= P else y
        assert int(out[0, i]) % P == (x + yc) % P, ("add_lc", hex(x), hex(y))
        assert int(out[1, i]) % P == (x - yc) % P, ("sub_lc", hex(x), hex(y))
        assert int(out[2, i]) % P == (x + y) % P, ("add_ll", hex(x), hex(y))
        assert int(out[3, i]) % P == (x - y) % P, ("sub_ll", hex(x), hex(y))
        assert int(out[4, i]) == x * yc * RINV % P, ("mul", hex(x), hex(y))


@pytest.mark.parametrize("log_n", list(range(1, 17)))
def test_structured_columns_all_transforms(ctx, orc, log_n):
    """forward / inverse, subgroup / coset NTT and the coset LDE on structured columns (the brainfuck MemValInv column —
    values 0, 1, 1/2, 1/3, 1/4 — exposed a spurious second carry in add_ll when two words sum to exactly 2^64)"""
    rng = np.random.default_rng(log_n)
    n = 1 << log_n
    cols = structured_columns(n, rng)
    k = cols.shape[0]
    for inverse in (False, True):
        for offset in (orc.ONE, orc.generator()):
            got = cols.copy()
            ctx.ntt_batch(got, ms.FP, log_n, k, inverse=inverse, offset=offset)
            assert np.array_equal(got, orc.ntt(cols, 1, log_n, offset, inverse=inverse)), (inverse, offset)
    polys = orc.ntt(cols, 1, log_n, inverse=True)
    for log_b in (1, 4):
        out = np.empty((k, n << log_b), dtype=np.uint64)
        ctx.lde_batch(polys, out, ms.FP, log_n, log_b, k, offset=ms.GENERATOR, bitrev=True)
        assert np.array_equal(out, orc.lde(polys, 1, log_n, log_b, orc.generator(), bitrev=True)), log_b
    # Fq3: the three lanes of a structured extension column
    q = np.ascontiguousarray(np.stack([cols[6], cols[2], cols[8]], axis=1).reshape(1, 3 * n))
    got = q.copy()
    ctx.ntt_batch(got, ms.FQ3, log_n, 1, inverse=True)
    assert np.array_equal(got, orc.ntt(q, 3, log_n, inverse=True))


@pytest.mark.parametrize("log_n,log_b,ncols,field", [(10, 3, 5, 1), (13, 3, 3, 1), (16, 2, 4, 1), (5, 3, 2, 1), (12, 3, 2, 3), (4, 1, 3, 1),
                                                     (16, 3, 32, 1)])     # the last one is large enough for the TMA pipeline (scatter through per-block tensor maps)
@pytest.mark.parametrize("world", [2, 4])
def test_lde_scatter_into_row_slabs(ctx, orc, log_n, log_b, ncols, field, world):
    """ms_lde_batch_scatter (the multi-GPU fused exchange) with the "peer" slabs on the same device: every coset block
    lands in the slab that owns its rows, at the column offset of this rank, plus a local copy of block 0"""
    torch = pytest.importorskip("torch")
    nb = 1 << log_b
    if nb % world:
        pytest.skip("world must divide the blow-up")
    n, N = 1 << log_n, 1 << (log_n + log_b)
    rows_per, per_rank = N // world, nb // world
    total_cols, lo = ncols + 3, 2                          # the local columns are global columns [lo, lo + ncols)
    coeffs = orc.rand_matrix(ncols, n, field, seed=log_n + world)
    want = orc.lde(coeffs, field, log_n, log_b, orc.generator(), True)
    d_coeffs = torch.from_numpy(coeffs.view(np.int64)).cuda()
    work = torch.zeros((ncols, N * field), dtype=torch.int64, device="cuda")
    slabs = [torch.zeros((total_cols, rows_per * field), dtype=torch.int64, device="cuda") for _ in range(world)]
    blocks = [slabs[q // per_rank].data_ptr() + (lo * rows_per + (q % per_rank) * n) * field * 8 for q in range(nb)]
    dups = [work.data_ptr() if q == 0 else 0 for q in range(nb)]
    ctx.lde_batch_scatter(d_coeffs, work, field, log_n, log_b, ncols, blocks, rows_per, dups, N)
    ctx.sync()
    for j in range(world):
        got = slabs[j].cpu().numpy().view(np.uint64)
        assert np.array_equal(got[lo:lo + ncols], want[:, j * rows_per * field:(j + 1) * rows_per * field]), j
        assert not got[:lo].any() and not got[lo + ncols:].any()          # other ranks' columns untouched
    assert np.array_equal(work.cpu().numpy().view(np.uint64)[:, :n * field], want[:, :n * field])


# ---- the persistent TMA pipeline (csrc/ntt_tma.cu) against the oracle and against the one-tile-per-CTA kernel --------------
@pytest.mark.parametrize("log_b,ncols", [(3, 8), (2, 16), (0, 64), (4, 5)])
def test_tma_pipeline_lde_2p16_vs_oracle(ctx, orc, log_b, ncols):
    """2^16 points = digits [8, 8]: a strided pass (with the coset pre-scale tile) + the contiguous pass, both on the TMA
    pipeline when it is switched on; bit-reversed LDE compared with the oracle word for word, and the two kernels with each other"""
    torch = pytest.importorskip("torch")
    log_n = 16
    n = 1 << log_n
    coeffs = orc.rand_matrix(ncols, n, 1, seed=300 + log_b)
    coeffs[0, :10] = [0, 1, ms.P - 1, ms.P - 2, 2**32 - 1, 2**32, 2**32 + 1, 0xFFFFFFFF00000000, 2**63, ms.P - 2**32]
    want = orc.lde(coeffs, 1, log_n, log_b, orc.generator(), bitrev=True)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        c2 = ms.Context(0, stream=stream.cuda_stream)
        dev = torch.from_numpy(coeffs.view(np.int64)).cuda()
        out = torch.empty((ncols, n << log_b), dtype=torch.int64, device="cuda")
        got = {}
        try:
            for tma in (1, 0):
                c2.set_option("ntt_tma", tma)
                out.zero_()
                c2.lde_batch(dev, out, ms.FP, log_n, log_b, ncols)
                c2.sync()
                got[tma] = out.cpu().numpy().view(np.uint64).copy()
        finally:
            c2.set_option("ntt_tma", 1)
    assert np.array_equal(got[1], want)
    assert np.array_equal(got[0], want)


@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("coset", [False, True])
def test_tma_pipeline_natural_order_ntt_2p16(ctx, orc, inverse, coset):
    """natural-order transforms: the strided pass runs on the TMA pipeline with the natural digit placement (and the
    inverse constants), the transposing last pass on the tile kernel"""
    torch = pytest.importorskip("torch")
    ncols, log_n = 64, 16
    offset = orc.generator() if coset else orc.ONE
    cols = orc.rand_matrix(ncols, 1 << log_n, 1, seed=5)
    want = orc.ntt(cols, 1, log_n, offset, inverse=inverse)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        c2 = ms.Context(0, stream=stream.cuda_stream)
        try:
            for tma in (1, 0):
                c2.set_option("ntt_tma", tma)
                d = torch.from_numpy(cols.view(np.int64)).cuda()
                c2.ntt_batch(d, ms.FP, log_n, ncols, inverse=inverse, offset=offset)
                c2.sync()
                assert np.array_equal(d.cpu().numpy().view(np.uint64), want)
        finally:
            c2.set_option("ntt_tma", 1)


def test_tma_pipeline_2p24_equals_tile_kernel_and_groups(ctx):
    """three passes at the config-3 transform size: TMA pipeline (2 and 3 consumer groups, a short stage ring) against the
    one-tile-per-CTA kernel, bit for bit, for the LDE and for natural-order forward / inverse transforms"""
    torch = pytest.importorskip("torch")
    log_n, log_b, ncols = 24, 3, 2
    n = 1 << log_n
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        c2 = ms.Context(0, stream=stream.cuda_stream)
        a = torch.empty((ncols, n), dtype=torch.int64, device="cuda")
        c2.fill_random(a, ncols * n, 11)
        ref = torch.empty((ncols, n << log_b), dtype=torch.int64, device="cuda")
        got = torch.empty_like(ref)
        try:
            c2.set_option("ntt_tma", 0)
            c2.lde_batch(a, ref, ms.FP, log_n, log_b, ncols)
            for groups, stages in ((2, 8), (3, 8), (2, 3)):
                c2.set_option("ntt_tma", 1)
                c2.set_option("ntt_tma_groups", groups)
                c2.set_option("ntt_tma_stages", stages)
                got.zero_()
                c2.lde_batch(a, got, ms.FP, log_n, log_b, ncols)
                c2.sync()
                assert torch.equal(got, ref), (groups, stages)
            c2.set_option("ntt_tma_groups", 2)
            c2.set_option("ntt_tma_stages", 8)
            for inverse in (True, False):
                outs = {}
                for tma in (0, 1):
                    c2.set_option("ntt_tma", tma)
                    d = a.clone()
                    c2.ntt_batch(d, ms.FP, log_n, ncols, inverse=inverse, offset=ms.GENERATOR)
                    c2.sync()
                    outs[tma] = d
                assert torch.equal(outs[0], outs[1])
        finally:
            c2.set_option("ntt_tma", 1)
            c2.set_option("ntt_tma_groups", 2)
            c2.set_option("ntt_tma_stages", 8)
