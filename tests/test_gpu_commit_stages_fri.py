"""GPU parity: SHA-256 row hashing + Merkle nodes, pointwise stages, sum_columns, FRI fold —
bit exact against the CPU oracle, through the C ABI."""
import hashlib

import numpy as np
import pytest

import ministark_b200 as ms

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    return ms.Context(0)


# ------------------------------------------------------------------ commitments
# row widths of the BASELINE configs (SURVEY.md §8a row 14): brainfuck base 17 Fp (136 B),
# extension 9 Fq3 (216 B), composition 16 Fq3 (384 B), config 3: 32 Fp (256 B), FRI rows ff x Fq3;
# plus the padding edge cases 55/56/64-byte messages (7, 8 words) and a single column.
@pytest.mark.parametrize("field,ncols", [(1, 1), (1, 3), (1, 6), (1, 7), (1, 8), (1, 17), (1, 32), (3, 1), (3, 2),
                                         (3, 8), (3, 9), (3, 16)])
@pytest.mark.parametrize("log_rows", [1, 5, 12])
def test_hash_rows_and_merkle(ctx, orc, field, ncols, log_rows):
    n = 1 << log_rows
    mat = orc.rand_matrix(ncols, n, field, seed=ncols * 10 + field)
    m = ms.Matrix(mat, field, ctx)
    leaves = m.hash_rows()
    want_leaves = orc.hash_rows(mat, field)
    assert np.array_equal(leaves, want_leaves)
    tree = ms.MatrixMerkleTree.from_matrix(m)
    want_nodes = orc.merkle_nodes(want_leaves)
    assert np.array_equal(tree.leaves, want_leaves)
    assert np.array_equal(tree.nodes, want_nodes)
    assert tree.root() == want_nodes[1].tobytes()
    assert not tree.nodes[0].any()                      # nodes[0] = Digest::default (src/merkle.rs:487)


def test_hash_row_against_hashlib(ctx):
    # leaf = SHA-256 of the canonical values, 8 bytes little-endian each (src/hash.rs:92-99)
    vals = [0, 1, 2, ms.P - 1, 2**32, 0xDEADBEEFCAFEF00D % ms.P]
    mat = np.array([[ms.to_mont(v), ms.to_mont(v + 1)] for v in vals], dtype=np.uint64)  # 6 columns x 2 rows
    got = ms.Matrix(mat, ms.FP, ctx).hash_rows()
    for i in range(2):
        msg = b"".join(int((v + i) % ms.P).to_bytes(8, "little") for v in vals)
        assert got[i].tobytes() == hashlib.sha256(msg).digest()


def test_merkle_errors(ctx):
    # MerkleTreeImpl::new errors (src/merkle.rs:113-128): < 2 leaves, not a power of two
    leaves = np.zeros((3, 32), dtype=np.uint8)
    nodes = np.zeros((3, 32), dtype=np.uint8)
    with pytest.raises(ms.MsError):
        ctx.merkle_nodes(leaves, nodes, 3)
    with pytest.raises(ms.MsError):
        ctx.merkle_nodes(leaves, nodes, 1)


def test_commit_pipeline_resident(ctx, orc):
    """trace -> iNTT -> LDE x8 (bit-reversed) -> root with everything resident on the device."""
    torch = pytest.importorskip("torch")
    log_n, log_b, ncols = 13, 3, 6
    trace = orc.rand_matrix(ncols, 1 << log_n, 1, seed=3)
    d = torch.from_numpy(trace.view(np.int64)).cuda()
    lde = torch.empty((ncols, 1 << (log_n + log_b)), dtype=torch.int64, device="cuda")
    ctx.ntt_batch(d, ms.FP, log_n, ncols, inverse=True)
    ctx.lde_batch(d, lde, ms.FP, log_n, log_b, ncols)
    root = ctx.merkle_commit(lde, ms.FP, 1 << (log_n + log_b), ncols)
    want = orc.lde(orc.ntt(trace, 1, log_n, inverse=True), 1, log_n, log_b, orc.generator(), True)
    assert root == orc.merkle_nodes(orc.hash_rows(want, 1))[1].tobytes()


# ------------------------------------------------------------------ pointwise stages
@pytest.mark.parametrize("op", ["mul", "add", "sub"])
@pytest.mark.parametrize("lf,rf", [(1, 1), (3, 1), (3, 3), (1, 3)])
@pytest.mark.parametrize("shift", [0, 5])
def test_binary_stages(ctx, orc, op, lf, rf, shift):
    n = 2048  # gpu/tests/fields.rs uses n = 2048
    a = orc.rand_matrix(1, n, lf, seed=1)[0]
    b = orc.rand_matrix(1, n, rf, seed=2)[0]
    df = max(lf, rf)
    dst = np.empty(n * df, dtype=np.uint64)
    ctx.pointwise(op, dst, df, a, lf, b, rf, n=n, shift=shift)
    assert np.array_equal(dst, orc.pointwise(op, a, lf, b, rf, shift=shift))
    if df == lf:  # *Assign form: lhs[i] op= rhs[(i+shift)%N]  (evaluation_shaders.h.metal:58-76)
        inplace = a.copy()
        ctx.pointwise(op, inplace, lf, inplace, lf, b, rf, n=n, shift=shift)
        assert np.array_equal(inplace, dst)


@pytest.mark.parametrize("field", [1, 3])
def test_unary_stages(ctx, orc, field):
    n = 2048
    a = orc.rand_matrix(1, n, field, seed=9)[0]
    a[: field] = ms.ONE if field == 1 else np.array([ms.ONE, 0, 0], dtype=np.uint64)
    for op, kw in (("inv", {}), ("neg", {}), ("exp", dict(exponent=3)), ("exp", dict(exponent=0)),
                   ("exp", dict(exponent=2**32 - 1))):
        dst = np.empty_like(a)
        ctx.pointwise(op, dst, field, a, field, n=n, **kw)
        assert np.array_equal(dst, orc.pointwise(op, a, field, **kw)), op
    # inverse really inverts (Fq3 inverse is missing in the reference: eval_gpu.rs:338)
    inv = np.empty_like(a)
    ctx.pointwise("inv", inv, field, a, field, n=n)
    prod = np.empty_like(a)
    ctx.pointwise("mul", prod, field, a, field, inv, field, n=n)
    one = np.zeros(field, dtype=np.uint64)
    one[0] = ms.ONE
    assert np.array_equal(prod.reshape(n, field), np.tile(one, (n, 1)))
    if field == 1:  # ConvertInto<Fq3, Fp>
        dst3 = np.empty(3 * n, dtype=np.uint64)
        ctx.pointwise("convert", dst3, 3, a, 1, n=n)
        assert np.array_equal(dst3, orc.pointwise("convert", a, 1, dfield=3))


def test_mulpow_stage(ctx, orc):
    # gpu/tests/fields.rs:17-117: lhs[i] *= rhs[(i+shift)%N]^e
    n = 2048
    for lf, rf, e in ((1, 1, 3), (3, 1, 2), (3, 3, 3)):
        a = orc.rand_matrix(1, n, lf, seed=4)[0]
        b = orc.rand_matrix(1, n, rf, seed=5)[0]
        dst = np.empty(n * max(lf, rf), dtype=np.uint64)
        ctx.pointwise("mulpow", dst, max(lf, rf), a, lf, b, rf, n=n, shift=1, exponent=e)
        assert np.array_equal(dst, orc.pointwise("mulpow", a, lf, b, rf, shift=1, exponent=e))


@pytest.mark.parametrize("op", ["mul", "add", "fill"])
@pytest.mark.parametrize("lf,cf", [(1, 1), (3, 1), (3, 3), (1, 3)])
def test_const_stages(ctx, orc, op, lf, cf):
    n = 1000
    a = orc.rand_matrix(1, n, lf, seed=6)[0]
    k = orc.rand_matrix(1, 1, cf, seed=8)[0]
    df = max(lf, cf)
    dst = np.empty(n * df, dtype=np.uint64)
    ctx.pointwise_const(op, dst, df, a, lf, k, cf, n)
    want = orc.pointwise_const(op, a, lf, k, cf, n=n, dfield=df)
    assert np.array_equal(dst, want)


def test_sum_columns(ctx, orc):
    for field, ncols, n in ((1, 1, 64), (1, 26, 4096), (3, 9, 2048)):
        mat = orc.rand_matrix(ncols, n, field, seed=ncols)
        got = ms.Matrix(mat, field, ctx).sum_columns().cols[0]
        assert np.array_equal(got, orc.sum_columns(mat, field))


def test_stage_argument_errors(ctx):
    a = np.zeros(8, dtype=np.uint64)
    with pytest.raises(ms.MsError):
        ctx.pointwise("mul", a, 1, a, 1, None, 1, n=8)           # binary op without rhs
    with pytest.raises(ms.MsError):
        ctx.pointwise("mul", a, 1, np.zeros(24, dtype=np.uint64), 3, a, 1, n=8)  # Fq3 result into Fp dst


def test_bit_reverse(ctx, orc):
    v = np.arange(16, dtype=np.uint64)
    ctx.bit_reverse(v, ms.FP, 4)
    assert v.tolist() == [0, 8, 4, 12, 2, 10, 6, 14, 1, 9, 5, 13, 3, 11, 7, 15]   # gpu/src/utils.rs:233-236
    for field, log_n in ((1, 10), (3, 9), (1, 0), (1, 1)):
        m = orc.rand_matrix(3, 1 << log_n, field, seed=log_n)
        got = m.copy()
        ctx.bit_reverse(got, field, log_n, ncols=3)
        for c in range(3):
            assert np.array_equal(got[c], orc.bit_reverse(m[c], field, log_n))


# ------------------------------------------------------------------ FRI
@pytest.mark.parametrize("field", [1, 3])
@pytest.mark.parametrize("log_ff", [1, 2, 3, 4])
@pytest.mark.parametrize("log_n", [4, 7, 11, 15])
def test_fri_fold_equals_apply_drp(ctx, orc, field, log_ff, log_n):
    ev = orc.rand_matrix(1, 1 << log_n, field, seed=log_n + log_ff)[0]
    alpha = orc.rand_matrix(1, 1, field, seed=99)[0]
    out = np.empty((field << log_n) >> log_ff, dtype=np.uint64)
    ctx.fri_fold(ev, out, field, log_n, log_ff, alpha)
    assert np.array_equal(out, orc.fri_apply_drp(ev, field, log_n, log_ff, alpha))


def test_fri_layer_sequence_and_commit(ctx, orc):
    """build_layers shape of BASELINE config 2 (src/fri.rs:179-231): 32768 -> 2048 -> 128, ff = 16,
    each layer committed as rows of ff Fq3 evaluations."""
    field, log_n, log_ff = 3, 15, 4
    ev = orc.rand_matrix(1, 1 << log_n, field, seed=2024)[0]
    want = ev
    got = ev
    for layer in range(2):
        ln = log_n - layer * log_ff
        alpha = orc.rand_matrix(1, 1, field, seed=50 + layer)[0]
        # layer matrix: row k = ff consecutive evaluations = ff columns of n/ff rows (Matrix::from_arrays)
        rows = got.reshape(-1, (1 << log_ff) * field)
        cols = np.ascontiguousarray(rows.reshape(rows.shape[0], 1 << log_ff, field).transpose(1, 0, 2)).reshape(1 << log_ff, -1)
        root = ctx.merkle_commit(cols, field, rows.shape[0], 1 << log_ff)
        assert root == orc.merkle_nodes(orc.hash_rows(cols, field))[1].tobytes()
        nxt = np.empty((field << ln) >> log_ff, dtype=np.uint64)
        ctx.fri_fold(got, nxt, field, ln, log_ff, alpha)
        want = orc.fri_apply_drp(want, field, ln, log_ff, alpha)
        assert np.array_equal(nxt, want)
        got = nxt


# ------------------------------------------------------------------ matrix plumbing + resident FRI layers
@pytest.mark.parametrize("field,k", [(1, 2), (3, 8), (3, 16)])
def test_from_rows_and_gather(ctx, orc, field, k):
    n = 512
    rows = orc.rand_matrix(1, n * k, field, seed=k)[0]            # n rows of k elements, row-major
    cols = np.empty((k, n * field), dtype=np.uint64)
    ctx.matrix_from_rows(rows, cols, field, n, k)
    want = np.ascontiguousarray(rows.reshape(n, k, field).transpose(1, 0, 2)).reshape(k, -1)
    assert np.array_equal(cols, want)                              # Matrix::from_arrays (src/matrix.rs:50-64)
    ids = [0, 5, n - 1, 17, 5]
    got = ctx.gather_rows(cols, field, n, k, ids)                  # Matrix::get_row (src/matrix.rs:288-294)
    for q, i in enumerate(ids):
        assert np.array_equal(got[q], rows.reshape(n, k * field)[i])
    with pytest.raises(ms.MsError):
        ctx.gather_rows(cols, field, n, k, [n])


@pytest.mark.parametrize("log_n", [12, 20])
def test_config4_fri_layers_resident(ctx, orc, log_n):
    """BASELINE config 4 shape: Fq3 codeword, ff = 8 (fib) — each layer committed in place (rows of ff
    consecutive evaluations) and folded on the device; roots and codewords equal the reference flow
    Matrix::from_arrays + from_matrix + apply_drp (src/fri.rs:199-231,526-567)."""
    torch = pytest.importorskip("torch")
    field, log_ff = 3, 3
    ev = orc.rand_matrix(1, 1 << log_n, field, seed=log_n)[0]
    cur = torch.from_numpy(ev.view(np.int64)).cuda()
    want = ev
    nlayers = 2 if log_n > 12 else 3
    for layer in range(nlayers):
        ln = log_n - layer * log_ff
        alpha = orc.rand_matrix(1, 1, field, seed=500 + layer)[0]
        nrows = 1 << (ln - log_ff)
        root = ctx.merkle_commit_rows(cur, (1 << log_ff) * field, nrows)
        rows = want.reshape(nrows, (1 << log_ff), field)
        cols = np.ascontiguousarray(rows.transpose(1, 0, 2)).reshape(1 << log_ff, -1)
        assert root == orc.merkle_nodes(orc.hash_rows(cols, field))[1].tobytes()
        nxt = torch.empty((field << ln) >> log_ff, dtype=torch.int64, device="cuda")
        ctx.fri_fold(cur, nxt, field, ln, log_ff, alpha)
        ctx.sync()
        want = orc.fri_apply_drp(want, field, ln, log_ff, alpha)
        assert np.array_equal(nxt.cpu().numpy().view(np.uint64), want)
        cur = nxt


def test_pow_grind_smallest_nonce(ctx, orc):
    # grind_fri_commitments (src/channel.rs:76-93); brainfuck uses grinding_factor 20 (examples/brainfuck/main.rs:95)
    for tag, bits in ((b"a", 0), (b"b", 8), (b"c", 16), (b"d", 20)):
        seed = hashlib.sha256(tag).digest()
        assert ctx.pow_grind(seed, bits) == orc.pow_grind(seed, bits)
    # each launch searches 2^24 nonces from `base` (1, 2^24 + 1, 2^25 + 1, ...): answers in the first, second and third
    # launch.  The nonces are the serial CPU oracle's, re-derived in tests/test_oracle_pins.py.
    for tag, bits, nonce in ((b"g0", 24, 10056532), (b"g2", 24, 28919286), (b"g5", 24, 41922605), (b"g3", 24, 45695959),
                             (b"g0", 0, 1)):
        seed = hashlib.sha256(tag).digest()
        assert ctx.pow_grind(seed, bits) == nonce, (tag, bits)
        digest = hashlib.sha256(seed + nonce.to_bytes(8, "big")).digest()
        assert 256 - int.from_bytes(digest, "big").bit_length() >= bits


@pytest.mark.parametrize("log_ff", [1, 2, 3, 4])
def test_fri_fold_structured_codewords(ctx, orc, log_ff):
    """few-valued codewords (constants, 2^63 / 2^62 pairs whose sums hit 2^64 exactly, 0/1 flags): the in-register
    inverse DFT of the fold starts with both-lazy additions"""
    log_n = 12
    n = 1 << log_n
    rng = np.random.default_rng(log_ff)
    pool = np.array([0, ms.ONE, 2**63, 2**62, ms.P - 1, ms.P - 2**63, 2**32, 2**32 - 2], dtype=np.uint64)
    alpha = orc.rand_matrix(1, 1, 3, seed=9)[0]
    for lanes in (1, 3):
        for pick in (pool[rng.integers(0, 4, size=n * lanes)], np.full(n * lanes, 2**63, dtype=np.uint64),
                     pool[(np.arange(n * lanes) // 3) % len(pool)]):
            ev = np.ascontiguousarray(pick, dtype=np.uint64)
            out = np.empty((n >> log_ff) * lanes, dtype=np.uint64)
            ctx.fri_fold(ev, out, lanes, log_n, log_ff, alpha)
            assert np.array_equal(out, orc.fri_apply_drp(ev, lanes, log_n, log_ff, alpha))
