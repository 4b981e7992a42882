"""GPU: the SHA-256 commitment kernels of csrc/hash.cu against hashlib, at every leaf shape a specialised kernel could
get wrong.  A leaf is SHA-256 of the row's canonical values, 8 bytes little-endian each (an Fq3 element is c0 || c1 || c2,
columns in order); a node is SHA-256 of its two children, nodes[0] is zero (src/hash.rs:58-100, src/merkle.rs:412-508).

  * ms_hash_rows_sha256 and ms_merkle_commit_sha256 over Fp rows of every width from 1 to 64 words and Fq3 rows of every
    width from 1 to 22 columns (3 to 66 words): 1 to 9 compression blocks, every message length mod 64 bytes, the 0x80
    marker and the bit length in the last data block or in the constant padding block; rows hold 0, 1, 2^32 - 1, 2^32,
    2^63, p - 2 and p - 1 at every word position; the leaves, the whole node heap and the root;
  * row counts 1, 2, 127, 128, 129, 1000 and 4097 (a partial last 128-thread CTA) at a one-block, a constant-padding and
    a multi-block width of each field, with the column stride equal to the row count and 5 elements larger (garbage in
    the gap), from host and from device memory;
  * ms_merkle_commit_rows_sha256 (FRI layers: rows of ff Fq3 evaluations) over rows of 1 to 48 words at 2, 64 and 4096
    rows;
  * the ALU-only instantiation of every SHA kernel (MS_SHA_FMA_ADDS=0), in a spawned process: leaves and heaps over Fp
    rows of 1 to 40 words and Fq3 rows of 1 to 16 columns, row-major commits at 24 and 48 words, ms_merkle_nodes_sha256
    and a 16-bit grind.
Every expected digest comes from hashlib."""
import hashlib
import os
import sys
import traceback

import numpy as np
import pytest
import torch

import ministark_b200 as ms
from ministark_b200 import FP, FQ3, P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EDGES = [0, 1, 2**32 - 1, 2**32, 2**63, P - 2, P - 1]


@pytest.fixture(scope="module")
def ctx():
    return ms.Context(0)


# ------------------------------------------------------------------ hashlib reference
def leaf(row):
    """SHA-256 of a row of canonical values, 8 bytes little-endian each"""
    return hashlib.sha256(b"".join(int(v).to_bytes(8, "little") for v in row)).digest()


def heap(leaves):
    """the (n, 32) uint8 node heap over n (a power of two) leaf digests: nodes[k] = SHA-256(child 2k || child 2k + 1),
    where children k >= n are leaves[k - n]; nodes[0] = 0"""
    n = len(leaves)
    nodes = [bytes(32)] * n
    child = lambda k: leaves[k - n] if k >= n else nodes[k]
    for k in range(n - 1, 0, -1):
        nodes[k] = hashlib.sha256(child(2 * k) + child(2 * k + 1)).digest()
    return np.frombuffer(b"".join(nodes), dtype=np.uint8).reshape(n, 32)


def smallest_nonce(seed, bits):
    """serial search: the smallest nonce >= 1 with leading_zeros(SHA-256(seed || nonce, 8 bytes big-endian)) >= bits"""
    nonce = 1
    while 256 - int.from_bytes(hashlib.sha256(seed + nonce.to_bytes(8, "big")).digest(), "big").bit_length() < bits:
        nonce += 1
    return nonce


def check(got, want, what):
    """got: digests as (k, 32) bytes (numpy or torch); want: k digests"""
    got = np.ascontiguousarray(got.cpu().numpy() if hasattr(got, "cpu") else got, dtype=np.uint8).reshape(-1, 32)
    want = [bytes(w) for w in want]
    assert got.shape[0] == len(want), f"{what}: {got.shape[0]} digests, want {len(want)}"
    bad = [i for i in range(len(want)) if got[i].tobytes() != want[i]]
    assert not bad, f"{what}: {len(bad)} of {len(want)} digests differ, the first at {bad[0]}"


# ------------------------------------------------------------------ inputs
def canonical_rows(nrows, words, seed):
    """(nrows, words) random canonical values; rows 0-6 hold one edge value in every word, rows 7-13 every edge value at
    every word position"""
    rows = np.random.default_rng(seed).integers(0, P, size=(nrows, words), dtype=np.uint64)
    for r in range(min(nrows, 14)):
        rows[r] = [EDGES[r if r < 7 else (r + j) % 7] for j in range(words)]
    return rows


def mont(rows):
    return np.array([ms.to_mont(v) for v in rows.reshape(-1).tolist()], dtype=np.uint64).reshape(rows.shape)


def column_major(mrows, field, stride, seed=1):
    """the (ncols, stride * field) matrix whose row i is mrows[i] (Montgomery words); the words past row nrows - 1 of
    each column are random garbage"""
    nrows, words = mrows.shape
    ncols = words // field
    mat = np.random.default_rng(seed).integers(0, 2**64, size=(ncols, stride * field), dtype=np.uint64)
    mat[:, :nrows * field] = mrows.reshape(nrows, ncols, field).transpose(1, 0, 2).reshape(ncols, nrows * field)
    return mat


def on_device(a):
    t = torch.from_numpy(a.view(np.int64)).cuda()
    torch.cuda.synchronize()            # the context reads it on its own stream
    return t


# ------------------------------------------------------------------ every width
NROWS = 256
WIDTHS = [(FP, w) for w in range(1, 65)] + [(FQ3, c) for c in range(1, 23)]


def _width_case(field, ncols):
    rows = canonical_rows(NROWS, ncols * field, seed=ncols * 4 + field)
    return column_major(mont(rows), field, NROWS), [leaf(r) for r in rows.tolist()]


@pytest.mark.parametrize("field,ncols", WIDTHS)
def test_leaves_and_heap_every_width(ctx, field, ncols):
    mat, want = _width_case(field, ncols)
    want_nodes = heap(want)
    got = np.empty((NROWS, 32), dtype=np.uint8)
    ctx.hash_rows(mat, got, field, NROWS, ncols)
    check(got, want, "hash_rows")
    leaves, nodes = np.empty((NROWS, 32), dtype=np.uint8), np.full((NROWS, 32), 0xAB, dtype=np.uint8)
    root = ctx.merkle_commit(mat, field, NROWS, ncols, leaves=leaves, nodes=nodes)
    check(leaves, want, "merkle_commit leaves")
    check(nodes, want_nodes, "merkle_commit nodes")
    assert root == want_nodes[1].tobytes()


# ------------------------------------------------------------------ row counts and column strides
# words per row: Fp 5 (one block), 8 (64 bytes: constant padding block), 17 (three blocks); Fq3 2 columns (6 words, one
# block), 8 columns (24 words: three data blocks and the constant padding block), 5 columns (15 words: 120 bytes, the
# length spills into a third block)
@pytest.mark.parametrize("field,ncols", [(FP, 5), (FP, 8), (FP, 17), (FQ3, 2), (FQ3, 8), (FQ3, 5)])
@pytest.mark.parametrize("nrows", [1, 2, 127, 128, 129, 1000, 4097])
@pytest.mark.parametrize("stride_pad", [0, 5])
def test_row_counts_and_strides(ctx, field, ncols, nrows, stride_pad):
    stride = nrows + stride_pad                         # in elements: 3 words each for Fq3
    rows = canonical_rows(nrows, ncols * field, seed=nrows * 8 + ncols * 2 + field)
    want = [leaf(r) for r in rows.tolist()]
    mat = column_major(mont(rows), field, stride, seed=nrows)
    got = np.empty((nrows, 32), dtype=np.uint8)
    ctx.hash_rows(mat, got, field, nrows, ncols, col_stride=stride)
    check(got, want, "host matrix")
    got = torch.zeros((nrows, 32), dtype=torch.uint8, device="cuda")
    d_mat = on_device(mat)
    ctx.hash_rows(d_mat, got, field, nrows, ncols, col_stride=stride)
    ctx.sync()
    check(got, want, "device matrix")


# ------------------------------------------------------------------ row-major commits (FRI layers)
# 6, 12, 24 and 48 words are rows of ff = 2, 4, 8 and 16 Fq3 evaluations; 24 and 48 take the constant padding block
@pytest.mark.parametrize("row_words", range(1, 49))
@pytest.mark.parametrize("nrows", [2, 64, 4096])
def test_row_major_commit(ctx, row_words, nrows):
    rows = canonical_rows(nrows, row_words, seed=row_words * 16 + nrows)
    want = [leaf(r) for r in rows.tolist()]
    want_nodes = heap(want)
    src = on_device(mont(rows))
    leaves = torch.zeros((nrows, 32), dtype=torch.uint8, device="cuda")
    nodes = torch.zeros((nrows, 32), dtype=torch.uint8, device="cuda")
    root = ctx.merkle_commit_rows(src, row_words, nrows, leaves=leaves, nodes=nodes)
    check(leaves, want, "leaves")
    check(nodes, want_nodes, "nodes")
    assert root == want_nodes[1].tobytes()


# ------------------------------------------------------------------ the ALU-only kernel variant
ALU_WIDTHS = [(FP, w) for w in range(1, 41)] + [(FQ3, c) for c in range(1, 17)]
ALU_ROW_WORDS, ALU_ROWS = (24, 48), 1024
GRIND_SEED = hashlib.sha256(b"alu").digest()


def _alu_variant_worker(jobs, rehearsal, q):
    """every job through a fresh library whose SHA kernels were chosen from MS_SHA_FMA_ADDS in this environment"""
    try:
        if rehearsal:                                   # the parent runs on the CPU build of the ABI: so does the worker
            sys.path.insert(0, os.path.join(ROOT, "tests"))
            import cpu_device
            cpu_device.install()
        ctx = ms.Context(0)
        out = dict(env=os.environ.get("MS_SHA_FMA_ADDS"))
        for field, ncols, mat in jobs["widths"]:
            leaves, nodes = np.empty((NROWS, 32), dtype=np.uint8), np.empty((NROWS, 32), dtype=np.uint8)
            root = ctx.merkle_commit(mat, field, NROWS, ncols, leaves=leaves, nodes=nodes)
            out[field, ncols] = (leaves, nodes, root)
        for row_words, rows in jobs["rows"]:
            leaves, nodes = np.empty((ALU_ROWS, 32), dtype=np.uint8), np.empty((ALU_ROWS, 32), dtype=np.uint8)
            root = ctx.merkle_commit_rows(rows, row_words, ALU_ROWS, leaves=leaves, nodes=nodes)
            out["rows", row_words] = (leaves, nodes, root)
        leaves = jobs["leaves"]
        nodes = np.empty_like(leaves)
        ctx.merkle_nodes(leaves, nodes, leaves.shape[0])
        out["nodes"] = nodes
        out["grind"] = ctx.pow_grind(GRIND_SEED, 16)
        q.put(out)
    except Exception:
        q.put(traceback.format_exc())


def test_alu_only_variant_equals_hashlib():
    import multiprocessing as mp
    jobs, want = dict(widths=[], rows=[]), {}
    for field, ncols in ALU_WIDTHS:
        mat, leaves = _width_case(field, ncols)
        jobs["widths"].append((field, ncols, mat))
        want[field, ncols] = leaves
    for row_words in ALU_ROW_WORDS:
        rows = canonical_rows(ALU_ROWS, row_words, seed=row_words)
        jobs["rows"].append((row_words, mont(rows)))
        want["rows", row_words] = [leaf(r) for r in rows.tolist()]
    rng = np.random.default_rng(5)
    jobs["leaves"] = rng.integers(0, 256, size=(1 << 12, 32), dtype=np.uint8)
    spawn = mp.get_context("spawn")
    q = spawn.Queue()
    p = spawn.Process(target=_alu_variant_worker, args=(jobs, getattr(ms._lib, "_cpu_device_installed", False), q))
    before = os.environ.get("MS_SHA_FMA_ADDS")
    os.environ["MS_SHA_FMA_ADDS"] = "0"                 # read once, at the worker's first SHA-256 launch
    try:
        p.start()
    finally:
        if before is None:
            del os.environ["MS_SHA_FMA_ADDS"]
        else:
            os.environ["MS_SHA_FMA_ADDS"] = before
    got = q.get(timeout=600)
    p.join(timeout=60)
    assert isinstance(got, dict), got
    assert got["env"] == "0"
    for key, leaves in want.items():
        nodes = heap(leaves)
        check(got[key][0], leaves, f"leaves {key}")
        check(got[key][1], nodes, f"nodes {key}")
        assert got[key][2] == nodes[1].tobytes(), key
    check(got["nodes"], heap([bytes(d) for d in jobs["leaves"]]), "merkle_nodes")
    assert got["grind"] == smallest_nonce(GRIND_SEED, 16)
