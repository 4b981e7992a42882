"""cosets.py — the coset-block structure of a bit-reversed LDE, shared by the provers that walk it block by block.

The bit-reversed LDE of n coefficients over offset * <g_N>, N = beta * n (src/matrix.rs:225-234), is beta blocks of n
rows; block q is the size-n transform of the same coefficients over the coset h_q * <g_n>, h_q = offset * g_N^bitrev(q).
The multi-GPU prover (prover_mgpu.py) gives each GPU a run of blocks; the streaming prover (prover.py) recomputes one
block at a time.  Both evaluate the composition constraints block by block with the same block-local program and answer
Merkle queries with the same index walk.
"""
from . import expr as E
from .air import domain_generator

P = E.P
_R = 2**64


def brev(v, bits):
    r = 0
    for _ in range(bits):
        r = (r << 1) | (v & 1)
        v >>= 1
    return r


def coset_offsets(log_n, log_b, blocks=None):
    """[(q, Montgomery word of h_q = 7 * g_N^bitrev(q))] for q in `blocks` (default: all 2^log_b blocks)"""
    gN = domain_generator(log_n + log_b)
    qs = range(1 << log_b) if blocks is None else blocks
    return [(q, 7 * pow(gN, brev(q, log_b), P) % P * _R % P) for q in qs]


def block_program(air):
    """the composition constraints evaluated over one block: inside a block the ce-domain stride is 1 and the domain has
    n points (compiled once per Air and cached on it)"""
    prog = getattr(air, "_block_program", None)
    if prog is None:
        prog = air._block_program = E.compile_program(air.composition_constraint, air.config.NUM_BASE_COLUMNS, lde_step=1,
                                                      log_ce=air.log_n, symbolic=True, batch_inverses=True)
    return prog


def heap_location(i, log_b):
    """where node i of the heap of a tree committed in 2^log_b blocks lives when the heap is split
    (include/ministark_host_nodes.h): (None, i) in the top heap of 2 * 2^log_b digests, else (block, index in the block's
    local heap).  Node i at level L = floor(log2 i) >= log_b + 1 is one of the 2^d, d = L - log_b, nodes block
    (i >> d) - 2^log_b owns on that level; in the block's heap the same level starts at 1 << d."""
    i = int(i)
    beta = 1 << log_b
    if i < 2 * beta:
        return None, i
    d = i.bit_length() - 1 - log_b
    return (i >> d) - beta, (1 << d) | (i & ((1 << d) - 1))


def merkle_walk(n_leaves, indices):
    """The index walk of MerkleTreeImpl::prove (src/merkle.rs:149-207; csrc/hash.cu ms_merkle_prove_sha256): which
    leaves and which heap nodes a batched proof names.  Returns (initial leaf indices, sibling leaf indices, node indices)."""
    idx = sorted(set(int(i) for i in indices))
    init, sib, path, node_q = [], [], [], []
    k = 0
    while k < len(idx):
        i = idx[k]
        init.append(i)
        node_q.append((n_leaves + i) >> 1)
        if k + 1 < len(idx) and (i ^ 1) == idx[k + 1]:
            init.append(idx[k + 1])
            k += 2
            continue
        sib.append(i ^ 1)
        k += 1
    head = 0
    while head < len(node_q):
        i = node_q[head]
        head += 1
        if i > 2:
            node_q.append(i >> 1)
        if head < len(node_q) and (i ^ 1) == node_q[head]:
            head += 1
            continue
        path.append(i ^ 1)
    return init, sib, path
