/*
 * ministark_rescue_merkle.h — examples/merkle on the device: the Rescue-Prime Merkle tree of 2^D leaves, and the trace
 * of K authentication paths through it (ministark_b200/examples/merkle.py, MerklePathsClaim).  A node is
 * merge(a, b) = words 0..3 of the Rescue-Prime permutation of (a, b, 0, 0, 0, 0): one permutation, capacity zero, no
 * padding.  The tree is a heap: node 1 is the root, node 2^D + i is leaf i, node v = merge(node 2 v, node 2 v + 1).
 * Conventions as in ministark_b200.h (column-major matrices, 0 on success, a negative MS_ERR_* otherwise; pointers may
 * be device or host memory unless a comment says otherwise).
 */
#ifndef MINISTARK_RESCUE_MERKLE_H
#define MINISTARK_RESCUE_MERKLE_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Writes `nodes`, the 2^(D + 1) x 4 heap of canonical words (row-major; row 0 is unused and written as zeros), from
 * `leaves`, 2^D x 4 canonical words (row-major), D = depth in 1..32.  One launch per level, one permutation per node;
 * the levels of at most 32 nodes are finished by one block.  Leaf words must be canonical (they are not checked).  Bad
 * arguments fail with MS_ERR_INVALID and a message in ms_last_error before anything is written.  Does not synchronise
 * unless an argument is host memory. */
int ms_rescue_merkle_tree(ms_ctx *ctx, const uint64_t *leaves, uint32_t depth, void *nodes);

/* Writes `out`, the (14, n) column-major matrix of Montgomery words, n = 8 K L with L the smallest power of two >= D:
 * K authentication paths through the heap `nodes` (as ms_rescue_merkle_tree writes it, depth D).  Path k holds rows
 * [8 L k, 8 L (k + 1)); permutation j = 0..L-1 of path k sits at rows 8 (L k + j) + r, its state before round r for
 * r < 7 and its output at r = 7 (columns 0..11).  With b_j = bit j of indices[k], sib_j = node
 * ((2^D + indices[k]) >> j) ^ 1 and cur the leaf (j = 0) or words 0..3 of permutation j - 1's output, permutation j
 * takes (cur, sib_j, 0^4) when b_j = 0 and (sib_j, cur, 0^4) when b_j = 1; the filler permutations j >= D take b_j = 0
 * and sib_j = 0.  Column 12 holds b_j and column 13 indices[k] >> j on all eight rows of permutation j.  So the root is
 * words 0..3 of row 8 (L k + D) - 1.
 * indices: K uint64 words; K a power of two, every index < 2^D, n <= 2^32.  Bad arguments fail with MS_ERR_INVALID and
 * a message in ms_last_error before anything is written.  Synchronises (the indices are checked first). */
int ms_rescue_merkle_paths(ms_ctx *ctx, const void *nodes, uint32_t depth, const uint64_t *indices, uint64_t K,
                           void *out);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_RESCUE_MERKLE_H */
