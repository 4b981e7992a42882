/*
 * ministark_rescue_merkle_updates.h — examples/merkle's write claim on the device: K ordered leaf writes into the
 * Rescue-Prime Merkle tree of include/ministark_rescue_merkle.h (ministark_b200/examples/merkle.py,
 * MerkleUpdatesClaim).  The node function and the heap layout are those of ms_rescue_merkle_tree: node 1 is the root,
 * node 2^D + i is leaf i, node v = merge(node 2 v, node 2 v + 1).  Conventions as in ministark_b200.h (column-major
 * matrices, 0 on success, a negative MS_ERR_* otherwise; pointers may be device or host memory).
 */
#ifndef MINISTARK_RESCUE_MERKLE_UPDATES_H
#define MINISTARK_RESCUE_MERKLE_UPDATES_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Applies K leaf writes to the heap `nodes` (as ms_rescue_merkle_tree writes it, depth D), one after another: write k
 * replaces leaf indices[k] with new_leaves[k] (four canonical words, K x 4 row-major).  An index may repeat; a later
 * write to the same leaf overwrites an earlier one.  Writes
 *   out:   the (15, n) column-major matrix of Montgomery words, n = 16 K L with L the smallest power of two >= D:
 *          the layout of ms_rescue_merkle_paths for 2 K paths.  Path 2 k is write k's old path: the leaf it replaces,
 *          then its siblings, as the tree stands before write k.  Path 2 k + 1 is its new path: new_leaves[k] with the
 *          same siblings.  Path g holds rows [8 L g, 8 L (g + 1)); its permutation j = 0..L-1 sits at rows
 *          8 (L g + j) + r, the state before round r for r < 7 and the output at r = 7 (columns 0..11).  Permutation j
 *          takes (cur, sib_j, 0^4) when b_j = 0 and (sib_j, cur, 0^4) when b_j = 1, b_j = bit j of indices[k] and sib_j
 *          node ((2^D + indices[k]) >> j) ^ 1 as the tree stands before write k; the filler permutations j >= D take
 *          b_j = 0 and sib_j = 0.  Column 12 holds b_j and column 13 indices[k] >> j on the eight rows of permutation j;
 *          column 14 (SIDE) is 0 on the old path's rows and 1 on the new path's.
 *   roots: (K + 1) x 4 canonical words: roots[0] the root before the first write, roots[k + 1] the root after write k.
 *   nodes: the heap after all K writes, in place, once every read of the original heap is done.
 * Level-parallel: level j resolves, for all K writes at once, which version of node ((2^D + indices[k]) >> j) ^ 1 and
 * (j = 0) of the leaf write k sees, the new value the latest earlier write through that node gave it or the heap's.
 * Per level j < D: one key fill, one stable radix sort of the writes by parent node (D - 1 - j key bits; none at the
 * top level), one mark fill, one max-scan, one resolve launch and one permutation launch; per filler level the
 * permutation launch only; then one scatter of the last writer's value of every touched node into the heap.
 * Permutations: 2 K L.  Bytes written: 15 n words of trace, at most 4 (D + 1) K heap words and 4 (K + 1) root words,
 * plus O(K) words of scratch per level.  Scratch is the context's own.
 * K a power of two, 1 <= D <= 32, n <= 2^32, every index < 2^D and every leaf word canonical (the last two checked on
 * the device).  Bad arguments fail with MS_ERR_INVALID and a message in ms_last_error before anything is written: the
 * heap is then untouched.  Synchronises (the indices and leaves are checked first). */
int ms_rescue_merkle_updates(ms_ctx *ctx, void *nodes, uint32_t depth, const uint64_t *indices,
                             const uint64_t *new_leaves, uint64_t K, void *out, uint64_t *roots);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_RESCUE_MERKLE_UPDATES_H */
