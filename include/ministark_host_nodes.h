/*
 * ministark_host_nodes.h — the entry point behind the "streamed_host" residency of the prover: a tree committed one coset
 * block at a time whose node heap lives in pinned host memory instead of device memory.  Conventions as in
 * ministark_b200.h (Montgomery words, column-major matrices, 0 on success, a negative MS_ERR_* otherwise).
 *
 * Split heap layout.  A tree of N = beta * 2^log_block_rows leaves, committed in beta blocks, is kept as
 *   - a top heap of 2 * beta digests: [beta, 2 beta) are the block roots, [1, beta) the nodes above them
 *     (ms_merkle_nodes_sha256 over the block roots) and slot 0 the unused default digest;
 *   - one local heap per block (this call's host_subtree): the heap ms_merkle_commit_sha256 builds for the block's
 *     2^log_block_rows rows, slot 0 unused (zero) and slot 1 the block root.
 * Global heap index i >= 2 beta lies in block (i >> d) - beta at local index (1 << d) | (i & ((1 << d) - 1)), where
 * d = floor(log2 i) - log2 beta (ministark_b200/cosets.py heap_location).
 *
 * The reference has no counterpart: its CPU prover keeps every tree in host memory.
 */
#ifndef MINISTARK_HOST_NODES_H
#define MINISTARK_HOST_NODES_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* hashes the 2^log_block_rows rows at cols (the block's first row) into context scratch, builds the block's local heap
 * in a device staging buffer of the context and enqueues its copy into host_subtree (2^log_block_rows x 32 B of PINNED
 * host memory; a range that begins or ends in pageable, managed or device memory is refused with MS_ERR_INVALID).
 * block_root (32 B, host or device) receives the block root; it is written when the call returns, the subtree is not.
 *
 * The copy runs on a copy stream of the context behind an event, and the staging buffer is double-buffered: the call
 * returns without waiting for the copy, and work the caller enqueues next on the context's stream runs beside it until
 * something synchronises the device.  host_subtree is complete after ms_ctx_sync, which also waits for these copies; it
 * must not be read or freed before. */
int ms_merkle_commit_block_sha256_host(ms_ctx *ctx, int field, const void *cols, size_t col_stride_elems, unsigned ncols,
                                       unsigned log_block_rows, void *host_subtree, void *block_root);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_HOST_NODES_H */
