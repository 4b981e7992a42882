/*
 * ministark_stream.h — the entry points of libministark_b200.so behind the streamed residency of the prover: a trace
 * whose bit-reversed LDE does not fit in device memory is committed one coset block at a time, and its query rows are
 * evaluated from the coefficients.  Conventions as in ministark_b200.h (Montgomery words, column-major matrices, any
 * pointer may be device or host memory, 0 on success, a negative MS_ERR_* otherwise).
 *
 * They have no counterpart in the reference, whose CPU prover keeps every LDE matrix in host memory.
 */
#ifndef MINISTARK_STREAM_H
#define MINISTARK_STREAM_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* one coset block of a tree committed block by block (no leaf array is kept): hashes the 2^log_block_rows rows at cols
 * (the block's first row) into context scratch and writes every heap node of the block's subtree at its global index in
 * `nodes`, the n x 32 B heap of the whole tree, n = 2^(log_block_rows + log_blocks).  block_root (32 B, host or device)
 * receives the subtree root = nodes[2^log_blocks + block]; with log_block_rows = 0 it is the leaf digest and no node is
 * written.  ms_merkle_nodes_sha256 over the 2^log_blocks block roots then fills nodes[0 .. 2^log_blocks): nodes[1..n)
 * and the root equal ms_merkle_commit_sha256's. */
int ms_merkle_commit_block_sha256(ms_ctx *ctx, int field, const void *cols, size_t col_stride_elems, unsigned ncols,
                                  unsigned log_block_rows, unsigned log_blocks, size_t block, void *nodes, void *block_root);

/* rows of a bit-reversed coset LDE without the LDE: out[(q * ncols + c) * field ..] is the element ms_lde_batch(...,
 * bitrev_out = 1) stores at row positions[q] of column c (the layout of ms_gather_rows), i.e. P_c(offset * g_N^bitrev(
 * positions[q])), N = 2^(log_n + log_blowup).  coeffs: ncols columns of 2^log_n coefficients; positions: host array
 * (any order, duplicates allowed).  The points are base-field elements: Fp arithmetic for Fp columns, Fq3 x Fp for Fq3. */
int ms_lde_rows(ms_ctx *ctx, int field, const void *coeffs, size_t col_stride_elems, unsigned ncols, unsigned log_n,
                unsigned log_blowup, uint64_t offset_mont, const uint64_t *positions, unsigned npos, void *out);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_STREAM_H */
