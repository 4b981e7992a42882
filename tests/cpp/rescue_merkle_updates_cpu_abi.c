/*
 * rescue_merkle_updates_cpu_abi.c — CPU build of examples/merkle's write entry point
 * (include/ministark_rescue_merkle_updates.h).  TEST INFRASTRUCTURE ONLY, compiled by
 * tests/test_rescue_merkle_updates_cpu.py into a temporary directory.
 *
 * The CPU build of the tree and the paths (tests/cpp/rescue_merkle_cpu_abi.c, which brings the chains trace, the
 * oracle's CPU ABI, the streamed residency, the constraint check and ms_extension_columns) is extended by
 * ms_rescue_merkle_updates, so that `merkle.update(..., device=...)` and whole proofs of its trace run on the CPU
 * harness (tests/cpu_device.py).  The writes are applied one after another to the heap, each with its old and its new
 * path hashed by the permutation written out plainly; none of the device's level-parallel resolution is used.  The
 * product never loads this library.
 */
#include "rescue_merkle_cpu_abi.c"
#include "../../include/ministark_rescue_merkle_updates.h"

/* one permutation of a path: its eight rows from `row` on, from the state s, the output left in s */
static void update_rows(const u64 *mds, const u64 *rc, u64 *s, u64 *o, u64 n, u64 row) {
    for (int r = 0; r < RN; r++) {
        for (int w = 0; w < RW; w++) o[(u64)w * n + row + r] = s[w];
        for (int w = 0; w < RW; w++) s[w] = fp_pow(s[w], 7);
        rescue_mds_mul(mds, s);
        for (int w = 0; w < RW; w++) s[w] = fp_pow(fp_add(s[w], rc[2 * RW * r + w]), MS_RESCUE_ALPHA_INV);
        rescue_mds_mul(mds, s);
        for (int w = 0; w < RW; w++) s[w] = fp_add(s[w], rc[2 * RW * r + RW + w]);
    }
    for (int w = 0; w < RW; w++) o[(u64)w * n + row + 7] = s[w];
}

int ms_rescue_merkle_updates(ms_ctx *c, void *nodes, uint32_t depth, const uint64_t *indices,
                             const uint64_t *new_leaves, uint64_t K, void *out, uint64_t *roots) {
    if (!c) return MS_ERR_INVALID;
    if (!nodes || !indices || !new_leaves || !out || !roots)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: null argument");
    if (!K || (K & (K - 1)))
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: K = %llu is not a power of two", (unsigned long long)K);
    if (depth < 1 || depth > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: depth %u is outside 1..32", (unsigned)depth);
    u64 L = 1;
    while (L < depth) L *= 2;
    if (__builtin_ctzll(K) + __builtin_ctzll(L) + 4 > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: 16 K L rows (K = %llu, depth %u) exceed 2^32",
                    (unsigned long long)K, (unsigned)depth);
    for (u64 k = 0; k < K; k++)
        if (indices[k] >> depth)
            return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: index %llu of write %llu is not below 2^%u",
                        (unsigned long long)indices[k], (unsigned long long)k, (unsigned)depth);
    for (u64 i = 0; i < 4 * K; i++)
        if (new_leaves[i] >= GL_P)
            return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: word %llu of new leaf %llu (%llu) is not canonical",
                        (unsigned long long)(i % 4), (unsigned long long)(i / 4), (unsigned long long)new_leaves[i]);
    const u64 n = 16 * K * L;
    u64 mds[RW * RW], rc[2 * RW * RN];
    merkle_params(mds, rc);
    u64 *heap = (u64 *)nodes, *o = (u64 *)out;
    memcpy(roots, heap + 4, 4 * 8);
    for (u64 k = 0; k < K; k++) {
        const u64 idx = indices[k], leaf = (1ull << depth) + idx;
        u64 cur[2][4];                                 /* the old and the new path's current node (Montgomery) */
        for (int w = 0; w < 4; w++) {
            cur[0][w] = fp_from_canon(heap[4 * leaf + w]);
            cur[1][w] = fp_from_canon(new_leaves[4 * k + w]);
        }
        for (u64 j = 0; j < L; j++) {
            const int bit = j < depth && ((idx >> j) & 1);
            u64 sib[4] = {0};
            if (j < depth) {
                for (int w = 0; w < 4; w++) sib[w] = fp_from_canon(heap[4 * ((leaf >> j) ^ 1) + w]);
                for (int w = 0; w < 4; w++) heap[4 * (leaf >> j) + w] = fp_to_canon(cur[1][w]);   /* the write */
            }
            for (int blk = 0; blk < 2; blk++) {                 /* path 2 k + blk */
                const u64 row = 8 * (L * (2 * k + blk) + j);
                u64 s[RW] = {0};
                for (int w = 0; w < 4; w++) {
                    s[w] = bit ? sib[w] : cur[blk][w];
                    s[4 + w] = bit ? cur[blk][w] : sib[w];
                }
                update_rows(mds, rc, s, o, n, row);
                memcpy(cur[blk], s, sizeof cur[blk]);
                for (int r = 0; r < 8; r++) {
                    o[(u64)RW * n + row + r] = bit ? GL_ONE : 0;
                    o[(u64)(RW + 1) * n + row + r] = fp_from_canon(idx >> j);
                    o[(u64)(RW + 2) * n + row + r] = blk ? GL_ONE : 0;
                }
            }
            if (j + 1 == depth) {
                for (int w = 0; w < 4; w++) heap[4 + w] = roots[4 * (k + 1) + w] = fp_to_canon(cur[1][w]);
            }
        }
    }
    return MS_OK;
}
