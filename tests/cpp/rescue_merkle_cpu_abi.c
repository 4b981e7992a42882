/*
 * rescue_merkle_cpu_abi.c — CPU build of the examples/merkle entry points (include/ministark_rescue_merkle.h).  TEST
 * INFRASTRUCTURE ONLY, compiled by tests/test_rescue_merkle_cpu.py into a temporary directory.
 *
 * The CPU build of the chains trace (tests/cpp/rescue_cpu_abi.c, which brings the oracle's CPU ABI, the streamed
 * residency, the constraint check and ms_extension_columns) is extended by ms_rescue_merkle_tree and
 * ms_rescue_merkle_paths, so that `merkle.tree(..., device=...)`, `merkle.gen_trace(..., device=...)` and whole proofs of
 * its trace run on the CPU harness (tests/cpu_device.py).  Nodes and paths run one after another with the permutation
 * written out plainly, as in rescue_cpu_abi.c.  The product never loads this library.
 */
#include "rescue_cpu_abi.c"
#include "../../include/ministark_rescue_merkle.h"

/* the permutation of a Montgomery state, in place */
static void merkle_permute(const u64 *mds, const u64 *rc, u64 *s) {
    for (int r = 0; r < RN; r++) {
        for (int w = 0; w < RW; w++) s[w] = fp_pow(s[w], 7);
        rescue_mds_mul(mds, s);
        for (int w = 0; w < RW; w++) s[w] = fp_pow(fp_add(s[w], rc[2 * RW * r + w]), MS_RESCUE_ALPHA_INV);
        rescue_mds_mul(mds, s);
        for (int w = 0; w < RW; w++) s[w] = fp_add(s[w], rc[2 * RW * r + RW + w]);
    }
}

static void merkle_params(u64 *mds, u64 *rc) {
    for (int i = 0; i < RW * RW; i++) mds[i] = fp_from_canon(rescue_mds[i]);
    for (int i = 0; i < 2 * RW * RN; i++) rc[i] = fp_from_canon(rescue_rc[i]);
}

int ms_rescue_merkle_tree(ms_ctx *c, const uint64_t *leaves, uint32_t depth, void *nodes) {
    if (!c) return MS_ERR_INVALID;
    if (!leaves || !nodes) return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_tree: null argument");
    if (depth < 1 || depth > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_tree: depth %u is outside 1..32", (unsigned)depth);
    u64 mds[RW * RW], rc[2 * RW * RN];
    merkle_params(mds, rc);
    const u64 count = 1ull << depth;
    u64 *o = (u64 *)nodes;
    memset(o, 0, 4 * 8);
    memcpy(o + 4 * count, leaves, count * 4 * 8);
    for (u64 v = count - 1; v >= 1; v--) {
        u64 s[RW] = {0};
        for (int w = 0; w < 8; w++) s[w] = fp_from_canon(o[8 * v + w]);
        merkle_permute(mds, rc, s);
        for (int w = 0; w < 4; w++) o[4 * v + w] = fp_to_canon(s[w]);
    }
    return MS_OK;
}

int ms_rescue_merkle_paths(ms_ctx *c, const void *nodes, uint32_t depth, const uint64_t *indices, uint64_t K, void *out) {
    if (!c) return MS_ERR_INVALID;
    if (!nodes || !indices || !out) return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_paths: null argument");
    if (!K || (K & (K - 1)))
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_paths: K = %llu is not a power of two", (unsigned long long)K);
    if (depth < 1 || depth > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_paths: depth %u is outside 1..32", (unsigned)depth);
    u64 L = 1;
    while (L < depth) L *= 2;
    if (__builtin_ctzll(K) + __builtin_ctzll(L) + 3 > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_paths: 8 K L rows (K = %llu, depth %u) exceed 2^32",
                    (unsigned long long)K, (unsigned)depth);
    for (u64 k = 0; k < K; k++)
        if (indices[k] >> depth)
            return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_paths: index %llu of path %llu is not below 2^%u",
                        (unsigned long long)indices[k], (unsigned long long)k, (unsigned)depth);
    const u64 n = 8 * K * L;
    u64 mds[RW * RW], rc[2 * RW * RN];
    merkle_params(mds, rc);
    const u64 *heap = (const u64 *)nodes;
    u64 *o = (u64 *)out;
    for (u64 k = 0; k < K; k++) {
        const u64 idx = indices[k], leaf = (1ull << depth) + idx;
        u64 cur[4];
        for (int w = 0; w < 4; w++) cur[w] = fp_from_canon(heap[4 * leaf + w]);
        for (u64 j = 0; j < L; j++) {
            const u64 row = 8 * (L * k + j);
            const int bit = j < depth && ((idx >> j) & 1);
            u64 sib[4] = {0}, s[RW] = {0};
            if (j < depth)
                for (int w = 0; w < 4; w++) sib[w] = fp_from_canon(heap[4 * ((leaf >> j) ^ 1) + w]);
            for (int w = 0; w < 4; w++) {
                s[w] = bit ? sib[w] : cur[w];
                s[4 + w] = bit ? cur[w] : sib[w];
            }
            for (int r = 0; r < 8; r++) {
                o[(u64)RW * n + row + r] = bit ? GL_ONE : 0;
                o[(u64)(RW + 1) * n + row + r] = fp_from_canon(idx >> j);
            }
            for (int r = 0; r < RN; r++) {
                for (int w = 0; w < RW; w++) o[(u64)w * n + row + r] = s[w];
                for (int w = 0; w < RW; w++) s[w] = fp_pow(s[w], 7);
                rescue_mds_mul(mds, s);
                for (int w = 0; w < RW; w++) s[w] = fp_pow(fp_add(s[w], rc[2 * RW * r + w]), MS_RESCUE_ALPHA_INV);
                rescue_mds_mul(mds, s);
                for (int w = 0; w < RW; w++) s[w] = fp_add(s[w], rc[2 * RW * r + RW + w]);
            }
            for (int w = 0; w < RW; w++) o[(u64)w * n + row + 7] = s[w];
            memcpy(cur, s, sizeof cur);
        }
    }
    return MS_OK;
}
