/*
 * rescue_rollup_cpu_abi.c — CPU build of examples/rollup's transfer entry point (include/ministark_rescue_rollup.h).
 * TEST INFRASTRUCTURE ONLY, compiled by tests/test_rescue_rollup_cpu.py into a temporary directory.
 *
 * The CPU build of the write entry point (tests/cpp/rescue_merkle_updates_cpu_abi.c, which brings the tree, the paths,
 * the chains trace, the oracle's CPU ABI, the streamed residency, the constraint check and ms_extension_columns) is
 * extended by ms_rescue_rollup, so that `rollup.apply(..., device=...)` and whole proofs of its trace run on the CPU
 * harness (tests/cpu_device.py).  The transfers are applied one after another in plain sequential code; none of the
 * device's sort and scans is used.  The tests link it with tests/cpp/lookup_cpu_abi.c, which fills the range lookup's
 * multiplicities.  The product never loads this library.
 */
#include "rescue_merkle_updates_cpu_abi.c"
#include "../../include/ministark_rescue_rollup.h"

int ms_rescue_rollup(ms_ctx *c, void *nodes, uint32_t depth, const uint64_t *transfers, uint64_t K, void *out,
                     uint64_t *roots) {
    if (!c) return MS_ERR_INVALID;
    if (!nodes || !transfers || !out || !roots) return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: null argument");
    if (!K || (K & (K - 1)))
        return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: K = %llu is not a power of two", (unsigned long long)K);
    if (depth < 1 || depth > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: depth %u is outside 1..32", (unsigned)depth);
    u64 L = 1;
    while (L < depth) L *= 2;
    const int log_n = __builtin_ctzll(K) + __builtin_ctzll(L) + 5;
    if (log_n > 32 || log_n < 8)
        return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: 32 K L rows (K = %llu, depth %u) are not in 2^8..2^32",
                    (unsigned long long)K, (unsigned)depth);
    for (u64 i = 0; i < 2 * K; i++)
        if (transfers[3 * (i / 2) + i % 2] >> depth)
            return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: %s %llu of transfer %llu is not below 2^%u",
                        i % 2 ? "receiver" : "sender", (unsigned long long)transfers[3 * (i / 2) + i % 2],
                        (unsigned long long)(i / 2), (unsigned)depth);
    for (u64 k = 0; k < K; k++)
        if (transfers[3 * k + 2] >> 32)
            return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: amount %llu of transfer %llu is not below 2^32",
                        (unsigned long long)transfers[3 * k + 2], (unsigned long long)k);
    const u64 n = 1ull << log_n, W = 2 * K;
    u64 *heap = (u64 *)nodes, *o = (u64 *)out;
    /* the accounts as the writes leave them, on a copy of the leaves so that a refused batch writes nothing */
    u64 *leaves = (u64 *)malloc((size_t)(1ull << depth) * 32), *idx = (u64 *)malloc(W * 8),
        *vals = (u64 *)malloc(W * 32), *delta = (u64 *)malloc(W * 8), *wroots = (u64 *)malloc((W + 1) * 32);
    memcpy(leaves, heap + 4 * (1ull << depth), (size_t)(1ull << depth) * 32);
    int rc = MS_OK;
    for (u64 w = 0; w < W && rc == MS_OK; w++) {
        const u64 k = w / 2, acc = transfers[3 * k + w % 2], amount = transfers[3 * k + 2];
        u64 *lf = leaves + 4 * acc;
        idx[w] = acc;
        delta[w] = w % 2 ? amount : (GL_P - amount) % GL_P;
        lf[0] = fp_to_canon(fp_add(fp_from_canon(lf[0]), fp_from_canon(delta[w])));
        if (w % 2 == 0) lf[1] = fp_to_canon(fp_add(fp_from_canon(lf[1]), fp_from_canon(1)));
        if (lf[0] >> 32)
            rc = fail(c, MS_ERR_INVALID, "ms_rescue_rollup: the %s step of transfer %llu leaves account %llu with balance "
                      "%llu, not below 2^32", w % 2 ? "receiver" : "sender", (unsigned long long)k,
                      (unsigned long long)acc, (unsigned long long)lf[0]);
        memcpy(vals + 4 * w, lf, 32);
    }
    if (rc == MS_OK) rc = ms_rescue_merkle_updates(c, heap, depth, idx, vals, W, o, wroots);
    if (rc == MS_OK) {
        for (u64 k = 0; k <= K; k++) memcpy(roots + 4 * k, wroots + 8 * k, 32);
        for (u64 i = 0; i < n; i++) {
            for (int col = RW + 3; col < RW + 10; col++) o[(u64)col * n + i] = 0;
            o[(u64)(RW + 10) * n + i] = fp_from_canon(i < 255 ? i : 255);
        }
        for (u64 w = 0; w < W; w++) {
            const u64 row = 16 * L * w, b = vals[4 * w];
            o[(u64)(RW + 3) * n + row] = fp_from_canon(delta[w]);
            o[(u64)(RW + 4) * n + row] = w % 2 ? 0 : GL_ONE;
            for (int q = 0; q < 4; q++) o[(u64)(RW + 5 + q) * n + row] = fp_from_canon((b >> (8 * q)) & 255);
        }
    }
    free(leaves);
    free(idx);
    free(vals);
    free(delta);
    free(wroots);
    return rc;
}
