/*
 * rescue_hash_cpu_abi.c — CPU build of the examples/rescue hash-trace entry point (include/ministark_rescue_hash.h).
 * TEST INFRASTRUCTURE ONLY, compiled by tests/test_rescue_hash_cpu.py into a temporary directory.
 *
 * The CPU build of the chains trace (tests/cpp/rescue_cpu_abi.c, which brings the oracle's CPU ABI, the streamed
 * residency, the constraint check and ms_extension_columns) is extended by ms_rescue_hash, so that
 * `rescue.gen_hash_trace(..., device=...)` and whole proofs of its trace run on the CPU harness (tests/cpu_device.py).
 * The messages run one after another with the permutation written out plainly, as in rescue_cpu_abi.c.  The product
 * never loads this library.
 */
#include "rescue_cpu_abi.c"
#include "../../include/ministark_rescue_hash.h"

int ms_rescue_hash(ms_ctx *c, const uint64_t *messages, uint64_t K, uint64_t length, void *out) {
    if (!c) return MS_ERR_INVALID;
    if (!out || (!messages && length)) return fail(c, MS_ERR_INVALID, "ms_rescue_hash: null argument");
    if (!K || (K & (K - 1))) return fail(c, MS_ERR_INVALID, "ms_rescue_hash: K = %llu is not a power of two", (unsigned long long)K);
    const u64 B = length / 8 + 1;
    u64 L = 1;
    while (L < B) L *= 2;
    if (__builtin_ctzll(K) + __builtin_ctzll(L) + 3 > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_hash: 8 K L rows (K = %llu, length = %llu) exceed 2^32",
                    (unsigned long long)K, (unsigned long long)length);
    const u64 n = 8 * K * L;
    u64 mds[RW * RW], rc[2 * RW * RN];
    for (int i = 0; i < RW * RW; i++) mds[i] = fp_from_canon(rescue_mds[i]);
    for (int i = 0; i < 2 * RW * RN; i++) rc[i] = fp_from_canon(rescue_rc[i]);
    u64 *o = (u64 *)out;
    for (u64 k = 0; k < K; k++) {
        u64 s[RW] = {0};
        for (u64 j = 0; j < L; j++) {
            const u64 row = 8 * (L * k + j);
            for (int i = 0; i < 8; i++) {
                const u64 p = 8 * j + i;
                const u64 m = p < length ? fp_from_canon(messages[k * length + p]) : p == length ? GL_ONE : 0;
                o[(u64)RW * n + row + i] = m;
                s[i] = fp_add(s[i], m);
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
        }
    }
    return MS_OK;
}
