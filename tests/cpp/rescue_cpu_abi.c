/*
 * rescue_cpu_abi.c — CPU build of the examples/rescue trace entry point (include/ministark_rescue.h).  TEST
 * INFRASTRUCTURE ONLY, compiled by tests/test_rescue_cpu.py into a temporary directory.
 *
 * The CPU build of the declared extension columns (tests/cpp/extension_cpu_abi.c: the oracle's CPU ABI, the streamed
 * residency, the constraint check and ms_extension_columns) is extended by ms_rescue_chains, so that
 * `rescue.gen_trace(..., device=...)` and whole proofs of its trace run on the CPU harness (tests/cpu_device.py).  The
 * chains run one after another, word by word, with the permutation written out plainly: x^7, the MDS product as a
 * matrix-vector loop, and x^(1/7) by square-and-multiply over the exponent's bits.  The product never loads this library.
 */
#include "extension_cpu_abi.c"
#include "../../include/ministark_rescue.h"
#include "../../ministark_b200/csrc/rescue_params.cuh"

enum { RW = MS_RESCUE_WIDTH, RN = MS_RESCUE_ROUNDS };

static const u64 rescue_rc[2 * RW * RN] = MS_RESCUE_RC;
static const u64 rescue_mds[RW * RW] = MS_RESCUE_MDS;

static void rescue_mds_mul(const u64 *m, u64 *s) {
    u64 t[RW];
    for (int i = 0; i < RW; i++) {
        t[i] = 0;
        for (int j = 0; j < RW; j++) t[i] = fp_add(t[i], fp_mul(m[i * RW + j], s[j]));
    }
    memcpy(s, t, sizeof t);
}

int ms_rescue_chains(ms_ctx *c, const uint64_t *seed, uint64_t K, uint64_t L, void *out) {
    if (!c) return MS_ERR_INVALID;
    if (!seed || !out) return fail(c, MS_ERR_INVALID, "ms_rescue_chains: null argument");
    if (!K || (K & (K - 1)) || !L || (L & (L - 1)))
        return fail(c, MS_ERR_INVALID, "ms_rescue_chains: K = %llu and L = %llu must be powers of two",
                    (unsigned long long)K, (unsigned long long)L);
    if (__builtin_ctzll(K) + __builtin_ctzll(L) + 3 > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_chains: 8 K L rows (K = %llu, L = %llu) exceed 2^32",
                    (unsigned long long)K, (unsigned long long)L);
    for (int w = 0; w < 4; w++)
        if (seed[w] >= GL_P) return fail(c, MS_ERR_INVALID, "ms_rescue_chains: seed word %d (%llu) is not canonical", w,
                                         (unsigned long long)seed[w]);
    const u64 n = 8 * K * L;
    u64 mds[RW * RW], rc[2 * RW * RN];
    for (int i = 0; i < RW * RW; i++) mds[i] = fp_from_canon(rescue_mds[i]);
    for (int i = 0; i < 2 * RW * RN; i++) rc[i] = fp_from_canon(rescue_rc[i]);
    const u64 root = fp_pow(fp_from_canon(GL_TWO_ADIC_ROOT_CANON), 1ull << (32 - __builtin_ctzll(K)));
    u64 *o = (u64 *)out, tag = GL_ONE;
    for (u64 k = 0; k < K; k++, tag = fp_mul(tag, root)) {
        u64 s[RW] = {0};
        for (int w = 0; w < 4; w++) s[w] = fp_from_canon(seed[w]);
        s[4] = tag;
        for (u64 j = 0; j < L; j++) {
            const u64 row = 8 * (L * k + j);
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
