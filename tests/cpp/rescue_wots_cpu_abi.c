/*
 * rescue_wots_cpu_abi.c — CPU build of examples/wots's entry points (include/ministark_rescue_wots.h).  TEST
 * INFRASTRUCTURE ONLY, compiled by tests/test_rescue_wots_cpu.py into a temporary directory.
 *
 * The CPU build of the transfer entry point (tests/cpp/rescue_rollup_cpu_abi.c, which brings the write, tree, paths
 * and chains entry points, the oracle's CPU ABI, the streamed residency, the constraint check and
 * ms_extension_columns) is extended by ms_rescue_wots_sign and ms_rescue_wots_trace, so that
 * `wots.sign_batch(..., device=...)`, `wots.gen_trace(..., device=...)` and whole proofs of its trace run on the CPU
 * harness (tests/cpu_device.py).  Keys, chains and blocks are processed one after another with the permutation written
 * out plainly; the trace is built in a buffer of its own and copied out only once every root has matched.  The product
 * never loads this library.
 */
#include "rescue_rollup_cpu_abi.c"
#include "../../include/ministark_rescue_wots.h"

enum { WOTS_CHAINS = 67, WOTS_STEPS = 15 };

static unsigned wots_digit_cpu(const u64 *m, unsigned i) {
    if (i < 64) return (unsigned)(m[i / 16] >> (4 * (i % 16))) & 15;
    unsigned c = 0;
    for (unsigned j = 0; j < 64; j++) c += 15 - wots_digit_cpu(m, j);
    return (c >> (4 * (i - 64))) & 15;
}

/* the Montgomery state (x || tail || tweak, i, rho_0, rho_1) from canonical words */
static void wots_state(u64 *s, const u64 *x, const u64 *tail, u64 tweak, u64 i, const u64 *rho) {
    for (int w = 0; w < 4; w++) {
        s[w] = x[w];
        s[4 + w] = tail ? tail[w] : 0;
    }
    s[8] = fp_from_canon(tweak);
    s[9] = fp_from_canon(i);
    s[10] = rho ? fp_from_canon(rho[0]) : 0;
    s[11] = rho ? fp_from_canon(rho[1]) : 0;
}

static int wots_first_bad(const u64 *v, u64 count) {
    for (u64 t = 0; t < count; t++)
        if (v[t] >= GL_P) return (int)t;
    return -1;
}

int ms_rescue_wots_sign(ms_ctx *c, const uint64_t *secrets, const uint64_t *seeds, const uint64_t *messages, uint64_t K,
                        void *signatures, void *public_keys) {
    if (!c) return MS_ERR_INVALID;
    if (!secrets || !seeds || !messages || !signatures || !public_keys)
        return fail(c, MS_ERR_INVALID, "ms_rescue_wots_sign: null argument");
    if (K < 1 || K > MS_WOTS_MAX_KEYS)
        return fail(c, MS_ERR_INVALID, "ms_rescue_wots_sign: K = %llu is outside 1..%u", (unsigned long long)K,
                    MS_WOTS_MAX_KEYS);
    const u64 *arrays[3] = {secrets, seeds, messages}, sizes[3] = {4 * K, 2 * K, 4 * K}, widths[3] = {4, 2, 4};
    const char *names[3] = {"secret", "seed", "message"};
    for (int q = 0; q < 3; q++) {
        const int t = wots_first_bad(arrays[q], sizes[q]);
        if (t >= 0)
            return fail(c, MS_ERR_INVALID, "ms_rescue_wots_sign: word %llu of %s %llu (%llu) is not canonical",
                        (unsigned long long)(t % widths[q]), names[q], (unsigned long long)(t / widths[q]),
                        (unsigned long long)arrays[q][t]);
    }
    u64 mds[RW * RW], rc[2 * RW * RN];
    merkle_params(mds, rc);
    u64 *sig = (u64 *)signatures, *pk = (u64 *)public_keys;
    for (u64 k = 0; k < K; k++) {
        u64 acc[4] = {0, 0, 0, 0};
        for (unsigned i = 0; i < WOTS_CHAINS; i++) {
            const unsigned d = wots_digit_cpu(messages + 4 * k, i);
            u64 x[4], s[RW];
            for (int w = 0; w < 4; w++) x[w] = fp_from_canon(secrets[4 * k + w]);
            wots_state(s, x, NULL, 16, i, seeds + 2 * k);
            merkle_permute(mds, rc, s);
            for (unsigned st = 0; st <= WOTS_STEPS; st++) {
                if (st == d)
                    for (int w = 0; w < 4; w++) sig[4 * (WOTS_CHAINS * k + i) + w] = fp_to_canon(s[w]);
                if (st == WOTS_STEPS) break;
                memcpy(x, s, 32);
                wots_state(s, x, NULL, 1 + st, i, seeds + 2 * k);
                merkle_permute(mds, rc, s);
            }
            memcpy(x, s, 32);
            wots_state(s, x, acc, 0, i, seeds + 2 * k);
            merkle_permute(mds, rc, s);
            memcpy(acc, s, 32);
        }
        pk[6 * k] = seeds[2 * k];
        pk[6 * k + 1] = seeds[2 * k + 1];
        for (int w = 0; w < 4; w++) pk[6 * k + 2 + w] = fp_to_canon(acc[w]);
    }
    return MS_OK;
}

int ms_rescue_wots_trace(ms_ctx *c, const uint64_t *public_keys, const uint64_t *messages, const uint64_t *signatures,
                         uint64_t K, void *out) {
    if (!c) return MS_ERR_INVALID;
    if (!public_keys || !messages || !signatures || !out)
        return fail(c, MS_ERR_INVALID, "ms_rescue_wots_trace: null argument");
    if (K < 1 || K > MS_WOTS_MAX_KEYS)
        return fail(c, MS_ERR_INVALID, "ms_rescue_wots_trace: K = %llu is outside 1..%u", (unsigned long long)K,
                    MS_WOTS_MAX_KEYS);
    const u64 *arrays[3] = {public_keys, messages, signatures}, sizes[3] = {6 * K, 4 * K, 4 * WOTS_CHAINS * K},
              widths[3] = {6, 4, 4};
    const char *names[3] = {"public key", "message", "signature element"};
    for (int q = 0; q < 3; q++) {
        const int t = wots_first_bad(arrays[q], sizes[q]);
        if (t < 0) continue;
        const u64 item = (u64)t / widths[q];
        if (q == 2)
            return fail(c, MS_ERR_INVALID, "ms_rescue_wots_trace: word %llu of element %llu of signature %llu (%llu) is "
                        "not canonical", (unsigned long long)(t % 4), (unsigned long long)(item % WOTS_CHAINS),
                        (unsigned long long)(item / WOTS_CHAINS), (unsigned long long)arrays[q][t]);
        return fail(c, MS_ERR_INVALID, "ms_rescue_wots_trace: word %llu of %s %llu (%llu) is not canonical",
                    (unsigned long long)(t % widths[q]), names[q], (unsigned long long)item,
                    (unsigned long long)arrays[q][t]);
    }
    u64 B = 1;
    while (B < WOTS_CHAINS * K) B *= 2;
    const u64 n = 128 * B;
    u64 mds[RW * RW], rc[2 * RW * RN];
    merkle_params(mds, rc);
    u64 *o = (u64 *)calloc((size_t)(RW + 3) * n, 8);
    u64 acc[4] = {0, 0, 0, 0};
    int rc_out = MS_OK;
    for (u64 b = 0; b < B && rc_out == MS_OK; b++) {
        const u64 k = b / WOTS_CHAINS;
        const int real = k < K;
        const unsigned i = real ? (unsigned)(b % WOTS_CHAINS) : 0, d = real ? wots_digit_cpu(messages + 4 * k, i) : 0;
        const u64 *rho = real ? public_keys + 6 * k : NULL;
        const u64 last = !real || i == WOTS_CHAINS - 1 ? GL_ONE : 0;     /* padding blocks have LAST = 1 */
        u64 x[4] = {0, 0, 0, 0}, s[RW];
        for (int w = 0; w < 4 && real; w++) x[w] = fp_from_canon(signatures[4 * b + w]);
        for (unsigned st = 0; st <= WOTS_STEPS; st++) {
            const u64 row = 128 * b + 8 * st;
            wots_state(s, x, st == WOTS_STEPS ? acc : NULL, st == WOTS_STEPS ? 0 : 1 + st, i, rho);
            update_rows(mds, rc, s, o, n, row);
            if (st < WOTS_STEPS && st >= d) memcpy(x, s, 32);
            for (int r = 0; r < 8; r++) {
                o[(u64)RW * n + row + r] = st < WOTS_STEPS && st >= d ? GL_ONE : 0;
                o[(u64)(RW + 1) * n + row + r] = fp_from_canon(st < d ? d - st : 0);
                o[(u64)(RW + 2) * n + row + r] = last;
            }
        }
        for (int w = 0; w < 4; w++) acc[w] = last ? 0 : s[w];
        if (last && real)
            for (int w = 0; w < 4; w++)
                if (fp_to_canon(s[w]) != public_keys[6 * k + 2 + w]) {
                    rc_out = fail(c, MS_ERR_INVALID, "ms_rescue_wots_trace: signature %llu does not verify: its root "
                                  "differs from its public key", (unsigned long long)k);
                    break;
                }
    }
    if (rc_out == MS_OK) memcpy(out, o, (size_t)(RW + 3) * n * 8);
    free(o);
    return rc_out;
}
