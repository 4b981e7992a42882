/*
 * ministark_rescue_wots.h — examples/wots on the device: K Winternitz one-time signatures over Rescue-Prime
 * (ministark_b200/examples/wots.py, SignaturesClaim).  w = 16, 67 chains of 15 steps; the permutation, the digits, the
 * key derivation, the chain steps and the fold are those of the module docstring.  Words are canonical Goldilocks
 * elements unless said otherwise.  Conventions as in ministark_b200.h (column-major matrices, 0 on success, a negative
 * MS_ERR_* otherwise; pointers may be device or host memory).
 */
#ifndef MINISTARK_RESCUE_WOTS_H
#define MINISTARK_RESCUE_WOTS_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The largest K: 67 K chain blocks of 128 rows, rounded up to a power of two, fit a trace of 2^32 rows. */
#define MS_WOTS_MAX_KEYS 500812u

/* Signs messages[k] with key k for k = 0..K-1.  secrets: K x 4, seeds: K x 2 (rho_0, rho_1), messages: K x 4 row-major
 * words.  Writes signatures, K x 67 x 4 words (element i of signature k at 4 (67 k + i)), and public_keys, K x 6 words
 * (rho_0, rho_1, root_0..3).  One chain per 16 lanes derives sk_i, runs all 15 steps and keeps the value after step
 * d_i - 1; a second launch runs the K sequential 67-step folds.  1 <= K <= MS_WOTS_MAX_KEYS; a word that is not
 * canonical fails with MS_ERR_INVALID naming it, before anything is written.  Scratch is the context's own. */
int ms_rescue_wots_sign(ms_ctx *ctx, const uint64_t *secrets, const uint64_t *seeds, const uint64_t *messages,
                        uint64_t K, void *signatures, void *public_keys);

/* Writes out, the (15, n) column-major matrix of Montgomery words of SignaturesClaim(public_keys, messages) for the
 * signatures given (layouts as ms_rescue_wots_sign writes them): B = 2^ceil(log2 67 K) blocks of 128 rows, n = 128 B.
 * Block b < 67 K is chain i = b mod 67 of signature k = b div 67; row 8 s + r of it holds slot s's permutation state
 * before round r (r < 7) or its output (r = 7) in columns 0..11; column 12 is ACT ([s >= d_i] on chain slot s < 15, 0
 * on the fold slot), column 13 CNT (max(d_i - s, 0)), column 14 LAST (1 on every row of chain 66).  Blocks 67 K .. B - 1
 * are padding: digit 0, start value 0, i = rho = 0 and LAST = 1, so each is the same block, its fold on 0^4.
 * The chain ends and the roots are computed into scratch first: a signature whose root differs from its key's fails
 * with MS_ERR_INVALID, ms_last_error naming the lowest such k, and out is not written.  So do bad arguments and words
 * that are not canonical.  1 <= K <= MS_WOTS_MAX_KEYS.  Synchronises (the roots are checked first). */
int ms_rescue_wots_trace(ms_ctx *ctx, const uint64_t *public_keys, const uint64_t *messages, const uint64_t *signatures,
                         uint64_t K, void *out);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_RESCUE_WOTS_H */
