/*
 * ministark_rescue_hash.h — the trace of examples/rescue's hash claim built on the device: K messages of one length
 * absorbed by the Rescue-Prime sponge over Goldilocks (state width 12, rate 8, capacity 4, 7 rounds;
 * ministark_b200/examples/rescue.py, RescueHashClaim).  Conventions as in ministark_b200.h (Montgomery words,
 * column-major matrices, 0 on success, a negative MS_ERR_* otherwise; pointers may be device or host memory unless a
 * comment says otherwise).
 */
#ifndef MINISTARK_RESCUE_HASH_H
#define MINISTARK_RESCUE_HASH_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Writes `out`, the (13, n) column-major matrix of Montgomery words with n = 8 K L, B = length / 8 + 1 blocks per
 * padded message and L the smallest power of two >= B.  Message k (rows [8 L k, 8 L (k + 1))) is padded with one 1 and
 * zeros to B blocks of 8 words, then zero blocks up to L; the sponge starts from the all-zero state and, for j = 0..L-1,
 * adds block j into words 0..7 and permutes.  Columns 0..11: row 8 (L k + j) + r holds permutation j's state before
 * round r for r < 7 (block j added) and its output at r = 7, so message k's digest is words 0..3 of row
 * 8 L k + 8 B - 1.  Column 12: row 8 (L k + j) + i holds word i of block j.
 * messages: K x length canonical words, row-major; may be null when length = 0.  K: a power of two with n <= 2^32.  Bad
 * arguments fail with MS_ERR_INVALID and a message in ms_last_error before anything is written.  Does not synchronise. */
int ms_rescue_hash(ms_ctx *ctx, const uint64_t *messages, uint64_t K, uint64_t length, void *out);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_RESCUE_HASH_H */
