/*
 * ministark_rescue.h — the trace of examples/rescue built on the device: K chains of L Rescue-Prime permutations over
 * Goldilocks (state width 12, capacity 4, 7 rounds; ministark_b200/examples/rescue.py).  Conventions as in
 * ministark_b200.h (Montgomery words, column-major matrices, 0 on success, a negative MS_ERR_* otherwise; pointers may be
 * device or host memory unless a comment says otherwise).
 */
#ifndef MINISTARK_RESCUE_H
#define MINISTARK_RESCUE_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Writes `out`, the (12, n) column-major matrix of Montgomery words with n = 8 K L: chain k (rows [8 L k, 8 L (k + 1)))
 * starts from (seed[0], seed[1], seed[2], seed[3], w_K^k, 0, ..., 0), w_K the generator of the order-K subgroup of Fp*
 * (ark-ff's root of unity of order K), and applies the permutation L times; row 8 (L k + j) + r holds permutation j's
 * state before round r for r < 7 and its output at r = 7.  seed: host array of four canonical words (< p).  K and L:
 * powers of two with 8 K L <= 2^32.  Bad arguments fail with MS_ERR_INVALID and a message in ms_last_error before
 * anything is written.  Does not synchronise. */
int ms_rescue_chains(ms_ctx *ctx, const uint64_t *seed, uint64_t K, uint64_t L, void *out);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_RESCUE_H */
