/*
 * ministark_rescue_rollup.h — examples/rollup's state transition on the device: K balance transfers over the accounts
 * of a Rescue-Prime Merkle tree (ministark_b200/examples/rollup.py, TransfersClaim).  The tree, its node function and
 * its heap layout are those of include/ministark_rescue_merkle.h: node 1 is the root, node 2^D + i is leaf i.  Leaf i
 * is account i, four canonical words (balance, nonce, owner_0, owner_1).  Conventions as in ministark_b200.h
 * (column-major matrices, 0 on success, a negative MS_ERR_* otherwise; pointers may be device or host memory).
 */
#ifndef MINISTARK_RESCUE_ROLLUP_H
#define MINISTARK_RESCUE_ROLLUP_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Applies K transfers to the heap `nodes` (depth D), one after another.  transfers: K x 3 row-major words (sender,
 * receiver, amount), both accounts < 2^D and amount < 2^32; sender == receiver is allowed.  Transfer k is two leaf
 * writes: write 2 k (the sender step) sets the sender's balance to balance - amount and its nonce to nonce + 1, then
 * write 2 k + 1 (the receiver step) sets the receiver's balance to balance + amount; both keep the owner words, and
 * arithmetic is mod p.  Writes
 *   out:   the (23, n) column-major matrix of Montgomery words, n = 32 K L with L the smallest power of two >= D.
 *          Columns 0..14 are exactly what ms_rescue_merkle_updates writes for the 2 K writes (write w's old path at rows
 *          16 L w, its new path at 16 L w + 8 L).  On row 16 L w (write w's old path's first row), and 0 on every other
 *          row: column 15 DELTA, -amount (sender) or +amount (receiver) as a field element; column 16 NINC, 1 (sender)
 *          or 0; columns 17..20 B0..B3, the four 8-bit limbs of write w's new balance, least significant first.
 *          Column 21 (M, the range lookup's multiplicities) is 0 for the prover to fill.  Column 22 (TBL) is
 *          min(row, 255).
 *   roots: (K + 1) x 4 canonical words: roots[0] the root before transfer 0, roots[k + 1] the root after transfer k.
 *   nodes: the heap after all K transfers, in place.
 * Balances are resolved for all 2 K writes at once: a stable radix sort of the writes by account (D key bits), one
 * segmented inclusive scan of (delta, nonce increment) in write order within each account, then one launch that forms
 * every new leaf and finds the first write whose new balance is not below 2^32.  The trace then comes from
 * ms_rescue_merkle_updates on the 2 K writes, and one launch fills columns 15..22.
 * K a power of two, 1 <= D <= 32 and 256 <= n <= 2^32.  Bad arguments, an account index >= 2^D or an amount >= 2^32
 * fail with MS_ERR_INVALID.  So does an invalid batch: when a write leaves a balance that is not below 2^32 as a
 * canonical field element, ms_last_error names the first such write's transfer, its step (sender or receiver), the
 * account and the balance.  Every failure comes before anything is written: the heap, out and roots are untouched.
 * Scratch is the context's own.  Synchronises (the arguments and the balances are checked first). */
int ms_rescue_rollup(ms_ctx *ctx, void *nodes, uint32_t depth, const uint64_t *transfers, uint64_t K, void *out,
                     uint64_t *roots);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_RESCUE_ROLLUP_H */
