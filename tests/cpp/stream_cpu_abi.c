/*
 * stream_cpu_abi.c — CPU build of the streamed-residency entry points (include/ministark_stream.h).  TEST
 * INFRASTRUCTURE ONLY, compiled by tests/test_stream_prover_cpu.py into a temporary directory.
 *
 * The CPU build of the C ABI (oracle/cpu_abi.c, included whole below) is extended by the two entry points of the
 * streamed prover, so that `GpuProver`'s streamed path runs end to end on the CPU harness (tests/cpu_device.py) and is
 * byte-compared with the restated reference prover.  The product never loads this library.
 */
#include "../../oracle/cpu_abi.c"
#include "../../include/ministark_stream.h"

/* one coset block of a tree committed block by block: the block's own heap, then each of its levels copied to its run of
 * the global heap (local level [cnt, 2 cnt) -> global [cnt * beta + block * cnt, ...)) */
int ms_merkle_commit_block_sha256(ms_ctx *c, int field, const void *cols, size_t stride, unsigned ncols, unsigned log_block_rows,
                                  unsigned log_blocks, size_t block, void *nodes, void *block_root) {
    if (!c || !cols || !nodes || !block_root) return MS_ERR_INVALID;
    if (bad_field(field)) return fail(c, MS_ERR_INVALID, "unknown field id %d", field);
    if (ncols == 0) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256: no columns");
    if (log_block_rows + log_blocks > 40) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256: tree too large");
    if (block >> log_blocks) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256: block %zu of %zu", block, (size_t)1 << log_blocks);
    const size_t nb = (size_t)1 << log_block_rows, beta = (size_t)1 << log_blocks;
    uint8_t *lv = (uint8_t *)malloc(nb * 32), *loc = (uint8_t *)malloc(nb * 32);
    if (!lv || !loc) { free(lv); free(loc); return fail(c, MS_ERR_NOMEM, "out of host memory"); }
    const double t0 = now_s();
    orc_hash_rows((const u64 *)cols, stride * field, ncols, (unsigned)field, nb, lv);
    if (nb == 1) {
        memcpy(block_root, lv, 32);
    } else {
        orc_merkle_nodes(lv, nb, loc);
        for (size_t cnt = nb / 2; cnt >= 1; cnt >>= 1)
            memcpy((uint8_t *)nodes + 32 * (cnt * beta + block * cnt), loc + 32 * cnt, 32 * cnt);
        memcpy(block_root, loc + 32, 32);
    }
    free(lv);
    free(loc);
    return done(c, "ms_merkle_commit_block", t0);
}
/* rows of the bit-reversed coset LDE by their definition: P_c(offset * g_N^bitrev(pos)), one Horner per (row, column) */
int ms_lde_rows(ms_ctx *c, int field, const void *coeffs, size_t stride, unsigned ncols, unsigned log_n, unsigned log_blowup, uint64_t offset,
                const uint64_t *positions, unsigned npos, void *out) {
    if (!c || !coeffs || !positions || !out) return MS_ERR_INVALID;
    if (bad_field(field)) return fail(c, MS_ERR_INVALID, "unknown field id %d", field);
    if (log_n + log_blowup > 32) return fail(c, MS_ERR_INVALID, "ms_lde_rows: log_n + log_blowup > 32");
    int rc = check_offset(c, offset);
    if (rc) return rc;
    const unsigned log_N = log_n + log_blowup;
    const size_t n = (size_t)1 << log_n;
    for (unsigned q = 0; q < npos; q++)
        if (positions[q] >> log_N) return fail(c, MS_ERR_INVALID, "ms_lde_rows: row %llu out of range", (unsigned long long)positions[q]);
    const double t0 = now_s();
    const u64 g = orc_root_of_unity(log_N);
    const size_t f = (size_t)field;
    #pragma omp parallel for schedule(dynamic)
    for (size_t job = 0; job < (size_t)npos * ncols; job++) {
        const size_t q = job / ncols, col = job % ncols;
        const u64 pt[3] = {fp_mul(offset, fp_pow(g, log_N ? bitrev(positions[q], log_N) : 0)), 0, 0};
        u64 r[3];
        orc_horner((const u64 *)coeffs + col * stride * f, (unsigned)field, n, pt, r);
        memcpy((u64 *)out + job * f, r, 8 * f);
    }
    return done(c, "ms_lde_rows", t0);
}

