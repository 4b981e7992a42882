/*
 * host_nodes_cpu_abi.c — CPU build of include/ministark_host_nodes.h.  TEST INFRASTRUCTURE ONLY, compiled by
 * tests/test_host_nodes_cpu.py into a temporary directory.
 *
 * The top of the CPU ABI chain (tests/cpp/device_cpu_abi.c: the oracle's CPU ABI with the streamed residency, the
 * constraint check, the brainfuck trace and ms_device_memory) is extended by the host-heap block commitment, so that the
 * "streamed_host" residency of the Python and C++ provers runs end to end without a GPU.  Every buffer is host memory
 * here, so the subtree is written in place and there is nothing to overlap or refuse.  The product never loads this
 * library.
 */
#include "device_cpu_abi.c"
#include "../../include/ministark_host_nodes.h"

/* the block's local heap (slot 0 zero, slot 1 the block root), as ms_merkle_commit_sha256 lays out a 2^log_block_rows-row tree */
int ms_merkle_commit_block_sha256_host(ms_ctx *c, int field, const void *cols, size_t stride, unsigned ncols, unsigned log_block_rows,
                                       void *host_subtree, void *block_root) {
    if (!c || !cols || !host_subtree || !block_root) return MS_ERR_INVALID;
    if (bad_field(field)) return fail(c, MS_ERR_INVALID, "unknown field id %d", field);
    if (ncols == 0) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256_host: no columns");
    if (log_block_rows > 36) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256_host: block too large");
    const size_t nb = (size_t)1 << log_block_rows;
    if (ncols > 1 && stride < nb) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256_host: stride < block rows");
    uint8_t *lv = (uint8_t *)malloc(nb * 32);
    if (!lv) return fail(c, MS_ERR_NOMEM, "out of host memory");
    const double t0 = now_s();
    orc_hash_rows((const u64 *)cols, stride * field, ncols, (unsigned)field, nb, lv);
    if (nb == 1) {
        memset(host_subtree, 0, 32);
        memcpy(block_root, lv, 32);
    } else {
        orc_merkle_nodes(lv, nb, (uint8_t *)host_subtree);     /* slot 0 zeroed */
        memcpy(block_root, (uint8_t *)host_subtree + 32, 32);
    }
    free(lv);
    return done(c, "ms_merkle_commit_block_host", t0);
}
