// ctx.cuh — context object behind the C ABI (include/ministark_b200.h): device, stream,
// scratch arena, cached NTT plans.  The CUDA counterpart of the reference's Planner
// singleton (gpu/src/plan.rs:327-350): one device, one in-order queue.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <deque>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/ministark_b200.h"
#include "ntt.cuh"

namespace ms {

using gl::u32;
using gl::u64;

struct NttPlanDev;

struct Scratch {
    void *ptr = nullptr;
    size_t cap = 0;
};

}  // namespace ms

namespace ms {
struct PtrTable {
    std::vector<void *> host;   // block pointers then duplicate pointers (ms_lde_batch_scatter)
    void *dev = nullptr;
};
}  // namespace ms

struct ms_ctx {
    int device = 0;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    std::string err;
    uint64_t launches = 0;
    ms::Scratch scratch[4];            // grow-only device arenas (0: ntt tmp, 1: staging in, 2: staging out, 3: misc)
    ms::u64 *t4096[2] = {nullptr, nullptr};  // omega_4096^e forward / inverse
    std::map<std::tuple<int, unsigned, int, uint64_t, unsigned, int>, std::shared_ptr<ms::NttPlanDev>> plans;
    int64_t ntt_table_words = -1;      // "ntt_table_words": cap in words on each full table a new plan builds (-1: built-in limits)
    std::deque<ms::PtrTable> ptr_tables;       // cached device copies of LDE scatter pointer tables (deque: stable addresses)
    std::map<unsigned, ms::u64 *> tw_tables;   // log_n -> two-level g_n^e table (4096 + n/4096 words), ntt_plan_tables
    // ms_merkle_commit_block_sha256_host: block heaps are built in node_stage[k] and copied to pinned host memory on
    // node_copy_stream; node_copied[k] marks the end of the last copy out of node_stage[k] (created on first use)
    cudaStream_t node_copy_stream = nullptr;
    ms::Scratch node_stage[2];
    cudaEvent_t node_built[2] = {nullptr, nullptr}, node_copied[2] = {nullptr, nullptr};
    int node_stage_next = 0;
};

namespace ms {

int fail(ms_ctx *c, int code, const char *fmt, ...);
// failures of ms_bf_run, which takes no context: the message is ms_last_error(NULL) until the thread's next ms_bf_run
int fail_noctx(int code, const char *fmt, ...);
void clear_noctx_error();
#define MS_CUDA(ctx, expr)                                                                          \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) return ms::fail(ctx, MS_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
    } while (0)
#define MS_CHECK_LAUNCH(ctx) MS_CUDA(ctx, cudaGetLastError())

// device scratch arena `slot`, at least `bytes`
int scratch_get(ms_ctx *c, int slot, size_t bytes, void **out);
// true if the pointer is directly usable by kernels without crossing PCIe (device / managed)
bool is_device_ptr(const void *p);
// waits for the node heap copies of ms_merkle_commit_block_sha256_host; with release, also frees their staging buffers,
// stream and events (hash.cu)
int host_nodes_drain(ms_ctx *c, bool release);

// RAII staging of a possibly-host buffer: gives a device pointer, copies in/out as asked.
struct Staged {
    ms_ctx *ctx;
    void *user;
    void *dev;
    size_t bytes;
    bool staged, copy_out;
    int rc;
    Staged(ms_ctx *c, const void *p, size_t bytes, bool copy_in, bool copy_out);
    ~Staged();
    int finish();  // copies back (if needed) and frees; returns status
    template <class T>
    T *as() { return reinterpret_cast<T *>(dev); }
};

// NTT job description (api_ntt.cu)
struct NttJob {
    int field;              // 1 | 3
    unsigned log_n;
    bool inverse;
    bool bitrev_out;        // LDE mode
    unsigned log_blowup;    // cosets = 2^log_blowup (bitrev_out only; 0 otherwise)
    u64 offset;             // Montgomery
};
int ntt_get_plan(ms_ctx *c, const NttJob &job, std::shared_ptr<NttPlanDev> *out);
// two-level table of g_n^e (forward root of unity of order 2^log_n): e = 4096*e1 + e0
int ntt_plan_tables(ms_ctx *c, unsigned log_n, const u64 **tw_lo, const u64 **tw_hi, u32 *hi_len);
void ntt_drop_plans(ms_ctx *c);
// run: natural mode: in == out allowed (uses scratch 0).  LDE mode: in -> out.
// LDE scatter (ms_lde_batch_scatter): the LAST pass writes coset block q of column 0 at block_ptr[q] (device array of
// 2^log_blowup pointers, entries may be peer-device memory) with column stride block_col_stride, and a second copy at
// dup_ptr[q] (where non-null) with column stride dup_col_stride; earlier passes work in `out` as usual.
struct LdeScatter {
    u64 *const *block_ptr;
    size_t block_col_stride_words;
    u64 *const *dup_ptr;
    size_t dup_col_stride_words;
    void *const *host_block_ptr = nullptr;   // the same tables on the host (2^log_blowup entries each; dup may be null)
    void *const *host_dup_ptr = nullptr;
};
int ntt_run(ms_ctx *c, NttPlanDev &plan, const u64 *in, size_t in_col_stride_words, u64 *out,
            size_t out_col_stride_words, unsigned ncols, const LdeScatter *scatter = nullptr);

}  // namespace ms
