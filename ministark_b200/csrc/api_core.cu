// api_core.cu — context, memory, staging and small utility kernels behind the C ABI.
#include <cstring>

#include "../../include/ministark_device.h"
#include "ctx.cuh"

namespace ms {

int fail(ms_ctx *c, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (c) c->err = buf;
    return code;
}

// the message of the context-free entry point ms_bf_run on this thread, if its last call failed: ms_last_error(NULL)
static thread_local std::string t_noctx_err;

int fail_noctx(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    t_noctx_err = buf;
    return code;
}

void clear_noctx_error() { t_noctx_err.clear(); }

int scratch_get(ms_ctx *c, int slot, size_t bytes, void **out) {
    Scratch &s = c->scratch[slot];
    if (s.cap < bytes) {
        if (s.ptr) {
            MS_CUDA(c, cudaStreamSynchronize(c->stream));
            MS_CUDA(c, cudaFree(s.ptr));
            s.ptr = nullptr;
            s.cap = 0;
        }
        size_t want = bytes + (bytes >> 3);
        cudaError_t e = cudaMalloc(&s.ptr, want);
        if (e != cudaSuccess) {
            want = bytes;
            e = cudaMalloc(&s.ptr, want);
        }
        if (e != cudaSuccess) {
            s.ptr = nullptr;
            cudaGetLastError();
            return fail(c, MS_ERR_NOMEM, "scratch %d: cudaMalloc(%zu) failed: %s", slot, bytes, cudaGetErrorString(e));
        }
        s.cap = want;
    }
    *out = s.ptr;
    return MS_OK;
}

bool is_device_ptr(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

Staged::Staged(ms_ctx *c, const void *p, size_t nbytes, bool copy_in, bool copy_out_)
    : ctx(c), user(const_cast<void *>(p)), dev(nullptr), bytes(nbytes), staged(false), copy_out(copy_out_), rc(MS_OK) {
    cudaSetDevice(c->device);   // every entry point builds a Staged first: the context's device becomes current
    if (p == nullptr || nbytes == 0 || is_device_ptr(p)) {
        dev = user;
        return;
    }
    staged = true;
    cudaError_t e = cudaMalloc(&dev, nbytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        dev = nullptr;
        rc = fail(c, MS_ERR_NOMEM, "staging cudaMalloc(%zu): %s", nbytes, cudaGetErrorString(e));
        return;
    }
    if (copy_in) {
        e = cudaMemcpyAsync(dev, user, nbytes, cudaMemcpyHostToDevice, c->stream);
        if (e != cudaSuccess) rc = fail(c, MS_ERR_CUDA, "staging H2D: %s", cudaGetErrorString(e));
    }
}
int Staged::finish() {
    if (!staged || dev == nullptr) return rc;
    if (rc == MS_OK && copy_out) {
        cudaError_t e = cudaMemcpyAsync(user, dev, bytes, cudaMemcpyDeviceToHost, ctx->stream);
        if (e != cudaSuccess) rc = fail(ctx, MS_ERR_CUDA, "staging D2H: %s", cudaGetErrorString(e));
    }
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess && rc == MS_OK) rc = fail(ctx, MS_ERR_CUDA, "staging sync: %s", cudaGetErrorString(e));
    cudaFree(dev);
    dev = nullptr;
    return rc;
}
Staged::~Staged() {
    if (staged && dev) {
        cudaStreamSynchronize(ctx->stream);
        cudaFree(dev);
    }
}

// ------------------------------------------------------------------------------------------
__global__ void fill_random_kernel(u64 *dst, size_t n, u64 seed) {
    // one splitmix64 stream per word (seeded by (seed, i)), rejecting draws >= p: uniform over
    // F_p and independent of the launch shape.
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    u64 s = seed ^ (0xD1B54A32D192ED03ULL * (u64)(i + 1));
    u64 z;
    do {
        s += 0x9E3779B97F4A7C15ULL;
        z = s;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
        z ^= z >> 31;
    } while (z >= gl::P);
    dst[i] = gl::to_mont(z);
}

template <int EW>
__global__ void bit_reverse_kernel(u64 *data, unsigned log_n, size_t col_stride_words) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    size_t n = (size_t)1 << log_n;
    if (i >= n) return;
    size_t j = log_n ? (__brevll(i) >> (64 - log_n)) : 0;
    if (j <= i) return;
    u64 *col = data + (size_t)blockIdx.y * col_stride_words;
#pragma unroll
    for (int w = 0; w < EW; w++) {
        u64 a = col[i * EW + w], b = col[j * EW + w];
        col[i * EW + w] = b;
        col[j * EW + w] = a;
    }
}

}  // namespace ms

using namespace ms;

extern "C" {

const char *ms_version(void) { return "ministark_b200 0.1 (sm_90a)"; }

int ms_ctx_create(int device, ms_ctx **out) {
    if (!out) return MS_ERR_INVALID;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
        cudaGetLastError();
        return MS_ERR_NODEVICE;
    }
    if (device < 0 || device >= count) return MS_ERR_INVALID;
    if (cudaSetDevice(device) != cudaSuccess) return MS_ERR_CUDA;
    ms_ctx *c = new ms_ctx();
    c->device = device;
    if (cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete c;
        return MS_ERR_CUDA;
    }
    c->stream = c->own_stream;
    // omega_4096^e tables, forward and inverse
    {
        std::vector<u64> h(2 * 4096);
        u64 w = gl::to_mont(1753635133440165772ULL);
        for (int i = 12; i < 32; i++) w = gl::sqr(w);
        u64 wi = gl::inv(w);
        u64 a = gl::ONE, b = gl::ONE;
        for (int e = 0; e < 4096; e++) {
            h[e] = a;
            h[4096 + e] = b;
            a = gl::mul(a, w);
            b = gl::mul(b, wi);
        }
        // on the context's own stream and waited for: a synchronous copy from pageable memory may return before its
        // DMA lands, and this context's kernels run on a non-blocking stream
        u64 *d = nullptr;
        if (cudaMalloc(&d, h.size() * 8) != cudaSuccess ||
            cudaMemcpyAsync(d, h.data(), h.size() * 8, cudaMemcpyHostToDevice, c->own_stream) != cudaSuccess ||
            cudaStreamSynchronize(c->own_stream) != cudaSuccess) {
            delete c;
            return MS_ERR_CUDA;
        }
        c->t4096[0] = d;
        c->t4096[1] = d + 4096;
    }
    if (cudaGetLastError() != cudaSuccess) {
        delete c;
        return MS_ERR_CUDA;
    }
    *out = c;
    return MS_OK;
}

int ms_ctx_destroy(ms_ctx *c) {
    if (!c) return MS_ERR_INVALID;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    ms::host_nodes_drain(c, true);
    c->plans.clear();
    for (auto &t : c->tw_tables) cudaFree(t.second);
    for (auto &e : c->ptr_tables) cudaFree(e.dev);
    c->ptr_tables.clear();
    c->tw_tables.clear();
    for (auto &s : c->scratch)
        if (s.ptr) cudaFree(s.ptr);
    if (c->t4096[0]) cudaFree(c->t4096[0]);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    delete c;
    return MS_OK;
}

int ms_ctx_set_stream(ms_ctx *c, void *s) {
    if (!c) return MS_ERR_INVALID;
    cudaStreamSynchronize(c->stream);
    c->stream = s ? (cudaStream_t)s : c->own_stream;
    return MS_OK;
}

int ms_ctx_sync(ms_ctx *c) {
    if (!c) return MS_ERR_INVALID;
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    return ms::host_nodes_drain(c, false);     // node heaps still crossing to host memory
}

// tuning / A-B switches (process-wide): "ntt_tma" 0|1, "ntt_tma_groups" 2|3, "ntt_tma_stages" 3..8, "ntt_wide_index" 0|1;
// per context: "ntt_table_words"
int ms_set_option(ms_ctx *c, const char *name, int64_t value) {
    if (!name) return MS_ERR_INVALID;
    if (!strcmp(name, "ntt_tma")) { msntt::tma_configure(value ? 1 : 0, 0, 0); return MS_OK; }
    if (!strcmp(name, "ntt_wide_index")) { msntt::wide_index_configure(value ? 1 : 0); return MS_OK; }
    if (!strcmp(name, "ntt_table_words")) {   // cap on the full tables of this context's plans; cached plans are dropped
        if (!c) return MS_ERR_INVALID;
        if (value < -1) return fail(c, MS_ERR_INVALID, "ntt_table_words must be -1 (built-in limits) or >= 0");
        cudaSetDevice(c->device);
        ms::ntt_drop_plans(c);
        c->ntt_table_words = value;
        return MS_OK;
    }
    if (!strcmp(name, "ntt_tma_groups")) {
        if (value != 2 && value != 3) return fail(c, MS_ERR_INVALID, "ntt_tma_groups must be 2 or 3");
        msntt::tma_configure(-1, (int)value, 0);
        return MS_OK;
    }
    if (!strcmp(name, "ntt_tma_stages")) {
        if (value < 3 || value > 8) return fail(c, MS_ERR_INVALID, "ntt_tma_stages must be in [3, 8]");
        msntt::tma_configure(-1, 0, (int)value);
        return MS_OK;
    }
    if (!strcmp(name, "drop_plans")) {   // free the cached NTT plans and their big tables (rebuilt on demand)
        if (!c) return MS_ERR_INVALID;
        cudaSetDevice(c->device);
        ms::ntt_drop_plans(c);
        return MS_OK;
    }
    if (!strcmp(name, "drop_scratch")) {   // free the context's scratch arenas and node staging (regrown on demand)
        if (!c) return MS_ERR_INVALID;
        cudaSetDevice(c->device);
        MS_CUDA(c, cudaStreamSynchronize(c->stream));
        if (int rc = ms::host_nodes_drain(c, true)) return rc;
        for (ms::Scratch &s : c->scratch) {
            if (s.ptr) MS_CUDA(c, cudaFree(s.ptr));
            s.ptr = nullptr;
            s.cap = 0;
        }
        return MS_OK;
    }
    return fail(c, MS_ERR_INVALID, "unknown option %s", name);
}

const char *ms_last_error(ms_ctx *c) { return c ? c->err.c_str() : t_noctx_err.empty() ? "null context" : t_noctx_err.c_str(); }
uint64_t ms_launch_count(ms_ctx *c) { return c ? c->launches : 0; }

int ms_alloc_device(ms_ctx *c, size_t bytes, void **out) {
    if (!c || !out) return MS_ERR_INVALID;
    cudaSetDevice(c->device);
    cudaError_t e = cudaMalloc(out, bytes ? bytes : 1);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(c, MS_ERR_NOMEM, "cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e));
    }
    return MS_OK;
}
int ms_device_memory(ms_ctx *c, size_t *free_bytes, size_t *total_bytes) {
    if (!c) return MS_ERR_INVALID;
    cudaSetDevice(c->device);
    size_t f = 0, t = 0;
    MS_CUDA(c, cudaMemGetInfo(&f, &t));
    if (free_bytes) *free_bytes = f;
    if (total_bytes) *total_bytes = t;
    return MS_OK;
}
int ms_alloc_host_pinned(ms_ctx *c, size_t bytes, void **out) {
    if (!c || !out) return MS_ERR_INVALID;
    cudaError_t e = cudaMallocHost(out, bytes ? bytes : 1);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(c, MS_ERR_NOMEM, "cudaMallocHost(%zu): %s", bytes, cudaGetErrorString(e));
    }
    return MS_OK;
}
int ms_free(ms_ctx *c, void *p) {
    if (!c) return MS_ERR_INVALID;
    if (!p) return MS_OK;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return fail(c, MS_ERR_INVALID, "ms_free: unknown pointer");
    }
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if (a.type == cudaMemoryTypeHost)
        MS_CUDA(c, cudaFreeHost(p));
    else if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged)
        MS_CUDA(c, cudaFree(p));
    else
        return fail(c, MS_ERR_INVALID, "ms_free: not a CUDA allocation");
    return MS_OK;
}
int ms_copy(ms_ctx *c, void *dst, const void *src, size_t bytes) {
    if (!c) return MS_ERR_INVALID;
    MS_CUDA(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    return MS_OK;
}

int ms_fill_random(ms_ctx *c, void *dst, size_t nwords, uint64_t seed) {
    if (!c || !dst) return MS_ERR_INVALID;
    Staged d(c, dst, nwords * 8, false, true);
    if (d.rc) return d.rc;
    if (nwords) {
        fill_random_kernel<<<(unsigned)((nwords + 255) / 256), 256, 0, c->stream>>>(d.as<u64>(), nwords, seed);
        c->launches++;
        MS_CHECK_LAUNCH(c);
    }
    return d.finish();
}

int ms_bit_reverse(ms_ctx *c, int field, void *data, size_t col_stride_elems, unsigned ncols, unsigned log_n) {
    if (!c || !data || (field != MS_FIELD_FP && field != MS_FIELD_FQ3) || log_n > 32 || ncols == 0)
        return fail(c, MS_ERR_INVALID, "ms_bit_reverse: bad argument");
    const size_t n = (size_t)1 << log_n;
    if (ncols > 1 && col_stride_elems < n) return fail(c, MS_ERR_INVALID, "ms_bit_reverse: stride < n");
    const size_t span = ((size_t)(ncols - 1) * col_stride_elems + n) * field * 8;
    Staged d(c, data, span, true, true);
    if (d.rc) return d.rc;
    dim3 grid((unsigned)((n + 255) / 256), ncols);
    if (field == MS_FIELD_FP)
        bit_reverse_kernel<1><<<grid, 256, 0, c->stream>>>(d.as<u64>(), log_n, col_stride_elems);
    else
        bit_reverse_kernel<3><<<grid, 256, 0, c->stream>>>(d.as<u64>(), log_n, col_stride_elems * 3);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    return d.finish();
}

}  // extern "C"
