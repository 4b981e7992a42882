// api_ntt.cu — NTT plans (GpuFft / GpuIfft, gpu/src/plan.rs:236-325,378-462) and the resident
// batched forms used by Matrix::{into_polynomials,into_evaluations,into_bit_reversed_evaluations}
// (src/matrix.rs:101-251).
//
// A plan is the pass list of msntt (ntt.cu) plus small device tables:
//   tw_lo/tw_hi : omega_N^e two-level table (<= 4096 + N/4096 words) — the reference builds and
//                 bit-reverses an n/2-word twiddle vector and an n-word scale vector on the CPU
//                 for every plan (plan.rs:395-398, stage.rs:255-259); plans here are cached.
//   sc_lo/sc_hi : powers of the coset offset (forward) or of offset^-1 times n^-1 (inverse).
#include <algorithm>
#include <cstring>

#include "ctx.cuh"

namespace ms {

using msntt::PassParams;

struct NttPlanDev {
    NttJob job;
    u64 N = 0;
    unsigned estride = 1, lanes = 1, ncos = 1;
    bool naive = false;
    u64 root = 0;
    std::vector<PassParams> passes;
    std::vector<unsigned> ntiles;
    u64 *dev = nullptr;  // one allocation holding the small tables
    std::vector<u64 *> big;  // full twiddle / scale tables
    msntt::Tables tb{};
    ~NttPlanDev() {
        if (dev) cudaFree(dev);
        for (u64 *b : big) cudaFree(b);
    }
};

static u64 root_of_unity(unsigned log_n) {
    u64 r = gl::to_mont(1753635133440165772ULL);
    for (unsigned i = log_n; i < 32; i++) r = gl::sqr(r);
    return r;
}
static unsigned brev_bits(unsigned v, unsigned bits) {
    unsigned r = 0;
    for (unsigned b = 0; b < bits; b++) r |= ((v >> b) & 1u) << (bits - 1 - b);
    return r;
}
static int ilog2(u64 v) {
    int l = 0;
    while ((1ull << l) < v) l++;
    return l;
}

int ntt_get_plan(ms_ctx *c, const NttJob &job, std::shared_ptr<NttPlanDev> *out) {
    auto key = std::make_tuple(job.field, job.log_n, (int)job.inverse, job.offset, job.log_blowup, (int)job.bitrev_out);
    auto it = c->plans.find(key);
    if (it != c->plans.end()) {
        *out = it->second;
        return MS_OK;
    }
    auto P = std::make_shared<NttPlanDev>();
    P->job = job;
    const unsigned log_n = job.log_n;
    const u64 N = 1ull << log_n;
    P->N = N;
    P->estride = P->lanes = (unsigned)job.field;
    P->ncos = job.bitrev_out ? (1u << job.log_blowup) : 1u;
    u64 root = root_of_unity(log_n);
    if (job.inverse) root = gl::inv(root);
    P->root = root;
    P->naive = log_n < 4;

    // ---- digits and strides
    std::vector<int> d;
    if (!P->naive) d = msntt::choose_digits(log_n);
    const int m = (int)d.size();
    std::vector<u64> S(m), Pw(m);
    {
        u64 s = 1;
        for (int l = m - 1; l >= 0; l--) { S[l] = s; s <<= d[l]; }
        u64 p = 1;
        for (int l = 0; l < m; l++) { Pw[l] = p; p <<= d[l]; }
    }
    const bool has_pre = !P->naive && !job.inverse && (job.offset != gl::ONE || P->ncos > 1);
    const bool has_post = !P->naive && job.inverse;
    const u32 hi_len = (u32)std::max<u64>(1, N >> 12);

    for (int k = 0; k < m; k++) {
        PassParams p;
        memset(&p, 0, sizeof p);
        const u64 R = 1ull << d[k];
        p.log_r = d[k];
        p.n_mask = N - 1;
        p.hi_len = hi_len;
        p.bitrev_digit = job.bitrev_out ? 1 : 0;
        p.lanes = P->lanes;
        p.ncos = P->ncos;
        p.estride = P->estride;
        u64 W;
        if (m == 1) {
            W = 1;
            p.in_rs = p.out_rs = 1;
            p.in_r_fast = p.out_r_fast = 1;
            p.ndims = 0;
        } else if (k < m - 1) {  // strided pass, position preserving
            W = std::min<u64>(1ull << (msntt::kTileLog - d[k]), S[k]);
            p.in_rs = p.out_rs = S[k];
            p.in_cs = p.out_cs = 1;
            p.low_cs = 1;
            p.ndims = 2;
            p.dims[0] = msntt::Dim{(u32)(S[k] / W), 0, W, W, W};
            p.dims[1] = msntt::Dim{(u32)(N / (R * S[k])), 0, R * S[k], R * S[k], 0};
            p.has_outer = 1;
            p.outer_mult = N / (R * S[k]);
        } else if (!job.bitrev_out) {  // last pass, natural order: transposing write
            W = std::min<u64>(1ull << (msntt::kTileLog - d[k]), 1ull << d[0]);
            p.in_rs = 1;
            p.in_cs = S[0];
            p.out_rs = Pw[k];
            p.out_cs = 1;
            p.in_r_fast = 1;
            p.out_r_fast = 0;
            p.ndims = 1;
            p.dims[0] = msntt::Dim{(u32)((1ull << d[0]) / W), 0, W * S[0], W, 0};
            for (int l = 1; l < m - 1; l++) p.dims[p.ndims++] = msntt::Dim{(u32)(1ull << d[l]), 0, S[l], Pw[l], 0};
        } else {  // last pass, bit-reversed order: contiguous, in place
            const u64 Rprev = 1ull << d[k - 1];
            W = std::min<u64>(1ull << (msntt::kTileLog - d[k]), Rprev);
            p.in_rs = p.out_rs = 1;
            p.in_cs = p.out_cs = R;
            p.in_r_fast = p.out_r_fast = 1;
            p.ndims = 2;
            p.dims[0] = msntt::Dim{(u32)(Rprev / W), 0, W * R, W * R, 0};
            p.dims[1] = msntt::Dim{(u32)(N / (R * Rprev)), 0, R * Rprev, R * Rprev, 0};
        }
        p.log_w = (u32)ilog2(W);
        for (u32 dd = 0; dd < p.ndims; dd++) p.dims[dd].log_ext = (u32)ilog2(p.dims[dd].ext);
        p.log_ncos = (u32)ilog2(P->ncos);
        p.has_pre = (k == 0 && has_pre) ? 1 : 0;
        p.has_post = (k == m - 1 && has_post) ? 1 : 0;
        P->passes.push_back(p);
        P->ntiles.push_back((unsigned)(N / (R * W)));
    }

    // ---- tables
    const size_t lo_len = 4096;
    const size_t n_tw = lo_len + hi_len;
    const size_t n_sc = (has_pre || has_post) ? (size_t)P->ncos * (lo_len + hi_len + 1) : 0;
    std::vector<u64> h(n_tw + n_sc);
    {
        u64 a = gl::ONE;
        for (size_t e = 0; e < lo_len; e++) { h[e] = a; a = gl::mul(a, root); }
        // a == root^4096 now
        u64 b = gl::ONE;
        for (size_t e = 0; e < hi_len; e++) { h[lo_len + e] = b; b = gl::mul(b, a); }
    }
    u64 post_step = gl::ONE;
    if (n_sc) {
        int st[3], nst;
        u64 *sc_lo = h.data() + n_tw;
        u64 *sc_hi = sc_lo + (size_t)P->ncos * lo_len;
        u64 *pre_step = sc_hi + (size_t)P->ncos * hi_len;
        const u64 gN = job.bitrev_out ? root_of_unity(log_n + job.log_blowup) : gl::ONE;
        for (unsigned q = 0; q < P->ncos; q++) {
            u64 base, cst;
            if (has_post) {
                base = gl::inv(job.offset);
                cst = gl::inv(gl::to_mont(N));
            } else {
                // block q of a bit-reversed LDE holds the coset offset * g_N^r, r = bitrev(q)
                const unsigned r = brev_bits(q, job.log_blowup);
                base = gl::mul(job.offset, gl::pow(gN, r));
                cst = gl::ONE;
            }
            u64 a = gl::ONE;
            for (size_t e = 0; e < lo_len; e++) { sc_lo[q * lo_len + e] = a; a = gl::mul(a, base); }
            u64 b = cst;
            for (size_t e = 0; e < hi_len; e++) { sc_hi[(size_t)q * hi_len + e] = b; b = gl::mul(b, a); }
            if (hi_len == 1) {  // single-level lookup: fold the constant into the low table
                for (size_t e = 0; e < lo_len; e++) sc_lo[q * lo_len + e] = gl::mul(sc_lo[q * lo_len + e], cst);
            }
            // first step of the first pass walks the transform index in units of 2^(log_r - A)
            msntt::steps_of(P->passes[0].log_r, st, &nst);
            pre_step[q] = gl::pow(base, P->passes[0].in_rs << (P->passes[0].log_r - st[0]));
            if (has_post) {
                const PassParams &lp = P->passes.back();
                msntt::steps_of(lp.log_r, st, &nst);
                post_step = gl::pow(base, lp.out_rs << (lp.log_r - st[nst - 1]));
            }
        }
    }
    if (!P->passes.empty()) P->passes.back().post_step = post_step;
    cudaError_t e = cudaMalloc(&P->dev, h.size() * 8);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(c, MS_ERR_NOMEM, "plan tables cudaMalloc: %s", cudaGetErrorString(e));
    }
    MS_CUDA(c, cudaMemcpyAsync(P->dev, h.data(), h.size() * 8, cudaMemcpyHostToDevice, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    P->tb.t4096 = c->t4096[job.inverse ? 1 : 0];
    P->tb.tw_lo = P->dev;
    P->tb.tw_hi = P->dev + lo_len;
    if (n_sc) {
        P->tb.sc_lo = P->dev + n_tw;
        P->tb.sc_hi = P->tb.sc_lo + (size_t)P->ncos * lo_len;
        P->tb.pre_step = P->tb.sc_hi + (size_t)P->ncos * hi_len;
    }
    // ---- full tables where they are affordable (one multiplication per element instead of the two of
    //      the on-the-fly geometric progression); skipped silently if memory is short
    {
        auto try_alloc = [&](size_t words) -> u64 * {
            u64 *d = nullptr;
            if (cudaMalloc(&d, words * 8) != cudaSuccess) {
                cudaGetLastError();
                return nullptr;
            }
            P->big.push_back(d);
            return d;
        };
        size_t kOuterMax = (size_t)64 << 20, kPreMax = (size_t)256 << 20;  // words (512 MiB / 2 GiB)
        if (c->ntt_table_words >= 0) {  // "ntt_table_words": a lower cap; 0 leaves every factor to the progressions
            kOuterMax = std::min(kOuterMax, (size_t)c->ntt_table_words);
            kPreMax = std::min(kPreMax, (size_t)c->ntt_table_words);
        }
        for (size_t k = 0; k < P->passes.size(); k++) {
            PassParams &p = P->passes[k];
            if (p.has_outer) {
                const u64 R = 1ull << p.log_r, S = p.in_rs;
                if (R * S <= kOuterMax) {
                    if (u64 *d = try_alloc(R * S)) {
                        msntt::build_outer_table(d, R, S, p.outer_mult, p.n_mask, P->tb.tw_lo, P->tb.tw_hi, hi_len, c->stream);
                        c->launches++;
                        p.outer_tab = d;
                        p.outer_S = S;
                    }
                }
            }
            if (p.has_pre && (size_t)P->ncos * N <= kPreMax) {
                if (u64 *d = try_alloc((size_t)P->ncos * N)) {
                    for (unsigned q = 0; q < P->ncos; q++) {
                        msntt::build_pow_table(d + (size_t)q * N, N, P->tb.sc_lo + (size_t)q * lo_len,
                                               P->tb.sc_hi + (size_t)q * hi_len, hi_len, c->stream);
                        c->launches++;
                    }
                    p.pre_tab = d;
                    p.pre_cos_stride = N;
                }
            }
            if (p.has_post && N <= kOuterMax) {
                if (u64 *d = try_alloc(N)) {
                    msntt::build_pow_table(d, N, P->tb.sc_lo, P->tb.sc_hi, hi_len, c->stream);
                    c->launches++;
                    p.post_tab = d;
                }
            }
        }
        MS_CUDA(c, cudaStreamSynchronize(c->stream));
    }
    c->plans[key] = P;
    *out = P;
    return MS_OK;
}

// Two-level table of g_n^e only (what the FRI fold, the evaluator's X leaf and the scans need): a few KiB per size,
// cached per context — NOT a full transform plan, whose inter-pass and scale tables run to hundreds of MiB.
int ntt_plan_tables(ms_ctx *c, unsigned log_n, const u64 **tw_lo, const u64 **tw_hi, u32 *hi_len) {
    const u32 hl = (u32)std::max<u64>(1, (1ull << log_n) >> 12);
    auto it = c->tw_tables.find(log_n);
    if (it == c->tw_tables.end()) {
        // reuse a full plan's tables when one exists already
        auto key = std::make_tuple((int)MS_FIELD_FP, log_n, 0, (uint64_t)gl::ONE, 0u, 0);
        auto pit = c->plans.find(key);
        if (pit != c->plans.end()) {
            *tw_lo = pit->second->tb.tw_lo;
            *tw_hi = pit->second->tb.tw_hi;
            *hi_len = hl;
            return MS_OK;
        }
        const size_t lo_len = 4096;
        std::vector<u64> h(lo_len + hl);
        const u64 root = root_of_unity(log_n);
        u64 a = gl::ONE;
        for (size_t e = 0; e < lo_len; e++) { h[e] = a; a = gl::mul(a, root); }
        u64 b = gl::ONE;
        for (size_t e = 0; e < hl; e++) { h[lo_len + e] = b; b = gl::mul(b, a); }
        u64 *d = nullptr;
        cudaError_t e = cudaMalloc(&d, h.size() * 8);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(c, MS_ERR_NOMEM, "twiddle table cudaMalloc: %s", cudaGetErrorString(e));
        }
        MS_CUDA(c, cudaMemcpyAsync(d, h.data(), h.size() * 8, cudaMemcpyHostToDevice, c->stream));
        MS_CUDA(c, cudaStreamSynchronize(c->stream));
        it = c->tw_tables.emplace(log_n, d).first;
    }
    *tw_lo = it->second;
    *tw_hi = it->second + 4096;
    *hi_len = hl;
    return MS_OK;
}

// drop every cached plan (and its big tables); plans are rebuilt on demand
void ntt_drop_plans(ms_ctx *c) {
    cudaStreamSynchronize(c->stream);
    c->plans.clear();
}

__global__ void copy_strided_kernel(const u64 *src, size_t src_stride, u64 *dst, size_t dst_stride, size_t words) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < words) dst[blockIdx.y * dst_stride + i] = src[blockIdx.y * src_stride + i];
}

int ntt_run(ms_ctx *c, NttPlanDev &P, const u64 *in, size_t in_cs, u64 *out, size_t out_cs, unsigned ncols, const LdeScatter *sc) {
    if (ncols == 0) return MS_OK;
    const u64 N = P.N;
    const size_t col_words = (size_t)N * P.estride;
    const bool lde = P.job.bitrev_out;
    const size_t tmp_budget = (size_t)1 << 30;
    unsigned max_tiles = 1;
    for (unsigned t : P.ntiles) max_tiles = std::max(max_tiles, t);
    // 1-D grid of ntiles * nbatch blocks (naive path: grid.y = columns * lanes)
    unsigned max_cols = P.naive ? 65535u / P.lanes
                                : (unsigned)std::max<u64>(1, 0x7FFFFFFFull / (P.lanes * P.ncos));
    (void)max_tiles;
    const int m = (int)P.passes.size();
    const bool need_tmp = P.naive ? (in == out) : (!lde && m >= 2);
    if (need_tmp) max_cols = (unsigned)std::max<size_t>(1, std::min<size_t>(max_cols, tmp_budget / (col_words * 8)));
    for (unsigned c0 = 0; c0 < ncols; c0 += max_cols) {
        const unsigned nc = std::min(max_cols, ncols - c0);
        const u64 *src = in + (size_t)c0 * in_cs;
        u64 *dst = out + (size_t)c0 * out_cs;
        u64 *tmp = nullptr;
        if (need_tmp) {
            void *t;
            int rc = scratch_get(c, 0, (size_t)nc * col_words * 8, &t);
            if (rc) return rc;
            tmp = (u64 *)t;
        }
        if (P.naive) {
            if (lde) return fail(c, MS_ERR_INVALID, "internal: naive plan in LDE mode");
            u64 *o = need_tmp ? tmp : dst;
            const size_t ocs = need_tmp ? col_words : out_cs;
            msntt::launch_naive(src, in_cs, o, ocs, P.job.log_n, P.estride, P.lanes, nc, P.job.inverse, P.root,
                                P.job.offset, c->stream);
            c->launches++;
            MS_CHECK_LAUNCH(c);
            if (need_tmp) {
                dim3 g((unsigned)((col_words + 255) / 256), nc);
                copy_strided_kernel<<<g, 256, 0, c->stream>>>(tmp, col_words, dst, out_cs, col_words);
                c->launches++;
                MS_CHECK_LAUNCH(c);
            }
            continue;
        }
        for (int k = 0; k < m; k++) {
            PassParams p = P.passes[k];
            const u64 *pin;
            u64 *pout;
            if (lde) {
                pin = (k == 0) ? src : dst;
                pout = dst;
                p.in_col_stride = (k == 0) ? in_cs : out_cs;
                p.out_col_stride = out_cs;
                p.in_cos_stride = (k == 0) ? 0 : col_words;
                p.out_cos_stride = col_words;
                if (sc && k == m - 1) {
                    // fused exchange: the last pass stores every coset block where its rows are needed
                    if (c0 != 0) return fail(c, MS_ERR_INVALID, "internal: scatter LDE must run in one column batch");
                    p.out_cos_ptr = sc->block_ptr;
                    p.out_col_stride = sc->block_col_stride_words;
                    p.out_dup_ptr = sc->dup_ptr;
                    p.dup_col_stride = sc->dup_col_stride_words;
                    p.host_cos_ptr = sc->host_block_ptr;
                    p.host_dup_ptr = sc->host_dup_ptr;
                }
            } else if (m == 1) {
                pin = src;
                pout = dst;
                p.in_col_stride = in_cs;
                p.out_col_stride = out_cs;
            } else {
                pin = (k == 0) ? src : tmp;
                pout = (k == m - 1) ? dst : tmp;
                p.in_col_stride = (k == 0) ? in_cs : col_words;
                p.out_col_stride = (k == m - 1) ? out_cs : col_words;
            }
            p.nbatch = nc * P.lanes * P.ncos;
            if (msntt::launch_pass_tma(p, P.tb, P.job.inverse, pin, pout, P.ntiles[k], nc, c->stream)) {
                c->launches++;
                MS_CHECK_LAUNCH(c);
                continue;
            }
            msntt::launch_pass(p, P.tb, P.job.inverse, pin, pout, P.ntiles[k], p.nbatch, c->stream);
            c->launches++;
            MS_CHECK_LAUNCH(c);
        }
    }
    return MS_OK;
}

static int check_field(ms_ctx *c, int field) {
    if (field != MS_FIELD_FP && field != MS_FIELD_FQ3) return fail(c, MS_ERR_INVALID, "unknown field id %d", field);
    return MS_OK;
}

}  // namespace ms

using namespace ms;

struct ms_ntt_plan {
    ms_ctx *ctx;
    std::shared_ptr<NttPlanDev> plan;
    std::vector<void *> queue;
};

extern "C" {

int ms_ntt_plan_create(ms_ctx *c, int field, unsigned log_n, int direction, uint64_t offset_mont, ms_ntt_plan **out) {
    if (!c || !out) return MS_ERR_INVALID;
    if (int rc = check_field(c, field)) return rc;
    if (log_n > 32) return fail(c, MS_ERR_INVALID, "log_n %u out of range [0, 32]", log_n);
    if (direction != MS_NTT_FORWARD && direction != MS_NTT_INVERSE) return fail(c, MS_ERR_INVALID, "bad direction");
    if (offset_mont >= gl::P || offset_mont == 0) return fail(c, MS_ERR_INVALID, "offset must be a non-zero canonical word");
    cudaSetDevice(c->device);
    NttJob job{field, log_n, direction == MS_NTT_INVERSE, false, 0, offset_mont};
    auto *pl = new ms_ntt_plan();
    pl->ctx = c;
    int rc = ntt_get_plan(c, job, &pl->plan);
    if (rc) {
        delete pl;
        return rc;
    }
    *out = pl;
    return MS_OK;
}

int ms_ntt_encode(ms_ntt_plan *pl, void *column) {
    if (!pl || !column) return MS_ERR_INVALID;
    pl->queue.push_back(column);
    return MS_OK;
}

int ms_ntt_execute(ms_ntt_plan *pl) {
    if (!pl) return MS_ERR_INVALID;
    ms_ctx *c = pl->ctx;
    cudaSetDevice(c->device);
    NttPlanDev &P = *pl->plan;
    const size_t col_words = (size_t)P.N * P.estride;
    std::vector<void *> host_cols, dev_cols;
    for (void *p : pl->queue) (is_device_ptr(p) ? dev_cols : host_cols).push_back(p);
    pl->queue.clear();
    int rc = MS_OK;
    for (void *p : dev_cols) {
        rc = ntt_run(c, P, (const u64 *)p, col_words, (u64 *)p, col_words, 1);
        if (rc) return rc;
    }
    if (!host_cols.empty()) {
        // stage all host columns into one device matrix, one batched transform, copy back
        const size_t tmp_budget = (size_t)4 << 30;
        const size_t per = std::max<size_t>(1, tmp_budget / (col_words * 8));
        for (size_t i0 = 0; i0 < host_cols.size(); i0 += per) {
            const size_t nc = std::min(per, host_cols.size() - i0);
            void *stage;
            rc = scratch_get(c, 1, nc * col_words * 8, &stage);
            if (rc) return rc;
            for (size_t i = 0; i < nc; i++)
                MS_CUDA(c, cudaMemcpyAsync((u64 *)stage + i * col_words, host_cols[i0 + i], col_words * 8,
                                           cudaMemcpyHostToDevice, c->stream));
            rc = ntt_run(c, P, (const u64 *)stage, col_words, (u64 *)stage, col_words, (unsigned)nc);
            if (rc) return rc;
            for (size_t i = 0; i < nc; i++)
                MS_CUDA(c, cudaMemcpyAsync(host_cols[i0 + i], (u64 *)stage + i * col_words, col_words * 8,
                                           cudaMemcpyDeviceToHost, c->stream));
            MS_CUDA(c, cudaStreamSynchronize(c->stream));
        }
    }
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    return MS_OK;
}

int ms_ntt_plan_destroy(ms_ntt_plan *pl) {
    if (!pl) return MS_ERR_INVALID;
    delete pl;
    return MS_OK;
}

int ms_ntt_batch(ms_ctx *c, int field, void *data, size_t col_stride_elems, unsigned ncols, unsigned log_n,
                 int direction, uint64_t offset_mont) {
    if (!c || !data) return MS_ERR_INVALID;
    if (int rc = check_field(c, field)) return rc;
    if (log_n > 32 || ncols == 0) return fail(c, MS_ERR_INVALID, "ms_ntt_batch: bad size");
    if (offset_mont >= gl::P || offset_mont == 0) return fail(c, MS_ERR_INVALID, "offset must be a non-zero canonical word");
    const size_t n = (size_t)1 << log_n;
    if (ncols > 1 && col_stride_elems < n) return fail(c, MS_ERR_INVALID, "ms_ntt_batch: stride < n");
    NttJob job{field, log_n, direction == MS_NTT_INVERSE, false, 0, offset_mont};
    std::shared_ptr<NttPlanDev> P;
    if (int rc = ntt_get_plan(c, job, &P)) return rc;
    const size_t span = ((size_t)(ncols - 1) * col_stride_elems + n) * field * 8;
    Staged d(c, data, span, true, true);
    if (d.rc) return d.rc;
    int rc = ntt_run(c, *P, d.as<u64>(), col_stride_elems * field, d.as<u64>(), col_stride_elems * field, ncols);
    if (rc) return rc;
    return d.finish();
}

int ms_ntt_batch_to(ms_ctx *c, int field, const void *src, size_t src_stride_elems, void *dst, size_t dst_stride_elems,
                    unsigned ncols, unsigned log_n, int direction, uint64_t offset_mont) {
    if (!c || !src || !dst) return MS_ERR_INVALID;
    if (src == dst && src_stride_elems == dst_stride_elems)
        return ms_ntt_batch(c, field, dst, dst_stride_elems, ncols, log_n, direction, offset_mont);
    if (src == dst && ncols > 1) return fail(c, MS_ERR_INVALID, "ms_ntt_batch_to: src == dst with different strides");
    if (int rc = check_field(c, field)) return rc;
    if (log_n > 32 || ncols == 0) return fail(c, MS_ERR_INVALID, "ms_ntt_batch_to: bad size");
    if (offset_mont >= gl::P || offset_mont == 0) return fail(c, MS_ERR_INVALID, "offset must be a non-zero canonical word");
    const size_t n = (size_t)1 << log_n;
    if (ncols > 1 && (src_stride_elems < n || dst_stride_elems < n)) return fail(c, MS_ERR_INVALID, "ms_ntt_batch_to: stride < n");
    NttJob job{field, log_n, direction == MS_NTT_INVERSE, false, 0, offset_mont};
    std::shared_ptr<NttPlanDev> P;
    if (int rc = ntt_get_plan(c, job, &P)) return rc;
    Staged in(c, src, ((size_t)(ncols - 1) * src_stride_elems + n) * field * 8, true, false);
    if (in.rc) return in.rc;
    // a staged host destination is copied back as one span: with gaps between the columns (stride > n) the gaps must
    // hold the caller's bytes, so they are copied in first
    Staged out(c, dst, ((size_t)(ncols - 1) * dst_stride_elems + n) * field * 8, ncols > 1 && dst_stride_elems != n, true);
    if (out.rc) return out.rc;
    int rc = ntt_run(c, *P, in.as<u64>(), src_stride_elems * field, out.as<u64>(), dst_stride_elems * field, ncols);
    if (rc) return rc;
    if ((rc = in.finish())) return rc;
    return out.finish();
}

__global__ void pad_copy_kernel(const u64 *src, size_t src_stride, u64 *dst, size_t dst_stride, size_t n_words,
                                size_t N_words) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < N_words) dst[blockIdx.y * dst_stride + i] = i < n_words ? src[blockIdx.y * src_stride + i] : 0;
}

int ms_lde_batch(ms_ctx *c, int field, const void *coeffs, size_t in_stride_elems, void *evals, size_t out_stride_elems,
                 unsigned ncols, unsigned log_n, unsigned log_blowup, uint64_t offset_mont, int bitrev_out) {
    if (!c || !coeffs || !evals) return MS_ERR_INVALID;
    if (int rc = check_field(c, field)) return rc;
    if (log_n + log_blowup > 32 || log_blowup > 6 || ncols == 0) return fail(c, MS_ERR_INVALID, "ms_lde_batch: bad size");
    if (offset_mont >= gl::P || offset_mont == 0) return fail(c, MS_ERR_INVALID, "offset must be a non-zero canonical word");
    const size_t n = (size_t)1 << log_n, N = n << log_blowup;
    if (ncols > 1 && (in_stride_elems < n || out_stride_elems < N)) return fail(c, MS_ERR_INVALID, "ms_lde_batch: stride too small");
    Staged in(c, coeffs, ((size_t)(ncols - 1) * in_stride_elems + n) * field * 8, true, false);
    if (in.rc) return in.rc;
    Staged out(c, evals, ((size_t)(ncols - 1) * out_stride_elems + N) * field * 8, ncols > 1 && out_stride_elems != N, true);
    if (out.rc) return out.rc;
    int rc;
    if (bitrev_out && log_n >= 4) {
        NttJob job{field, log_n, false, true, log_blowup, offset_mont};
        std::shared_ptr<NttPlanDev> P;
        if ((rc = ntt_get_plan(c, job, &P))) return rc;
        rc = ntt_run(c, *P, in.as<u64>(), in_stride_elems * field, out.as<u64>(), out_stride_elems * field, ncols);
        if (rc) return rc;
    } else {
        // natural order (Matrix::into_evaluations, src/matrix.rs:192-208: resize with zeros, then
        // a full-size coset NTT), or a tiny transform: zero-pad on device and run the size-N plan.
        dim3 g((unsigned)((N * field + 255) / 256), ncols);
        pad_copy_kernel<<<g, 256, 0, c->stream>>>(in.as<u64>(), in_stride_elems * field, out.as<u64>(),
                                                  out_stride_elems * field, n * field, N * field);
        c->launches++;
        MS_CHECK_LAUNCH(c);
        NttJob job{field, log_n + log_blowup, false, false, 0, offset_mont};
        std::shared_ptr<NttPlanDev> P;
        if ((rc = ntt_get_plan(c, job, &P))) return rc;
        rc = ntt_run(c, *P, out.as<u64>(), out_stride_elems * field, out.as<u64>(), out_stride_elems * field, ncols);
        if (rc) return rc;
        if (bitrev_out) {
            rc = ms_bit_reverse(c, field, out.dev, out_stride_elems, ncols, log_n + log_blowup);
            if (rc) return rc;
        }
    }
    if ((rc = in.finish())) return rc;
    return out.finish();
}

// ---- fused LDE + exchange (multi-GPU commit, SURVEY.md §8e "fusion opportunity") ---------------------------------
// The bit-reversed LDE is 2^log_blowup coset blocks of n rows; with G GPUs (G | 2^log_blowup) the row slab of GPU j is
// a run of whole blocks.  Instead of LDE -> all-to-all, the last NTT pass stores block q of every local column straight
// into the slab of the GPU that hashes those rows: block_ptrs[q] = address (possibly peer memory mapped with
// ms_ipc_open) of block q of LOCAL column 0 inside that slab, consecutive local columns block_col_stride_elems apart.
// dup_ptrs (optional, entries may be NULL): a second copy of block q — e.g. the local copy of the ce-domain prefix the
// constraint evaluation of this rank's columns reads.  work: ncols x work_stride_elems scratch for the earlier passes.
int ms_lde_batch_scatter(ms_ctx *c, int field, const void *coeffs, size_t in_stride_elems, unsigned ncols, unsigned log_n,
                         unsigned log_blowup, uint64_t offset_mont, void *work, size_t work_stride_elems, void *const *block_ptrs,
                         size_t block_col_stride_elems, void *const *dup_ptrs, size_t dup_col_stride_elems) {
    if (!c || !coeffs || !work || !block_ptrs) return MS_ERR_INVALID;
    if (int rc = check_field(c, field)) return rc;
    if (log_n < 4 || log_n + log_blowup > 32 || log_blowup > 6 || ncols == 0) return fail(c, MS_ERR_INVALID, "ms_lde_batch_scatter: bad size");
    if (offset_mont >= gl::P || offset_mont == 0) return fail(c, MS_ERR_INVALID, "offset must be a non-zero canonical word");
    const size_t n = (size_t)1 << log_n, N = n << log_blowup;
    const unsigned nb = 1u << log_blowup;
    if (ncols > 1 && (in_stride_elems < n || work_stride_elems < N || block_col_stride_elems < n))
        return fail(c, MS_ERR_INVALID, "ms_lde_batch_scatter: stride too small");
    if (!is_device_ptr(coeffs) || !is_device_ptr(work)) return fail(c, MS_ERR_INVALID, "ms_lde_batch_scatter: resident buffers only");
    for (unsigned q = 0; q < nb; q++)
        if (!block_ptrs[q]) return fail(c, MS_ERR_INVALID, "ms_lde_batch_scatter: block pointer %u is null", q);
    cudaSetDevice(c->device);
    NttJob job{field, log_n, false, true, log_blowup, offset_mont};
    std::shared_ptr<NttPlanDev> P;
    int rc;
    if ((rc = ntt_get_plan(c, job, &P))) return rc;
    // the block-pointer table: a small per-context device buffer that is re-uploaded only when its contents change (the
    // slabs of a run keep their addresses per column chunk), from a host copy that outlives the call — no stream sync
    std::vector<void *> host(2 * nb, nullptr);
    for (unsigned q = 0; q < nb; q++) {
        host[q] = block_ptrs[q];
        host[nb + q] = dup_ptrs ? dup_ptrs[q] : nullptr;
    }
    void *tab = nullptr;
    for (auto &e : c->ptr_tables)
        if (e.host == host) tab = e.dev;
    if (!tab) {
        if (c->ptr_tables.size() >= 64) {            // bounded: drop the oldest tables
            MS_CUDA(c, cudaStreamSynchronize(c->stream));
            for (auto &e : c->ptr_tables) cudaFree(e.dev);
            c->ptr_tables.clear();
        }
        c->ptr_tables.emplace_back();
        auto &e = c->ptr_tables.back();
        e.host = host;
        cudaError_t ce = cudaMalloc(&e.dev, (size_t)nb * 16);
        if (ce != cudaSuccess) {
            cudaGetLastError();
            c->ptr_tables.pop_back();
            return fail(c, MS_ERR_NOMEM, "pointer table cudaMalloc: %s", cudaGetErrorString(ce));
        }
        MS_CUDA(c, cudaMemcpyAsync(e.dev, e.host.data(), (size_t)nb * 16, cudaMemcpyHostToDevice, c->stream));
        tab = e.dev;
    }
    LdeScatter sc{(u64 *const *)tab, block_col_stride_elems * field, dup_ptrs ? (u64 *const *)tab + nb : nullptr,
                  dup_col_stride_elems * field, host.data(), dup_ptrs ? host.data() + nb : nullptr};
    return ntt_run(c, *P, (const u64 *)coeffs, in_stride_elems * field, (u64 *)work, work_stride_elems * field, ncols, &sc);
}

// CUDA IPC plumbing for the peer slabs (one process per GPU): export a cudaMalloc'ed buffer of this process, map a
// buffer exported by a peer process.  handle: 64 bytes (cudaIpcMemHandle_t).
int ms_ipc_export(ms_ctx *c, const void *dev_ptr, uint8_t *handle64) {
    if (!c || !dev_ptr || !handle64) return MS_ERR_INVALID;
    cudaSetDevice(c->device);
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    cudaIpcMemHandle_t h;
    MS_CUDA(c, cudaIpcGetMemHandle(&h, const_cast<void *>(dev_ptr)));
    memcpy(handle64, &h, 64);
    return MS_OK;
}
int ms_ipc_open(ms_ctx *c, const uint8_t *handle64, void **peer_ptr) {
    if (!c || !handle64 || !peer_ptr) return MS_ERR_INVALID;
    cudaSetDevice(c->device);
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    MS_CUDA(c, cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return MS_OK;
}
int ms_ipc_close(ms_ctx *c, void *peer_ptr) {
    if (!c || !peer_ptr) return MS_ERR_INVALID;
    cudaSetDevice(c->device);
    MS_CUDA(c, cudaIpcCloseMemHandle(peer_ptr));
    return MS_OK;
}

}  // extern "C"
