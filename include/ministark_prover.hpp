// ministark_prover.hpp — `default_prove` (src/prover.rs:25-174) in C++ on top of the C ABI: the compiled-language
// counterpart of ministark_b200/prover.py (same transcript order, same calls), including the extension-trace phase
// (prover.rs:56-72) through a device-side column builder; bf::device_extension below builds the nine brainfuck
// extension columns from the resident base trace with the fused evaluator + ms_scan_affine.
//
// Three residencies, chosen per proof as GpuProver (prover.py) chooses them: resident keeps every LDE matrix and tree in
// device memory; streamed keeps the coefficients and the tree node heaps and recomputes one coset block of the LDE at a
// time (commitment, constraint evaluation, DEEP), answering queries from the coefficients; streamed_host is streamed with
// the node heaps in pinned host memory (ministark_host_nodes.h).  All emit the same bytes.
//
// Host logic (coin, AIR, programs, wire format) comes from ministark_host.hpp and is CPU-tested.  This file only strings
// the ms_* calls together; linked against the CPU build of the ABI it is byte-compared with the CPU restatement of the
// reference prover, and on a GPU with the Python driver (tests/test_zz_gpu_cpp_prover.py,
// tests/test_gpu_cpp_stream_prover.py).
#pragma once
#include <chrono>
#include <cstdio>
#include <memory>
#include <stdexcept>

#include "ministark_b200.h"
#include "ministark_bf.h"
#include "ministark_device.h"
#include "ministark_examples.hpp"
#include "ministark_host.hpp"
#include "ministark_host_nodes.h"
#include "ministark_stream.h"

// ministark_b200.h is the ABI every library build exports.  The entry points of the headers beside it are referenced
// weakly, so that this layer also links against a build that exports the core alone: without ms_device_memory only
// GpuProver::memory_budget limits a proof, and the streamed residency and the device-built brainfuck trace throw when the
// library lacks their entry points.
#pragma weak ms_device_memory
#pragma weak ms_merkle_commit_block_sha256
#pragma weak ms_lde_rows
#pragma weak ms_merkle_commit_block_sha256_host
#pragma weak ms_bf_run
#pragma weak ms_bf_trace_sizes
#pragma weak ms_bf_trace_fill
#pragma weak ms_bf_helper_columns

namespace mshost {

// number of ms_alloc_device calls made through DeviceBuf by this process
inline u64 &device_allocations() {
    static u64 count = 0;
    return count;
}

struct DeviceBuf {   // RAII over ms_alloc_device
    ms_ctx *ctx = nullptr;
    void *p = nullptr;
    DeviceBuf() = default;
    DeviceBuf(ms_ctx *c, size_t bytes) : ctx(c) {
        device_allocations()++;
        if (ms_alloc_device(c, bytes, &p) != MS_OK) throw std::runtime_error(std::string("ms_alloc_device: ") + ms_last_error(c));
    }
    DeviceBuf(const DeviceBuf &) = delete;
    DeviceBuf &operator=(const DeviceBuf &) = delete;
    DeviceBuf(DeviceBuf &&o) noexcept : ctx(o.ctx), p(o.p) { o.p = nullptr; }
    DeviceBuf &operator=(DeviceBuf &&o) noexcept {
        if (this != &o) { release(); ctx = o.ctx; p = o.p; o.p = nullptr; }
        return *this;
    }
    ~DeviceBuf() { release(); }
    void release() { if (p) ms_free(ctx, p); p = nullptr; }
    u64 *words() const { return static_cast<u64 *>(p); }
};

inline void ck(ms_ctx *c, int rc, const char *what) {
    if (rc != MS_OK) throw std::runtime_error(std::string(what) + ": " + ms_last_error(c));   // the reference panics
}

// DEEP composition as a symbolic expression over LDE columns [base..., composition...] (ministark_b200/deep.py), with the
// terms grouped by their out-of-domain point:
//     sum_j a_j (P_j(x) - P_j(z_k)) / (x - z_k)  =  (sum_j a_j P_j(x) - K_k) / (x - z_k),      K_k = sum_j a_j P_j(z_k)
// one multiplication by a_j per column and one Fq x Fq product per distinct point (z^m and z*g^o per trace offset o).
// Hints, in order of first use: per group the alphas of its columns, the constant K_k and the point; then the two
// degree coefficients.
struct DeepKey { int kind; int64_t index; bool operator<(const DeepKey &o) const { return std::tie(kind, index) < std::tie(o.kind, o.index); } };
enum { DK_ZM, DK_KZM, DK_CALPHA, DK_ZPT, DK_KZ, DK_TALPHA, DK_DALPHA, DK_DBETA };
inline Expr deep_expression(Graph &g, const std::vector<std::pair<u64, int64_t>> &trace_arguments, u32 num_trace_cols,
                            u32 num_composition_cols, std::vector<DeepKey> &keys) {
    std::map<DeepKey, u64> index;
    auto H = [&](int kind, int64_t i) {
        DeepKey k{kind, i};
        if (!index.count(k)) { index[k] = keys.size(); keys.push_back(k); }
        return Hint(g, index[k]);
    };
    Expr x = X(g), one = Constant(g, 1), total;
    bool first = true;
    auto add_group = [&](const std::vector<std::pair<u64, DeepKey>> &members, const DeepKey &konst, const DeepKey &point) {
        if (members.empty()) return;
        Expr acc;
        bool f = true;
        for (const auto &m : members) {
            Expr term = Trace(g, m.first, 0) * H(m.second.kind, m.second.index);
            acc = f ? term : acc + term;
            f = false;
        }
        Expr term = (acc - H(konst.kind, konst.index)) * (one / (x - H(point.kind, point.index)));
        total = first ? term : total + term;
        first = false;
    };
    std::vector<std::pair<u64, DeepKey>> members;
    for (u32 j = 0; j < num_composition_cols; j++) members.push_back({num_trace_cols + j, DeepKey{DK_CALPHA, (int64_t)j}});
    add_group(members, DeepKey{DK_KZM, 0}, DeepKey{DK_ZM, 0});
    std::set<int64_t> offsets;
    for (const auto &ta : trace_arguments) offsets.insert(ta.second);
    for (int64_t off : offsets) {
        members.clear();
        for (size_t i = 0; i < trace_arguments.size(); i++)
            if (trace_arguments[i].second == off) members.push_back({trace_arguments[i].first, DeepKey{DK_TALPHA, (int64_t)i}});
        add_group(members, DeepKey{DK_KZ, off}, DeepKey{DK_ZPT, off});
    }
    return total * (H(DK_DALPHA, 0) + x * H(DK_DBETA, 0));
}

// ------------------------------------------------------------------------------------------------ residency
// Device memory the estimates leave free: NTT plans with their twiddle and scale tables, the NTT temporary and the
// context's scratch arenas (prover.py MEMORY_RESERVE).
constexpr u64 MEMORY_RESERVE = (u64)3 << 30;

// device bytes of each residency, and the pinned host bytes of streamed_host (its node heaps)
struct PeakBytes { u64 resident, streamed, streamed_host, host; };

// Peak bytes of one proof in each residency, from the shapes (prover.py peak_bytes).  lanes: 1 for Fq = Fp, 3 for
// Fq3; ce_blowup: the composition blow-up; ff: the FRI folding factor.
inline PeakBytes peak_bytes(u64 n, u64 beta, u64 nbase, u64 next, u64 lanes, u64 ce_blowup, u64 ff = 2) {
    const u64 N = n * beta, M = n * ce_blowup;
    const u64 words = nbase + lanes * (next + ce_blowup);
    const u64 ntrees = next ? 3 : 2;
    const u64 fri = (8 * lanes + 64) * N / (ff - 1);
    const u64 common = 8 * words * n + 8 * N * lanes + fri + ((u64)16 << 20);
    const u64 blocks = common + 8 * words * n + 32 * n;
    return {common + 8 * M * lanes + 8 * words * N + 64 * ntrees * N, blocks + 32 * ntrees * N, blocks + 64 * n, 32 * ntrees * N};
}

inline std::string gib(long double b) {
    char s[64];
    snprintf(s, sizeof s, "%.2Lf GiB", b / (long double)((u64)1 << 30));
    return s;
}

// ------------------------------------------------------------------------------------------------ coset blocks
// ministark_b200/cosets.py: block q of the bit-reversed LDE over 7 * <g_N> is the size-n transform over the coset
// h_q * <g_n>, h_q = 7 * g_N^bitrev(q).  Returns the Montgomery words of h_0 .. h_(2^log_b - 1).
inline u64 bit_reverse_bits(u64 v, unsigned bits) {
    u64 r = 0;
    for (unsigned i = 0; i < bits; i++, v >>= 1) r = (r << 1) | (v & 1);
    return r;
}
inline std::vector<u64> coset_offsets(unsigned log_n, unsigned log_b) {
    const u64 gN = domain_generator(log_n + log_b);
    std::vector<u64> h;
    for (u64 q = 0; q < ((u64)1 << log_b); q++) h.push_back(to_mont(mulm(GENERATOR, powm(gN, bit_reverse_bits(q, log_b)))));
    return h;
}

// The index walk of MerkleTreeImpl::prove (src/merkle.rs:149-207): which leaves and which heap nodes a batched proof of
// `indices` names (cosets.py merkle_walk).
struct MerkleWalk { std::vector<u64> init, sib, path; };
inline MerkleWalk merkle_walk(u64 n_leaves, const std::vector<u64> &indices) {
    const std::set<u64> s(indices.begin(), indices.end());
    const std::vector<u64> idx(s.begin(), s.end());
    MerkleWalk w;
    std::vector<u64> node_q;
    for (size_t k = 0; k < idx.size();) {
        const u64 i = idx[k];
        w.init.push_back(i);
        node_q.push_back((n_leaves + i) >> 1);
        if (k + 1 < idx.size() && (i ^ 1) == idx[k + 1]) {
            w.init.push_back(idx[k + 1]);
            k += 2;
            continue;
        }
        w.sib.push_back(i ^ 1);
        k++;
    }
    for (size_t head = 0; head < node_q.size();) {
        const u64 i = node_q[head++];
        if (i > 2) node_q.push_back(i >> 1);
        if (head < node_q.size() && (i ^ 1) == node_q[head]) {
            head++;
            continue;
        }
        w.path.push_back(i ^ 1);
    }
    return w;
}

// Where node i of a tree committed in 2^log_b blocks lives in the split heap of ministark_host_nodes.h (cosets.py
// heap_location): block -1 and index i in the top heap of 2 * 2^log_b digests, else the block and the index in its local
// heap.
struct HeapLocation { int64_t block; u64 index; };
inline HeapLocation heap_location(u64 i, unsigned log_b) {
    const u64 beta = (u64)1 << log_b;
    if (i < 2 * beta) return {-1, i};
    const unsigned d = 63 - (unsigned)__builtin_clzll(i) - log_b;
    return {(int64_t)((i >> d) - beta), ((u64)1 << d) | (i & (((u64)1 << d) - 1))};
}

class GpuProver {
    ms_ctx *ctx = nullptr;
    void *pinned = nullptr;     // streamed_host's node heaps (ms_alloc_host_pinned), kept for the next proof
    u64 pinned_size = 0;

public:
    // bytes one proof may use on the device; 0: whatever the device has free
    u64 memory_budget = 0;
    // pinned host bytes one proof may hold (streamed_host's node heaps); 0: none.  Heaps pinned under a larger budget are
    // freed when the next proof starts.
    u64 host_memory_budget = 0;
    // "resident", "streamed" or "streamed_host": what the last proof ran (empty before the first)
    std::string last_residency;
    // the lowest free device memory ms_device_memory reported between the phases of the last proof
    u64 lowest_free_bytes = 0;
    // seconds the last proof spent pinning host memory (0 when it reused the held heaps or needed none)
    double last_pin_seconds = 0;

    explicit GpuProver(int device = 0) {
        if (ms_ctx_create(device, &ctx) != MS_OK) throw std::runtime_error("ms_ctx_create failed (no CUDA device? there is no CPU fallback)");
    }
    ~GpuProver() {
        if (!ctx) return;
        release_host_memory();
        ms_ctx_destroy(ctx);
    }
    GpuProver(const GpuProver &) = delete;
    GpuProver &operator=(const GpuProver &) = delete;

    // builds the extension columns (num_extension_columns x n elements of Fq, column-major, device) from the resident base
    // trace and the challenges: Trace::build_extension_columns (src/trace.rs:27-34)
    using ExtensionBuilder = std::function<DeviceBuf(ms_ctx *, const u64 *base_dev, u64 n, const std::vector<Fq> &challenges)>;
    ms_ctx *context() const { return ctx; }

    // free device memory as the driver reports it (SIZE_MAX where the library has no device limit or no ms_device_memory)
    u64 free_memory() const {
        if (!ms_device_memory) return SIZE_MAX;
        size_t f = 0;
        ck(ctx, ms_device_memory(ctx, &f, nullptr), "ms_device_memory");
        return f;
    }
    // bytes a proof may allocate: free device memory minus MEMORY_RESERVE, capped by memory_budget (prover.py
    // memory_available; there is no allocator cache to add back).  Negative when the device is nearly full.
    int64_t memory_available() const {
        const u64 f = free_memory();
        const int64_t avail = (f >= (u64)INT64_MAX ? INT64_MAX : (int64_t)f) - (int64_t)MEMORY_RESERVE;
        return memory_budget ? std::min<int64_t>((int64_t)memory_budget, avail) : avail;
    }
    // "resident" if its estimate fits, else "streamed" if that fits, else "streamed_host" if its device estimate fits and
    // its node heaps fit host_memory_budget, else the refusal (nothing is allocated yet)
    std::string choose_residency(const PeakBytes &est) const {
        const int64_t budget = memory_available();
        if ((int64_t)est.resident <= budget) return "resident";
        if ((int64_t)est.streamed <= budget) return "streamed";
        if (host_memory_budget && (int64_t)est.streamed_host <= budget && est.host <= host_memory_budget) return "streamed_host";
        std::string msg = "the proof does not fit on the device: it needs about " + gib(est.resident) + " resident or " +
                          gib(est.streamed) + " streamed, and " + gib(budget) + " is available";
        if (host_memory_budget)
            msg += "; with the Merkle node heaps in pinned host memory it needs about " + gib(est.streamed_host) + " on the device and " +
                   gib(est.host) + " of host memory, and " + gib(host_memory_budget) + " of host memory is allowed";
        throw std::runtime_error(msg);
    }

    // pinned host memory held for streamed_host's node heaps (0 before its first such proof)
    u64 pinned_bytes() const { return pinned_size; }
    // frees the pinned node heaps; the next streamed_host proof pins them again
    void release_host_memory() {
        if (!pinned) return;
        ms_ctx_sync(ctx);
        ms_free(ctx, pinned);
        pinned = nullptr;
        pinned_size = 0;
    }

    // base_trace: num_base_columns x n Montgomery words, column-major, HOST memory.  public_inputs: handed to gen_hints;
    // public_inputs_bytes: their CanonicalSerialize form for the coin seed (empty: the Fq elements back to back, as for
    // examples/fib's single claimed value).  The trace is not read when the proof does not fit (std::runtime_error).
    Proof prove(const AirConfig &cfg, ProofOptions options, const u64 *base_trace, u64 n, const std::vector<Fq> &public_inputs,
                const Bytes &public_inputs_bytes = {}, const ExtensionBuilder &ext_builder = nullptr) {
        DeviceBuf none;
        return prove_any(cfg, options, base_trace, none, n, public_inputs, public_inputs_bytes, ext_builder);
    }
    // the same from a DEVICE trace (num_base_columns x n, column-major, allocated on this prover's context), whose
    // ownership passes to the prover: it is freed as soon as the extension columns are built (ministark_b200's
    // release_base_columns), so the proof's peak device memory is the host trace's.
    Proof prove(const AirConfig &cfg, ProofOptions options, DeviceBuf base_trace, u64 n, const std::vector<Fq> &public_inputs,
                const Bytes &public_inputs_bytes = {}, const ExtensionBuilder &ext_builder = nullptr) {
        if (!base_trace.p || base_trace.ctx != ctx) throw std::runtime_error("the device trace must be allocated on this prover's context");
        return prove_any(cfg, options, nullptr, base_trace, n, public_inputs, public_inputs_bytes, ext_builder);
    }

private:
    struct Run {                    // per-proof state shared by the phases of both residencies
        const AirConfig &cfg;
        ProofOptions options;
        Air air;
        const std::vector<Fq> &public_inputs;
        const ExtensionBuilder &ext_builder;
        PublicCoin coin;
        Proof proof;
        int fq, lanes;
        unsigned log_n, log_b, log_N, log_ce;
        u64 n, N, ce, M, GEN, ONE;
        u32 nbase, next;
        const u64 *host_trace;      // exactly one of host_trace / device_trace holds the base trace
        DeviceBuf &device_trace;
        u8 *host_heaps = nullptr;   // streamed_host: the node heaps of the trees, N x 32 B each, in commitment order
    };

    void note_memory() { lowest_free_bytes = std::min<u64>(lowest_free_bytes, free_memory()); }

    Proof prove_any(const AirConfig &cfg, ProofOptions options, const u64 *host_trace, DeviceBuf &device_trace, u64 n,
                    const std::vector<Fq> &public_inputs, const Bytes &public_inputs_bytes, const ExtensionBuilder &ext_builder) {
        const u32 next = cfg.num_extension_columns;
        if (next && !ext_builder) throw std::runtime_error("this AIR has extension columns: pass an ExtensionBuilder");
        const int lanes = cfg.fq_is_fp ? 1 : 3;
        // gen_public_coin (examples/fib/main.rs:166-172)
        Bytes seed = public_inputs_bytes;
        if (seed.empty())
            for (const Fq &v : public_inputs) put_elem(seed, v, lanes);
        put_u64_le(seed, n);
        for (u8 b : options.to_bytes()) seed.push_back(b);
        Run r{cfg, options, Air(cfg, n, options), public_inputs, ext_builder, PublicCoin(sha256({seed}), lanes), Proof{},
              cfg.fq_is_fp ? MS_FIELD_FP : MS_FIELD_FQ3, lanes, 0, 0, 0, 0, n, 0, 0, 0, to_mont(GENERATOR), to_mont(1),
              cfg.num_base_columns, next, host_trace, device_trace};
        const unsigned beta = options.lde_blowup_factor;
        r.log_n = r.air.log_n;
        r.log_b = 31 - (unsigned)__builtin_clz(beta);
        r.log_N = r.log_n + r.log_b;
        r.N = n << r.log_b;
        r.ce = r.air.ce_blowup_factor;
        r.M = n * r.ce;
        r.log_ce = r.log_n + (63 - (unsigned)__builtin_clzll(r.ce));
        r.proof.options = options;
        r.proof.trace_len = n;
        const PeakBytes est = peak_bytes(n, beta, r.nbase, next, lanes, r.ce, options.fri_folding_factor);
        if (pinned_size > host_memory_budget) release_host_memory();   // heaps pinned under a larger budget are not held past a lower one
        last_residency = choose_residency(est);
        last_pin_seconds = 0;
        lowest_free_bytes = UINT64_MAX;
        note_memory();
        if (last_residency == "streamed_host") r.host_heaps = host_heaps(est.host);
        if (last_residency == "resident") prove_resident(r);
        else prove_streamed(r);
        note_memory();
        return std::move(r.proof);
    }

    // at least `bytes` of pinned host memory: the held allocation while it is large enough
    u8 *host_heaps(u64 bytes) {
        if (!ms_merkle_commit_block_sha256_host) throw std::runtime_error("the library lacks the host node heaps (ministark_host_nodes.h)");
        if (pinned_size < bytes) {
            release_host_memory();
            const auto t0 = std::chrono::steady_clock::now();
            ck(ctx, ms_alloc_host_pinned(ctx, bytes, &pinned), "ms_alloc_host_pinned");
            pinned_size = bytes;
            last_pin_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        }
        return static_cast<u8 *>(pinned);
    }

    // the base trace on the device: the handed-over device matrix, or a fresh upload of the host one
    DeviceBuf device_base(Run &r) {
        if (r.device_trace.p) return std::move(r.device_trace);
        DeviceBuf d(ctx, (size_t)r.nbase * r.n * 8);
        ck(ctx, ms_copy(ctx, d.p, r.host_trace, (size_t)r.nbase * r.n * 8), "upload");
        return d;
    }

    // challenges drawn after the base commitment, then the extension columns built from the natural-order base matrix,
    // which is freed as soon as they exist
    DeviceBuf extension_columns(Run &r, DeviceBuf &d_trace, std::vector<Fq> &challenges, std::vector<Fq> &hints) {
        for (u64 i = 0; i < r.air.num_challenges(); i++) challenges.push_back(r.coin.draw());
        hints = r.cfg.gen_hints ? r.cfg.gen_hints(r.n, r.public_inputs, challenges) : std::vector<Fq>{};
        DeviceBuf ext;
        if (r.next) ext = r.ext_builder(ctx, d_trace.words(), r.n, challenges);
        d_trace.release();
        return ext;
    }

    void prove_resident(Run &r) {
        const u64 n = r.n, N = r.N, ce = r.ce, M = r.M, GEN = r.GEN, ONE = r.ONE;
        const unsigned log_n = r.log_n, log_b = r.log_b, log_N = r.log_N, log_ce = r.log_ce;
        const u32 nbase = r.nbase, next = r.next;
        const int fq = r.fq, lanes = r.lanes;
        Proof &proof = r.proof;

        // ---- base trace commitment (prover.rs:46-55)
        DeviceBuf d_trace = device_base(r), base_polys(ctx, (size_t)nbase * n * 8), base_lde(ctx, (size_t)nbase * N * 8);
        DeviceBuf base_leaves(ctx, N * 32), base_nodes(ctx, N * 32);
        ck(ctx, ms_ntt_batch_to(ctx, MS_FIELD_FP, d_trace.p, n, base_polys.p, n, nbase, log_n, MS_NTT_INVERSE, ONE), "interpolate");
        ck(ctx, ms_lde_batch(ctx, MS_FIELD_FP, base_polys.p, n, base_lde.p, N, nbase, log_n, log_b, GEN, 1), "lde");
        proof.base_trace_commitment.resize(32);
        ck(ctx, ms_merkle_commit_sha256(ctx, MS_FIELD_FP, base_lde.p, N, nbase, N, base_leaves.p, base_nodes.p, proof.base_trace_commitment.data()), "commit");
        r.coin.reseed_with_digest(proof.base_trace_commitment);
        note_memory();

        // ---- extension trace commitment (prover.rs:56-72)
        std::vector<Fq> challenges, hints;
        DeviceBuf ext = extension_columns(r, d_trace, challenges, hints);
        DeviceBuf ext_polys, ext_lde, ext_leaves, ext_nodes;
        if (next) {
            ext_polys = DeviceBuf(ctx, (size_t)next * n * lanes * 8);
            ext_lde = DeviceBuf(ctx, (size_t)next * N * lanes * 8);
            ext_leaves = DeviceBuf(ctx, N * 32);
            ext_nodes = DeviceBuf(ctx, N * 32);
            ck(ctx, ms_ntt_batch_to(ctx, fq, ext.p, n, ext_polys.p, n, next, log_n, MS_NTT_INVERSE, ONE), "extension interpolate");
            ck(ctx, ms_lde_batch(ctx, fq, ext_polys.p, n, ext_lde.p, N, next, log_n, log_b, GEN, 1), "extension lde");
            proof.has_extension = true;
            proof.extension_trace_commitment.resize(32);
            ck(ctx, ms_merkle_commit_sha256(ctx, fq, ext_lde.p, N, next, N, ext_leaves.p, ext_nodes.p, proof.extension_trace_commitment.data()),
               "extension commit");
            r.coin.reseed_with_digest(proof.extension_trace_commitment);
        }
        ext.release();
        note_memory();

        // ---- constraint evaluation over the ce domain, read in place from the bit-reversed LDE prefix (prover.rs:75-108)
        std::vector<Fq> ccoefs;
        for (u64 i = 0; i < r.air.num_composition_constraint_coeffs(); i++) ccoefs.push_back(r.coin.draw());
        const Program prog = r.air.composition_program(nbase).bind(challenges, hints, ccoefs);
        DeviceBuf comp_evals(ctx, M * lanes * 8);
        ck(ctx, ms_eval_constraints(ctx, &prog.code[0][0], (unsigned)prog.code.size(), &prog.consts[0][0], (unsigned)prog.consts.size(),
                                    base_lde.p, N, nbase, next ? ext_lde.p : nullptr, N, next, fq, log_ce, GEN, 1, 0, comp_evals.p), "eval_constraints");
        note_memory();

        // ---- composition trace (prover.rs:110-125)
        ck(ctx, ms_ntt_batch(ctx, fq, comp_evals.p, M, 1, log_ce, MS_NTT_INVERSE, GEN), "composition iNTT");
        DeviceBuf comp_split;
        void *comp_polys = comp_evals.p;
        if (ce > 1) {
            comp_split = DeviceBuf(ctx, M * lanes * 8);
            ck(ctx, ms_matrix_from_rows(ctx, fq, comp_evals.p, n, (unsigned)ce, comp_split.p, n), "composition split");
            comp_polys = comp_split.p;
        }
        DeviceBuf comp_lde(ctx, ce * N * lanes * 8), comp_leaves(ctx, N * 32), comp_nodes(ctx, N * 32);
        ck(ctx, ms_lde_batch(ctx, fq, comp_polys, n, comp_lde.p, N, (unsigned)ce, log_n, log_b, GEN, 1), "composition lde");
        proof.composition_trace_commitment.resize(32);
        ck(ctx, ms_merkle_commit_sha256(ctx, fq, comp_lde.p, N, (unsigned)ce, N, comp_leaves.p, comp_nodes.p, proof.composition_trace_commitment.data()),
           "composition commit");
        r.coin.reseed_with_digest(proof.composition_trace_commitment);
        note_memory();

        // ---- DEEP composition evaluated over the LDE domain (composer.rs:89-188 in evaluation form)
        const Program dprog = bind_deep(r, base_polys.p, ext_polys.p, comp_polys);
        std::vector<const void *> cols;
        std::vector<int> is_q;
        for (u32 c = 0; c < nbase; c++) { cols.push_back(base_lde.words() + (size_t)c * N); is_q.push_back(0); }
        for (u32 c = 0; c < next; c++) { cols.push_back(ext_lde.words() + (size_t)c * N * lanes); is_q.push_back(1); }
        for (u64 j = 0; j < ce; j++) { cols.push_back(comp_lde.words() + (size_t)j * N * lanes); is_q.push_back(1); }
        DeviceBuf cur(ctx, N * lanes * 8);
        ck(ctx, ms_eval_constraints_ptrs(ctx, &dprog.code[0][0], (unsigned)dprog.code.size(), &dprog.consts[0][0], (unsigned)dprog.consts.size(),
                                         cols.data(), is_q.data(), (unsigned)cols.size(), fq, log_N, GEN, 1, 1, cur.p), "deep composition");
        note_memory();

        // ---- FRI, proof of work, FRI queries; then the trace rows and their paths from the resident trees
        const std::vector<u64> positions = fri_and_queries(r, cur);
        std::vector<u64> brow(positions.size() * nbase), crow(positions.size() * ce * lanes);
        ck(ctx, ms_gather_rows(ctx, MS_FIELD_FP, base_lde.p, N, nbase, N, positions.data(), (unsigned)positions.size(), brow.data()), "base rows");
        ck(ctx, ms_gather_rows(ctx, fq, comp_lde.p, N, (unsigned)ce, N, positions.data(), (unsigned)positions.size(), crow.data()), "composition rows");
        proof.trace_queries.base_trace_values = canon_vec(brow, 1);
        proof.trace_queries.composition_trace_values = canon_vec(crow, lanes);
        if (next) {
            std::vector<u64> erow(positions.size() * next * lanes);
            ck(ctx, ms_gather_rows(ctx, fq, ext_lde.p, N, next, N, positions.data(), (unsigned)positions.size(), erow.data()), "extension rows");
            proof.trace_queries.extension_trace_values = canon_vec(erow, lanes);
            proof.trace_queries.has_extension = true;
            proof.trace_queries.extension_trace_proof = view_of(ext_leaves, ext_nodes, N, positions);
        }
        proof.trace_queries.base_trace_proof = view_of(base_leaves, base_nodes, N, positions);
        proof.trace_queries.composition_trace_proof = view_of(comp_leaves, comp_nodes, N, positions);
    }

    // ---- streamed residency: coefficients and tree nodes stay, coset blocks are recomputed
    // coset block with offset h of the bit-reversed LDE of every column of `polys`, into `blk`.  Its NTT plan is dropped at
    // once: every block has its own offset, and beta cached plans with their full tables would take back the memory
    // streaming saves.
    void lde_block(const void *polys, void *blk, int field, unsigned ncols, unsigned log_n, u64 h) {
        const u64 n = (u64)1 << log_n;
        ck(ctx, ms_lde_batch(ctx, field, polys, n, blk, n, ncols, log_n, 0, h, 1), "block lde");
        ck(ctx, ms_set_option(ctx, "drop_plans", 1), "drop_plans");
    }

    // a tree's node heap: whole on the device, or split (ministark_host_nodes.h) into the top heap here and the blocks'
    // local heaps in pinned host memory
    struct NodeHeap {
        DeviceBuf dev;
        std::vector<u8> top;
        const u8 *host = nullptr;
    };

    // Merkle commitment of the bit-reversed LDE of `polys`, one coset block at a time: block q is transformed into `blk`
    // and hashed into its subtree of the node heap; the top log_b levels come from the block roots.  Returns the node heap
    // and writes the root.  With host_heap (N x 32 B pinned), block q's subtree is the local heap at host_heap + q * n * 32.
    NodeHeap commit_blocks(Run &r, const void *polys, void *blk, int field, unsigned ncols, const std::vector<u64> &offsets, Bytes &root,
                           u8 *host_heap = nullptr) {
        const u64 beta = (u64)1 << r.log_b;
        DeviceBuf nodes(ctx, (host_heap ? 2 * beta : r.N) * 32), own_roots;
        u8 *roots = static_cast<u8 *>(nodes.p) + 32 * beta;          // the top heap's last level
        if (!host_heap) {
            own_roots = DeviceBuf(ctx, beta * 32);
            roots = static_cast<u8 *>(own_roots.p);
        }
        for (u64 q = 0; q < beta; q++) {
            lde_block(polys, blk, field, ncols, r.log_n, offsets[q]);
            if (host_heap)
                ck(ctx, ms_merkle_commit_block_sha256_host(ctx, field, blk, r.n, ncols, r.log_n, host_heap + q * r.n * 32, roots + 32 * q),
                   "block commit (host heap)");
            else
                ck(ctx, ms_merkle_commit_block_sha256(ctx, field, blk, r.n, ncols, r.log_n, r.log_b, q, nodes.p, roots + 32 * q), "block commit");
        }
        if (beta > 1) ck(ctx, ms_merkle_nodes_sha256(ctx, roots, beta, nodes.p), "block roots");
        const u8 zero[32] = {0};          // the unused default digest (named by a walk over a 2-leaf tree)
        ck(ctx, ms_copy(ctx, nodes.p, zero, 32), "node 0");
        root.resize(32);
        ck(ctx, ms_copy(ctx, root.data(), static_cast<u8 *>(nodes.p) + 32, 32), "root");
        NodeHeap h;
        if (host_heap) {
            h.top.resize(2 * beta * 32);
            ck(ctx, ms_copy(ctx, h.top.data(), nodes.p, h.top.size()), "top heap");
            h.host = host_heap;
        } else {
            h.dev = std::move(nodes);
        }
        return h;
    }

    // the rows at `positions` and their MerkleView without the LDE: rows and leaf digests from the coefficients
    // (ms_lde_rows), path nodes gathered from the node heap (on the device, or split between here and pinned host memory)
    MerkleView streamed_rows(Run &r, const void *polys, int field, unsigned ncols, const NodeHeap &nodes, const std::vector<u64> &positions,
                             std::vector<u64> &rows) {
        const MerkleWalk w = merkle_walk(r.N, positions);
        std::vector<u64> ids = positions;
        ids.insert(ids.end(), w.init.begin(), w.init.end());
        ids.insert(ids.end(), w.sib.begin(), w.sib.end());
        const size_t row_words = (size_t)ncols * field;
        std::vector<u64> all(ids.size() * row_words);
        ck(ctx, ms_lde_rows(ctx, field, polys, r.n, ncols, r.log_n, r.log_b, r.GEN, ids.data(), (unsigned)ids.size(), all.data()), "lde rows");
        rows.assign(all.begin(), all.begin() + positions.size() * row_words);
        MerkleView v;
        for (size_t k = positions.size(); k < ids.size(); k++) {   // hash_rows: canonical words, 8 bytes little-endian each
            Bytes ser;
            for (size_t j = 0; j < row_words; j++) put_u64_le(ser, from_mont(all[k * row_words + j]));
            (k < positions.size() + w.init.size() ? v.initial_leaves : v.sibling_leaves).push_back(sha256({ser}));
        }
        if (!w.path.empty() && nodes.host) {
            ck(ctx, ms_ctx_sync(ctx), "sync");    // the last subtrees' copies to host memory
            for (u64 i : w.path) {
                const HeapLocation at = heap_location(i, r.log_b);
                const u8 *d = at.block < 0 ? nodes.top.data() + 32 * at.index : nodes.host + ((u64)at.block * r.n + at.index) * 32;
                v.nodes.emplace_back(d, d + 32);
            }
        } else if (!w.path.empty()) {
            std::vector<u8> path(w.path.size() * 32);
            ck(ctx, ms_gather_rows_rowmajor(ctx, nodes.dev.p, 4, r.N, w.path.data(), (unsigned)w.path.size(), path.data()), "path nodes");
            for (size_t i = 0; i < w.path.size(); i++) v.nodes.emplace_back(path.begin() + 32 * i, path.begin() + 32 * i + 32);
        }
        v.height = r.log_N;
        return v;
    }

    void prove_streamed(Run &r) {
        const u64 n = r.n, N = r.N, ce = r.ce, M = r.M, GEN = r.GEN, ONE = r.ONE;
        const unsigned log_n = r.log_n, log_ce = r.log_ce;
        const u32 nbase = r.nbase, next = r.next;
        const int fq = r.fq, lanes = r.lanes;
        Proof &proof = r.proof;
        if (!ms_merkle_commit_block_sha256 || !ms_lde_rows) throw std::runtime_error("the library lacks the streamed residency (ministark_stream.h)");
        const std::vector<u64> offsets = coset_offsets(log_n, r.log_b);
        auto host_heap = [&](u64 tree) { return r.host_heaps ? r.host_heaps + tree * N * 32 : nullptr; };   // streamed_host

        // ---- base trace commitment: coefficients stay, the LDE passes through one block buffer
        DeviceBuf d_trace = device_base(r), base_polys(ctx, (size_t)nbase * n * 8), base_blk(ctx, (size_t)nbase * n * 8);
        ck(ctx, ms_ntt_batch_to(ctx, MS_FIELD_FP, d_trace.p, n, base_polys.p, n, nbase, log_n, MS_NTT_INVERSE, ONE), "interpolate");
        NodeHeap base_nodes = commit_blocks(r, base_polys.p, base_blk.p, MS_FIELD_FP, nbase, offsets, proof.base_trace_commitment, host_heap(0));
        r.coin.reseed_with_digest(proof.base_trace_commitment);
        note_memory();

        // ---- extension trace commitment
        std::vector<Fq> challenges, hints;
        DeviceBuf ext = extension_columns(r, d_trace, challenges, hints);
        DeviceBuf ext_polys, ext_blk;
        NodeHeap ext_nodes;
        if (next) {
            ext_polys = DeviceBuf(ctx, (size_t)next * n * lanes * 8);
            ck(ctx, ms_ntt_batch_to(ctx, fq, ext.p, n, ext_polys.p, n, next, log_n, MS_NTT_INVERSE, ONE), "extension interpolate");
            ext.release();
            ext_blk = DeviceBuf(ctx, (size_t)next * n * lanes * 8);
            ext_nodes = commit_blocks(r, ext_polys.p, ext_blk.p, fq, next, offsets, proof.extension_trace_commitment, host_heap(1));
            proof.has_extension = true;
            r.coin.reseed_with_digest(proof.extension_trace_commitment);
        }
        note_memory();

        auto trace_block = [&](u64 h) {
            lde_block(base_polys.p, base_blk.p, MS_FIELD_FP, nbase, log_n, h);
            std::vector<const void *> cols;
            for (u32 c = 0; c < nbase; c++) cols.push_back(base_blk.words() + (size_t)c * n);
            if (next) {
                lde_block(ext_polys.p, ext_blk.p, fq, next, log_n, h);
                for (u32 c = 0; c < next; c++) cols.push_back(ext_blk.words() + (size_t)c * n * lanes);
            }
            return cols;
        };

        // ---- constraint evaluation, block by block: the blocks q < ce_blowup of the LDE are the ce domain
        std::vector<Fq> ccoefs;
        for (u64 i = 0; i < r.air.num_composition_constraint_coeffs(); i++) ccoefs.push_back(r.coin.draw());
        const Program prog = r.air.block_program(nbase).bind(challenges, hints, ccoefs);
        DeviceBuf comp_evals(ctx, M * lanes * 8);
        std::vector<int> is_q(nbase, 0);
        is_q.resize(nbase + next, 1);
        for (u64 q = 0; q < ce; q++) {
            const std::vector<const void *> cols = trace_block(offsets[q]);
            ck(ctx, ms_eval_constraints_ptrs(ctx, &prog.code[0][0], (unsigned)prog.code.size(), &prog.consts[0][0], (unsigned)prog.consts.size(),
                                             cols.data(), is_q.data(), (unsigned)cols.size(), fq, log_n, offsets[q], 1, 1,
                                             comp_evals.words() + q * n * lanes), "eval_constraints (block)");
        }
        note_memory();

        // ---- composition trace: the bit-reversed ce-domain column -> coefficients -> ce_blowup columns
        ck(ctx, ms_bit_reverse(ctx, fq, comp_evals.p, M, 1, log_ce), "composition bit reverse");
        ck(ctx, ms_ntt_batch(ctx, fq, comp_evals.p, M, 1, log_ce, MS_NTT_INVERSE, GEN), "composition iNTT");
        DeviceBuf comp_split;
        if (ce > 1) {
            comp_split = DeviceBuf(ctx, M * lanes * 8);
            ck(ctx, ms_matrix_from_rows(ctx, fq, comp_evals.p, n, (unsigned)ce, comp_split.p, n), "composition split");
            comp_evals.release();
        }
        const void *comp_polys = ce > 1 ? comp_split.p : comp_evals.p;
        ck(ctx, ms_set_option(ctx, "drop_scratch", 1), "drop_scratch");   // the size-M transform's temporary
        DeviceBuf comp_blk(ctx, ce * n * lanes * 8);
        NodeHeap comp_nodes = commit_blocks(r, comp_polys, comp_blk.p, fq, (unsigned)ce, offsets, proof.composition_trace_commitment,
                                            host_heap(next ? 2 : 1));
        r.coin.reseed_with_digest(proof.composition_trace_commitment);
        note_memory();

        // ---- DEEP composition polynomial: every block of the three matrices recomputed once more
        const Program dprog = bind_deep(r, base_polys.p, ext_polys.p, comp_polys);
        DeviceBuf deep(ctx, N * lanes * 8);
        is_q.resize(nbase + next + ce, 1);
        for (u64 q = 0; q < offsets.size(); q++) {
            std::vector<const void *> cols = trace_block(offsets[q]);
            lde_block(comp_polys, comp_blk.p, fq, (unsigned)ce, log_n, offsets[q]);
            for (u64 j = 0; j < ce; j++) cols.push_back(comp_blk.words() + j * n * lanes);
            ck(ctx, ms_eval_constraints_ptrs(ctx, &dprog.code[0][0], (unsigned)dprog.code.size(), &dprog.consts[0][0], (unsigned)dprog.consts.size(),
                                             cols.data(), is_q.data(), (unsigned)cols.size(), fq, log_n, offsets[q], 1, 1,
                                             deep.words() + q * n * lanes), "deep composition (block)");
        }
        note_memory();                  // the high point: the codeword and one block of every matrix besides the rest
        base_blk.release();
        ext_blk.release();
        comp_blk.release();

        // ---- FRI, proof of work, FRI queries; then rows and leaf digests from the coefficients, paths from the node heaps
        const std::vector<u64> positions = fri_and_queries(r, deep);
        std::vector<u64> rows;
        Queries &tq = proof.trace_queries;
        tq.base_trace_proof = streamed_rows(r, base_polys.p, MS_FIELD_FP, nbase, base_nodes, positions, rows);
        tq.base_trace_values = canon_vec(rows, 1);
        tq.composition_trace_proof = streamed_rows(r, comp_polys, fq, (unsigned)ce, comp_nodes, positions, rows);
        tq.composition_trace_values = canon_vec(rows, lanes);
        if (next) {
            tq.extension_trace_proof = streamed_rows(r, ext_polys.p, fq, next, ext_nodes, positions, rows);
            tq.extension_trace_values = canon_vec(rows, lanes);
            tq.has_extension = true;
        }
    }

    // ---- phases both residencies share
    static std::vector<Fq> canon_vec(const std::vector<u64> &w, int l) {
        std::vector<Fq> o;
        for (size_t i = 0; i < w.size(); i += l) {
            Fq v;
            for (int k = 0; k < l; k++) v.c[k] = from_mont(w[i + k]);
            o.push_back(v);
        }
        return o;
    }

    MerkleView view_of(const DeviceBuf &leaves, const DeviceBuf &nodes, u64 nleaves, const std::vector<u64> &idx) {
        const unsigned height = 63 - (unsigned)__builtin_clzll(nleaves);
        std::vector<u8> init(idx.size() * 32), sib(idx.size() * 32), path(idx.size() * (height ? height : 1) * 32);
        unsigned counts[3];
        ck(ctx, ms_merkle_prove_sha256(ctx, leaves.p, nodes.p, nleaves, idx.data(), (unsigned)idx.size(), init.data(), sib.data(), path.data(), counts),
           "merkle prove");
        MerkleView v;
        auto take = [](const std::vector<u8> &b, unsigned k) { std::vector<Bytes> o; for (unsigned i = 0; i < k; i++) o.emplace_back(b.begin() + 32 * i, b.begin() + 32 * i + 32); return o; };
        v.initial_leaves = take(init, counts[0]);
        v.sibling_leaves = take(sib, counts[1]);
        v.nodes = take(path, counts[2]);
        v.height = height;
        return v;
    }

    // out-of-domain evaluations (composer.rs:43-86) from the coefficients, into the proof and the coin; then the DEEP
    // coefficients are drawn and bound into the DEEP program
    Program bind_deep(Run &r, const void *base_polys, const void *ext_polys, const void *comp_polys) {
        const u64 n = r.n, ce = r.ce;
        const u32 nbase = r.nbase, next = r.next;
        const int fq = r.fq, lanes = r.lanes;
        Proof &proof = r.proof;
        const Fq z = r.coin.draw();
        const auto trace_args = r.air.trace_arguments();
        std::vector<int64_t> offsets;
        for (const auto &ta : trace_args)
            if (std::find(offsets.begin(), offsets.end(), ta.second) == offsets.end()) offsets.push_back(ta.second);
        std::sort(offsets.begin(), offsets.end());
        const u64 g = domain_generator(r.log_n), g_inv = invm(g);
        std::vector<Fq> z_points;
        std::vector<u64> pts;
        for (int64_t o : offsets) {
            const Fq p = fq_scale(z, powm(o >= 0 ? g : g_inv, (u64)(o >= 0 ? o : -o)));
            z_points.push_back(p);
            for (int l = 0; l < 3; l++) pts.push_back(to_mont(p.c[l]));
        }
        const Fq z_m = fq_pow(z, ce);
        std::vector<u64> base_ood((size_t)nbase * offsets.size() * 3), comp_ood(ce * 3);
        ck(ctx, ms_poly_eval(ctx, MS_FIELD_FP, base_polys, n, nbase, n, pts.data(), (unsigned)offsets.size(), base_ood.data()), "ood (trace)");
        std::vector<u64> ext_ood((size_t)next * offsets.size() * 3);
        if (next) ck(ctx, ms_poly_eval(ctx, fq, ext_polys, n, next, n, pts.data(), (unsigned)offsets.size(), ext_ood.data()), "ood (extension)");
        const u64 zm_w[3] = {to_mont(z_m.c[0]), to_mont(z_m.c[1]), to_mont(z_m.c[2])};
        ck(ctx, ms_poly_eval(ctx, fq, comp_polys, n, (unsigned)ce, n, zm_w, 1, comp_ood.data()), "ood (composition)");
        auto canon3 = [&](const u64 *w) {
            Fq v(from_mont(w[0]), from_mont(w[1]), from_mont(w[2]));
            if (lanes == 1 && (v.c[1] || v.c[2])) throw std::runtime_error("out-of-domain value left the base field although Fq = Fp");
            return v;
        };
        for (const auto &ta : trace_args) {
            const size_t k = std::find(offsets.begin(), offsets.end(), ta.second) - offsets.begin();
            if (ta.first < nbase) proof.execution_trace_ood_evals.push_back(canon3(&base_ood[(ta.first * offsets.size() + k) * 3]));
            else if (ta.first < nbase + next) proof.execution_trace_ood_evals.push_back(canon3(&ext_ood[((ta.first - nbase) * offsets.size() + k) * 3]));
            else throw std::runtime_error("trace argument names a column that does not exist");
        }
        for (u64 j = 0; j < ce; j++) proof.composition_trace_ood_evals.push_back(canon3(&comp_ood[j * 3]));
        std::vector<Fq> all_oods = proof.execution_trace_ood_evals;
        all_oods.insert(all_oods.end(), proof.composition_trace_ood_evals.begin(), proof.composition_trace_ood_evals.end());
        r.coin.reseed_with_field_elements(all_oods);

        std::vector<Fq> ex_alphas, co_alphas;
        for (size_t i = 0; i < trace_args.size(); i++) ex_alphas.push_back(r.coin.draw());
        for (u64 j = 0; j < ce; j++) co_alphas.push_back(r.coin.draw());
        const Fq d_alpha = r.coin.draw(), d_beta = r.coin.draw();
        Graph dg;
        std::vector<DeepKey> keys;
        const Expr dexpr = deep_expression(dg, trace_args, nbase + next, (u32)ce, keys);
        std::vector<Fq> dhints;
        for (const DeepKey &k : keys) {
            switch (k.kind) {
                case DK_ZM: dhints.push_back(z_m); break;
                case DK_KZM: {      // sum_j alpha'_j H_j(z^m)
                    Fq acc;
                    for (u64 j = 0; j < ce; j++) acc = fq_add(acc, fq_mul(co_alphas[j], proof.composition_trace_ood_evals[j]));
                    dhints.push_back(acc);
                    break;
                }
                case DK_CALPHA: dhints.push_back(co_alphas[k.index]); break;
                case DK_ZPT: dhints.push_back(z_points[std::find(offsets.begin(), offsets.end(), k.index) - offsets.begin()]); break;
                case DK_KZ: {       // sum over the arguments with this offset of alpha * T(z g^o)
                    Fq acc;
                    for (size_t i = 0; i < trace_args.size(); i++)
                        if (trace_args[i].second == k.index) acc = fq_add(acc, fq_mul(ex_alphas[i], proof.execution_trace_ood_evals[i]));
                    dhints.push_back(acc);
                    break;
                }
                case DK_TALPHA: dhints.push_back(ex_alphas[k.index]); break;
                case DK_DALPHA: dhints.push_back(d_alpha); break;
                default: dhints.push_back(d_beta);
            }
        }
        return compile_program(dg, dexpr.id, nbase, 1, (int)r.log_N, /*batch_inverses=*/true).bind({}, dhints, {});
    }

    // FRI layers (fri.rs:179-249), the remainder, the proof of work, the query positions and the FRI layers' query
    // answers; `cur` is the DEEP codeword over the LDE domain in bit-reversed order.  Returns the query positions.
    std::vector<u64> fri_and_queries(Run &r, DeviceBuf &cur) {
        const ProofOptions &options = r.options;
        const int fq = r.fq, lanes = r.lanes;
        const u64 ONE = r.ONE;
        Proof &proof = r.proof;
        const unsigned ff = options.fri_folding_factor, log_ff = 31 - (unsigned)__builtin_clz(ff);
        struct Layer { DeviceBuf evals, leaves, nodes; Bytes root; u64 nrows; };
        std::vector<Layer> layers;
        unsigned ln = r.log_N;
        for (unsigned l = 0; l < options.fri_num_layers(r.N); l++) {
            Layer L;
            if (ln < log_ff) throw std::runtime_error("FRI: the evaluation domain is smaller than the folding factor");
            L.nrows = (u64)1 << (ln - log_ff);
            L.leaves = DeviceBuf(ctx, L.nrows * 32);
            L.nodes = DeviceBuf(ctx, L.nrows * 32);
            L.root.resize(32);
            ck(ctx, ms_merkle_commit_rows_sha256(ctx, cur.p, ff * lanes, L.nrows, L.leaves.p, L.nodes.p, L.root.data()), "fri layer commit");
            r.coin.reseed_with_digest(L.root);
            const Fq alpha = r.coin.draw();
            const u64 aw[3] = {to_mont(alpha.c[0]), to_mont(alpha.c[1]), to_mont(alpha.c[2])};
            DeviceBuf nxt(ctx, L.nrows * lanes * 8);
            ck(ctx, ms_fri_fold(ctx, fq, cur.p, ln, log_ff, ONE, aw, nxt.p), "fri fold");
            L.evals = std::move(cur);
            cur = std::move(nxt);
            layers.push_back(std::move(L));
            ln -= log_ff;
        }
        {   // set_remainder (fri.rs:233-249)
            const u64 rem_size = (u64)1 << ln;
            ck(ctx, ms_bit_reverse(ctx, fq, cur.p, rem_size, 1, ln), "remainder bit reverse");
            ck(ctx, ms_ntt_batch(ctx, fq, cur.p, rem_size, 1, ln, MS_NTT_INVERSE, ONE), "remainder iNTT");
            std::vector<u64> w(rem_size * lanes);
            ck(ctx, ms_copy(ctx, w.data(), cur.p, w.size() * 8), "remainder download");
            const u64 keep = rem_size / options.lde_blowup_factor;
            for (u64 i = 0; i < rem_size; i++) {
                Fq v;
                for (int l = 0; l < lanes; l++) v.c[l] = from_mont(w[i * lanes + l]);
                if (i < keep) proof.fri_proof.remainder_coeffs.push_back(v);
                else if (!v.is_zero()) throw std::runtime_error("FRI remainder is not low degree");
            }
            r.coin.reseed_with_field_elements(proof.fri_proof.remainder_coeffs);
        }
        note_memory();
        // ---- proof of work + queries
        if (options.grinding_factor) {
            ck(ctx, ms_pow_grind_sha256(ctx, r.coin.seed.data(), options.grinding_factor, &proof.pow_nonce), "pow");
            if (!r.coin.verify_proof_of_work(options.grinding_factor, proof.pow_nonce)) throw std::runtime_error("bad nonce");
            r.coin.reseed_with_int(proof.pow_nonce);
        }
        const std::vector<u64> positions = r.coin.draw_queries(options.num_queries, r.N);
        std::vector<u64> folded = positions;
        for (Layer &L : layers) {
            std::set<u64> s;
            for (u64 p : folded) s.insert(p / ff);
            folded.assign(s.begin(), s.end());
            std::vector<u64> rows(folded.size() * ff * lanes);
            ck(ctx, ms_gather_rows_rowmajor(ctx, L.evals.p, ff * lanes, L.nrows, folded.data(), (unsigned)folded.size(), rows.data()), "fri rows");
            LayerProof lp;
            lp.flattenend_rows = canon_vec(rows, lanes);
            lp.merkle_proof = view_of(L.leaves, L.nodes, L.nrows, folded);
            lp.commitment = L.root;
            proof.fri_proof.layers.push_back(std::move(lp));
        }
        return positions;
    }
};

// ------------------------------------------------------------------------------------------------ examples/brainfuck
namespace bf {

// public inputs of the brainfuck claim as ark-serialize writes them (main.rs:56-61): String, Vec<u8>, Vec<u8>
inline Bytes claim_bytes(const std::string &source, const Bytes &input, const Bytes &output) {
    Bytes o;
    put_u64_le(o, source.size());
    o.insert(o.end(), source.begin(), source.end());
    put_u64_le(o, input.size());
    o.insert(o.end(), input.begin(), input.end());
    put_u64_le(o, output.size());
    o.insert(o.end(), output.begin(), output.end());
    return o;
}

// The nine Fq3 extension columns (examples/brainfuck/trace.rs:108-279) on the device, as in
// ministark_b200/examples/brainfuck.py::_device_extension: every column is x_0 = init, x_(i+1) = x_i * a_i + b_i with
// per-row factors that are pointwise expressions of the base row (fused evaluator over the resident trace + eight 0/1
// helper columns derived from the integer rows), then one ms_scan_affine.  instr_initial / mem_initial: the two
// permutation start values (the reference draws them from ark_std::test_rng()).
// d_aux: the eight helper columns ((8, n) Montgomery words on the device) of BrainfuckTrace.helper_columns().
inline DeviceBuf device_extension(ms_ctx *ctx, u64 n, const DeviceBuf &d_aux, const u64 *base_dev, const std::vector<Fq> &ch,
                                  const Fq &instr_initial, const Fq &mem_initial) {
    const unsigned log_n = 63 - (unsigned)__builtin_clzll(n);
    const u64 ONE = to_mont(1);
    std::vector<const void *> cols;
    std::vector<int> is_q(25, 0);
    for (u32 c = 0; c < 17; c++) cols.push_back(base_dev + (u64)c * n);
    for (u32 k = 0; k < 8; k++) cols.push_back(d_aux.words() + (u64)k * n);
    auto evaluate = [&](Graph &g, const Expr &e) {
        DeviceBuf out(ctx, n * 24);
        const Program p = compile_program(g, e.id, 25, 1, (int)log_n).bind(ch, {}, {});
        ck(ctx, ms_eval_constraints_ptrs(ctx, &p.code[0][0], (unsigned)p.code.size(), &p.consts[0][0], (unsigned)p.consts.size(), cols.data(),
                                         is_q.data(), 25, MS_FIELD_FQ3, log_n, ONE, 0, 0, out.p), "extension factors");
        return out;
    };
    Graph g;
    auto T = [&](u32 c) { return Trace(g, c, 0); };
    auto AUX = [&](u32 k) { return Trace(g, 17 + k, 0); };
    auto CH = [&](u64 i) { return Challenge(g, i); };
    const Expr one = Constant(g, 1);
    auto instr_fp = [&](u32 ip, u32 c, u32 nx) { return CH(CH_ALPHA) - CH(CH_A) * T(ip) - CH(CH_B) * T(c) - CH(CH_C) * T(nx); };
    auto mem_fp = [&](u32 cy, u32 mp, u32 v) { return CH(CH_BETA) - CH(CH_D) * T(cy) - CH(CH_E) * T(mp) - CH(CH_F) * T(v); };
    auto gated = [&](const Expr &mask, const Expr &factor) { return one + mask * (factor - one); };   // factor where mask = 1, else 1
    DeviceBuf ext(ctx, (size_t)9 * n * 24);
    auto words3 = [](const Fq &v) { return std::array<u64, 3>{to_mont(v.c[0]), to_mont(v.c[1]), to_mont(v.c[2])}; };
    const std::array<u64, 3> zero3 = {0, 0, 0}, ii = words3(instr_initial), mi = words3(mem_initial);
    auto scan = [&](u32 k, const std::array<u64, 3> &init, const void *a, const u64 *a_const, const void *b, int b_field, int inclusive) {
        ck(ctx, ms_scan_affine(ctx, MS_FIELD_FQ3, a, MS_FIELD_FQ3, a_const, b, b_field, n, init.data(), inclusive, ext.words() + (u64)k * n * 3), "scan");
    };
    { DeviceBuf a = evaluate(g, gated(AUX(0), instr_fp(IP, CURR_INSTR, NEXT_INSTR))); scan(0, ii, a.p, nullptr, nullptr, 1, 0); }
    { DeviceBuf a = evaluate(g, gated(AUX(0), mem_fp(CYCLE, MP, MEM_VAL))); scan(1, mi, a.p, nullptr, nullptr, 1, 0); }
    { DeviceBuf a = evaluate(g, gated(AUX(1), CH(CH_GAMMA))); scan(2, zero3, a.p, nullptr, d_aux.words() + 2 * n, MS_FIELD_FP, 0); }
    { DeviceBuf a = evaluate(g, gated(AUX(3), CH(CH_DELTA))); scan(3, zero3, a.p, nullptr, d_aux.words() + 4 * n, MS_FIELD_FP, 0); }
    { DeviceBuf a = evaluate(g, gated(AUX(5), mem_fp(M_CYCLE, M_MP, M_MEM_VAL))); scan(4, mi, a.p, nullptr, nullptr, 1, 0); }
    { DeviceBuf a = evaluate(g, gated(AUX(6), instr_fp(I_IP, I_CURR_INSTR, I_NEXT_INSTR))); scan(5, ii, a.p, nullptr, nullptr, 1, 1); }
    {
        DeviceBuf a = evaluate(g, gated(AUX(7), CH(CH_ETA)));
        DeviceBuf b = evaluate(g, AUX(7) * (CH(CH_A) * T(I_IP) + CH(CH_B) * T(I_CURR_INSTR) + CH(CH_C) * T(I_NEXT_INSTR)));
        scan(6, zero3, a.p, nullptr, b.p, MS_FIELD_FQ3, 1);
    }
    const std::array<u64, 3> gamma = words3(ch.at(CH_GAMMA)), delta = words3(ch.at(CH_DELTA));
    scan(7, zero3, nullptr, gamma.data(), base_dev + (u64)IN_VALUE * n, MS_FIELD_FP, 1);
    scan(8, zero3, nullptr, delta.data(), base_dev + (u64)OUT_VALUE * n, MS_FIELD_FP, 1);
    ck(ctx, ms_ctx_sync(ctx), "extension sync");       // the factor buffers above are freed when their scopes end
    return ext;
}

// the helper columns computed on the host from the integer rows of a host trace
inline DeviceBuf device_extension(ms_ctx *ctx, const VmTrace &t, const u64 *base_dev, const std::vector<Fq> &ch, const Fq &instr_initial,
                                  const Fq &mem_initial) {
    const u64 n = t.n;
    std::vector<u64> aux(8 * n);    // Montgomery words
    for (u64 r = 0; r < n; r++) {
        const u64 ci = t.at(CURR_INSTR, r), nxt_mv = t.at(MEM_VAL, (r + 1) % n), iip = t.at(I_IP, r);
        const bool same_ip = r > 0 && iip == t.at(I_IP, r - 1);
        const u64 v[8] = {ci != 0, ci == ',', ci == ',' ? nxt_mv : 0, ci == '.', ci == '.' ? nxt_mv : 0, t.at(M_DUMMY, r) == 0,
                          (u64)(t.at(I_CURR_INSTR, r) != 0 && same_ip), (u64)!same_ip};
        for (int k = 0; k < 8; k++) aux[(u64)k * n + r] = to_mont(v[k]);
    }
    DeviceBuf d_aux(ctx, aux.size() * 8);
    ck(ctx, ms_copy(ctx, d_aux.p, aux.data(), aux.size() * 8), "helper columns upload");
    return device_extension(ctx, n, d_aux, base_dev, ch, instr_initial, mem_initial);
}

// the helper columns computed on the device from the filled base matrix (ms_bf_helper_columns), as for a device trace
inline DeviceBuf device_extension(ms_ctx *ctx, u64 n, const u64 *base_dev, const std::vector<Fq> &ch, const Fq &instr_initial,
                                  const Fq &mem_initial) {
    if (!ms_bf_helper_columns) throw std::runtime_error("the library lacks ms_bf_helper_columns (ministark_bf.h)");
    DeviceBuf d_aux(ctx, (size_t)8 * n * 8);
    ck(ctx, ms_bf_helper_columns(ctx, base_dev, n, d_aux.p), "helper columns");
    return device_extension(ctx, n, d_aux, base_dev, ch, instr_initial, mem_initial);
}

// The trace of one run with its 17 base columns on the device (ministark_b200/examples/brainfuck.py::simulate with a
// device): the VM on the host (ms_bf_run), its records uploaded, the table lengths (ms_bf_trace_sizes) and the tables
// (ms_bf_trace_fill).  The matrix is complete when this returns.  VM errors (the memory pointer leaves the tape, the input
// runs out, max_cycles cycles do not end the program) throw std::runtime_error with the library's message.
struct DeviceTrace {
    DeviceBuf base;                 // (17, n) column-major Montgomery words
    u64 n = 0;
    Bytes output;
};
inline DeviceTrace simulate_device(ms_ctx *ctx, const std::string &source, const Bytes &input = {}, u64 max_cycles = (u64)1 << 26) {
    if (!ms_bf_run || !ms_bf_trace_sizes || !ms_bf_trace_fill) throw std::runtime_error("the library lacks the brainfuck trace (ministark_bf.h)");
    std::vector<uint32_t> program;
    for (u64 w : compile(source)) program.push_back((uint32_t)w);
    // room for the longest run; pages the run does not reach are never touched
    std::unique_ptr<uint64_t[]> log(new uint64_t[max_cycles + 1]);
    std::unique_ptr<uint8_t[]> out(new uint8_t[max_cycles ? max_cycles : 1]);
    uint64_t counts[2] = {0, 0};
    if (ms_bf_run(program.data(), program.size(), input.data(), input.size(), max_cycles, log.get(), out.get(), counts) != MS_OK)
        throw std::runtime_error(ms_last_error(nullptr));
    const size_t nrec = counts[0] + 1;
    DeviceTrace t;
    t.output.assign(out.get(), out.get() + counts[1]);
    DeviceBuf d_prog(ctx, program.size() * 4), d_log(ctx, nrec * 8);
    ck(ctx, ms_copy(ctx, d_prog.p, program.data(), program.size() * 4), "program upload");
    ck(ctx, ms_copy(ctx, d_log.p, log.get(), nrec * 8), "records upload");
    uint64_t sizes[MS_BF_NSIZES];
    ck(ctx, ms_bf_trace_sizes(ctx, static_cast<const uint32_t *>(d_prog.p), program.size(), d_log.words(), nrec, sizes), "trace sizes");
    t.n = sizes[MS_BF_N];
    t.base = DeviceBuf(ctx, (size_t)17 * t.n * 8);
    DeviceBuf work(ctx, sizes[MS_BF_WORK_BYTES]);
    ck(ctx, ms_bf_trace_fill(ctx, static_cast<const uint32_t *>(d_prog.p), program.size(), d_log.words(), nrec, sizes, work.p, t.base.p),
       "trace fill");
    ck(ctx, ms_ctx_sync(ctx), "trace sync");    // the fill is done before its inputs are freed and the matrix handed over
    return t;
}

// ---- ark_std::test_rng(): ChaCha12 seeded as the reference seeds it, Fq3 elements drawn as Fq3::rand draws them
// (ministark_b200/examples/brainfuck.py::test_rng_fq3).  The reference takes the two permutation start values of the
// extension columns from it.
inline void chacha_block(const uint32_t key[8], u64 counter, uint32_t out[16], int rounds = 12) {
    uint32_t st[16] = {0x61707865, 0x3320646E, 0x79622D32, 0x6B206574};
    for (int i = 0; i < 8; i++) st[4 + i] = key[i];
    st[12] = (uint32_t)counter;
    st[13] = (uint32_t)(counter >> 32);
    st[14] = st[15] = 0;          // rand_chacha: 64-bit block counter in words 12-13, stream id 0 in words 14-15
    uint32_t w[16];
    for (int i = 0; i < 16; i++) w[i] = st[i];
    auto rot = [](uint32_t v, int r) { return (v << r) | (v >> (32 - r)); };
    auto qr = [&](int a, int b, int c, int d) {
        w[a] += w[b]; w[d] = rot(w[d] ^ w[a], 16);
        w[c] += w[d]; w[b] = rot(w[b] ^ w[c], 12);
        w[a] += w[b]; w[d] = rot(w[d] ^ w[a], 8);
        w[c] += w[d]; w[b] = rot(w[b] ^ w[c], 7);
    };
    for (int i = 0; i < rounds / 2; i++) {
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15);
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14);
    }
    for (int i = 0; i < 16; i++) out[i] = w[i] + st[i];
}
inline std::vector<Fq> test_rng_fq3(size_t count) {
    const uint8_t seed[32] = {1, 0, 0, 0, 23, 0, 0, 0, 200, 1, 0, 0, 210, 30, 0, 0};
    uint32_t key[8];
    for (int i = 0; i < 8; i++) key[i] = (uint32_t)seed[4 * i] | (uint32_t)seed[4 * i + 1] << 8 | (uint32_t)seed[4 * i + 2] << 16 | (uint32_t)seed[4 * i + 3] << 24;
    std::vector<uint32_t> words;
    u64 ctr = 0;
    size_t at = 0;
    auto next_u64 = [&]() {
        if (words.size() - at < 2) {
            words.erase(words.begin(), words.begin() + at);
            at = 0;
            uint32_t blk[16];
            chacha_block(key, ctr++, blk);
            words.insert(words.end(), blk, blk + 16);
        }
        const u64 lo = words[at], hi = words[at + 1];
        at += 2;
        return hi << 32 | lo;
    };
    auto fp = [&]() {
        for (;;) {
            const u64 w = next_u64();
            if (w < P) return from_mont(w);     // a raw u64 below p is taken as the Montgomery word
        }
    };
    std::vector<Fq> out;
    for (size_t i = 0; i < count; i++) {
        const u64 c0 = fp(), c1 = fp(), c2 = fp();
        out.push_back(Fq(c0, c1, c2));
    }
    return out;
}

}  // namespace bf
}  // namespace mshost
