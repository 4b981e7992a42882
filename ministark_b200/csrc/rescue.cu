// rescue.cu — the traces of examples/rescue and examples/merkle, side by side on the device: K independent chains of L
// Rescue-Prime permutations (include/ministark_rescue.h), K messages absorbed by the Rescue-Prime sponge
// (include/ministark_rescue_hash.h), and the Rescue-Prime Merkle tree with K authentication paths through it
// (include/ministark_rescue_merkle.h).
//
// One chain (or message, tree node, path) per 16 lanes (two per warp), one state word per lane; lanes 12-15 compute along on word 11's
// parameters and write nothing.  A lane keeps its row of the MDS matrix and its 14 round constants in registers, so the
// MDS product is 12 shuffles and 12 multiply-adds per lane.  The S-box is x^7 (4 multiplications), the inverse S-box
// x^(1/7) a fixed addition chain of 63 squarings and 9 multiplications.  A chain is one long dependent sequence (7 L
// rounds of about 100 field multiplications each), so the kernel is bound by the latency of that sequence, not by HBM:
// 12 n words are written in all (13 n by the hash, whose lanes 0..7 also write the absorbed words), each lane storing
// its own column's rows in order.  The hash is meant for many short messages: from K = 2^16 on, its grid fills the GPU.
#include "../../include/ministark_rescue.h"
#include "../../include/ministark_rescue_hash.h"
#include "../../include/ministark_rescue_merkle.h"
#include "ctx.cuh"
#include "rescue_params.cuh"

namespace ms {

constexpr int kW = MS_RESCUE_WIDTH, kRounds = MS_RESCUE_ROUNDS;
constexpr unsigned kLanes = 16;         // lanes per chain
constexpr unsigned kThreads = 128;      // 8 chains per block

static __constant__ u64 kRc[2 * kW * kRounds] = MS_RESCUE_RC;      // canonical words
static __constant__ u64 kMds[kW * kW] = MS_RESCUE_MDS;

// the exponent the chain of inv_sbox computes: e3 = 0b100100 = 36, e4 = e3 * 2^6 + e3, e5 = e4 * 2^12 + e4,
// e6 = e5 * 2^6 + e3, e7 = e6 * 2^31 + e6, then ((e7 * 2 + e6) * 4) + 7
constexpr u64 chain_exponent() {
    const u64 e3 = 36, e4 = (e3 << 6) + e3, e5 = (e4 << 12) + e4, e6 = (e5 << 6) + e3, e7 = (e6 << 31) + e6;
    return (((e7 << 1) + e6) << 2) + 7;
}
static_assert(chain_exponent() == MS_RESCUE_ALPHA_INV, "the inverse S-box chain must compute x^(1/7)");

template <int K>
__device__ __forceinline__ u64 exp_acc(u64 base, u64 tail) {     // base^(2^K) * tail
#pragma unroll
    for (int i = 0; i < K; i++) base = gl::sqr(base);
    return gl::mul(base, tail);
}

__device__ __forceinline__ u64 inv_sbox(u64 x) {
    const u64 t1 = gl::sqr(x), t2 = gl::sqr(t1);
    const u64 t3 = exp_acc<3>(t2, t2);
    const u64 t4 = exp_acc<6>(t3, t3);
    const u64 t5 = exp_acc<12>(t4, t4);
    const u64 t6 = exp_acc<6>(t5, t3);
    const u64 t7 = exp_acc<31>(t6, t6);
    const u64 a = gl::sqr(gl::sqr(gl::mul(gl::sqr(t7), t6)));
    return gl::mul(a, gl::mul(gl::mul(t1, t2), x));
}

// word `lane` of MDS v, v spread over the chain's 16 lanes one word each
__device__ __forceinline__ u64 mds_apply(const u64 (&row)[kW], u64 v) {
    u64 acc = 0;
#pragma unroll
    for (int j = 0; j < kW; j++) acc = gl::add(acc, gl::mul(row[j], __shfl_sync(~0u, v, j, kLanes)));
    return acc;
}

// the lane's MDS row and round constants (Montgomery), word w of the state
__device__ __forceinline__ void load_params(unsigned w, u64 (&row)[kW], u64 (&c1)[kRounds], u64 (&c2)[kRounds]) {
#pragma unroll
    for (int j = 0; j < kW; j++) row[j] = gl::to_mont(kMds[w * kW + j]);
#pragma unroll
    for (int r = 0; r < kRounds; r++) {
        c1[r] = gl::to_mont(kRc[2 * kW * r + w]);
        c2[r] = gl::to_mont(kRc[2 * kW * r + kW + w]);
    }
}

// one round on the chain's 16 lanes: S-box, MDS, the first constants, inverse S-box, MDS, the second constants
__device__ __forceinline__ u64 rescue_round(const u64 (&row)[kW], u64 c1, u64 c2, u64 s) {
    const u64 x3 = gl::mul(gl::sqr(s), s);
    s = gl::add(mds_apply(row, gl::mul(gl::sqr(x3), s)), c1);
    return gl::add(mds_apply(row, inv_sbox(s)), c2);
}

struct ChainArgs {
    u64 seed[4];        // Montgomery
    u64 tag_root;       // Montgomery w_K
    u64 K, L, n;
    u64 *out;
};

__global__ void __launch_bounds__(kThreads) rescue_chains_kernel(ChainArgs a) {
    const unsigned lane = threadIdx.x % kLanes;
    const u64 chain = (blockIdx.x * (u64)kThreads + threadIdx.x) / kLanes;
    const bool live = chain < a.K && lane < (unsigned)kW;       // every lane runs: the shuffles take the whole warp
    const unsigned w = lane < (unsigned)kW ? lane : kW - 1;
    u64 row[kW], c1[kRounds], c2[kRounds];
    load_params(w, row, c1, c2);
    u64 s = 0;
    if (lane < 4) s = lane == 0 ? a.seed[0] : lane == 1 ? a.seed[1] : lane == 2 ? a.seed[2] : a.seed[3];
    else if (lane == 4) s = gl::pow(a.tag_root, chain < a.K ? chain : 0);
    u64 *col = a.out + (u64)w * a.n + (chain < a.K ? chain : 0) * 8 * a.L;
    for (u64 j = 0; j < a.L; j++, col += 8) {
#pragma unroll
        for (int r = 0; r < kRounds; r++) {
            if (live) col[r] = s;
            s = rescue_round(row, c1[r], c2[r], s);
        }
        if (live) col[kRounds] = s;
    }
}

struct HashArgs {
    const u64 *messages;    // K x length canonical words
    u64 K, length, L, n;
    u64 *out;
};

// the sponge of one message per 16 lanes: before permutation j, lanes 0..7 take word `lane` of block j (a message word,
// the padding's 1, or 0 in the padding and the filler blocks j >= B), write it to column 12 and add it into the state
__global__ void __launch_bounds__(kThreads) rescue_hash_kernel(HashArgs a) {
    const unsigned lane = threadIdx.x % kLanes;
    const u64 msg = (blockIdx.x * (u64)kThreads + threadIdx.x) / kLanes;
    const bool live = msg < a.K && lane < (unsigned)kW;
    const unsigned w = lane < (unsigned)kW ? lane : kW - 1;
    u64 row[kW], c1[kRounds], c2[kRounds];
    load_params(w, row, c1, c2);
    const u64 k = msg < a.K ? msg : 0;
    const u64 *words = a.messages + k * a.length;
    u64 *col = a.out + (u64)w * a.n + k * 8 * a.L;
    u64 *mcol = a.out + (u64)kW * a.n + k * 8 * a.L;
    u64 s = 0;
    for (u64 j = 0; j < a.L; j++, col += 8, mcol += 8) {
        if (lane < 8) {
            const u64 p = 8 * j + lane;
            const u64 m = p < a.length ? gl::to_mont(words[p]) : p == a.length ? gl::ONE : 0;
            if (live) mcol[lane] = m;
            s = gl::add(s, m);
        }
#pragma unroll
        for (int r = 0; r < kRounds; r++) {
            if (live) col[r] = s;
            s = rescue_round(row, c1[r], c2[r], s);
        }
        if (live) col[kRounds] = s;
    }
}

// ------------------------------------------------------------------------------------------------- examples/merkle
// merge(node 2 v, node 2 v + 1): the two children are the 8 canonical words at nodes + 8 v, lanes 0..7 take one each,
// the capacity starts at zero; words 0..3 of the output end on lanes 0..3 (Montgomery)
__device__ __forceinline__ u64 merge_children(const u64 (&row)[kW], const u64 (&c1)[kRounds], const u64 (&c2)[kRounds],
                                              const u64 *nodes, u64 v, unsigned lane) {
    u64 s = lane < 8 ? gl::to_mont(nodes[8 * v + lane]) : 0;
#pragma unroll
    for (int r = 0; r < kRounds; r++) s = rescue_round(row, c1[r], c2[r], s);
    return s;
}

// one level of the tree: nodes [first, 2 first), one per 16 lanes
__global__ void __launch_bounds__(kThreads) merkle_level_kernel(u64 *nodes, u64 first) {
    const unsigned lane = threadIdx.x % kLanes;
    const u64 g = (blockIdx.x * (u64)kThreads + threadIdx.x) / kLanes;
    u64 row[kW], c1[kRounds], c2[kRounds];
    load_params(lane < (unsigned)kW ? lane : kW - 1, row, c1, c2);
    const u64 v = first + (g < first ? g : 0);
    const u64 s = merge_children(row, c1, c2, nodes, v, lane);
    if (g < first && lane < 4) nodes[4 * v + lane] = gl::from_mont(s);
}

constexpr unsigned kTopThreads = 512;                          // 32 nodes at once
constexpr unsigned kTopLevels = 6;                             // levels 0..5, of 1..32 nodes

// levels `levels` - 1 .. 0 of the tree in one block: one launch in place of six tiny ones
__global__ void __launch_bounds__(kTopThreads) merkle_top_kernel(u64 *nodes, unsigned levels) {
    const unsigned lane = threadIdx.x % kLanes, g = threadIdx.x / kLanes;
    u64 row[kW], c1[kRounds], c2[kRounds];
    load_params(lane < (unsigned)kW ? lane : kW - 1, row, c1, c2);
    for (int l = (int)levels - 1; l >= 0; l--) {
        const unsigned count = 1u << l;
        const u64 v = count + (g < count ? g : 0);
        const u64 s = merge_children(row, c1, c2, nodes, v, lane);
        if (g < count && lane < 4) nodes[4 * v + lane] = gl::from_mont(s);
        __syncthreads();                                       // level l is written before level l - 1 reads it
    }
}

__global__ void merkle_check_indices_kernel(const u64 *indices, u64 K, u64 bound, unsigned long long *first_bad) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < K; i += (u64)gridDim.x * blockDim.x)
        if (indices[i] >= bound) atomicMin(first_bad, (unsigned long long)i);
}

struct PathArgs {
    const u64 *nodes;       // the heap, canonical words
    const u64 *indices;
    u64 K, L, n;
    unsigned D;
    u64 *out;
};

// one path per 16 lanes: before permutation j, lanes 0..3 and 4..7 take the current node (words 0..3 of the previous
// output, or the leaf) and the sibling, in the order bit j of the index gives; lane 12 writes BIT, lane 13 IDX
__global__ void __launch_bounds__(kThreads) rescue_merkle_paths_kernel(PathArgs a) {
    const unsigned lane = threadIdx.x % kLanes;
    const u64 path = (blockIdx.x * (u64)kThreads + threadIdx.x) / kLanes;
    const bool in_range = path < a.K, live = in_range && lane < (unsigned)kW;
    const unsigned w = lane < (unsigned)kW ? lane : kW - 1;
    u64 row[kW], c1[kRounds], c2[kRounds];
    load_params(w, row, c1, c2);
    const u64 k = in_range ? path : 0;
    const u64 idx = a.indices[k];
    const u64 leaf = (1ull << a.D) + idx;
    u64 s = lane < 4 ? gl::to_mont(a.nodes[4 * leaf + lane]) : 0;
    u64 *col = a.out + (u64)w * a.n + k * 8 * a.L;
    u64 *bcol = a.out + (u64)kW * a.n + k * 8 * a.L, *icol = bcol + a.n;
    for (u64 j = 0; j < a.L; j++, col += 8, bcol += 8, icol += 8) {
        const bool bit = j < a.D && ((idx >> j) & 1);
        u64 sib = 0;
        if (j < a.D && lane < 8) sib = gl::to_mont(a.nodes[4 * ((leaf >> j) ^ 1) + (lane & 3)]);
        const u64 cur = __shfl_sync(~0u, s, lane & 3, kLanes);
        s = lane < 8 ? ((lane < 4) != bit ? cur : sib) : 0;
#pragma unroll
        for (int r = 0; r < kRounds; r++) {
            if (live) col[r] = s;
            s = rescue_round(row, c1[r], c2[r], s);
        }
        if (live) col[kRounds] = s;
        if (in_range && lane == kW) {
#pragma unroll
            for (int r = 0; r < 8; r++) bcol[r] = bit ? gl::ONE : 0;
        } else if (in_range && lane == kW + 1) {
            const u64 v = gl::to_mont(idx >> j);
#pragma unroll
            for (int r = 0; r < 8; r++) icol[r] = v;
        }
    }
}

static bool pow2(u64 v) { return v && !(v & (v - 1)); }
static unsigned log2u(u64 v) { return 63 - __builtin_clzll(v); }

}  // namespace ms

using namespace ms;

extern "C" int ms_rescue_chains(ms_ctx *c, const uint64_t *seed, uint64_t K, uint64_t L, void *out) {
    if (!c) return MS_ERR_INVALID;
    if (!seed || !out) return fail(c, MS_ERR_INVALID, "ms_rescue_chains: null argument");
    if (!pow2(K) || !pow2(L))
        return fail(c, MS_ERR_INVALID, "ms_rescue_chains: K = %llu and L = %llu must be powers of two",
                    (unsigned long long)K, (unsigned long long)L);
    if (log2u(K) + log2u(L) + 3 > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_chains: 8 K L rows (K = %llu, L = %llu) exceed 2^32",
                    (unsigned long long)K, (unsigned long long)L);
    for (int w = 0; w < 4; w++)
        if (seed[w] >= gl::P)
            return fail(c, MS_ERR_INVALID, "ms_rescue_chains: seed word %d (%llu) is not canonical", w, (unsigned long long)seed[w]);
    const u64 n = 8 * K * L;
    ChainArgs a;
    for (int w = 0; w < 4; w++) a.seed[w] = gl::to_mont(seed[w]);
    // ark-ff's root of unity of order 2^32 (7^((p - 1) / 2^32)), raised to 2^(32 - log2 K)
    constexpr u64 kTwoAdicRoot = 1753635133440165772ull;
    a.tag_root = gl::pow(gl::to_mont(kTwoAdicRoot), 1ull << (32 - log2u(K)));
    a.K = K;
    a.L = L;
    a.n = n;
    Staged O(c, out, (size_t)kW * n * 8, false, true);
    if (O.rc) return O.rc;
    a.out = O.as<u64>();
    const u64 blocks = (K * kLanes + kThreads - 1) / kThreads;
    rescue_chains_kernel<<<(unsigned)blocks, kThreads, 0, c->stream>>>(a);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    return O.finish();
}

extern "C" int ms_rescue_hash(ms_ctx *c, const uint64_t *messages, uint64_t K, uint64_t length, void *out) {
    if (!c) return MS_ERR_INVALID;
    if (!out || (!messages && length)) return fail(c, MS_ERR_INVALID, "ms_rescue_hash: null argument");
    if (!pow2(K)) return fail(c, MS_ERR_INVALID, "ms_rescue_hash: K = %llu is not a power of two", (unsigned long long)K);
    const u64 B = length / 8 + 1;                               // the padding always appends its 1
    const unsigned log_l = B == 1 ? 0 : log2u(B - 1) + 1;       // L = 2^log_l, the smallest power of two >= B
    if (log2u(K) + log_l + 3 > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_hash: 8 K L rows (K = %llu, length = %llu) exceed 2^32",
                    (unsigned long long)K, (unsigned long long)length);
    const u64 L = 1ull << log_l;
    HashArgs a;
    a.K = K;
    a.length = length;
    a.L = L;
    a.n = 8 * K * L;
    Staged O(c, out, (size_t)(kW + 1) * a.n * 8, false, true);
    if (O.rc) return O.rc;
    Staged M(c, messages, (size_t)K * length * 8, true, false);
    if (M.rc) return M.rc;
    a.out = O.as<u64>();
    a.messages = M.as<u64>();
    const u64 blocks = (K * kLanes + kThreads - 1) / kThreads;
    rescue_hash_kernel<<<(unsigned)blocks, kThreads, 0, c->stream>>>(a);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    const int rc = M.finish();
    const int rc_out = O.finish();
    return rc ? rc : rc_out;
}

extern "C" int ms_rescue_merkle_tree(ms_ctx *c, const uint64_t *leaves, uint32_t depth, void *nodes) {
    if (!c) return MS_ERR_INVALID;
    if (!leaves || !nodes) return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_tree: null argument");
    if (depth < 1 || depth > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_tree: depth %u is outside 1..32", (unsigned)depth);
    const u64 leaves_n = 1ull << depth;
    Staged N(c, nodes, (size_t)(2 * leaves_n) * 4 * 8, false, true);
    if (N.rc) return N.rc;
    u64 *heap = N.as<u64>();
    MS_CUDA(c, cudaMemsetAsync(heap, 0, 4 * 8, c->stream));
    MS_CUDA(c, cudaMemcpyAsync(heap + 4 * leaves_n, leaves, (size_t)leaves_n * 4 * 8, cudaMemcpyDefault, c->stream));
    for (unsigned l = depth; l-- > kTopLevels;) {
        const u64 blocks = ((1ull << l) * kLanes + kThreads - 1) / kThreads;
        merkle_level_kernel<<<(unsigned)blocks, kThreads, 0, c->stream>>>(heap, 1ull << l);
        c->launches++;
        MS_CHECK_LAUNCH(c);
    }
    merkle_top_kernel<<<1, kTopThreads, 0, c->stream>>>(heap, depth < kTopLevels ? depth : kTopLevels);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    return N.finish();
}

extern "C" int ms_rescue_merkle_paths(ms_ctx *c, const void *nodes, uint32_t depth, const uint64_t *indices, uint64_t K,
                                      void *out) {
    if (!c) return MS_ERR_INVALID;
    if (!nodes || !indices || !out) return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_paths: null argument");
    if (!pow2(K)) return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_paths: K = %llu is not a power of two", (unsigned long long)K);
    if (depth < 1 || depth > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_paths: depth %u is outside 1..32", (unsigned)depth);
    const unsigned log_l = depth == 1 ? 0 : log2u(depth - 1) + 1;     // L = 2^log_l, the smallest power of two >= D
    if (log2u(K) + log_l + 3 > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_paths: 8 K L rows (K = %llu, depth %u) exceed 2^32",
                    (unsigned long long)K, (unsigned)depth);
    Staged I(c, indices, (size_t)K * 8, true, false);
    if (I.rc) return I.rc;
    void *flag = nullptr;
    if (int rc = scratch_get(c, 3, 8, &flag)) return rc;
    MS_CUDA(c, cudaMemsetAsync(flag, 0xFF, 8, c->stream));
    const u64 check_blocks = (K + 255) / 256 < 1024 ? (K + 255) / 256 : 1024;
    merkle_check_indices_kernel<<<(unsigned)check_blocks, 256, 0, c->stream>>>(I.as<u64>(), K, 1ull << depth,
                                                                               (unsigned long long *)flag);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    u64 bad = 0, value = 0;
    MS_CUDA(c, cudaMemcpyAsync(&bad, flag, 8, cudaMemcpyDeviceToHost, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if (bad != ~0ull) {
        MS_CUDA(c, cudaMemcpy(&value, I.as<u64>() + bad, 8, cudaMemcpyDefault));
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_paths: index %llu of path %llu is not below 2^%u",
                    (unsigned long long)value, (unsigned long long)bad, (unsigned)depth);
    }
    const u64 L = 1ull << log_l;
    PathArgs a;
    a.K = K;
    a.L = L;
    a.n = 8 * K * L;
    a.D = depth;
    Staged N(c, nodes, (size_t)(2ull << depth) * 4 * 8, true, false);
    if (N.rc) return N.rc;
    Staged O(c, out, (size_t)(kW + 2) * a.n * 8, false, true);
    if (O.rc) return O.rc;
    a.nodes = N.as<u64>();
    a.indices = I.as<u64>();
    a.out = O.as<u64>();
    const u64 blocks = (K * kLanes + kThreads - 1) / kThreads;
    rescue_merkle_paths_kernel<<<(unsigned)blocks, kThreads, 0, c->stream>>>(a);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    const int rc_i = I.finish(), rc_n = N.finish(), rc_o = O.finish();
    return rc_i ? rc_i : rc_n ? rc_n : rc_o;
}
