// rescue.cu — the traces of examples/rescue and examples/merkle, side by side on the device: K independent chains of L
// Rescue-Prime permutations (include/ministark_rescue.h), K messages absorbed by the Rescue-Prime sponge
// (include/ministark_rescue_hash.h), the Rescue-Prime Merkle tree with K authentication paths through it
// (include/ministark_rescue_merkle.h), K ordered leaf writes into that tree (include/ministark_rescue_merkle_updates.h),
// K balance transfers between the accounts that are its leaves (include/ministark_rescue_rollup.h), and K Winternitz
// one-time signatures over the permutation (include/ministark_rescue_wots.h).
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
#include "../../include/ministark_rescue_merkle_updates.h"
#include "../../include/ministark_rescue_rollup.h"
#include "../../include/ministark_rescue_wots.h"
#include "ctx.cuh"
#include "rescue_params.cuh"

#include <cub/cub.cuh>

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

// ------------------------------------------------------------------------------- examples/merkle: ordered writes
// Level j of K writes: write k passes node v_k = (2^D + i_k) >> j, side b_k = bit j of i_k, parent v_k >> 1.  Sorting
// the writes stably by parent puts both children of a parent in one run, in write order.  Within a run, the sibling
// write k sees is the new value of the latest earlier entry on the other side, and (level 0) the leaf it replaces the
// new value of the latest earlier entry on its own side; without one, the heap's.  Marks hold 1-based positions: an
// inclusive max-scan of (run start, last side-0 entry, last side-1 entry) gives each, and an entry found before the
// run start belongs to another run.
struct UpdateMarks {
    u32 start, last[2];
};

struct UpdateMarksMax {
    __device__ __forceinline__ UpdateMarks operator()(const UpdateMarks &a, const UpdateMarks &b) const {
        return {a.start > b.start ? a.start : b.start, {a.last[0] > b.last[0] ? a.last[0] : b.last[0],
                                                        a.last[1] > b.last[1] ? a.last[1] : b.last[1]}};
    }
};

constexpr unsigned kUpdateThreads = 256;

// the indices below 2^D and the leaf words canonical (the first failing position of each, atomically), and the new
// leaves in Montgomery form into cur (the new paths' level-0 inputs)
__global__ void update_check_kernel(const u64 *indices, const u64 *leaves, u64 K, u64 bound, u64 *cur,
                                    unsigned long long *first_bad) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < 4 * K; i += (u64)gridDim.x * blockDim.x) {
        if (i < K && indices[i] >= bound) atomicMin(first_bad, (unsigned long long)i);
        const u64 w = leaves[i];
        if (w >= gl::P) atomicMin(first_bad + 1, (unsigned long long)i);
        cur[i] = gl::to_mont(w < gl::P ? w : 0);
    }
}

__global__ void update_keys_kernel(const u64 *indices, u64 K, unsigned shift, u32 *keys, u32 *vals) {
    const u64 k = blockIdx.x * (u64)kUpdateThreads + threadIdx.x;
    if (k >= K) return;
    keys[k] = (u32)(indices[k] >> shift);
    vals[k] = (u32)k;
}

__global__ void update_marks_kernel(const u32 *keys, const u32 *order, const u64 *indices, u64 K, unsigned j,
                                    UpdateMarks *marks) {
    const u64 t = blockIdx.x * (u64)kUpdateThreads + threadIdx.x;
    if (t >= K) return;
    const unsigned b = (indices[order[t]] >> j) & 1;
    UpdateMarks m;
    m.start = t == 0 || keys[t] != keys[t - 1] ? (u32)(t + 1) : 0;
    m.last[0] = b ? 0 : (u32)(t + 1);
    m.last[1] = b ? (u32)(t + 1) : 0;
    marks[t] = m;
}

struct ResolveArgs {
    const u64 *nodes;           // the original heap, canonical
    const u64 *indices;
    const u32 *order;           // sorted position -> write
    const UpdateMarks *scan;    // inclusive max-scan of the marks
    const u64 *cur_new;         // K x 4 Montgomery: each write's new value of its level-j node
    u64 *sib;                   // K x 4 Montgomery: the sibling each write sees
    u64 *cur_old;               // level 0 only: K x 4 Montgomery, the leaf each write replaces
    unsigned char *last;        // K flags of level j: cleared for every write a later one in the same node follows
    u64 K;
    unsigned D, j;
};

__global__ void update_resolve_kernel(ResolveArgs a) {
    const u64 t = blockIdx.x * (u64)kUpdateThreads + threadIdx.x;
    if (t >= a.K) return;
    const u32 k = a.order[t];
    const u64 v = ((1ull << a.D) + a.indices[k]) >> a.j;
    const unsigned b = v & 1;
    const u32 start = a.scan[t].start;
    const UpdateMarks before = t ? a.scan[t - 1] : UpdateMarks{0, {0, 0}};
    const u32 other = b ? before.last[0] : before.last[1], same = b ? before.last[1] : before.last[0];
    if (other >= start) {
        const u32 k2 = a.order[other - 1];
        for (int w = 0; w < 4; w++) a.sib[4 * (u64)k + w] = a.cur_new[4 * (u64)k2 + w];
    } else {
        for (int w = 0; w < 4; w++) a.sib[4 * (u64)k + w] = gl::to_mont(a.nodes[4 * (v ^ 1) + w]);
    }
    if (same >= start) a.last[a.order[same - 1]] = 0;
    if (a.j == 0) {
        if (same >= start) {
            const u32 k2 = a.order[same - 1];
            for (int w = 0; w < 4; w++) a.cur_old[4 * (u64)k + w] = a.cur_new[4 * (u64)k2 + w];
        } else {
            for (int w = 0; w < 4; w++) a.cur_old[4 * (u64)k + w] = gl::to_mont(a.nodes[4 * v + w]);
        }
    }
}

struct UpdateArgs {
    const u64 *indices;
    const u64 *cur_in[2];       // K x 4 Montgomery inputs of the old (0) and new (1) paths at this level
    u64 *cur_out[2];            // their outputs, words 0..3: the inputs of the next level
    const u64 *sib;             // K x 4 Montgomery siblings (nullptr on filler levels)
    u64 *roots;                 // (K + 1) x 4 canonical, written at level D - 1
    u64 K, L, n;
    unsigned D, j;
    u64 *out;
};

// one path per 16 lanes, the old (even group) and the new (odd group) path of one write side by side in a warp, path
// g = 2 k + side at rows 8 (L g + j) + r: lanes 0..3 and 4..7 take the path's current node and the sibling in the order
// bit j gives; lane 12 writes BIT, lane 13 IDX and lane 14 SIDE
__global__ void __launch_bounds__(kThreads) rescue_merkle_update_kernel(UpdateArgs a) {
    const unsigned lane = threadIdx.x % kLanes;
    const u64 g = (blockIdx.x * (u64)kThreads + threadIdx.x) / kLanes;
    const bool in_range = g < 2 * a.K, live = in_range && lane < (unsigned)kW;
    const unsigned w = lane < (unsigned)kW ? lane : kW - 1;
    u64 row[kW], c1[kRounds], c2[kRounds];
    load_params(w, row, c1, c2);
    const u64 k = in_range ? g >> 1 : 0;
    const unsigned side = g & 1;
    const u64 idx = a.indices[k];
    const bool bit = a.j < a.D && ((idx >> a.j) & 1);
    u64 s = 0;
    if (lane < 8) {
        const u64 cur = (side ? a.cur_in[1] : a.cur_in[0])[4 * k + (lane & 3)];
        const u64 sib = a.sib ? a.sib[4 * k + (lane & 3)] : 0;
        s = (lane < 4) != bit ? cur : sib;
    }
    const u64 at = 8 * (a.L * (2 * k + side) + a.j);
    u64 *col = a.out + (u64)w * a.n + at;
#pragma unroll
    for (int r = 0; r < kRounds; r++) {
        if (live) col[r] = s;
        s = rescue_round(row, c1[r], c2[r], s);
    }
    if (live) col[kRounds] = s;
    if (in_range && lane < 4) {
        (side ? a.cur_out[1] : a.cur_out[0])[4 * k + lane] = s;
        if (a.j + 1 == a.D && (side || k == 0)) a.roots[4 * (side ? k + 1 : 0) + lane] = gl::from_mont(s);
    }
    if (in_range && lane == kW) {
        u64 *bcol = a.out + (u64)kW * a.n + at;
#pragma unroll
        for (int r = 0; r < 8; r++) bcol[r] = bit ? gl::ONE : 0;
    } else if (in_range && lane == kW + 1) {
        u64 *icol = a.out + (u64)(kW + 1) * a.n + at;
        const u64 v = gl::to_mont(idx >> a.j);
#pragma unroll
        for (int r = 0; r < 8; r++) icol[r] = v;
    } else if (in_range && lane == kW + 2) {
        u64 *scol = a.out + (u64)(kW + 2) * a.n + at;
#pragma unroll
        for (int r = 0; r < 8; r++) scol[r] = side ? gl::ONE : 0;
    }
}

// the heap after the writes: node (2^D + i_k) >> j gets its last writer's new value, read from the new path (its input
// at level j < D, its output at level D - 1 for the root, which only write K - 1 sets)
__global__ void update_scatter_kernel(const u64 *indices, const unsigned char *last, const u64 *out, u64 K, u64 L,
                                      u64 n, unsigned D, u64 *nodes) {
    const u64 t = blockIdx.x * (u64)kUpdateThreads + threadIdx.x;
    if (t >= (D + 1) * K) return;
    const unsigned j = (unsigned)(t / K);
    const u64 k = t % K;
    if (j < D ? !last[t] : k != K - 1) return;
    const u64 idx = indices[k], v = ((1ull << D) + idx) >> j;
    const u64 row = j < D ? 8 * (L * (2 * k + 1) + j) : 8 * (L * (2 * k + 1) + D) - 1;
    const unsigned half = j < D && ((idx >> j) & 1) ? 4 : 0;
    for (int w = 0; w < 4; w++) nodes[4 * v + w] = gl::from_mont(out[(u64)(half + w) * n + row]);
}

// ------------------------------------------------------------------------------------ examples/rollup: transfers
// Transfer k is write 2 k (the sender step: delta = -amount, nonce + 1) then write 2 k + 1 (the receiver step: delta =
// +amount).  Sorting the 2 K writes stably by account puts each account's writes in one run, in write order; an
// inclusive scan of (delta, nonce increment) within the run then gives what the account's balance and nonce have
// gained after each of its writes.
struct RollupStep {
    u64 delta, ninc;
};

struct RollupStepAdd {
    __device__ __forceinline__ RollupStep operator()(const RollupStep &a, const RollupStep &b) const {
        return {gl::add(a.delta, b.delta), gl::add(a.ninc, b.ninc)};
    }
};

// the accounts below 2^D (the first failing 3 k + side) and the amounts below 2^32 (the first failing k), atomically;
// per write w: its account as the updates' index and as the sort key, w as the sort value, and its delta
__global__ void rollup_check_kernel(const u64 *transfers, u64 K, u64 bound, u64 *account, u32 *keys, u32 *vals,
                                    u64 *delta, unsigned long long *first_bad) {
    const u64 w = blockIdx.x * (u64)kUpdateThreads + threadIdx.x;
    if (w >= 2 * K) return;
    const u64 k = w >> 1, side = w & 1;
    const u64 acc = transfers[3 * k + side], amount = transfers[3 * k + 2];
    if (acc >= bound) atomicMin(first_bad, (unsigned long long)(3 * k + side));
    if (side == 0 && amount >> 32) atomicMin(first_bad + 1, (unsigned long long)k);
    const u64 a = acc < bound ? acc : 0, m = amount >> 32 ? 0 : amount;
    account[w] = a;
    keys[w] = (u32)a;
    vals[w] = (u32)w;
    delta[w] = side ? m : gl::sub(0, m);
}

__global__ void rollup_gather_kernel(const u32 *order, const u64 *delta, u64 n2, RollupStep *steps) {
    const u64 t = blockIdx.x * (u64)kUpdateThreads + threadIdx.x;
    if (t >= n2) return;
    const u32 w = order[t];
    steps[t] = {delta[w], (w & 1) ? 0ull : 1ull};
}

// write w's new leaf (balance + scanned delta, nonce + scanned increment, the owner words kept) and its new balance;
// the lowest write whose new balance is not below 2^32, atomically
__global__ void rollup_resolve_kernel(const u64 *nodes, const u32 *skeys, const u32 *order, const RollupStep *scan,
                                      u64 n2, unsigned D, u64 *leaves, u64 *balance, unsigned long long *first_bad) {
    const u64 t = blockIdx.x * (u64)kUpdateThreads + threadIdx.x;
    if (t >= n2) return;
    const u32 w = order[t];
    const u64 *old = nodes + 4 * ((1ull << D) + skeys[t]);
    const u64 bal = gl::add(old[0], scan[t].delta);
    leaves[4 * (u64)w] = bal;
    leaves[4 * (u64)w + 1] = gl::add(old[1], scan[t].ninc);
    leaves[4 * (u64)w + 2] = old[2];
    leaves[4 * (u64)w + 3] = old[3];
    balance[w] = bal;
    if (bal >> 32) atomicMin(first_bad, (unsigned long long)w);
}

// columns 15..22 of row i: on row 16 L w, write w's DELTA, NINC and balance limbs; M = 0; TBL = min(i, 255)
__global__ void rollup_fill_kernel(const u64 *delta, const u64 *balance, u64 n, unsigned log_16l, u64 *out) {
    const u64 i = blockIdx.x * (u64)kUpdateThreads + threadIdx.x;
    if (i >= n) return;
    u64 *col = out + (u64)(kW + 3) * n + i;
    u64 v[6] = {0, 0, 0, 0, 0, 0};
    if ((i & ((1ull << log_16l) - 1)) == 0) {
        const u64 w = i >> log_16l, b = balance[w];
        v[0] = gl::to_mont(delta[w]);
        v[1] = (w & 1) ? 0 : gl::ONE;
        for (int q = 0; q < 4; q++) v[2 + q] = gl::to_mont((b >> (8 * q)) & 255);
    }
#pragma unroll
    for (int c = 0; c < 6; c++) col[(u64)c * n] = v[c];
    col[6 * n] = 0;
    col[7 * n] = gl::to_mont(i < 255 ? i : 255);
}

// ------------------------------------------------------------------------- examples/wots: one-time signatures
// One chain (signature element, trace block) per 16 lanes, as above.  Chain step s of chain i under seed rho permutes
// (x || 0^4 || 1 + s, i, rho_0, rho_1), the chain secret (sigma || 0^4 || 16, i, rho), the fold (end || acc || 0, i, rho).
constexpr unsigned kWotsChains = 67, kWotsSteps = 15, kWotsBlock = 128;

// digit i of a four-word message: its nibbles for i < 64, then those of the checksum sum_(j<64) (15 - d_j)
__device__ __forceinline__ unsigned wots_digit(const u64 *m, unsigned i) {
    if (i < 64) return (unsigned)(m[i >> 4] >> (4 * (i & 15))) & 15;
    unsigned c = 0;
    for (unsigned j = 0; j < 64; j++) c += 15 - ((unsigned)(m[j >> 4] >> (4 * (j & 15))) & 15);
    return (c >> (4 * (i - 64))) & 15;
}

// a permutation input on the group's lanes (all Montgomery): x on lanes 0..3, tail on 4..7, then the tweak, i, rho_0
// and rho_1; lanes 12..15 take 0
__device__ __forceinline__ u64 wots_input(unsigned lane, u64 x, u64 tail, u64 tweak, u64 i, u64 r0, u64 r1) {
    return lane < 4 ? x : lane < 8 ? tail : lane == 8 ? tweak : lane == 9 ? i : lane == 10 ? r0 : lane == 11 ? r1 : 0;
}

// the permutation, its eight states written to col[0..7] when `live`
__device__ __forceinline__ u64 wots_permute(const u64 (&row)[kW], const u64 (&c1)[kRounds], const u64 (&c2)[kRounds],
                                            u64 s, u64 *col, bool live) {
#pragma unroll
    for (int r = 0; r < kRounds; r++) {
        if (live) col[r] = s;
        s = rescue_round(row, c1[r], c2[r], s);
    }
    if (live) col[kRounds] = s;
    return s;
}

__global__ void wots_check_kernel(const u64 *v, u64 count, unsigned long long *first_bad) {
    for (u64 t = blockIdx.x * (u64)blockDim.x + threadIdx.x; t < count; t += (u64)gridDim.x * blockDim.x)
        if (v[t] >= gl::P) atomicMin(first_bad, (unsigned long long)t);
}

struct WotsSignArgs {
    const u64 *secrets, *seeds, *messages;
    u64 K;
    u64 *signatures;            // K x 67 x 4 canonical
    u64 *ends;                  // 67 K x 4 Montgomery
};

// chain c = 67 k + i: sk_i, then all 15 steps; the value before step d_i is signature element i
__global__ void __launch_bounds__(kThreads) wots_sign_kernel(WotsSignArgs a) {
    const unsigned lane = threadIdx.x % kLanes;
    const u64 g = (blockIdx.x * (u64)kThreads + threadIdx.x) / kLanes;
    const bool in_range = g < kWotsChains * a.K, out = in_range && lane < 4;
    u64 row[kW], c1[kRounds], c2[kRounds];
    load_params(lane < (unsigned)kW ? lane : kW - 1, row, c1, c2);
    const u64 c = in_range ? g : 0, k = c / kWotsChains;
    const unsigned i = (unsigned)(c % kWotsChains), d = wots_digit(a.messages + 4 * k, i);
    const u64 ti = gl::to_mont(i), r0 = gl::to_mont(a.seeds[2 * k]), r1 = gl::to_mont(a.seeds[2 * k + 1]);
    u64 x = lane < 4 ? gl::to_mont(a.secrets[4 * k + lane]) : 0;
    x = wots_permute(row, c1, c2, wots_input(lane, x, 0, gl::to_mont(16), ti, r0, r1), nullptr, false);
    for (unsigned s = 0; s < kWotsSteps; s++) {
        if (s == d && out) a.signatures[4 * c + lane] = gl::from_mont(x);
        x = wots_permute(row, c1, c2, wots_input(lane, x, 0, gl::to_mont(1 + s), ti, r0, r1), nullptr, false);
    }
    if (d == kWotsSteps && out) a.signatures[4 * c + lane] = gl::from_mont(x);
    if (out) a.ends[4 * c + lane] = x;
}

struct WotsFoldArgs {
    const u64 *ends;            // 67 K x 4 Montgomery: the chain ends
    const u64 *seeds;           // rho of key k at seeds[seed_stride k]
    u64 seed_stride, K;
    u64 *accs;                  // 67 K x 4 Montgomery: each fold's acc input (or nullptr)
    u64 *public_keys;           // K x 6: (rho_0, rho_1, root) per key (or nullptr)
    const u64 *expect;          // K x 6: the root each key must reach (or nullptr)
    unsigned long long *first_bad;
};

// one key's 67 folds per 16 lanes, in order: acc <- words 0..3 of permute(end_i || acc || 0, i, rho), from acc = 0
__global__ void __launch_bounds__(kThreads) wots_fold_kernel(WotsFoldArgs a) {
    const unsigned lane = threadIdx.x % kLanes;
    const u64 g0 = (blockIdx.x * (u64)kThreads + threadIdx.x) / kLanes;
    const bool in_range = g0 < a.K, out = in_range && lane < 4;
    u64 row[kW], c1[kRounds], c2[kRounds];
    load_params(lane < (unsigned)kW ? lane : kW - 1, row, c1, c2);
    const u64 g = in_range ? g0 : 0;
    const u64 r0 = gl::to_mont(a.seeds[a.seed_stride * g]), r1 = gl::to_mont(a.seeds[a.seed_stride * g + 1]);
    u64 acc = 0;
    for (unsigned i = 0; i < kWotsChains; i++) {
        const u64 b = kWotsChains * g + i;
        if (out && a.accs) a.accs[4 * b + lane] = acc;
        const u64 x = lane < 4 ? a.ends[4 * b + lane] : 0;
        const u64 tail = __shfl_sync(~0u, acc, lane & 3, kLanes);
        acc = wots_permute(row, c1, c2, wots_input(lane, x, tail, 0, gl::to_mont(i), r0, r1), nullptr, false);
    }
    const u64 root = gl::from_mont(acc);
    if (out && a.public_keys) {
        a.public_keys[6 * g + 2 + lane] = root;
        if (lane < 2) a.public_keys[6 * g + lane] = a.seeds[a.seed_stride * g + lane];
    }
    if (out && a.expect && a.expect[6 * g + 2 + lane] != root) atomicMin(a.first_bad, (unsigned long long)g);
}

struct WotsTraceArgs {
    const u64 *public_keys, *messages, *signatures;
    u64 K, B, n;
    const u64 *accs;            // per block, Montgomery (kWrite)
    u64 *ends;                  // per block, Montgomery (!kWrite)
    u64 *out;
};

// block b per 16 lanes: the 15 chain slots from the signature element (0 for padding), each step applied from slot
// d on.  kWrite = false: the chain end into ends.  kWrite = true: the block's rows, the fold on accs[b] included (on 0^4
// for padding, which has LAST = 1 and so follows a block with LAST = 1); lane 12 writes ACT, lane 13 CNT, lane 14 LAST
template <bool kWrite>
__global__ void __launch_bounds__(kThreads) wots_trace_kernel(WotsTraceArgs a) {
    const unsigned lane = threadIdx.x % kLanes;
    const u64 g = (blockIdx.x * (u64)kThreads + threadIdx.x) / kLanes;
    const bool in_range = g < a.B, live = kWrite && in_range && lane < (unsigned)kW;
    const unsigned w = lane < (unsigned)kW ? lane : kW - 1;
    u64 row[kW], c1[kRounds], c2[kRounds];
    load_params(w, row, c1, c2);
    const u64 b = in_range ? g : 0, k = b / kWotsChains;
    const bool real = k < a.K;
    const unsigned i = real ? (unsigned)(b % kWotsChains) : 0, d = real ? wots_digit(a.messages + 4 * k, i) : 0;
    const u64 last = !real || i == kWotsChains - 1 ? gl::ONE : 0;
    const u64 ti = gl::to_mont(i), r0 = real ? gl::to_mont(a.public_keys[6 * k]) : 0,
              r1 = real ? gl::to_mont(a.public_keys[6 * k + 1]) : 0;
    u64 x = real && lane < 4 ? gl::to_mont(a.signatures[4 * b + lane]) : 0;
    u64 *col = kWrite ? a.out + (u64)w * a.n + kWotsBlock * b : nullptr;
    u64 *aux = kWrite ? a.out + (u64)(lane < kW + 3 ? lane : kW) * a.n + kWotsBlock * b : nullptr;
    const bool aux_live = kWrite && in_range && lane >= (unsigned)kW && lane < (unsigned)kW + 3;
    for (unsigned s = 0; s < kWotsSteps; s++, col += 8, aux += 8) {
        const u64 y = wots_permute(row, c1, c2, wots_input(lane, x, 0, gl::to_mont(1 + s), ti, r0, r1), col, live);
        if (s >= d) x = y;
        if (aux_live) {
            const u64 v = lane == (unsigned)kW ? (s >= d ? gl::ONE : 0)
                          : lane == (unsigned)kW + 1 ? gl::to_mont(s < d ? d - s : 0)
                          : last;
#pragma unroll
            for (int r = 0; r < 8; r++) aux[r] = v;
        }
    }
    if (!kWrite) {
        if (in_range && lane < 4) a.ends[4 * b + lane] = x;
        return;
    }
    const u64 tail = real && lane >= 4 && lane < 8 ? a.accs[4 * b + lane - 4] : 0;
    wots_permute(row, c1, c2, wots_input(lane, x, tail, 0, ti, r0, r1), col, live);
    if (aux_live) {
        const u64 v = lane == (unsigned)kW + 2 ? last : 0;
#pragma unroll
        for (int r = 0; r < 8; r++) aux[r] = v;
    }
}

static bool pow2(u64 v) { return v && !(v & (v - 1)); }
static unsigned log2u(u64 v) { return 63 - __builtin_clzll(v); }
static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

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

extern "C" int ms_rescue_merkle_updates(ms_ctx *c, void *nodes, uint32_t depth, const uint64_t *indices,
                                        const uint64_t *new_leaves, uint64_t K, void *out, uint64_t *roots) {
    if (!c) return MS_ERR_INVALID;
    if (!nodes || !indices || !new_leaves || !out || !roots)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: null argument");
    if (!pow2(K)) return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: K = %llu is not a power of two", (unsigned long long)K);
    if (depth < 1 || depth > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: depth %u is outside 1..32", (unsigned)depth);
    const unsigned log_l = depth == 1 ? 0 : log2u(depth - 1) + 1;     // L = 2^log_l, the smallest power of two >= D
    if (log2u(K) + log_l + 4 > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: 16 K L rows (K = %llu, depth %u) exceed 2^32",
                    (unsigned long long)K, (unsigned)depth);
    const u64 L = 1ull << log_l, n = 16 * K * L;
    const size_t kw = (size_t)K * 4 * 8;                               // one K x 4 word buffer
    // scratch arena 3: the check flags, the sort's keys and values (double-buffered), the marks and their scan, the
    // siblings, the old and new paths' inputs (double-buffered), the last-writer flags of levels 0..D-1, cub's storage
    size_t sort_b = 0, scan_b = 0;
    MS_CUDA(c, cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const u32 *)nullptr, (u32 *)nullptr, (const u32 *)nullptr,
                                               (u32 *)nullptr, (int)K, 0, 32, c->stream));
    MS_CUDA(c, cub::DeviceScan::InclusiveScan(nullptr, scan_b, (const UpdateMarks *)nullptr, (UpdateMarks *)nullptr,
                                              UpdateMarksMax(), (int)K, c->stream));
    const size_t u32s = align256((size_t)K * 4), marks_b = align256((size_t)K * sizeof(UpdateMarks));
    const size_t off_keys = 256, off_marks = off_keys + 4 * u32s, off_sib = off_marks + 2 * marks_b,
                 off_cur = off_sib + align256(kw), off_last = off_cur + 4 * align256(kw),
                 off_temp = off_last + align256((size_t)K * depth), total = off_temp + (sort_b > scan_b ? sort_b : scan_b);
    void *scr = nullptr;
    if (int rc = scratch_get(c, 3, total, &scr)) return rc;
    char *sb = (char *)scr;
    unsigned long long *flag = (unsigned long long *)sb;
    u32 *keys[2] = {(u32 *)(sb + off_keys), (u32 *)(sb + off_keys + u32s)};
    u32 *vals[2] = {(u32 *)(sb + off_keys + 2 * u32s), (u32 *)(sb + off_keys + 3 * u32s)};
    UpdateMarks *marks = (UpdateMarks *)(sb + off_marks), *scan = (UpdateMarks *)(sb + off_marks + marks_b);
    u64 *sib = (u64 *)(sb + off_sib);
    u64 *cur_old[2] = {(u64 *)(sb + off_cur), (u64 *)(sb + off_cur + align256(kw))};
    u64 *cur_new[2] = {(u64 *)(sb + off_cur + 2 * align256(kw)), (u64 *)(sb + off_cur + 3 * align256(kw))};
    unsigned char *last = (unsigned char *)(sb + off_last);
    void *temp = sb + off_temp;

    Staged I(c, indices, (size_t)K * 8, true, false);
    if (I.rc) return I.rc;
    Staged V(c, new_leaves, kw, true, false);
    if (V.rc) return V.rc;
    const u64 *idx = I.as<u64>();
    MS_CUDA(c, cudaMemsetAsync(flag, 0xFF, 16, c->stream));
    const u64 check_blocks = (4 * K + 255) / 256 < 1024 ? (4 * K + 255) / 256 : 1024;
    update_check_kernel<<<(unsigned)check_blocks, 256, 0, c->stream>>>(idx, V.as<u64>(), K, 1ull << depth, cur_new[0], flag);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    u64 bad[2] = {0, 0}, value = 0;
    MS_CUDA(c, cudaMemcpyAsync(bad, flag, 16, cudaMemcpyDeviceToHost, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if (bad[0] != ~0ull) {
        MS_CUDA(c, cudaMemcpy(&value, idx + bad[0], 8, cudaMemcpyDefault));
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: index %llu of write %llu is not below 2^%u",
                    (unsigned long long)value, (unsigned long long)bad[0], (unsigned)depth);
    }
    if (bad[1] != ~0ull) {
        MS_CUDA(c, cudaMemcpy(&value, V.as<u64>() + bad[1], 8, cudaMemcpyDefault));
        return fail(c, MS_ERR_INVALID, "ms_rescue_merkle_updates: word %llu of new leaf %llu (%llu) is not canonical",
                    (unsigned long long)(bad[1] % 4), (unsigned long long)(bad[1] / 4), (unsigned long long)value);
    }

    Staged N(c, nodes, (size_t)(2ull << depth) * 4 * 8, true, true);
    if (N.rc) return N.rc;
    Staged O(c, out, (size_t)(kW + 3) * n * 8, false, true);
    if (O.rc) return O.rc;
    Staged R(c, roots, (size_t)(K + 1) * 4 * 8, false, true);
    if (R.rc) return R.rc;
    u64 *heap = N.as<u64>();
    MS_CUDA(c, cudaMemsetAsync(last, 1, (size_t)K * depth, c->stream));
    const unsigned kblocks = (unsigned)((K + kUpdateThreads - 1) / kUpdateThreads);
    const unsigned pblocks = (unsigned)((2 * K * kLanes + kThreads - 1) / kThreads);
    UpdateArgs u;
    u.indices = idx;
    u.roots = R.as<u64>();
    u.K = K;
    u.L = L;
    u.n = n;
    u.D = depth;
    u.out = O.as<u64>();
    int in = 0;                                                        // cur_*[in] holds this level's inputs
    for (unsigned j = 0; j < L; j++) {
        if (j < depth) {
            const int bits = (int)depth - 1 - (int)j;                   // the parent's index below the top level
            update_keys_kernel<<<kblocks, kUpdateThreads, 0, c->stream>>>(idx, K, j + 1, keys[0], vals[0]);
            c->launches++;
            MS_CHECK_LAUNCH(c);
            const u32 *skeys = keys[0], *order = vals[0];
            if (bits > 0) {
                MS_CUDA(c, cub::DeviceRadixSort::SortPairs(temp, sort_b, keys[0], keys[1], vals[0], vals[1], (int)K, 0,
                                                           bits, c->stream));
                skeys = keys[1];
                order = vals[1];
            }
            update_marks_kernel<<<kblocks, kUpdateThreads, 0, c->stream>>>(skeys, order, idx, K, j, marks);
            c->launches++;
            MS_CHECK_LAUNCH(c);
            MS_CUDA(c, cub::DeviceScan::InclusiveScan(temp, scan_b, marks, scan, UpdateMarksMax(), (int)K, c->stream));
            ResolveArgs r;
            r.nodes = heap;
            r.indices = idx;
            r.order = order;
            r.scan = scan;
            r.cur_new = cur_new[in];
            r.sib = sib;
            r.cur_old = cur_old[in];
            r.last = last + (size_t)j * K;
            r.K = K;
            r.D = depth;
            r.j = j;
            update_resolve_kernel<<<kblocks, kUpdateThreads, 0, c->stream>>>(r);
            c->launches++;
            MS_CHECK_LAUNCH(c);
        }
        u.cur_in[0] = cur_old[in];
        u.cur_in[1] = cur_new[in];
        u.cur_out[0] = cur_old[in ^ 1];
        u.cur_out[1] = cur_new[in ^ 1];
        u.sib = j < depth ? sib : nullptr;
        u.j = j;
        rescue_merkle_update_kernel<<<pblocks, kThreads, 0, c->stream>>>(u);
        c->launches++;
        MS_CHECK_LAUNCH(c);
        in ^= 1;
    }
    const u64 sblocks = ((u64)(depth + 1) * K + kUpdateThreads - 1) / kUpdateThreads;
    update_scatter_kernel<<<(unsigned)sblocks, kUpdateThreads, 0, c->stream>>>(idx, last, O.as<u64>(), K, L, n, depth, heap);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    const int rc_i = I.finish(), rc_v = V.finish(), rc_n = N.finish(), rc_o = O.finish(), rc_r = R.finish();
    return rc_i ? rc_i : rc_v ? rc_v : rc_n ? rc_n : rc_o ? rc_o : rc_r;
}

extern "C" int ms_rescue_rollup(ms_ctx *c, void *nodes, uint32_t depth, const uint64_t *transfers, uint64_t K,
                                void *out, uint64_t *roots) {
    if (!c) return MS_ERR_INVALID;
    if (!nodes || !transfers || !out || !roots) return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: null argument");
    if (!pow2(K)) return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: K = %llu is not a power of two", (unsigned long long)K);
    if (depth < 1 || depth > 32)
        return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: depth %u is outside 1..32", (unsigned)depth);
    const unsigned log_l = depth == 1 ? 0 : log2u(depth - 1) + 1;     // L = 2^log_l, the smallest power of two >= D
    const unsigned log_n = log2u(K) + log_l + 5;
    if (log_n > 32 || log_n < 8)
        return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: 32 K L rows (K = %llu, depth %u) are not in 2^8..2^32",
                    (unsigned long long)K, (unsigned)depth);
    const u64 n = 1ull << log_n, n2 = 2 * K;
    // scratch arena 2 (ms_rescue_merkle_updates takes arena 3): the check flags, the sort's keys and values
    // (double-buffered), the accounts, the deltas, the steps and their scan, the new leaves and balances, the 2 K + 1
    // roots of the writes, cub's storage
    size_t sort_b = 0, scan_b = 0;
    MS_CUDA(c, cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const u32 *)nullptr, (u32 *)nullptr, (const u32 *)nullptr,
                                               (u32 *)nullptr, (int)n2, 0, (int)depth, c->stream));
    MS_CUDA(c, cub::DeviceScan::InclusiveScanByKey(nullptr, scan_b, (const u32 *)nullptr, (const RollupStep *)nullptr,
                                                   (RollupStep *)nullptr, RollupStepAdd(), (int)n2, cuda::std::equal_to<>(),
                                                   c->stream));
    const size_t u32s = align256(n2 * 4), words = align256(n2 * 8), steps_b = align256(n2 * sizeof(RollupStep));
    const size_t off_keys = 256, off_acc = off_keys + 4 * u32s, off_delta = off_acc + words,
                 off_steps = off_delta + words, off_leaves = off_steps + 2 * steps_b, off_bal = off_leaves + 4 * words,
                 off_roots = off_bal + words, off_temp = off_roots + align256((n2 + 1) * 32),
                 total = off_temp + (sort_b > scan_b ? sort_b : scan_b);
    void *scr = nullptr;
    if (int rc = scratch_get(c, 2, total, &scr)) return rc;
    char *sb = (char *)scr;
    unsigned long long *flag = (unsigned long long *)sb;
    u32 *keys[2] = {(u32 *)(sb + off_keys), (u32 *)(sb + off_keys + u32s)};
    u32 *vals[2] = {(u32 *)(sb + off_keys + 2 * u32s), (u32 *)(sb + off_keys + 3 * u32s)};
    u64 *account = (u64 *)(sb + off_acc), *delta = (u64 *)(sb + off_delta);
    RollupStep *steps = (RollupStep *)(sb + off_steps), *scan = (RollupStep *)(sb + off_steps + steps_b);
    u64 *leaves = (u64 *)(sb + off_leaves), *balance = (u64 *)(sb + off_bal), *wroots = (u64 *)(sb + off_roots);
    void *temp = sb + off_temp;

    Staged T(c, transfers, (size_t)K * 3 * 8, true, false);
    if (T.rc) return T.rc;
    const unsigned blocks = (unsigned)((n2 + kUpdateThreads - 1) / kUpdateThreads);
    MS_CUDA(c, cudaMemsetAsync(flag, 0xFF, 24, c->stream));
    rollup_check_kernel<<<blocks, kUpdateThreads, 0, c->stream>>>(T.as<u64>(), K, 1ull << depth, account, keys[0],
                                                                    vals[0], delta, flag);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    u64 bad[3] = {0, 0, 0}, value = 0;
    MS_CUDA(c, cudaMemcpyAsync(bad, flag, 16, cudaMemcpyDeviceToHost, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if (bad[0] != ~0ull) {
        MS_CUDA(c, cudaMemcpy(&value, T.as<u64>() + bad[0], 8, cudaMemcpyDefault));
        return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: %s %llu of transfer %llu is not below 2^%u",
                    bad[0] % 3 ? "receiver" : "sender", (unsigned long long)value, (unsigned long long)(bad[0] / 3),
                    (unsigned)depth);
    }
    if (bad[1] != ~0ull) {
        MS_CUDA(c, cudaMemcpy(&value, T.as<u64>() + 3 * bad[1] + 2, 8, cudaMemcpyDefault));
        return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: amount %llu of transfer %llu is not below 2^32",
                    (unsigned long long)value, (unsigned long long)bad[1]);
    }

    Staged N(c, nodes, (size_t)(2ull << depth) * 4 * 8, true, true);
    if (N.rc) return N.rc;
    const u64 *heap = N.as<u64>();
    MS_CUDA(c, cub::DeviceRadixSort::SortPairs(temp, sort_b, keys[0], keys[1], vals[0], vals[1], (int)n2, 0, (int)depth,
                                               c->stream));
    rollup_gather_kernel<<<blocks, kUpdateThreads, 0, c->stream>>>(vals[1], delta, n2, steps);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    MS_CUDA(c, cub::DeviceScan::InclusiveScanByKey(temp, scan_b, keys[1], steps, scan, RollupStepAdd(), (int)n2,
                                                   cuda::std::equal_to<>(), c->stream));
    rollup_resolve_kernel<<<blocks, kUpdateThreads, 0, c->stream>>>(heap, keys[1], vals[1], scan, n2, depth, leaves,
                                                                      balance, flag + 2);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    MS_CUDA(c, cudaMemcpyAsync(bad + 2, flag + 2, 8, cudaMemcpyDeviceToHost, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if (bad[2] != ~0ull) {
        u64 acc = 0;
        MS_CUDA(c, cudaMemcpy(&acc, account + bad[2], 8, cudaMemcpyDeviceToHost));
        MS_CUDA(c, cudaMemcpy(&value, balance + bad[2], 8, cudaMemcpyDeviceToHost));
        return fail(c, MS_ERR_INVALID, "ms_rescue_rollup: the %s step of transfer %llu leaves account %llu with balance "
                    "%llu, not below 2^32", bad[2] & 1 ? "receiver" : "sender", (unsigned long long)(bad[2] / 2),
                    (unsigned long long)acc, (unsigned long long)value);
    }

    Staged O(c, out, (size_t)(kW + 11) * n * 8, false, true);
    if (O.rc) return O.rc;
    Staged R(c, roots, (size_t)(K + 1) * 4 * 8, false, true);
    if (R.rc) return R.rc;
    // columns 0..14 of the (23, n) matrix are a (15, n) matrix: the updates trace of the 2 K writes
    if (int rc = ms_rescue_merkle_updates(c, N.as<u64>(), depth, (const uint64_t *)account,
                                          (const uint64_t *)leaves, n2, O.as<u64>(), (uint64_t *)wroots))
        return rc;
    MS_CUDA(c, cudaMemcpy2DAsync(R.as<u64>(), 32, wroots, 64, 32, K + 1, cudaMemcpyDeviceToDevice, c->stream));
    const u64 fblocks = (n + kUpdateThreads - 1) / kUpdateThreads;
    rollup_fill_kernel<<<(unsigned)fblocks, kUpdateThreads, 0, c->stream>>>(delta, balance, n, log_l + 4, O.as<u64>());
    c->launches++;
    MS_CHECK_LAUNCH(c);
    const int rc_t = T.finish(), rc_n = N.finish(), rc_o = O.finish(), rc_r = R.finish();
    return rc_t ? rc_t : rc_n ? rc_n : rc_o ? rc_o : rc_r;
}

// the lowest index of each of `count` arrays whose word is not canonical, into flag[0..count), ~0 where none
static int wots_check_words(ms_ctx *c, const u64 *const *arrays, const u64 *sizes, int count, unsigned long long *flag,
                            u64 *bad) {
    MS_CUDA(c, cudaMemsetAsync(flag, 0xFF, 8 * count, c->stream));
    for (int q = 0; q < count; q++) {
        const u64 blocks = (sizes[q] + 255) / 256 < 1024 ? (sizes[q] + 255) / 256 : 1024;
        wots_check_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(arrays[q], sizes[q], flag + q);
        c->launches++;
        MS_CHECK_LAUNCH(c);
    }
    MS_CUDA(c, cudaMemcpyAsync(bad, flag, 8 * count, cudaMemcpyDeviceToHost, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    return MS_OK;
}

static int wots_fold(ms_ctx *c, const WotsFoldArgs &a) {
    const u64 blocks = (a.K * kLanes + kThreads - 1) / kThreads;
    wots_fold_kernel<<<(unsigned)blocks, kThreads, 0, c->stream>>>(a);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    return MS_OK;
}

extern "C" int ms_rescue_wots_sign(ms_ctx *c, const uint64_t *secrets, const uint64_t *seeds, const uint64_t *messages,
                                   uint64_t K, void *signatures, void *public_keys) {
    if (!c) return MS_ERR_INVALID;
    if (!secrets || !seeds || !messages || !signatures || !public_keys)
        return fail(c, MS_ERR_INVALID, "ms_rescue_wots_sign: null argument");
    if (K < 1 || K > MS_WOTS_MAX_KEYS)
        return fail(c, MS_ERR_INVALID, "ms_rescue_wots_sign: K = %llu is outside 1..%u", (unsigned long long)K,
                    MS_WOTS_MAX_KEYS);
    const u64 chains = kWotsChains * K;
    // scratch arena 3: the check flags, then the chain ends
    void *scr = nullptr;
    if (int rc = scratch_get(c, 3, 256 + align256(chains * 32), &scr)) return rc;
    unsigned long long *flag = (unsigned long long *)scr;
    u64 *ends = (u64 *)((char *)scr + 256);
    Staged S(c, secrets, (size_t)K * 32, true, false);
    if (S.rc) return S.rc;
    Staged D(c, seeds, (size_t)K * 16, true, false);
    if (D.rc) return D.rc;
    Staged M(c, messages, (size_t)K * 32, true, false);
    if (M.rc) return M.rc;
    const u64 *arrays[3] = {S.as<u64>(), D.as<u64>(), M.as<u64>()}, sizes[3] = {4 * K, 2 * K, 4 * K};
    const char *names[3] = {"secret", "seed", "message"};
    const unsigned widths[3] = {4, 2, 4};
    u64 bad[3], value = 0;
    if (int rc = wots_check_words(c, arrays, sizes, 3, flag, bad)) return rc;
    for (int q = 0; q < 3; q++)
        if (bad[q] != ~0ull) {
            MS_CUDA(c, cudaMemcpy(&value, arrays[q] + bad[q], 8, cudaMemcpyDefault));
            return fail(c, MS_ERR_INVALID, "ms_rescue_wots_sign: word %llu of %s %llu (%llu) is not canonical",
                        (unsigned long long)(bad[q] % widths[q]), names[q], (unsigned long long)(bad[q] / widths[q]),
                        (unsigned long long)value);
        }
    Staged G(c, signatures, (size_t)chains * 32, false, true);
    if (G.rc) return G.rc;
    Staged Pk(c, public_keys, (size_t)K * 48, false, true);
    if (Pk.rc) return Pk.rc;
    WotsSignArgs s{S.as<u64>(), D.as<u64>(), M.as<u64>(), K, G.as<u64>(), ends};
    wots_sign_kernel<<<(unsigned)((chains * kLanes + kThreads - 1) / kThreads), kThreads, 0, c->stream>>>(s);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    if (int rc = wots_fold(c, {ends, D.as<u64>(), 2, K, nullptr, Pk.as<u64>(), nullptr, nullptr}))
        return rc;
    const int rc_s = S.finish(), rc_d = D.finish(), rc_m = M.finish(), rc_g = G.finish(), rc_p = Pk.finish();
    return rc_s ? rc_s : rc_d ? rc_d : rc_m ? rc_m : rc_g ? rc_g : rc_p;
}

extern "C" int ms_rescue_wots_trace(ms_ctx *c, const uint64_t *public_keys, const uint64_t *messages,
                                    const uint64_t *signatures, uint64_t K, void *out) {
    if (!c) return MS_ERR_INVALID;
    if (!public_keys || !messages || !signatures || !out)
        return fail(c, MS_ERR_INVALID, "ms_rescue_wots_trace: null argument");
    if (K < 1 || K > MS_WOTS_MAX_KEYS)
        return fail(c, MS_ERR_INVALID, "ms_rescue_wots_trace: K = %llu is outside 1..%u", (unsigned long long)K,
                    MS_WOTS_MAX_KEYS);
    const u64 chains = kWotsChains * K, B = 1ull << (log2u(chains - 1) + 1), n = kWotsBlock * B;
    // scratch arena 3: the check flags, the signatures' chain ends, their folds' acc inputs (padding blocks need
    // neither: each is the same block, its fold on 0^4)
    void *scr = nullptr;
    if (int rc = scratch_get(c, 3, 256 + 2 * align256(chains * 32), &scr)) return rc;
    unsigned long long *flag = (unsigned long long *)scr;
    u64 *ends = (u64 *)((char *)scr + 256), *accs = (u64 *)((char *)scr + 256 + align256(chains * 32));
    Staged Pk(c, public_keys, (size_t)K * 48, true, false);
    if (Pk.rc) return Pk.rc;
    Staged M(c, messages, (size_t)K * 32, true, false);
    if (M.rc) return M.rc;
    Staged S(c, signatures, (size_t)chains * 32, true, false);
    if (S.rc) return S.rc;
    const u64 *arrays[3] = {Pk.as<u64>(), M.as<u64>(), S.as<u64>()}, sizes[3] = {6 * K, 4 * K, 4 * chains};
    const char *names[3] = {"public key", "message", "signature element"};
    const unsigned widths[3] = {6, 4, 4};
    u64 bad[3], value = 0;
    if (int rc = wots_check_words(c, arrays, sizes, 3, flag, bad)) return rc;
    for (int q = 0; q < 3; q++)
        if (bad[q] != ~0ull) {
            MS_CUDA(c, cudaMemcpy(&value, arrays[q] + bad[q], 8, cudaMemcpyDefault));
            const u64 item = bad[q] / widths[q];
            if (q == 2)
                return fail(c, MS_ERR_INVALID, "ms_rescue_wots_trace: word %llu of element %llu of signature %llu (%llu) "
                            "is not canonical", (unsigned long long)(bad[q] % 4), (unsigned long long)(item % kWotsChains),
                            (unsigned long long)(item / kWotsChains), (unsigned long long)value);
            return fail(c, MS_ERR_INVALID, "ms_rescue_wots_trace: word %llu of %s %llu (%llu) is not canonical",
                        (unsigned long long)(bad[q] % widths[q]), names[q], (unsigned long long)item,
                        (unsigned long long)value);
        }
    WotsTraceArgs t{Pk.as<u64>(), M.as<u64>(), S.as<u64>(), K, chains, n, accs, ends, nullptr};
    wots_trace_kernel<false><<<(unsigned)((chains * kLanes + kThreads - 1) / kThreads), kThreads, 0, c->stream>>>(t);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    MS_CUDA(c, cudaMemsetAsync(flag, 0xFF, 8, c->stream));
    if (int rc = wots_fold(c, {ends, Pk.as<u64>(), 6, K, accs, nullptr, Pk.as<u64>(), flag})) return rc;
    MS_CUDA(c, cudaMemcpyAsync(bad, flag, 8, cudaMemcpyDeviceToHost, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if (bad[0] != ~0ull)
        return fail(c, MS_ERR_INVALID, "ms_rescue_wots_trace: signature %llu does not verify: its root differs from its "
                    "public key", (unsigned long long)bad[0]);
    Staged O(c, out, (size_t)(kW + 3) * n * 8, false, true);
    if (O.rc) return O.rc;
    t.B = B;
    t.out = O.as<u64>();
    wots_trace_kernel<true><<<(unsigned)((B * kLanes + kThreads - 1) / kThreads), kThreads, 0, c->stream>>>(t);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    const int rc_p = Pk.finish(), rc_m = M.finish(), rc_s = S.finish(), rc_o = O.finish();
    return rc_p ? rc_p : rc_m ? rc_m : rc_s ? rc_s : rc_o;
}
