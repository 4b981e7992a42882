// hash.cu — SHA-256 Merkle commitment of a column-major field matrix.
//
// Replaces the reference's CPU path (it never hashes on the GPU, SURVEY.md §0 fact 5):
//   hash_rows            src/merkle.rs:412-436   leaf_i = SHA-256(row i serialized)
//   hash_elements        src/hash.rs:92-99       ark-serialize: canonical value, 8 bytes LE each,
//                                                Fq3 = c0 || c1 || c2
//   build_merkle_nodes   src/merkle.rs:438-508   heap layout, nodes[k] = H(nodes[2k] || nodes[2k+1])
//   merge                src/hash.rs:77-82       SHA-256 over the 64 digest bytes
//
// One thread per row: the column-major LDE is read directly (coalesced across threads since
// consecutive threads take consecutive rows), each word is taken out of Montgomery form with
// one reduction, byte-swapped into the big-endian SHA message schedule and compressed.  This
// kernel is INT32-ALU bound (about 2k instructions per 64-byte block), not HBM bound.
#include <mutex>
#include <cstring>
#include "ctx.cuh"
#include "../../include/ministark_stream.h"
#include "../../include/ministark_host_nodes.h"
#include <algorithm>
#include <cstring>
#include <deque>
#include <vector>

namespace ms {

__constant__ u32 c_K[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
    0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
    0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};

__device__ __forceinline__ u32 bswap(u32 x) { return __byte_perm(x, 0, 0x0123); }

// SHA-256 is bound by the INT32 ALU pipe (SHF/LOP3/IADD3).  Moving the rotations to the FMA pipe (x * 2^(32-r) as
// IMAD.WIDE, hi ^ lo) is slower: IMAD.WIDE issues at half rate and the instruction count grows, so they stay funnel
// shifts.
__device__ __forceinline__ u32 rotr(u32 x, int r) { return __funnelshift_r(x, x, r); }
__device__ __forceinline__ u32 big_sigma1(u32 e) { return rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25); }
__device__ __forceinline__ u32 big_sigma0(u32 a) { return rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22); }
__device__ __forceinline__ u32 small_sigma0(u32 w) { return rotr(w, 7) ^ rotr(w, 18) ^ (w >> 3); }
__device__ __forceinline__ u32 small_sigma1(u32 w) { return rotr(w, 17) ^ rotr(w, 19) ^ (w >> 10); }

// K[i] + W[i] of the constant second block of a 64-byte message (0x80, zeros, bit length 512): the
// Merkle node hash needs no message schedule for it.
__constant__ u32 c_KW_pad64[64];
// same for the padding block that follows a leaf row whose length is a multiple of 64 bytes: per-LAUNCH state, passed
// as a __grid_constant__ kernel argument (constant bank, compile-time indices) — a __constant__ symbol would be shared by
// every context and stream of the device and could be re-uploaded under a kernel still in flight
struct KW64 {
    u32 v[64];
};

// Pipe balancing: SHF/LOP3/IADD3 all issue on the 64-lane ALU pipe while the FMA pipe idles.  fma_add() forces
// an addition onto the FMA pipe as IMAD (x * c_one + y); c_one lives in constant memory so ptxas cannot fold it
// back into an IADD3.  V is a bit mask: 1 message-schedule adds, 2 the t1 chain, 4 t2 / e / a, 8 K+W, 16 sigma shifts.
__constant__ u32 c_one = 1;
template <int ON>
__device__ __forceinline__ u32 fma_add(u32 a, u32 b) {
    if constexpr (ON) {
        u32 d;
        asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(c_one), "r"(b));
        return d;
    } else {
        return a + b;
    }
}

// logical right shift on the FMA pipe: x >> r = mulhi(x, 2^(32-r)), the multiplier read from constant memory
__constant__ u32 c_pow2[33] = {0, 1u << 31, 1u << 30, 1u << 29, 1u << 28, 1u << 27, 1u << 26, 1u << 25, 1u << 24, 1u << 23, 1u << 22,
                               1u << 21, 1u << 20, 1u << 19, 1u << 18, 1u << 17, 1u << 16, 1u << 15, 1u << 14, 1u << 13, 1u << 12,
                               1u << 11, 1u << 10, 1u << 9, 1u << 8, 1u << 7, 1u << 6, 1u << 5, 1u << 4, 1u << 3, 1u << 2, 1u << 1, 1};
template <int ON, int R>
__device__ __forceinline__ u32 shr_fma(u32 x) {
    if constexpr (ON) {
        u32 d;
        asm("mul.hi.u32 %0, %1, %2;" : "=r"(d) : "r"(x), "r"(c_pow2[R]));
        return d;
    } else {
        return x >> R;
    }
}
template <int V> __device__ __forceinline__ u32 small_sigma0_v(u32 w) { return rotr(w, 7) ^ rotr(w, 18) ^ shr_fma<((V & 16) != 0), 3>(w); }
template <int V> __device__ __forceinline__ u32 small_sigma1_v(u32 w) { return rotr(w, 17) ^ rotr(w, 19) ^ shr_fma<((V & 16) != 0), 10>(w); }

template <int V>
struct ShaT {
    u32 h[8];
    __device__ __forceinline__ void init() {
        h[0] = 0x6a09e667; h[1] = 0xbb67ae85; h[2] = 0x3c6ef372; h[3] = 0xa54ff53a;
        h[4] = 0x510e527f; h[5] = 0x9b05688c; h[6] = 0x1f83d9ab; h[7] = 0x5be0cd19;
    }
    // w: 16 message words (big-endian interpreted), destroyed
    __device__ __forceinline__ void compress(u32 (&w)[16]) {
        u32 a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll
        for (int i = 0; i < 64; i++) {
            if (i >= 16)
                w[i & 15] = fma_add<((V & 1) != 0)>(fma_add<((V & 1) != 0)>(w[i & 15], small_sigma0_v<V>(w[(i + 1) & 15])),
                                              fma_add<((V & 1) != 0)>(w[(i + 9) & 15], small_sigma1_v<V>(w[(i + 14) & 15])));
            u32 ch = (e & f) ^ (~e & g);
            u32 t1 = fma_add<((V & 2) != 0)>(fma_add<((V & 2) != 0)>(hh, big_sigma1(e)), fma_add<((V & 2) != 0)>(ch, fma_add<((V & 8) != 0)>(w[i & 15], c_K[i])));
            u32 mj = (a & b) ^ (a & c) ^ (b & c);
            u32 t2 = fma_add<((V & 4) != 0)>(big_sigma0(a), mj);
            hh = g; g = f; f = e; e = fma_add<((V & 4) != 0)>(d, t1); d = c; c = b; b = a; a = fma_add<((V & 4) != 0)>(t1, t2);
        }
        h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
    }
    // compression of the constant padding block that follows a 64-byte message
    __device__ __forceinline__ void compress_pad64() { compress_const(c_KW_pad64); }
    __device__ __forceinline__ void compress_const(const u32 (&kw)[64]) {
        u32 a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll
        for (int i = 0; i < 64; i++) {
            u32 ch = (e & f) ^ (~e & g);
            u32 t1 = fma_add<((V & 2) != 0)>(fma_add<((V & 2) != 0)>(hh, big_sigma1(e)), fma_add<((V & 8) != 0)>(ch, kw[i]));
            u32 mj = (a & b) ^ (a & c) ^ (b & c);
            u32 t2 = fma_add<((V & 4) != 0)>(big_sigma0(a), mj);
            hh = g; g = f; f = e; e = fma_add<((V & 4) != 0)>(d, t1); d = c; c = b; b = a; a = fma_add<((V & 4) != 0)>(t1, t2);
        }
        h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
    }
    // digest bytes = big-endian state words
    __device__ __forceinline__ void store(u32 *out) const {
        uint4 lo = make_uint4(bswap(h[0]), bswap(h[1]), bswap(h[2]), bswap(h[3]));
        uint4 hi = make_uint4(bswap(h[4]), bswap(h[5]), bswap(h[6]), bswap(h[7]));
        reinterpret_cast<uint4 *>(out)[0] = lo;
        reinterpret_cast<uint4 *>(out)[1] = hi;
    }
};

using Sha = ShaT<0>;

// words_per_row = ncols * lanes 64-bit words; word t of row i lives at
// cols[(t / lanes) * col_stride_words + i * lanes + t % lanes].
template <int V>
__global__ void __launch_bounds__(128) hash_rows_kernel(const u64 *__restrict__ cols, size_t col_stride_words,
                                                         unsigned lanes, unsigned words_per_row, size_t nrows,
                                                         u32 *__restrict__ digests, int const_pad,
                                                         const __grid_constant__ KW64 kw_pad) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= nrows) return;
    ShaT<V> s;
    s.init();
    const unsigned msg_words32 = words_per_row * 2;
    const unsigned total32 = ((msg_words32 + 1 + 2 + 15) / 16) * 16;  // 0x80 marker + 64-bit length
    const u64 bitlen = (u64)words_per_row * 64;
    const u64 *row = cols + i * lanes;
    unsigned t = 0, cidx = 0, l = 0;  // running word index -> (column, lane)
    const unsigned data_blocks = const_pad ? msg_words32 / 16 : total32 / 16;   // const_pad: the last block is pure padding
    for (unsigned blk = 0; blk < data_blocks; blk++) {
        u32 w[16];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const unsigned g = blk * 16 + 2 * j;
            u32 lo = 0, hi = 0;
            if (t < words_per_row) {
                u64 x = gl::from_mont(row[(size_t)cidx * col_stride_words + l]);
                lo = bswap((u32)x);
                hi = bswap((u32)(x >> 32));
                t++;
                if (++l == lanes) { l = 0; cidx++; }
            } else {
                if (g == msg_words32) lo = 0x80000000u;
                if (g == total32 - 2) { lo = (u32)(bitlen >> 32); hi = (u32)bitlen; }
            }
            w[2 * j] = lo;
            w[2 * j + 1] = hi;
        }
        s.compress(w);
    }
    if (const_pad) s.compress_const(kw_pad.v);
    s.store(digests + i * 8);
}

// dst[k] = SHA-256(src[2k] || src[2k+1]) for k in [0, count): one Merkle level.
template <int V>
__global__ void __launch_bounds__(128) merkle_level_kernel(const u32 *__restrict__ src, u32 *__restrict__ dst,
                                                            size_t count) {
    const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (k >= count) return;
    ShaT<V> s;
    s.init();
    u32 w[16];
    const uint4 *p = reinterpret_cast<const uint4 *>(src + k * 16);
#pragma unroll
    for (int q = 0; q < 4; q++) {
        uint4 v = p[q];
        w[4 * q] = bswap(v.x); w[4 * q + 1] = bswap(v.y); w[4 * q + 2] = bswap(v.z); w[4 * q + 3] = bswap(v.w);
    }
    s.compress(w);
    s.compress_pad64();
    s.store(dst + k * 8);
}

// Proof-of-work grinding (PublicCoin::grind_proof_of_work, src/random.rs:48-55,129-132; called from
// ProverChannel::grind_fri_commitments, src/channel.rs:76-93): find a nonce with
// leading_zeros(SHA-256(seed || nonce.to_be_bytes())) >= bits.  The reference's parallel search returns ANY
// such nonce (rayon find_any), which makes proof bytes non-deterministic; here every batch of candidates is
// reduced with atomicMin, so the SMALLEST nonce >= 1 is returned — the value the reference's serial branch finds.
__global__ void __launch_bounds__(128) pow_grind_kernel(uint4 seed_lo, uint4 seed_hi, unsigned bits, u64 base, u64 count,
                                                         unsigned long long *best) {
    const u64 idx = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    if (idx >= count) return;
    const u64 nonce = base + idx;
    Sha s;
    s.init();
    u32 w[16] = {seed_lo.x, seed_lo.y, seed_lo.z, seed_lo.w, seed_hi.x, seed_hi.y, seed_hi.z, seed_hi.w,
                 (u32)(nonce >> 32), (u32)nonce, 0x80000000u, 0, 0, 0, 0, 320};
    s.compress(w);
    unsigned lz = __clz(s.h[0]);
    if (s.h[0] == 0) { lz = 32 + __clz(s.h[1]); if (s.h[1] == 0) lz = 64 + __clz(s.h[2]); }
    if (lz >= bits) atomicMin(best, (unsigned long long)nonce);
}

// multiproof gather: out[q] = (sel[q] >> 63 ? nodes : leaves)[sel[q] & mask]  (32-byte digests as 2 x uint4)
__global__ void gather_digests_kernel(const uint4 *__restrict__ leaves, const uint4 *__restrict__ nodes, const u64 *__restrict__ sel,
                                      unsigned count, uint4 *__restrict__ out) {
    const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * count) return;
    const u64 s = sel[t >> 1];
    const uint4 *src = (s >> 63) ? nodes : leaves;
    out[t] = src[2 * (s & ~(1ull << 63)) + (t & 1)];
}

// MS_SHA_FMA_ADDS=0 keeps every addition on the ALU pipe (the compiler's choice); the default mask 7 moves the
// schedule and round-function additions to the FMA pipe (profiles/exp_sha.py times a mask against another).
static int sha_variant() {
    static const int v = [] {
        const char *e = getenv("MS_SHA_FMA_ADDS");
        return (e && atoi(e) == 0) ? 0 : 7;
    }();
    return v;
}
#define MS_SHA_DISPATCH(KERNEL, GRID, ...)                                        \
    if (sha_variant() == 0) KERNEL<0><<<GRID, 128, 0, c->stream>>>(__VA_ARGS__);   \
    else KERNEL<7><<<GRID, 128, 0, c->stream>>>(__VA_ARGS__);

static int row_pad_schedule(unsigned row_words, KW64 *kw);
static int hash_rows_dev(ms_ctx *c, int field, const u64 *cols, size_t col_stride_elems, unsigned ncols, size_t nrows,
                         u32 *digests) {
    if (nrows == 0) return MS_OK;
    const unsigned threads = 128;
    KW64 kw;
    const int const_pad = row_pad_schedule(ncols * field, &kw);
    MS_SHA_DISPATCH(hash_rows_kernel, (unsigned)((nrows + threads - 1) / threads), cols, col_stride_elems * field, (unsigned)field,
                    ncols * field, nrows, digests, const_pad, kw);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    return MS_OK;
}

static u32 h_rotr(u32 x, int r) { return (x >> r) | (x << (32 - r)); }
// K[i] + W[i] for the block {0x80000000, 0, ..., bitlen_hi, bitlen_lo}
static void pad_schedule(unsigned long long bitlen, u32 kw[64]);
static int upload_pad_schedule(ms_ctx *c) {
    static bool done[64] = {false};
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);   // the constant is the same for every context: upload once per device
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 64 && done[dev]) return MS_OK;
    u32 kw[64];
    pad_schedule(512, kw);
    // complete before `done` is set: a synchronous copy from pageable memory may return before its DMA lands, and the
    // kernels of other contexts (other streams, other threads) read the constant as soon as `done` says so
    MS_CUDA(c, cudaMemcpyToSymbolAsync(c_KW_pad64, kw, sizeof kw, 0, cudaMemcpyHostToDevice, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if (dev >= 0 && dev < 64) done[dev] = true;
    return MS_OK;
}
// leaf rows: returns 1 (and fills the schedule) if row_words*8 bytes is a multiple of 64, else 0
static int row_pad_schedule(unsigned row_words, KW64 *kw) {
    memset(kw, 0, sizeof *kw);
    if (row_words % 8) return 0;
    pad_schedule((unsigned long long)row_words * 64, kw->v);
    return 1;
}
static void pad_schedule(unsigned long long bitlen, u32 kw[64]) {
    static const u32 K[64] = {
        0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
        0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
        0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
        0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
        0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
        0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
        0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
        0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
    u32 w[64] = {0};
    w[0] = 0x80000000u;
    w[14] = (u32)(bitlen >> 32);
    w[15] = (u32)bitlen;
    for (int i = 16; i < 64; i++) {
        u32 s0 = h_rotr(w[i - 15], 7) ^ h_rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
        u32 s1 = h_rotr(w[i - 2], 17) ^ h_rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
        w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
    for (int i = 0; i < 64; i++) kw[i] = K[i] + w[i];
}

static int merkle_nodes_dev(ms_ctx *c, const u32 *leaves, size_t n, u32 *nodes) {
    if (int rc = upload_pad_schedule(c)) return rc;
    MS_CUDA(c, cudaMemsetAsync(nodes, 0, 32, c->stream));
    const unsigned threads = 128;
    // leaf pairs -> nodes[n/2 .. n)
    MS_SHA_DISPATCH(merkle_level_kernel, (unsigned)((n / 2 + threads - 1) / threads), leaves, nodes + (n / 2) * 8, n / 2);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    for (size_t size = n / 4; size >= 1; size >>= 1) {
        // nodes[size .. 2 size) from nodes[2 size .. 4 size)
        MS_SHA_DISPATCH(merkle_level_kernel, (unsigned)((size + threads - 1) / threads), nodes + 2 * size * 8, nodes + size * 8, size);
        c->launches++;
        MS_CHECK_LAUNCH(c);
    }
    return MS_OK;
}

int host_nodes_drain(ms_ctx *c, bool release) {
    if (!c->node_copy_stream) return MS_OK;
    MS_CUDA(c, cudaStreamSynchronize(c->node_copy_stream));
    if (!release) return MS_OK;
    for (int k = 0; k < 2; k++) {
        if (c->node_stage[k].ptr) MS_CUDA(c, cudaFree(c->node_stage[k].ptr));
        c->node_stage[k] = Scratch{};
        if (c->node_built[k]) MS_CUDA(c, cudaEventDestroy(c->node_built[k]));
        if (c->node_copied[k]) MS_CUDA(c, cudaEventDestroy(c->node_copied[k]));
        c->node_built[k] = c->node_copied[k] = nullptr;
    }
    MS_CUDA(c, cudaStreamDestroy(c->node_copy_stream));
    c->node_copy_stream = nullptr;
    return MS_OK;
}

// both staging buffers of ms_merkle_commit_block_sha256_host at least `bytes`, with the copy stream and the events
static int host_nodes_staging(ms_ctx *c, size_t bytes) {
    if (!c->node_copy_stream) {
        MS_CUDA(c, cudaStreamCreateWithFlags(&c->node_copy_stream, cudaStreamNonBlocking));
        for (int k = 0; k < 2; k++) {
            MS_CUDA(c, cudaEventCreateWithFlags(&c->node_built[k], cudaEventDisableTiming));
            MS_CUDA(c, cudaEventCreateWithFlags(&c->node_copied[k], cudaEventDisableTiming));
        }
    }
    if (c->node_stage[0].cap >= bytes) return MS_OK;
    MS_CUDA(c, cudaStreamSynchronize(c->node_copy_stream));   // no copy may still read a buffer that is replaced
    for (Scratch &s : c->node_stage) {
        if (s.ptr) MS_CUDA(c, cudaFree(s.ptr));
        s = Scratch{};
        MS_CUDA(c, cudaMalloc(&s.ptr, bytes));
        s.cap = bytes;
    }
    return MS_OK;
}

}  // namespace ms

using namespace ms;

extern "C" {

// include/ministark_host_nodes.h.  Block b's heap is built in staging buffer k = b mod 2 on the compute stream, after the
// copy that last read that buffer (two blocks ago) has finished; the copy stream then moves it to host_subtree while the
// compute stream goes on with the next block.
int ms_merkle_commit_block_sha256_host(ms_ctx *c, int field, const void *cols, size_t col_stride_elems, unsigned ncols,
                                       unsigned log_block_rows, void *host_subtree, void *block_root) {
    if (!c || !cols || !host_subtree || !block_root) return MS_ERR_INVALID;
    if (field != MS_FIELD_FP && field != MS_FIELD_FQ3) return fail(c, MS_ERR_INVALID, "unknown field id %d", field);
    if (ncols == 0) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256_host: no columns");
    if (log_block_rows > 36) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256_host: block too large");
    const size_t nb = (size_t)1 << log_block_rows, bytes = nb * 32;
    if (ncols > 1 && col_stride_elems < nb) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256_host: stride < block rows");
    cudaSetDevice(c->device);
    // an asynchronous copy into pageable memory is staged by the driver and serialises with the compute stream.  Both ends
    // of the range are checked, so a pinned start whose range runs past its allocation is refused too.
    for (const char *p : {(const char *)host_subtree, (const char *)host_subtree + bytes - 1}) {
        cudaPointerAttributes a;
        MS_CUDA(c, cudaPointerGetAttributes(&a, p));
        if (a.type != cudaMemoryTypeHost)
            return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256_host: the subtree buffer is %s memory, not pinned host memory",
                        a.type == cudaMemoryTypeUnregistered ? "pageable host" : a.type == cudaMemoryTypeManaged ? "managed" : "device");
    }
    int rc = host_nodes_staging(c, bytes);
    if (rc) return rc;
    const int k = c->node_stage_next;
    c->node_stage_next ^= 1;
    u32 *heap = (u32 *)c->node_stage[k].ptr;
    Staged in(c, cols, ((size_t)(ncols - 1) * col_stride_elems + nb) * field * 8, true, false);
    if (in.rc) return in.rc;
    void *lv;
    if ((rc = scratch_get(c, 2, bytes, &lv))) return rc;
    if ((rc = hash_rows_dev(c, field, in.as<u64>(), col_stride_elems, ncols, nb, (u32 *)lv))) return rc;
    MS_CUDA(c, cudaStreamWaitEvent(c->stream, c->node_copied[k], 0));
    const u32 *root = (const u32 *)lv;                      // one row: the root is its leaf digest, slot 0 the whole heap
    if (nb == 1) {
        MS_CUDA(c, cudaMemsetAsync(heap, 0, 32, c->stream));
    } else {
        if ((rc = merkle_nodes_dev(c, (const u32 *)lv, nb, heap))) return rc;
        root = heap + 8;
    }
    MS_CUDA(c, cudaEventRecord(c->node_built[k], c->stream));
    MS_CUDA(c, cudaStreamWaitEvent(c->node_copy_stream, c->node_built[k], 0));
    MS_CUDA(c, cudaMemcpyAsync(host_subtree, heap, bytes, cudaMemcpyDeviceToHost, c->node_copy_stream));
    MS_CUDA(c, cudaEventRecord(c->node_copied[k], c->node_copy_stream));
    MS_CUDA(c, cudaMemcpyAsync(block_root, root, 32, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    return in.finish();
}

int ms_hash_rows_sha256(ms_ctx *c, int field, const void *cols, size_t col_stride_elems, unsigned ncols, size_t nrows,
                        void *digests) {
    if (!c || !cols || !digests) return MS_ERR_INVALID;
    if (field != MS_FIELD_FP && field != MS_FIELD_FQ3) return fail(c, MS_ERR_INVALID, "unknown field id %d", field);
    if (ncols == 0) return fail(c, MS_ERR_INVALID, "ms_hash_rows_sha256: no columns");
    if (ncols > 1 && col_stride_elems < nrows) return fail(c, MS_ERR_INVALID, "ms_hash_rows_sha256: stride < nrows");
    Staged in(c, cols, ((size_t)(ncols - 1) * col_stride_elems + nrows) * field * 8, true, false);
    if (in.rc) return in.rc;
    Staged out(c, digests, nrows * 32, false, true);
    if (out.rc) return out.rc;
    int rc = hash_rows_dev(c, field, in.as<u64>(), col_stride_elems, ncols, nrows, out.as<u32>());
    if (rc) return rc;
    if ((rc = in.finish())) return rc;
    return out.finish();
}

int ms_merkle_nodes_sha256(ms_ctx *c, const void *leaves, size_t n, void *nodes) {
    if (!c || !leaves || !nodes) return MS_ERR_INVALID;
    // MerkleTreeImpl::new: at least two leaves, power of two (src/merkle.rs:113-128)
    if (n < 2 || (n & (n - 1))) return fail(c, MS_ERR_INVALID, "merkle tree needs a power-of-two number of leaves >= 2, got %zu", n);
    Staged in(c, leaves, n * 32, true, false);
    if (in.rc) return in.rc;
    Staged out(c, nodes, n * 32, false, true);
    if (out.rc) return out.rc;
    int rc = merkle_nodes_dev(c, in.as<u32>(), n, out.as<u32>());
    if (rc) return rc;
    if ((rc = in.finish())) return rc;
    return out.finish();
}

int ms_merkle_commit_sha256(ms_ctx *c, int field, const void *cols, size_t col_stride_elems, unsigned ncols, size_t nrows,
                            void *leaves, void *nodes, void *root) {
    if (!c || !cols || !root) return MS_ERR_INVALID;
    if (field != MS_FIELD_FP && field != MS_FIELD_FQ3) return fail(c, MS_ERR_INVALID, "unknown field id %d", field);
    if (ncols == 0) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_sha256: no columns");
    if (nrows < 2 || (nrows & (nrows - 1))) return fail(c, MS_ERR_INVALID, "merkle tree needs a power-of-two number of leaves >= 2, got %zu", nrows);
    if (ncols > 1 && col_stride_elems < nrows) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_sha256: stride < nrows");
    Staged in(c, cols, ((size_t)(ncols - 1) * col_stride_elems + nrows) * field * 8, true, false);
    if (in.rc) return in.rc;
    int rc;
    void *lv = nullptr, *nd = nullptr;
    Staged lout(c, leaves, leaves ? nrows * 32 : 0, false, true);
    if (lout.rc) return lout.rc;
    Staged nout(c, nodes, nodes ? nrows * 32 : 0, false, true);
    if (nout.rc) return nout.rc;
    if (leaves) lv = lout.dev;
    else if ((rc = scratch_get(c, 2, nrows * 32, &lv))) return rc;
    if (nodes) nd = nout.dev;
    else if ((rc = scratch_get(c, 3, nrows * 32, &nd))) return rc;
    if ((rc = hash_rows_dev(c, field, in.as<u64>(), col_stride_elems, ncols, nrows, (u32 *)lv))) return rc;
    if ((rc = merkle_nodes_dev(c, (const u32 *)lv, nrows, (u32 *)nd))) return rc;
    MS_CUDA(c, cudaMemcpyAsync(root, (const char *)nd + 32, 32, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if ((rc = in.finish())) return rc;
    if ((rc = lout.finish())) return rc;
    return nout.finish();
}


// One coset block of a tree that is committed block by block (the streaming prover never holds the whole LDE): the
// 2^log_block_rows rows are hashed into scratch, and every subtree level is written straight into its run of the global
// heap.  Level d >= log_blocks of a tree with N = 2^(log_block_rows + log_blocks) leaves holds 2^d nodes at [2^d, 2^(d+1));
// block b owns the cnt = 2^(d - log_blocks) consecutive ones from 2^d + b * cnt, whose children are the block's run one
// level down.  So the leaf pairs go to [N/2 + b * nb/2, ...) and the subtree root lands at nodes[2^log_blocks + b].
int ms_merkle_commit_block_sha256(ms_ctx *c, int field, const void *cols, size_t col_stride_elems, unsigned ncols,
                                  unsigned log_block_rows, unsigned log_blocks, size_t block, void *nodes, void *block_root) {
    if (!c || !cols || !nodes || !block_root) return MS_ERR_INVALID;
    if (field != MS_FIELD_FP && field != MS_FIELD_FQ3) return fail(c, MS_ERR_INVALID, "unknown field id %d", field);
    if (ncols == 0) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256: no columns");
    if (log_block_rows + log_blocks > 40) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256: tree too large");
    if (block >> log_blocks) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256: block %zu of %zu", block, (size_t)1 << log_blocks);
    const size_t nb = (size_t)1 << log_block_rows, beta = (size_t)1 << log_blocks, N = nb << log_blocks;
    if (ncols > 1 && col_stride_elems < nb) return fail(c, MS_ERR_INVALID, "ms_merkle_commit_block_sha256: stride < block rows");
    Staged in(c, cols, ((size_t)(ncols - 1) * col_stride_elems + nb) * field * 8, true, false);
    if (in.rc) return in.rc;
    // a host heap is staged whole, both ways: the block writes only its own runs and the rest must survive
    Staged nd(c, nodes, log_block_rows ? N * 32 : 0, true, true);
    if (nd.rc) return nd.rc;
    void *lv;
    int rc = scratch_get(c, 2, nb * 32, &lv);
    if (rc) return rc;
    if ((rc = hash_rows_dev(c, field, in.as<u64>(), col_stride_elems, ncols, nb, (u32 *)lv))) return rc;
    const u32 *root = (const u32 *)lv;
    if (log_block_rows) {
        if ((rc = upload_pad_schedule(c))) return rc;
        const unsigned threads = 128;
        const u32 *src = (const u32 *)lv;
        for (size_t cnt = nb / 2; cnt >= 1; cnt >>= 1) {
            u32 *dst = nd.as<u32>() + (cnt * beta + block * cnt) * 8;
            MS_SHA_DISPATCH(merkle_level_kernel, (unsigned)((cnt + threads - 1) / threads), src, dst, cnt);
            c->launches++;
            MS_CHECK_LAUNCH(c);
            src = dst;
        }
        root = src;   // nodes[beta + block]
    }
    MS_CUDA(c, cudaMemcpyAsync(block_root, root, 32, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if ((rc = in.finish())) return rc;
    return nd.finish();
}

// Commitment of a ROW-MAJOR matrix (nrows rows of row_words contiguous words): FRI layers commit rows of
// `ff` consecutive evaluations (src/fri.rs:199-216 builds Matrix::from_arrays(chunks) only to hash those
// rows again); hashing the codeword in place gives the same leaves without the transpose.
int ms_merkle_commit_rows_sha256(ms_ctx *c, const void *rows, unsigned row_words, size_t nrows, void *leaves, void *nodes,
                                 void *root) {
    if (!c || !rows || !root || row_words == 0) return MS_ERR_INVALID;
    if (nrows < 2 || (nrows & (nrows - 1))) return fail(c, MS_ERR_INVALID, "merkle tree needs a power-of-two number of leaves >= 2, got %zu", nrows);
    Staged in(c, rows, nrows * row_words * 8, true, false);
    if (in.rc) return in.rc;
    int rc;
    void *lv = nullptr, *nd = nullptr;
    Staged lout(c, leaves, leaves ? nrows * 32 : 0, false, true);
    if (lout.rc) return lout.rc;
    Staged nout(c, nodes, nodes ? nrows * 32 : 0, false, true);
    if (nout.rc) return nout.rc;
    if (leaves) lv = lout.dev;
    else if ((rc = scratch_get(c, 2, nrows * 32, &lv))) return rc;
    if (nodes) nd = nout.dev;
    else if ((rc = scratch_get(c, 3, nrows * 32, &nd))) return rc;
    // one "column" whose element is the whole row: word t of row i at base + i*row_words + t
    const unsigned threads = 128;
    KW64 kw;
    const int const_pad = row_pad_schedule(row_words, &kw);
    MS_SHA_DISPATCH(hash_rows_kernel, (unsigned)((nrows + threads - 1) / threads), in.as<u64>(), (size_t)0, row_words, row_words, nrows,
                    (u32 *)lv, const_pad, kw);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    if ((rc = merkle_nodes_dev(c, (const u32 *)lv, nrows, (u32 *)nd))) return rc;
    MS_CUDA(c, cudaMemcpyAsync(root, (const char *)nd + 32, 32, cudaMemcpyDefault, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if ((rc = in.finish())) return rc;
    if ((rc = lout.finish())) return rc;
    return nout.finish();
}


int ms_pow_grind_sha256(ms_ctx *c, const uint8_t *seed, unsigned bits, uint64_t *nonce_out) {
    if (!c || !seed || !nonce_out) return MS_ERR_INVALID;
    if (bits > 64) return fail(c, MS_ERR_INVALID, "ms_pow_grind_sha256: at most 64 bits supported");
    cudaSetDevice(c->device);
    u32 sw[8];
    for (int i = 0; i < 8; i++)
        sw[i] = ((u32)seed[4 * i] << 24) | ((u32)seed[4 * i + 1] << 16) | ((u32)seed[4 * i + 2] << 8) | seed[4 * i + 3];
    void *best;
    int rc = scratch_get(c, 3, 64, &best);
    if (rc) return rc;
    const unsigned long long none = ~0ull;
    const u64 batch = 1ull << 24;
    for (u64 base = 1;; base += batch) {   // (1..u64::MAX), src/random.rs:50
        MS_CUDA(c, cudaMemcpyAsync(best, &none, 8, cudaMemcpyHostToDevice, c->stream));
        pow_grind_kernel<<<(unsigned)(batch / 128), 128, 0, c->stream>>>(make_uint4(sw[0], sw[1], sw[2], sw[3]),
                                                                         make_uint4(sw[4], sw[5], sw[6], sw[7]), bits, base, batch,
                                                                         (unsigned long long *)best);
        c->launches++;
        MS_CHECK_LAUNCH(c);
        unsigned long long got = none;
        MS_CUDA(c, cudaMemcpyAsync(&got, best, 8, cudaMemcpyDeviceToHost, c->stream));
        MS_CUDA(c, cudaStreamSynchronize(c->stream));
        if (got != none) {
            *nonce_out = got;
            return MS_OK;
        }
        if (base > (~0ull) - 2 * batch) return fail(c, MS_ERR_INVALID, "nonce not found");   // .expect("nonce not found")
    }
}

// MerkleTreeImpl::prove (src/merkle.rs:149-207): batched authentication paths for a set of leaves, read from the
// RESIDENT leaf and node arrays — only the <= n_indices * (height + 1) digests of the proof cross PCIe.
// The index walk (two queues, siblings merged when both are in the set) runs on the host; one gather kernel
// fetches every digest the walk names.
int ms_merkle_prove_sha256(ms_ctx *c, const void *leaves, const void *nodes, size_t n_leaves, const uint64_t *indices,
                           unsigned n_indices, uint8_t *initial_leaves, uint8_t *sibling_leaves, uint8_t *path_nodes,
                           unsigned counts[3]) {
    if (!c || !leaves || !nodes || !indices || !initial_leaves || !sibling_leaves || !path_nodes || !counts) return MS_ERR_INVALID;
    if (n_leaves < 2 || (n_leaves & (n_leaves - 1))) return fail(c, MS_ERR_INVALID, "ms_merkle_prove: leaf count must be a power of two >= 2");
    cudaSetDevice(c->device);
    std::vector<u64> idx(indices, indices + n_indices);
    for (u64 i : idx)
        if (i >= n_leaves) return fail(c, MS_ERR_INVALID, "leaf index `%llu` cannot exceed the number of leaves (`%llu`)",
                                       (unsigned long long)i, (unsigned long long)n_leaves);
    std::sort(idx.begin(), idx.end());
    idx.erase(std::unique(idx.begin(), idx.end()), idx.end());
    const u64 NODE = 1ull << 63;
    std::vector<u64> init, sib, path;
    std::deque<u64> node_q;
    for (size_t k = 0; k < idx.size(); k++) {
        const u64 i = idx[k];
        init.push_back(i);
        node_q.push_back((n_leaves + i) >> 1);
        if (k + 1 < idx.size() && (i ^ 1) == idx[k + 1]) {
            init.push_back(idx[++k]);
            continue;
        }
        sib.push_back(i ^ 1);
    }
    while (!node_q.empty()) {
        const u64 i = node_q.front();
        node_q.pop_front();
        if (i > 2) node_q.push_back(i >> 1);
        if (!node_q.empty() && (i ^ 1) == node_q.front()) {
            node_q.pop_front();
            continue;
        }
        path.push_back((i ^ 1) | NODE);      // (n_leaves == 2 names nodes[0], the unused default digest, as the reference does)
    }
    counts[0] = (unsigned)init.size();
    counts[1] = (unsigned)sib.size();
    counts[2] = (unsigned)path.size();
    std::vector<u64> sel(init);
    sel.insert(sel.end(), sib.begin(), sib.end());
    sel.insert(sel.end(), path.begin(), path.end());
    const unsigned total = (unsigned)sel.size();
    if (!total) return MS_OK;
    Staged lv(c, leaves, n_leaves * 32, true, false);
    if (lv.rc) return lv.rc;
    Staged nd(c, nodes, n_leaves * 32, true, false);
    if (nd.rc) return nd.rc;
    void *dsel, *dout;
    int rc;
    if ((rc = scratch_get(c, 2, (size_t)total * 8, &dsel))) return rc;
    if ((rc = scratch_get(c, 3, (size_t)total * 32, &dout))) return rc;
    MS_CUDA(c, cudaMemcpyAsync(dsel, sel.data(), (size_t)total * 8, cudaMemcpyHostToDevice, c->stream));
    gather_digests_kernel<<<(2 * total + 127) / 128, 128, 0, c->stream>>>(lv.as<uint4>(), nd.as<uint4>(), (const u64 *)dsel, total,
                                                                           (uint4 *)dout);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    std::vector<uint8_t> host((size_t)total * 32);
    MS_CUDA(c, cudaMemcpyAsync(host.data(), dout, host.size(), cudaMemcpyDeviceToHost, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    memcpy(initial_leaves, host.data(), init.size() * 32);
    memcpy(sibling_leaves, host.data() + init.size() * 32, sib.size() * 32);
    memcpy(path_nodes, host.data() + (init.size() + sib.size()) * 32, path.size() * 32);
    if ((rc = lv.finish())) return rc;
    return nd.finish();
}

}  // extern "C"
