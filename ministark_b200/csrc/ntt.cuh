// ntt.cuh — shared declarations of the multi-pass NTT engine (ntt.cu) used by api.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "field.cuh"

namespace msntt {

using gl::u32;
using gl::u64;

constexpr int kMaxDims = 4;
constexpr int kTileLog = 12;          // a CTA tile holds at most 4096 elements (32 KiB + padding)
constexpr int kElemsPerThread = 16;   // radix-16 register butterflies

struct Dim {
    u32 ext;      // number of values enumerated by the tile id (a power of two)
    u32 log_ext;
    u64 in_str;   // element strides
    u64 out_str;
    u64 low_str;  // contribution to the "lower index" of the outer twiddle
};

// One pass = every CTA runs W independent R-point sub-NTTs on a [R][W] tile held in
// shared memory (radix-16/8/4/2 register butterflies, smem exchange between steps),
// then multiplies by the inter-pass twiddles and writes the tile back.
struct PassParams {
    u32 log_r, log_w;
    u64 in_rs, in_cs, out_rs, out_cs;  // element strides of (transform index, lane) in / out
    u64 low_cs;                        // lower-index increment per lane
    u32 ndims;
    Dim dims[kMaxDims];
    u32 in_r_fast, out_r_fast;         // which tile dimension is contiguous in global memory
    u32 bitrev_digit;                  // 1: leave the digit bit-reversed in place (LDE), 0: natural
    u32 has_outer;
    u64 outer_mult;                    // exponent of omega_N = i_R * lower * outer_mult (mod N)
    u64 n_mask;
    u32 hi_len;                        // entries of tw_hi / sc_hi per table (1 => single-level)
    u32 has_pre, has_post;
    u64 post_step;                     // q^(out_rs << shift) (Montgomery), inverse transforms
    // batch decode: blockIdx.y -> (column, coset block, lane)
    u32 lanes, ncos;
    u64 in_col_stride, out_col_stride;   // words
    u64 in_cos_stride, out_cos_stride;   // words
    u32 estride;                         // words per element (1 Fp, 3 Fq3)
    u32 nbatch;                          // columns * coset blocks * lanes = gridDim.x (batch varies fastest)
    u32 log_ncos;
    // optional full tables (replace the per-thread geometric progressions: one multiplication per
    // element instead of two; shared by every column / coset of the batch, so they stay in L2)
    const u64 *outer_tab;                // [i_R * outer_S + lower] = omega_{N_k}^(i_R * lower)
    u64 outer_S;
    const u64 *pre_tab;                  // [cos * pre_cos_stride + j] = q_cos^j
    u64 pre_cos_stride;
    const u64 *post_tab;                 // [i] = c * q^i
    // LDE scatter (fused exchange, multi-GPU): when set, coset block `cos` of column 0 is written at out_cos_ptr[cos]
    // (a pointer that may live on a PEER device, reached over NVLink) instead of out + cos * out_cos_stride, and —
    // where out_dup_ptr[cos] is non-null — a second copy at out_dup_ptr[cos] with its own column stride.
    u64 *const *out_cos_ptr = nullptr;
    u64 *const *out_dup_ptr = nullptr;
    u64 dup_col_stride = 0;              // words
    // the same two tables as HOST arrays (valid for the duration of the launch call): the TMA pipeline encodes one
    // tensor map per destination block from them
    void *const *host_cos_ptr = nullptr;
    void *const *host_dup_ptr = nullptr;
};

struct Tables {
    const u64 *t4096;    // omega_4096^e, direction specific, Montgomery, canonical
    const u64 *tw_lo;    // omega_N^e0            e0 < min(N,4096)
    const u64 *tw_hi;    // omega_N^(4096 e1)     e1 < hi_len
    const u64 *sc_lo;    // per coset block: q^e0            [ncos][4096]
    const u64 *sc_hi;    // per coset block: c * q^(4096 e1) [ncos][hi_len]
    const u64 *pre_step; // per coset block: q^(in_rs << shift of first step)
};

// digit decomposition of a 2^log_n transform
std::vector<int> choose_digits(unsigned log_n);
// radix steps of one CTA-level sub-NTT of 2^log_r points
void steps_of(int log_r, int out[3], int *nsteps);

void launch_pass(const PassParams &p, const Tables &t, bool inverse, const u64 *in, u64 *out, unsigned ntiles,
                 unsigned nbatch, cudaStream_t stream);

// definition-based reference kernel, one thread per output; used for n < 16 and self checks
// (out of place: `in` and `out` must not overlap)
void launch_naive(const u64 *in, u64 in_stride_words, u64 *out, u64 out_stride_words, unsigned log_n, unsigned estride,
                  unsigned lanes, unsigned ncols, bool inverse, u64 root_mont, u64 offset_mont, cudaStream_t stream);

// persistent TMA pipeline (ntt_tma.cu) for the 256 x 16 tile passes of Fp transforms; false = shape not covered, nothing
// launched.  tma_configure: enabled (0/1, -1 keeps), consumer groups per CTA (2/3), cap on shared-memory stages.
bool launch_pass_tma(const PassParams &p, const Tables &t, bool inverse, const u64 *in, u64 *out, unsigned ntiles,
                     unsigned ncols, cudaStream_t stream);
void tma_configure(int enabled, int groups, int max_stages);
// wide_index_configure(1): launch_pass uses the 64-bit-offset instantiations (LW = -1) at every size instead of the
// compile-time (8,4) / (7,5) / (6,6) tile shapes, so that path can be compared with the oracle at small sizes
void wide_index_configure(int enabled);
// table builders (device kernels): dst[i] = lookup2(lo, hi, hi_len, i) and the outer-twiddle table
void build_pow_table(u64 *dst, u64 count, const u64 *lo, const u64 *hi, u32 hi_len, cudaStream_t stream);
void build_outer_table(u64 *dst, u64 R, u64 S, u64 mult, u64 n_mask, const u64 *lo, const u64 *hi, u32 hi_len,
                       cudaStream_t stream);

}  // namespace msntt
