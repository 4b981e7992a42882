// bf_trace.cu — the execution trace of examples/brainfuck (include/ministark_bf.h).
//
// ms_bf_run is the VM (examples/brainfuck/vm.rs:68-336) as a host loop writing one 8-byte record per processor row.
// Everything that turns those records into the 17 base columns is data-parallel and runs here on the device:
//   processor   (cols 0-7)   row r < P is record r; rows past P repeat the final state with the cycle counting on;
//   instruction (cols 12-14) every row with ip = k is (k, prog[k], prog[k+1]), so the table is the segments k = 0..L in
//                            order, segment k of length [k < L] + hist[k]: a histogram of ip, an exclusive scan, and a
//                            binary search per row; padding (L, 0, 0) continues segment L;
//   memory      (cols 8-11)  the first P - 1 records (curr != 0) are already in cycle order, so a stable sort by mp gives
//                            the reference's (mp, cycle) order; entry j is followed by cycle[j+1] - cycle[j] - 1 dummy
//                            rows when mp[j+1] == mp[j]: an exclusive scan of 1 + extra_j and a binary search per row;
//   input / output (15, 16)  stream compactions of the READ rows (value: the next record's mem_val) and WRITE rows.
// Every value is below 2^32, so its Montgomery word is v * (2^32 - 1) without a reduction; MemValInv comes from a table
// of the 255 inverses.
#include <algorithm>
#include <array>
#include <cub/cub.cuh>

#include "../../include/ministark_bf.h"
#include "ctx.cuh"

namespace ms {

constexpr u64 kMontOne = 0xFFFFFFFFull;     // Montgomery word of 1 = 2^64 mod p; v * kMontOne is the word of v < 2^32
constexpr u32 kTape = 1024;
constexpr u32 kInc = '+', kDec = '-', kLeft = '<', kRight = '>', kWrite = '.', kRead = ',', kLoop = '[', kEnd = ']';

__host__ __device__ __forceinline__ u32 rec_ip(u64 r) { return (u32)r; }
__host__ __device__ __forceinline__ u32 rec_mp(u64 r) { return (u32)(r >> 32) & 0xFFFF; }
__host__ __device__ __forceinline__ u32 rec_val(u64 r) { return (u32)(r >> 48) & 0xFF; }

// Montgomery words of 1/v for v = 0..255 (0 for v = 0, as BrainfuckTrace stores it)
static const u64 *inverse_table() {
    static const std::array<u64, 256> table = [] {
        using u128 = unsigned __int128;
        auto mulmod = [](u64 a, u64 b) { return (u64)((u128)a * b % gl::P); };
        std::array<u64, 256> t{};
        for (u64 v = 1; v < 256; v++) {
            u64 r = 1, b = v, e = gl::P - 2;
            for (; e; e >>= 1, b = mulmod(b, b))
                if (e & 1) r = mulmod(r, b);
            t[v] = (u64)(((u128)r << 64) % gl::P);
        }
        return t;
    }();
    return table.data();
}

// ---------------------------------------------------------------------------------------------------- phase 1: sizes
struct BfCounts {
    unsigned long long reads, writes, bad;
};

// per memory address the first and last cycle that touches it; READ / WRITE counts; records that cannot come from a run
__global__ void bf_scan_log_kernel(const u32 *prog, u64 L, const u64 *log, u64 nrec, u32 *first, u32 *last, BfCounts *cnt) {
    const u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    const bool live = i < nrec;
    const u64 rec = live ? log[i] : 0;
    const u32 ip = rec_ip(rec), mp = rec_mp(rec);
    const bool is_cycle = live && i + 1 < nrec;
    const bool bad = live && (mp >= kTape || (is_cycle ? ip >= L : ip != L));
    const bool cyc = is_cycle && !bad;
    const u32 curr = cyc ? prog[ip] : 0;
    const unsigned nread = __popc(__ballot_sync(~0u, curr == kRead)), nwrite = __popc(__ballot_sync(~0u, curr == kWrite));
    const unsigned nbad = __popc(__ballot_sync(~0u, bad));
    const unsigned lane = threadIdx.x & 31;
    if (lane == 0) {
        if (nread) atomicAdd(&cnt->reads, nread);
        if (nwrite) atomicAdd(&cnt->writes, nwrite);
        if (nbad) atomicAdd(&cnt->bad, nbad);
    }
    // one atomic per distinct address in the warp: the loops of a program touch few cells
    const unsigned peers = __match_any_sync(~0u, cyc ? mp : kTape);
    const u32 lo = __reduce_min_sync(peers, cyc ? (u32)i : ~0u), hi = __reduce_max_sync(peers, cyc ? (u32)i : 0u);
    if (cyc && lane == (unsigned)(__ffs(peers) - 1)) {
        atomicMin(first + mp, lo);
        atomicMax(last + mp, hi);
    }
}

// ----------------------------------------------------------------------------------------------------- phase 2: fill
// workspace of ms_bf_trace_fill: byte offsets of its arrays, each aligned to 256 bytes
struct BfWork {
    size_t inv, seg, istart, kin, kout, vin, vout, mlen, mstart, io, iopos, temp, temp_bytes, total;
};

static int bf_layout(ms_ctx *c, size_t L, size_t C, BfWork *w) {
    size_t sort_b = 0, scan32_a = 0, scan32_b = 0, scan64_b = 0;
    const int nc = (int)C, ns = (int)(L + 1);
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const uint16_t *)nullptr, (uint16_t *)nullptr,
                                                    (const u32 *)nullptr, (u32 *)nullptr, nc, 0, 10);
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(nullptr, scan32_a, (const u32 *)nullptr, (u32 *)nullptr, ns);
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(nullptr, scan32_b, (const u32 *)nullptr, (u32 *)nullptr, nc);
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(nullptr, scan64_b, (const u64 *)nullptr, (u64 *)nullptr, nc);
    if (e != cudaSuccess) return fail(c, MS_ERR_CUDA, "bf tables: temporary storage query: %s", cudaGetErrorString(e));
    size_t off = 0;
    auto take = [&](size_t bytes) {
        const size_t at = off;
        off += (bytes + 255) & ~(size_t)255;
        return at;
    };
    w->inv = take(256 * 8);
    w->seg = take((L + 1) * 4);
    w->istart = take((L + 1) * 4);
    w->kin = take(C * 2);
    w->kout = take(C * 2);
    w->vin = take(C * 4);
    w->vout = take(C * 4);
    w->mlen = take(C * 4);
    w->mstart = take(C * 4);
    w->io = take(C * 8);
    w->iopos = take(C * 8);
    w->temp_bytes = std::max(std::max(sort_b, scan32_a), std::max(scan32_b, scan64_b));
    w->temp = take(w->temp_bytes);
    w->total = off;
    return MS_OK;
}

__global__ void bf_seg_init_kernel(u32 *seg, u64 L) {
    const u64 k = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    if (k <= L) seg[k] = k < L;                  // the program listing's own row of address k
}

// seg[ip] += 1 for every record; sort keys / payloads and the packed READ | WRITE << 32 flags of every cycle
__global__ void bf_prep_kernel(const u32 *prog, u64 L, const u64 *log, u64 nrec, u32 *seg, uint16_t *kin, u32 *vin, u64 *io) {
    const u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    const bool live = i < nrec;
    const u64 rec = live ? log[i] : 0;
    const u32 ip = rec_ip(rec);
    const bool in_range = live && ip <= L;     // false only for a log ms_bf_trace_sizes did not accept: no fault
    const unsigned peers = __match_any_sync(~0u, in_range ? ip : ~0u);
    if (in_range && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(seg + ip, (u32)__popc(peers));
    if (live && i + 1 < nrec) {
        const u32 curr = ip < L ? prog[ip] : 0;
        kin[i] = (uint16_t)rec_mp(rec);
        vin[i] = (u32)i;
        io[i] = (u64)(curr == kRead) | ((u64)(curr == kWrite) << 32);
    }
}

// rows of memory entry j: itself and the dummy rows up to the next access of the same address
__global__ void bf_memlen_kernel(const uint16_t *key, const u32 *cyc, u64 C, u32 *len) {
    const u64 j = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    if (j >= C) return;
    len[j] = 1 + (j + 1 < C && key[j + 1] == key[j] ? cyc[j + 1] - cyc[j] - 1 : 0);
}

// the last index j < count with start[j] <= r (start[0] = 0 <= r)
__device__ __forceinline__ u64 segment_of(const u32 *start, u64 count, u64 r) {
    u64 lo = 0, hi = count;
    while (hi - lo > 1) {
        const u64 mid = (lo + hi) >> 1;
        if (start[mid] <= r) lo = mid;
        else hi = mid;
    }
    return lo;
}

struct BfFill {
    const u32 *prog;
    const u64 *log, *inv;
    const u32 *istart, *mstart, *mcyc;
    u64 L, P, M, n;
    u64 *out;
};

__global__ void bf_fill_kernel(BfFill f) {
    const u64 r = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    if (r >= f.n) return;
    u64 *o = f.out + r;
    const u64 n = f.n, C = f.P - 1;
    const auto prog_at = [&](u64 k) -> u64 { return k < f.L ? f.prog[k] : 0; };
    // processor: record r, or the final state with the cycle counting on
    {
        const u64 rec = f.log[r < f.P ? r : f.P - 1];
        const u64 ip = rec_ip(rec), mv = rec_val(rec);
        const u64 curr = prog_at(ip), next = prog_at(ip + 1);      // ip = L on the final state: both 0
        o[0 * n] = r * kMontOne;
        o[1 * n] = ip * kMontOne;
        o[2 * n] = curr * kMontOne;
        o[3 * n] = next * kMontOne;
        o[4 * n] = (u64)rec_mp(rec) * kMontOne;
        o[5 * n] = mv * kMontOne;
        o[6 * n] = f.inv[mv];
        o[7 * n] = curr == 0 ? kMontOne : 0;
    }
    // memory: entry j and its dummy rows; past M the last entry with the cycle counting on
    {
        const bool in_table = r < f.M;
        const u64 j = in_table ? segment_of(f.mstart, C, r) : C - 1;
        const u64 off = in_table ? r - f.mstart[j] : r - f.M + 1;
        const u64 cyc = f.mcyc[j];
        const u64 rec = f.log[cyc];
        o[8 * n] = (cyc + off) * kMontOne;
        o[9 * n] = (u64)rec_mp(rec) * kMontOne;
        o[10 * n] = (u64)rec_val(rec) * kMontOne;
        o[11 * n] = (!in_table || off) ? kMontOne : 0;
    }
    // instruction: segment k; past L + P the row (L, 0, 0) of segment L
    {
        const u64 k = r < f.L + f.P ? segment_of(f.istart, f.L + 1, r) : f.L;
        o[12 * n] = k * kMontOne;
        o[13 * n] = prog_at(k) * kMontOne;
        o[14 * n] = prog_at(k + 1) * kMontOne;
    }
    o[15 * n] = 0;                                   // input / output padding; bf_io_kernel writes the values
    o[16 * n] = 0;
}

__global__ void bf_io_kernel(const u32 *prog, u64 L, const u64 *log, u64 C, const u64 *pos, u64 *out, u64 n) {
    const u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    if (i >= C) return;
    const u64 rec = log[i];
    const u32 curr = rec_ip(rec) < L ? prog[rec_ip(rec)] : 0;
    if (curr == kRead) out[15 * n + (u32)pos[i]] = (u64)rec_val(log[i + 1]) * kMontOne;      // the value read
    else if (curr == kWrite) out[16 * n + (pos[i] >> 32)] = (u64)rec_val(rec) * kMontOne;
}

__global__ void bf_helper_kernel(const u64 *base, u64 n, u64 *aux) {
    const u64 r = blockIdx.x * (u64)blockDim.x + threadIdx.x;
    if (r >= n) return;
    const u64 ci = base[2 * n + r], next_mv = base[5 * n + (r + 1 == n ? 0 : r + 1)];
    const u64 iip = base[12 * n + r], ici = base[13 * n + r];
    const bool first = r == 0, same_ip = !first && base[12 * n + r - 1] == iip;
    const bool rd = ci == kRead * kMontOne, wr = ci == kWrite * kMontOne;
    aux[0 * n + r] = ci != 0 ? kMontOne : 0;
    aux[1 * n + r] = rd ? kMontOne : 0;
    aux[2 * n + r] = rd ? next_mv : 0;
    aux[3 * n + r] = wr ? kMontOne : 0;
    aux[4 * n + r] = wr ? next_mv : 0;
    aux[5 * n + r] = base[11 * n + r] == 0 ? kMontOne : 0;
    aux[6 * n + r] = ici != 0 && same_ip ? kMontOne : 0;
    aux[7 * n + r] = !same_ip ? kMontOne : 0;
}

static unsigned blocks(u64 count, unsigned threads) { return (unsigned)((count + threads - 1) / threads); }

}  // namespace ms

using namespace ms;

// ---------------------------------------------------------------------------------------------------------- the VM
extern "C" int ms_bf_run(const uint32_t *prog, size_t L, const uint8_t *input, size_t input_len, uint64_t max_cycles,
                         uint64_t *log, uint8_t *output, uint64_t *counts) {
    clear_noctx_error();
    if (!prog || !log || !counts || (input_len && !input) || (max_cycles && !output))
        return fail_noctx(MS_ERR_INVALID, "ms_bf_run: null argument");
    if (L == 0) return fail_noctx(MS_ERR_INVALID, "ms_bf_run: empty program");
    if (L >= 0xFFFFFFFFull) return fail_noctx(MS_ERR_INVALID, "ms_bf_run: program of %zu words is too long", L);
    uint8_t tape[kTape] = {0};
    u64 ip = 0, mp = 0, cycle = 0, nout = 0;
    size_t in = 0;
    while (ip < L) {
        if (cycle == max_cycles)
            return fail_noctx(MS_ERR_INVALID, "ms_bf_run: the cycle cap of %llu was reached at ip %llu",
                        (unsigned long long)max_cycles, (unsigned long long)ip);
        log[cycle] = ip | mp << 32 | (u64)tape[mp] << 48;
        const u32 op = prog[ip];
        if ((op == kLoop || op == kEnd) && ip + 1 >= L)
            return fail_noctx(MS_ERR_INVALID, "ms_bf_run: jump at ip %llu has no target", (unsigned long long)ip);
        switch (op) {
            case kLoop: ip = tape[mp] == 0 ? prog[ip + 1] : ip + 2; break;
            case kEnd: ip = tape[mp] != 0 ? prog[ip + 1] : ip + 2; break;
            case kLeft:
            case kRight:
                if (op == kLeft ? mp == 0 : mp == kTape - 1)
                    return fail_noctx(MS_ERR_INVALID, "ms_bf_run: the memory pointer leaves the %u-cell tape at cycle %llu (ip %llu)",
                                kTape, (unsigned long long)cycle, (unsigned long long)ip);
                mp = op == kLeft ? mp - 1 : mp + 1;
                ip++;
                break;
            case kInc: tape[mp]++; ip++; break;
            case kDec: tape[mp]--; ip++; break;
            case kWrite: output[nout++] = tape[mp]; ip++; break;
            case kRead:
                if (in == input_len)
                    return fail_noctx(MS_ERR_INVALID, "ms_bf_run: ',' at cycle %llu (ip %llu) finds the input exhausted",
                                (unsigned long long)cycle, (unsigned long long)ip);
                tape[mp] = input[in++];
                ip++;
                break;
            default:
                return fail_noctx(MS_ERR_INVALID, "ms_bf_run: unrecognized instruction %u at ip %llu", op, (unsigned long long)ip);
        }
        cycle++;
    }
    if (ip != L) return fail_noctx(MS_ERR_INVALID, "ms_bf_run: jump past the end of the program (ip %llu)", (unsigned long long)ip);
    log[cycle] = ip | mp << 32 | (u64)tape[mp] << 48;
    counts[0] = cycle;
    counts[1] = nout;
    return MS_OK;
}

// --------------------------------------------------------------------------------------------------------- the tables
extern "C" int ms_bf_trace_sizes(ms_ctx *c, const uint32_t *program, size_t L, const uint64_t *log, size_t nrec, uint64_t *sizes) {
    if (!c || !program || !log || !sizes) return MS_ERR_INVALID;
    if (L == 0 || nrec < 2) return fail(c, MS_ERR_INVALID, "ms_bf_trace_sizes: need a program and at least one cycle");
    if (nrec + L >= (1ull << 31)) return fail(c, MS_ERR_INVALID, "ms_bf_trace_sizes: %zu records of a %zu-word program are too many", nrec, L);
    Staged Pg(c, program, L * 4, true, false);
    if (Pg.rc) return Pg.rc;
    Staged Lg(c, log, nrec * 8, true, false);
    if (Lg.rc) return Lg.rc;
    void *meta;
    const size_t tab = kTape * 4;
    int rc = scratch_get(c, 3, 2 * tab + sizeof(BfCounts), &meta);
    if (rc) return rc;
    u32 *first = (u32 *)meta, *last = first + kTape;
    BfCounts *cnt = (BfCounts *)(last + kTape);
    MS_CUDA(c, cudaMemsetAsync(first, 0xff, tab, c->stream));
    MS_CUDA(c, cudaMemsetAsync(last, 0, tab + sizeof(BfCounts), c->stream));
    bf_scan_log_kernel<<<blocks(nrec, 256), 256, 0, c->stream>>>(Pg.as<u32>(), L, Lg.as<u64>(), nrec, first, last, cnt);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    std::vector<u32> h(2 * kTape);
    BfCounts hc;
    MS_CUDA(c, cudaMemcpyAsync(h.data(), first, 2 * tab, cudaMemcpyDeviceToHost, c->stream));
    MS_CUDA(c, cudaMemcpyAsync(&hc, cnt, sizeof hc, cudaMemcpyDeviceToHost, c->stream));
    MS_CUDA(c, cudaStreamSynchronize(c->stream));
    if ((rc = Pg.finish()) || (rc = Lg.finish())) return rc;
    if (hc.bad) return fail(c, MS_ERR_INVALID, "ms_bf_trace_sizes: %llu records are not states of a run of this program", hc.bad);
    u64 M = 0;                                   // an address's rows run from its first to its last access, dummies included
    for (u32 k = 0; k < kTape; k++)
        if (h[k] != ~0u) M += (u64)h[kTape + k] - h[k] + 1;
    const u64 P = nrec, IR = L + P, longest = std::max(IR, M);
    u64 n = 1;
    while (n < longest) n <<= 1;
    BfWork w;
    if ((rc = bf_layout(c, L, nrec - 1, &w))) return rc;
    sizes[MS_BF_PROC_ROWS] = P;
    sizes[MS_BF_INSTR_ROWS] = IR;
    sizes[MS_BF_MEM_ROWS] = M;
    sizes[MS_BF_READS] = hc.reads;
    sizes[MS_BF_WRITES] = hc.writes;
    sizes[MS_BF_N] = n;
    sizes[MS_BF_WORK_BYTES] = w.total;
    return MS_OK;
}

extern "C" int ms_bf_trace_fill(ms_ctx *c, const uint32_t *program, size_t L, const uint64_t *log, size_t nrec,
                                const uint64_t *sizes, void *work, void *out) {
    if (!c || !program || !log || !sizes || !work || !out) return MS_ERR_INVALID;
    if (L == 0 || nrec < 2 || sizes[MS_BF_PROC_ROWS] != nrec || sizes[MS_BF_INSTR_ROWS] != L + nrec)
        return fail(c, MS_ERR_INVALID, "ms_bf_trace_fill: sizes are not ms_bf_trace_sizes' for this program and log");
    const u64 n = sizes[MS_BF_N], M = sizes[MS_BF_MEM_ROWS], C = nrec - 1;
    if (n < std::max((u64)L + nrec, M) || (n & (n - 1)) || M < C)
        return fail(c, MS_ERR_INVALID, "ms_bf_trace_fill: inconsistent sizes");
    if (!is_device_ptr(work)) return fail(c, MS_ERR_INVALID, "ms_bf_trace_fill: the workspace must be device memory");
    BfWork w;
    int rc = bf_layout(c, L, C, &w);
    if (rc) return rc;
    if (w.total != sizes[MS_BF_WORK_BYTES]) return fail(c, MS_ERR_INVALID, "ms_bf_trace_fill: workspace size mismatch");
    Staged Pg(c, program, L * 4, true, false);
    if (Pg.rc) return Pg.rc;
    Staged Lg(c, log, nrec * 8, true, false);
    if (Lg.rc) return Lg.rc;
    Staged O(c, out, 17 * n * 8, false, true);
    if (O.rc) return O.rc;
    char *wb = (char *)work;
    u32 *seg = (u32 *)(wb + w.seg), *istart = (u32 *)(wb + w.istart), *vin = (u32 *)(wb + w.vin), *vout = (u32 *)(wb + w.vout);
    u32 *mlen = (u32 *)(wb + w.mlen), *mstart = (u32 *)(wb + w.mstart);
    uint16_t *kin = (uint16_t *)(wb + w.kin), *kout = (uint16_t *)(wb + w.kout);
    u64 *io = (u64 *)(wb + w.io), *iopos = (u64 *)(wb + w.iopos), *inv = (u64 *)(wb + w.inv);
    void *temp = wb + w.temp;
    size_t tb = w.temp_bytes;
    const u32 *prog = Pg.as<u32>();
    const u64 *lg = Lg.as<u64>();
    cudaStream_t s = c->stream;
    MS_CUDA(c, cudaMemcpyAsync(inv, inverse_table(), 256 * 8, cudaMemcpyHostToDevice, s));
    bf_seg_init_kernel<<<blocks(L + 1, 256), 256, 0, s>>>(seg, L);
    bf_prep_kernel<<<blocks(nrec, 256), 256, 0, s>>>(prog, L, lg, nrec, seg, kin, vin, io);
    c->launches += 2;
    MS_CHECK_LAUNCH(c);
    // the stable radix sort over the 10 address bits keeps cycle order within an address
    MS_CUDA(c, cub::DeviceScan::ExclusiveSum(temp, tb, seg, istart, (int)(L + 1), s));
    MS_CUDA(c, cub::DeviceRadixSort::SortPairs(temp, tb, kin, kout, vin, vout, (int)C, 0, 10, s));
    bf_memlen_kernel<<<blocks(C, 256), 256, 0, s>>>(kout, vout, C, mlen);
    c->launches++;
    MS_CHECK_LAUNCH(c);
    MS_CUDA(c, cub::DeviceScan::ExclusiveSum(temp, tb, mlen, mstart, (int)C, s));
    // READ and WRITE counts below 2^32 each: one 64-bit scan of READ | WRITE << 32 gives both output positions
    MS_CUDA(c, cub::DeviceScan::ExclusiveSum(temp, tb, io, iopos, (int)C, s));
    BfFill f;
    f.prog = prog;
    f.log = lg;
    f.inv = inv;
    f.istart = istart;
    f.mstart = mstart;
    f.mcyc = vout;
    f.L = L;
    f.P = nrec;
    f.M = M;
    f.n = n;
    f.out = O.as<u64>();
    bf_fill_kernel<<<blocks(n, 256), 256, 0, s>>>(f);
    bf_io_kernel<<<blocks(C, 256), 256, 0, s>>>(prog, L, lg, C, iopos, O.as<u64>(), n);
    c->launches += 2;
    MS_CHECK_LAUNCH(c);
    if ((rc = Pg.finish()) || (rc = Lg.finish())) return rc;
    return O.finish();
}

extern "C" int ms_bf_helper_columns(ms_ctx *c, const void *base, size_t n, void *aux) {
    if (!c || !base || !aux) return MS_ERR_INVALID;
    if (n == 0) return MS_OK;
    Staged B(c, base, 17 * n * 8, true, false);
    if (B.rc) return B.rc;
    Staged A(c, aux, 8 * n * 8, false, true);
    if (A.rc) return A.rc;
    bf_helper_kernel<<<blocks(n, 256), 256, 0, c->stream>>>(B.as<u64>(), n, A.as<u64>());
    c->launches++;
    MS_CHECK_LAUNCH(c);
    int rc = B.finish();
    return rc ? rc : A.finish();
}
