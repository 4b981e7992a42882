/*
 * bf_trace_cpu_abi.c — CPU build of the brainfuck trace entry points (include/ministark_bf.h).  TEST INFRASTRUCTURE ONLY,
 * compiled by tests/test_bf_trace_cpu.py into a temporary directory.
 *
 * The CPU build of the constraint check (tests/cpp/check_cpu_abi.c, itself the oracle's CPU ABI plus the streamed
 * residency) is extended by ms_bf_run and the table entry points, so that `simulate(..., device=...)` and whole proofs
 * from its trace run on the CPU harness (tests/cpu_device.py).  The tables are built the way the reference builds them
 * (examples/brainfuck/vm.rs:338-381): rows appended in order, the memory rows sorted by (mp, cycle), dummy rows inserted
 * between accesses of one address.  The product never loads this library.
 */
#define ms_last_error ms_last_error_of_context
#include "check_cpu_abi.c"
#undef ms_last_error
#include "../../include/ministark_bf.h"

static _Thread_local char bf_err[512] = "no context";

/* the oracle ABI keeps messages in the context; ms_bf_run has none */
const char *ms_last_error(ms_ctx *c) { return c ? ms_last_error_of_context(c) : bf_err; }

static int bf_fail(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(bf_err, sizeof bf_err, fmt, ap);
    va_end(ap);
    return MS_ERR_INVALID;
}

#define BF_MONT(v) ((u64)(v) * 0xFFFFFFFFull)
enum { BF_TAPE = 1024 };

int ms_bf_run(const uint32_t *prog, size_t len, const uint8_t *input, size_t input_len, uint64_t max_cycles, uint64_t *log,
              uint8_t *output, uint64_t *counts) {
    snprintf(bf_err, sizeof bf_err, "no context");
    if (!prog || !log || !counts || len == 0) return bf_fail("ms_bf_run: bad argument");
    uint8_t tape[BF_TAPE] = {0};
    u64 ip = 0, mp = 0, cycle = 0, nout = 0, in = 0;
    for (; ip < len; cycle++) {
        if (cycle == max_cycles) return bf_fail("ms_bf_run: cycle cap %llu reached", (unsigned long long)max_cycles);
        log[cycle] = ip | mp << 32 | (u64)tape[mp] << 48;
        const uint32_t op = prog[ip];
        if (op == '[') ip = tape[mp] ? ip + 2 : prog[ip + 1];
        else if (op == ']') ip = tape[mp] ? prog[ip + 1] : ip + 2;
        else if (op == '<' || op == '>') {
            if (op == '<' ? mp == 0 : mp == BF_TAPE - 1) return bf_fail("ms_bf_run: memory pointer leaves the tape");
            mp = op == '<' ? mp - 1 : mp + 1;
            ip++;
        } else if (op == '+') { tape[mp]++; ip++; }
        else if (op == '-') { tape[mp]--; ip++; }
        else if (op == '.') { output[nout++] = tape[mp]; ip++; }
        else if (op == ',') {
            if (in == input_len) return bf_fail("ms_bf_run: input exhausted");
            tape[mp] = input[in++];
            ip++;
        } else return bf_fail("ms_bf_run: unrecognized instruction");
    }
    if (ip != len) return bf_fail("ms_bf_run: jump past the end");
    log[cycle] = ip | mp << 32 | (u64)tape[mp] << 48;
    counts[0] = cycle;
    counts[1] = nout;
    return MS_OK;
}

#define R_IP(r) ((u64)(uint32_t)(r))
#define R_MP(r) (((r) >> 32) & 0xFFFF)
#define R_VAL(r) (((r) >> 48) & 0xFF)

/* the memory table's real rows in (mp, cycle) order (a counting sort, stable), then with the dummy rows: returns the
 * number of rows; rows == NULL only counts them */
static u64 bf_memory_rows(const uint64_t *log, u64 C, u64 (*rows)[4]) {
    u64 start[BF_TAPE + 1] = {0};
    for (u64 i = 0; i < C; i++) start[R_MP(log[i]) + 1]++;
    for (int k = 0; k < BF_TAPE; k++) start[k + 1] += start[k];
    u64 *order = (u64 *)malloc(8 * (C ? C : 1));
    for (u64 i = 0; i < C; i++) order[start[R_MP(log[i])]++] = i;
    u64 m = 0;
    for (u64 j = 0; j < C; j++) {
        const u64 cy = order[j], mp = R_MP(log[cy]), v = R_VAL(log[cy]);
        if (rows) { rows[m][0] = cy; rows[m][1] = mp; rows[m][2] = v; rows[m][3] = 0; }
        m++;
        if (j + 1 < C && R_MP(log[order[j + 1]]) == mp)
            for (u64 d = cy + 1; d < order[j + 1]; d++, m++)
                if (rows) { rows[m][0] = d; rows[m][1] = mp; rows[m][2] = v; rows[m][3] = 1; }
    }
    free(order);
    return m;
}

int ms_bf_trace_sizes(ms_ctx *c, const uint32_t *prog, size_t L, const uint64_t *log, size_t nrec, uint64_t *sizes) {
    if (!c || !prog || !log || !sizes || L == 0 || nrec < 2) return MS_ERR_INVALID;
    u64 reads = 0, writes = 0;
    for (u64 i = 0; i + 1 < nrec; i++) {
        if (R_IP(log[i]) >= L || R_MP(log[i]) >= BF_TAPE) return fail(c, MS_ERR_INVALID, "ms_bf_trace_sizes: bad record %llu", (unsigned long long)i);
        reads += prog[R_IP(log[i])] == ',';
        writes += prog[R_IP(log[i])] == '.';
    }
    if (R_IP(log[nrec - 1]) != L) return fail(c, MS_ERR_INVALID, "ms_bf_trace_sizes: the last record is not a final state");
    const u64 M = bf_memory_rows(log, nrec - 1, NULL), longest = L + nrec > M ? L + nrec : M;
    u64 n = 1;
    while (n < longest) n <<= 1;
    sizes[MS_BF_PROC_ROWS] = nrec;
    sizes[MS_BF_INSTR_ROWS] = L + nrec;
    sizes[MS_BF_MEM_ROWS] = M;
    sizes[MS_BF_READS] = reads;
    sizes[MS_BF_WRITES] = writes;
    sizes[MS_BF_N] = n;
    sizes[MS_BF_WORK_BYTES] = 0;         /* the CPU build allocates its own */
    return MS_OK;
}

int ms_bf_trace_fill(ms_ctx *c, const uint32_t *prog, size_t L, const uint64_t *log, size_t nrec, const uint64_t *sizes,
                     void *work, void *out) {
    (void)work;
    if (!c || !prog || !log || !sizes || !out) return MS_ERR_INVALID;
    const u64 n = sizes[MS_BF_N], C = nrec - 1;
    u64 *o = (u64 *)out;
    #define COL(k, r) o[(u64)(k) * n + (r)]
    #define PROG(k) ((k) < L ? (u64)prog[k] : 0)
    /* processor: the records, then the final state repeated with the cycle counting on */
    for (u64 r = 0; r < n; r++) {
        const u64 rec = log[r < nrec ? r : nrec - 1], ip = R_IP(rec), mv = R_VAL(rec);
        const u64 curr = r < nrec ? PROG(ip) : 0, next = r < nrec ? PROG(ip + 1) : 0;
        COL(0, r) = BF_MONT(r); COL(1, r) = BF_MONT(ip); COL(2, r) = BF_MONT(curr); COL(3, r) = BF_MONT(next);
        COL(4, r) = BF_MONT(R_MP(rec)); COL(5, r) = BF_MONT(mv);
        COL(6, r) = mv ? fp_inv(BF_MONT(mv)) : 0;
        COL(7, r) = curr == 0 ? BF_MONT(1) : 0;
    }
    /* memory */
    const u64 M = sizes[MS_BF_MEM_ROWS];
    u64 (*mem)[4] = (u64 (*)[4])malloc(32 * (M ? M : 1));
    if (!mem) return fail(c, MS_ERR_NOMEM, "out of host memory");
    bf_memory_rows(log, C, mem);
    for (u64 r = 0; r < n; r++) {
        const u64 *m = mem[r < M ? r : M - 1], extra = r < M ? 0 : r - M + 1;
        COL(8, r) = BF_MONT(m[0] + extra); COL(9, r) = BF_MONT(m[1]); COL(10, r) = BF_MONT(m[2]);
        COL(11, r) = BF_MONT(r < M ? m[3] : 1);
    }
    free(mem);
    /* instruction: the program listing and the processor rows, stably sorted by ip (a counting sort), then (L, 0, 0) */
    u64 *start = (u64 *)calloc(L + 2, 8);
    for (u64 k = 0; k < L; k++) start[k + 1]++;
    for (u64 i = 0; i < nrec; i++) start[R_IP(log[i]) + 1]++;
    for (u64 k = 0; k <= L; k++) start[k + 1] += start[k];
    for (u64 k = 0; k <= L; k++)
        for (u64 r = start[k]; r < start[k + 1]; r++) {
            COL(12, r) = BF_MONT(k); COL(13, r) = BF_MONT(PROG(k)); COL(14, r) = BF_MONT(PROG(k + 1));
        }
    for (u64 r = start[L + 1]; r < n; r++) { COL(12, r) = BF_MONT(L); COL(13, r) = 0; COL(14, r) = 0; }
    free(start);
    /* input / output */
    u64 nin = 0, nout = 0;
    for (u64 r = 0; r < n; r++) COL(15, r) = COL(16, r) = 0;
    for (u64 i = 0; i < C; i++) {
        const u64 op = PROG(R_IP(log[i]));
        if (op == ',') { COL(15, nin) = BF_MONT(R_VAL(log[i + 1])); nin++; }
        if (op == '.') { COL(16, nout) = BF_MONT(R_VAL(log[i])); nout++; }
    }
    #undef COL
    #undef PROG
    return MS_OK;
}

int ms_bf_helper_columns(ms_ctx *c, const void *base, size_t n, void *aux) {
    if (!c || !base || !aux) return MS_ERR_INVALID;
    const u64 *b = (const u64 *)base, one = BF_MONT(1);
    u64 *a = (u64 *)aux;
    for (u64 r = 0; r < n; r++) {
        const u64 ci = b[2 * n + r], nmv = b[5 * n + (r + 1) % n], iip = b[12 * n + r], ici = b[13 * n + r];
        const int same = r > 0 && b[12 * n + r - 1] == iip;
        a[0 * n + r] = ci ? one : 0;
        a[1 * n + r] = ci == BF_MONT(',') ? one : 0;
        a[2 * n + r] = ci == BF_MONT(',') ? nmv : 0;
        a[3 * n + r] = ci == BF_MONT('.') ? one : 0;
        a[4 * n + r] = ci == BF_MONT('.') ? nmv : 0;
        a[5 * n + r] = b[11 * n + r] == 0 ? one : 0;
        a[6 * n + r] = ici && same ? one : 0;
        a[7 * n + r] = same ? 0 : one;
    }
    return MS_OK;
}
