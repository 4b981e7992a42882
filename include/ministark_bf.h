/*
 * ministark_bf.h — the execution trace of examples/brainfuck built natively: the VM run on the host, every table of the
 * trace on the device.  Conventions as in ministark_b200.h (Montgomery words, column-major matrices, 0 on success, a
 * negative MS_ERR_* otherwise; pointers may be device or host memory unless a comment says otherwise).
 *
 * The reference runs the VM and builds the tables in one sequential pass (examples/brainfuck/vm.rs:68-381); here only the
 * VM loop is sequential.  It writes one 8-byte record per processor row, and the tables are data-parallel functions of
 * those records and the program: a pointwise gather (processor), a histogram of ip (instruction), a stable sort by
 * memory pointer plus dummy rows for cycle gaps (memory) and two stream compactions (input / output).
 *
 * A record packs the state at the start of a cycle: bits 0-31 ip, bits 32-47 mp, bits 48-55 mem_val = tape[mp].
 * A run of c cycles has c + 1 records; the last one is the final state, ip == program length.
 */
#ifndef MINISTARK_BF_H
#define MINISTARK_BF_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* entries of the `sizes` array of ms_bf_trace_sizes */
#define MS_BF_PROC_ROWS 0   /* processor rows P = cycles + 1 */
#define MS_BF_INSTR_ROWS 1  /* instruction rows: program length + P */
#define MS_BF_MEM_ROWS 2    /* memory rows, dummy rows included */
#define MS_BF_READS 3       /* input table rows */
#define MS_BF_WRITES 4      /* output table rows */
#define MS_BF_N 5           /* trace length: the longest table, rounded up to a power of two */
#define MS_BF_WORK_BYTES 6  /* device workspace ms_bf_trace_fill needs */
#define MS_BF_NSIZES 7

/* Runs the compiled program (examples/brainfuck/vm.rs:68-336; ministark_b200/examples/brainfuck.py::compile_program:
 * opcodes as ASCII, each '[' and ']' followed by its jump target) on a 1024-cell u8 tape that wraps on '+' and '-'.
 * Host memory only; takes no context and touches no device.  log: room for max_cycles + 1 records; output: room for
 * max_cycles bytes.  counts[0] receives the number of cycles (log holds counts[0] + 1 records), counts[1] the number of
 * output bytes.  Fails with MS_ERR_INVALID when the memory pointer would leave [0, 1024), when ',' finds the input
 * exhausted, when max_cycles cycles have run and the program has not halted, and on a malformed program; the message is
 * ms_last_error(NULL) on the calling thread until its next ms_bf_run call ("null context" after a success). */
int ms_bf_run(const uint32_t *program, size_t program_len, const uint8_t *input, size_t input_len, uint64_t max_cycles,
              uint64_t *log, uint8_t *output, uint64_t *counts);

/* Phase 1 of the tables: checks the nrec records of `log` against the program and computes the table lengths on the
 * device; sizes: host array of MS_BF_NSIZES entries (MS_BF_*).  Synchronises the context's stream once. */
int ms_bf_trace_sizes(ms_ctx *ctx, const uint32_t *program, size_t program_len, const uint64_t *log, size_t nrec,
                      uint64_t *sizes);

/* Phase 2: fills `out`, the (17, n) column-major matrix of Montgomery words of BrainfuckTrace.base_columns(), from the
 * same program and log; sizes: what ms_bf_trace_sizes returned for them; work: device memory of sizes[MS_BF_WORK_BYTES]
 * bytes, free again when the stream reaches the end of this call.  Does not synchronise. */
int ms_bf_trace_fill(ms_ctx *ctx, const uint32_t *program, size_t program_len, const uint64_t *log, size_t nrec,
                     const uint64_t *sizes, void *work, void *out);

/* The eight 0/1 helper columns of BrainfuckTrace.helper_columns() (Montgomery words, (8, n) column-major in `aux`) from
 * a filled (17, n) base matrix: processor row is real, READ and its next mem_val, WRITE and its next mem_val, memory row
 * is real, instruction permutation advances, program evaluation advances.  Does not synchronise. */
int ms_bf_helper_columns(ms_ctx *ctx, const void *base, size_t n, void *aux);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_BF_H */
