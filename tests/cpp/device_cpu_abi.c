/*
 * device_cpu_abi.c — CPU build of include/ministark_device.h.  TEST INFRASTRUCTURE ONLY, compiled by
 * tests/test_cpp_stream_prover_cpu.py into a temporary directory.
 *
 * The CPU build of the brainfuck trace entry points (tests/cpp/bf_trace_cpu_abi.c, itself the oracle's CPU ABI plus the
 * streamed residency and the constraint check) is extended by ms_device_memory, so that the C++ prover and the brainfuck
 * command line link and run end to end without a GPU.  The product never loads this library.
 */
#include <stdint.h>

#include "bf_trace_cpu_abi.c"
#include "../../include/ministark_device.h"

/* "unlimited": off a GPU only an explicit memory budget limits a proof */
int ms_device_memory(ms_ctx *c, size_t *free_bytes, size_t *total_bytes) {
    if (!c) return MS_ERR_INVALID;
    if (free_bytes) *free_bytes = SIZE_MAX;
    if (total_bytes) *total_bytes = SIZE_MAX;
    return MS_OK;
}
