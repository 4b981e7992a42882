/*
 * ministark_device.h — what a host needs to know about the device a context runs on before it sizes a proof.
 * Conventions as in ministark_b200.h (0 on success, a negative MS_ERR_* otherwise).
 *
 * The reference has no counterpart: its prover allocates unified memory and lets the driver page.
 */
#ifndef MINISTARK_DEVICE_H
#define MINISTARK_DEVICE_H
#include "ministark_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* free and total memory of the context's device in bytes (cudaMemGetInfo on that device), as the driver reports them at
 * the moment of the call: allocations of every process on the device count, and work still queued on the context's
 * stream does not (nothing is synchronised).  Either pointer may be NULL. */
int ms_device_memory(ms_ctx *ctx, size_t *free_bytes, size_t *total_bytes);

#ifdef __cplusplus
}
#endif
#endif /* MINISTARK_DEVICE_H */
