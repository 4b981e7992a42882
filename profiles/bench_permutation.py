#!/usr/bin/env python
"""What filling a permutation's target columns on the device costs (csrc/permutation.cu, ms_permutation_fill), against a
host numpy lexsort plus upload of the same tuples, and what share of a proof it takes.

    profiles/bench_permutation.py [--sizes 20 24] [--reps 10] [--out-dir profiles]

  * kernel: W = 1, 2, 3, 4 source words, each a plain base column (words 0 and 2 of 62 random bits, words 1 and 3 of a
    few values, so long runs share their leading words); ms_permutation_fill timed with CUDA events, minimum of --reps
    calls after two warm-up calls;
  * in the same run, the host route on the same canonical tuples: np.lexsort, the gather, the Montgomery conversion and
    the upload of the W target columns (wall clock ending in a synchronise); its words must equal the kernel's;
  * examples/memory's MemoryDeclaredClaim proves from a device trace (gen_trace(n, n / 16, device=0)),
    ProofOptions(16, 8, 4, 4, 8): one warm-up, then two proofs; timings["permutation_fill"] beside the whole prove, and the
    host route for its four-word tuple;
  * the card name and power limit are read in the same run (nvidia-smi, read-only query).
One JSON file per size: <out-dir>/bench_permutation_2p<log_n>_h100.json, and one JSON line per size on stdout."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import ministark_b200 as ms
from ministark_b200 import expr as E
from ministark_b200.air import ProofOptions
from ministark_b200.examples import memory as MM
from ministark_b200.examples.lookup import _to_mont
from ministark_b200.prover import GpuProver

P = E.P
T = E.Trace


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (v.strip() for v in out.split(",", 1))
        return name, limit
    except Exception as e:
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def host_route(words):
    """words (W, n) canonical uint64 below 2^62 -> the (W, n) target words on the device, and the wall seconds"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    order = np.lexsort(words[::-1])
    out = torch.from_numpy(_to_mont(words[:, order]).view(np.int64)).cuda()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def bench_kernel(ctx, stream, W, log_n, reps):
    n = 1 << log_n
    rng = np.random.default_rng(W + log_n)
    canon = np.stack([rng.integers(0, hi, size=n, dtype=np.uint64) for hi in (1 << 62, 5, 1 << 62, 3)[:W]])
    base = torch.from_numpy(_to_mont(canon).view(np.int64)).cuda()
    prog = E.compile_lookup_program(tuple(T(k) for k in range(W)), (), None, W, log_n)
    work = torch.empty(ctx.permutation_workspace_bytes(log_n, W), dtype=torch.uint8, device="cuda")
    out = torch.empty((W, n), dtype=torch.int64, device="cuda")
    cols, targets = [base[c] for c in range(W)], [out[k] for k in range(W)]
    torch.cuda.synchronize()
    times = []
    for k in range(reps + 2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)                # the fill is asynchronous on the context's stream: time it there
        ctx.permutation_fill(prog, targets, log_n, cols, W, work)
        b.record(stream)
        b.synchronize()
        if k >= 2:
            times.append(a.elapsed_time(b) / 1e3)
    want, t_host = host_route(canon)
    same = bool(torch.equal(out, want))
    assert same, "the kernel and the host route disagree"
    return {"kernel_s_min": min(times), "kernel_s_all": times, "host_lexsort_upload_s": t_host, "identical_words": same,
            "workspace_bytes": work.numel(), "width": W}


def bench_prove(ctx, log_n):
    n = 1 << log_n
    opts = ProofOptions(16, 8, 4, 4, 8)
    trace, reads = MM.MemoryDeclaredClaim.gen_trace(n, n // 16, seed=1, device=0)
    p, claim = GpuProver.shared(0), MM.MemoryDeclaredClaim(reads)
    p.prove(claim, opts, trace)
    runs = []
    for _ in range(2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        proof = p.prove(claim, opts, trace)
        wall = time.perf_counter() - t0
        runs.append({"prove_s": wall, "permutation_fill_s": proof.timings["permutation_fill"],
                     "lookup_multiplicities_s": proof.timings["lookup_multiplicities"], "timings": proof.timings,
                     "residency": p.last_residency})
    # the host route for the same (addr, clk, val, w) tuples: the log's canonical words (a Montgomery product with the
    # word 1), read back, sorted, converted and uploaded
    log = torch.stack([trace.base_columns()[c] for c in MM.LOG]).contiguous()
    ctx.pointwise_const("mul", log, ms.FP, log, ms.FP, [1], ms.FP, log.numel())
    torch.cuda.synchronize()
    _, t_host = host_route(log.cpu().numpy().view(np.uint64))
    return {"proofs": runs, "host_lexsort_upload_s": t_host, "rows": n, "addresses": n // 16, "reads": len(reads)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[20, 24])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    name, limit = card()
    stream = torch.cuda.Stream()
    ctx = ms.Context(0, stream=stream.cuda_stream)
    for log_n in args.sizes:
        res = {"card": name, "power_limit": limit, "log_n": log_n, "timing": "kernels: CUDA events, seconds; prove: wall",
               "kernels": {f"W{W}": bench_kernel(ctx, stream, W, log_n, args.reps) for W in (1, 2, 3, 4)},
               "memory_prove": bench_prove(ctx, log_n)}
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, f"bench_permutation_2p{log_n}_h100.json"), "w") as f:
            json.dump(res, f, indent=1)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
