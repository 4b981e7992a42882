#!/usr/bin/env python
"""examples/brainfuck: the execution trace built on the device against the host path.  One JSON line on stdout.

    profiles/bench_brainfuck_trace.py [--burner A B C] [--host]

  * the card name and power limit, read in the same run (nvidia-smi, read-only query);
  * the device path of `simulate(..., device=0)` split into the VM (ms_bf_run, host), the upload of the program and the
    records, and the two table phases (CUDA events, after a warm-up), plus the whole call; the table lengths;
  * the host `simulate` at the same size and the equality of the two traces, word for word: always up to 2^20 rows
    (about 9 s there), above that only with --host (about 2 minutes at 2^24);
  * source -> proof with the device trace (the default options), its residency, the torch peak of device memory over
    the proof and the proof's SHA-256."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import ministark_b200 as ms
from ministark_b200.examples import brainfuck as bf
from ministark_b200.prover import GpuProver


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (v.strip() for v in out.split(",", 1))
        return name, limit
    except Exception as e:          # the numbers still stand, but without their card they are incomplete
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def split_times(src, reps=3):
    """best of `reps`: VM, upload, sizes, fill.  Everything runs on one torch stream that the context also launches on, so
    the CUDA events around the two table phases bracket the device work itself."""
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    best = None
    with torch.cuda.stream(stream):
        for _ in range(reps + 1):                               # the first round warms up
            t = time.perf_counter()
            program = np.array(bf.compile_program(src), dtype=np.uint32)
            log, _ = ms.bf_run(program, b"")
            t_vm = time.perf_counter() - t
            stream.synchronize()
            t = time.perf_counter()
            d_prog = torch.from_numpy(program.view(np.int32)).to(dev)
            d_log = torch.from_numpy(log.view(np.int64)).to(dev)
            stream.synchronize()
            t_up = time.perf_counter() - t
            ctx = bf._context(dev)                              # queued on `stream`
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record(stream)
            sizes = ctx.bf_trace_sizes(d_prog, program.size, d_log, log.size)
            e[1].record(stream)
            base = torch.empty((17, sizes["n"]), dtype=torch.int64, device=dev)
            work = torch.empty(sizes["work_bytes"], dtype=torch.uint8, device=dev)
            ctx.bf_trace_fill(d_prog, program.size, d_log, log.size, sizes, work, base)
            e[2].record(stream)
            stream.synchronize()
            row = {"vm_s": t_vm, "upload_s": t_up, "sizes_s": e[0].elapsed_time(e[1]) / 1e3,
                   "fill_s": e[1].elapsed_time(e[2]) / 1e3}
            del base, work, d_log, d_prog
            best = row if best is None else {k: min(best[k], row[k]) for k in row}
    best["cycles"] = int(log.size - 1)
    best["work_mib"] = round(sizes["work_bytes"] / 2**20, 1)
    best["fill_GBps"] = round(17 * 8 * sizes["n"] / best["fill_s"] / 1e9, 1)     # the matrix written, per second
    return best, sizes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--burner", type=int, nargs=3, default=[40, 40, 60])
    ap.add_argument("--host", action="store_true", help="run the host simulate and compare above 2^20 rows too (about 2 min "
                    "at 2^24); up to 2^20 rows it always runs")
    args = ap.parse_args()
    name, power = card()
    a, b, c = args.burner
    src = bf.cycle_burner(a, b, c)
    res = {"bench": "brainfuck_trace", "gpu": name, "power_limit": power, "program": f"cycle_burner({a},{b},{c})"}
    res["device_split"], sizes = split_times(src)
    res["sizes"] = sizes
    walls = []
    for _ in range(3):
        torch.cuda.synchronize()
        t = time.perf_counter()
        trace, out = bf.simulate(src, device=0)
        walls.append(time.perf_counter() - t)
        del trace
    res["simulate_device_s"] = walls                          # the whole call, until the matrix is complete
    res["rows"] = sizes["n"]
    if args.host or sizes["n"] <= 1 << 20:
        t = time.perf_counter()
        host, out_h = bf.simulate(src)
        res["simulate_host_s"] = time.perf_counter() - t
        trace, out = bf.simulate(src, device=0)
        res["equal_to_host"] = bool(out == out_h and np.array_equal(trace.base_columns().cpu().numpy().view(np.uint64),
                                                                     host.base_columns()))
        del host, trace
    # source -> proof with the device trace (a warm-up proof first: AIR programs, plans, scratch)
    claim = bf.BrainfuckClaim(src, b"", out)
    prover = GpuProver(0)
    trace, _ = bf.simulate(src, device=0)
    prover.prove(claim, bf.OPTIONS, trace)
    del trace
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t = time.perf_counter()
    trace, _ = bf.simulate(src, device=0)
    t_sim = time.perf_counter() - t
    proof = prover.prove(claim, bf.OPTIONS, trace)
    torch.cuda.synchronize()
    res["source_to_proof_s"] = time.perf_counter() - t
    res["source_to_proof_simulate_s"] = t_sim
    res["residency"] = prover.last_residency
    res["torch_peak_gib"] = round(torch.cuda.max_memory_allocated() / 2**30, 2)
    res["budget_gib"] = round(prover.memory_available() / 2**30, 2)
    res["proof_sha256"] = hashlib.sha256(proof.to_bytes()).hexdigest()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
