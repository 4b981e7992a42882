#!/usr/bin/env python
"""examples/merkle: K ordered leaf writes into a Rescue-Prime Merkle tree, proved from the old root to the new one, with
the update trace built on the GPU.

    profiles/bench_rescue_merkle_updates.py [--shapes 16:15,24:14] [--reps 5] [--out-dir profiles]

Each shape is depth D : log2 K; the defaults are D = 16 with 2^15 writes (L = 16) and D = 24 with 2^14 writes (L = 32,
a 2^24-leaf tree), the (K, D) of the paths benchmark (profiles/bench_rescue_merkle.py).  The write trace holds two
paths per write, so it has n = 16 K L = 2^23 rows at both shapes.  Per shape:
  * update kernel: ms_rescue_merkle_updates alone (heap copy, indices, new leaves, trace and roots in device memory),
    timed by CUDA events after one warm-up, minimum of --reps calls; each call starts from a fresh copy of the heap,
    made outside the timed region.  The call synchronises once (its argument check), so the events span that too;
  * update kernel split: torch.profiler's device time of one call, per kernel name and summed into the permutation
    launches, the radix sorts, the max-scans and the rest (key and mark fills, resolves, check, scatter, copies);
  * paths kernel: ms_rescue_merkle_paths on the same (K, D) in the same run, timed the same way, for context (K L
    permutations, against the update's 2 K L and its per-level sorts);
  * update(): merkle.update(device=...) wall time up to a device synchronise (heap copy, uploads, kernel, roots);
  * prove: GpuProver from the device trace, one warm-up, then --reps proofs; wall time, proof.timings per phase and the
    torch peak of the fastest;
  * verify: Stark.verify of the proof on the host;
  * the card name, power limit and SM clock limit are read in the same run (nvidia-smi, read-only query).
One JSON line per arm on stdout; writes <out-dir>/bench_rescue_merkle_updates_2p23_h100.json (2p<log n> for other
shapes)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import numpy as np
import torch

from bench_rescue import card
from make_rescue_merkle_golden import leaves
from make_rescue_merkle_updates_golden import writes
from ministark_b200.examples import merkle as M
from ministark_b200.examples import rescue as R
from ministark_b200.prover import GpuProver

SEED = 5


def _events(fn, reps, ctx, stream, before=None):
    """minimum and all of --reps CUDA-event timings of fn() on `stream`, the context's, after one warm-up"""
    if before:
        before()
    fn()
    ctx.sync()
    times = []
    for _ in range(reps):
        if before:
            before()
        torch.cuda.synchronize()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record(stream)
        fn()
        stop.record(stream)
        stop.synchronize()
        times.append(start.elapsed_time(stop) / 1e3)
    return min(times), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="16:15,24:14", help="comma-separated depth : log2 K pairs")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    shapes = [tuple(int(v) for v in s.split(":")) for s in args.shapes.split(",")]
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = dict(card(), options=list(vars(M.OPTIONS).values()),
               timing="kernels: CUDA events; update(), prove, verify: wall clock up to a device synchronise; seconds",
               shapes=[])
    for depth, log_k in shapes:
        K = 1 << log_k
        L = 1 << (depth - 1).bit_length()
        log_n = (16 * K * L).bit_length() - 1
        shape = {"depth": depth, "K": K, "L": L, "log_n": log_n, "arms": []}
        res["shapes"].append(shape)

        def emit(a):
            shape["arms"].append(a)
            print(json.dumps(dict(a, card=res["card"], power_limit=res["power_limit"], depth=depth, K=K, log_n=log_n)),
                  flush=True)

        nodes = M.tree(leaves(depth, SEED), device=0)
        idx, new = writes(K, depth, SEED)
        didx = torch.from_numpy(idx.view(np.int64)).to(dev)
        dnew = torch.from_numpy(new.view(np.int64)).to(dev)
        heap = torch.empty_like(nodes)
        out = torch.empty((15, 16 * K * L), dtype=torch.int64, device=dev)
        roots = torch.empty((K + 1, 4), dtype=torch.int64, device=dev)
        stream = torch.cuda.Stream(dev)
        with torch.cuda.stream(stream):                         # the context queues on this stream, and the events too
            ctx = R._context(dev)
        torch.cuda.synchronize()
        u, us = _events(lambda: ctx.rescue_merkle_updates(heap, depth, didx, dnew, K, out, roots), args.reps, ctx,
                        stream, before=lambda: heap.copy_(nodes))
        emit({"arm": "update_kernel", "kernel_s_min": u, "kernel_s_all": us, "permutations": 2 * K * L,
              "permutations_per_s": 2 * K * L / u, "sort_levels": depth})
        heap.copy_(nodes)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            ctx.rescue_merkle_updates(heap, depth, didx, dnew, K, out, roots)
            ctx.sync()
        split, kernels = {"permutations": 0.0, "radix_sort": 0.0, "scan": 0.0, "other": 0.0}, {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            if not t:
                continue
            kernels[ev.key[:100]] = t / 1e6
            part = ("permutations" if "rescue_merkle_update_kernel" in ev.key else "radix_sort" if "RadixSort" in ev.key
                    else "scan" if "Scan" in ev.key else "other")
            split[part] += t / 1e6
        emit({"arm": "update_kernel_split", "device_s": split, "device_s_by_kernel": kernels,
              "timing": "torch.profiler device time of one call, summed per kernel name"})
        del out
        pout = torch.empty((14, 8 * K * L), dtype=torch.int64, device=dev)
        k, ks = _events(lambda: ctx.rescue_merkle_paths(nodes, depth, didx, K, pout), args.reps, ctx, stream)
        emit({"arm": "paths_kernel", "kernel_s_min": k, "kernel_s_all": ks, "permutations": K * L,
              "permutations_per_s": K * L / k})
        del pout, heap, roots
        torch.cuda.empty_cache()
        times = []
        for _ in range(args.reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            trace, new_nodes, rts = M.update(nodes, depth, idx, new, device=0)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            del trace, new_nodes
        emit({"arm": "update", "update_s_min": min(times[1:]), "update_s_all": times[1:]})
        trace, new_nodes, rts = M.update(nodes, depth, idx, new, device=0)
        assert rts[-1] == M.root(new_nodes)
        del new_nodes
        claim = M.MerkleUpdatesClaim(depth, rts[0], rts[-1], idx, new)
        p = GpuProver.shared(0)
        p.prove(claim, M.OPTIONS, trace)
        runs = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            t0 = time.perf_counter()
            proof = p.prove(claim, M.OPTIONS, trace)
            runs.append({"prove_s": time.perf_counter() - t0, "timings": proof.timings, "residency": p.last_residency,
                         "torch_peak_bytes": torch.cuda.max_memory_allocated(dev)})
        best = min(runs, key=lambda r: r["prove_s"])
        blob = proof.to_bytes()
        emit({"arm": "prove_1gpu", "prove_s_min": best["prove_s"], "prove_s_all": [r["prove_s"] for r in runs],
              "timings_of_min": best["timings"], "residency": best["residency"],
              "torch_peak_bytes": best["torch_peak_bytes"], "proof_bytes": len(blob)})
        t0 = time.perf_counter()
        claim.verify(blob, M.SECURITY_LEVEL)
        emit({"arm": "verify", "verify_s": time.perf_counter() - t0})
        del trace, nodes, didx, dnew
        torch.cuda.empty_cache()
    log_ns = sorted({s["log_n"] for s in res["shapes"]})
    name = f"bench_rescue_merkle_updates_2p{'_'.join(map(str, log_ns))}_h100.json"
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, name), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
