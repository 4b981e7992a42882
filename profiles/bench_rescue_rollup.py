#!/usr/bin/env python
"""examples/rollup: K balance transfers over a Rescue-Prime account tree, proved from the old root to the new one, with
the balances resolved and the trace built on the GPU.

    profiles/bench_rescue_rollup.py [--shapes 16:14,24:13] [--reps 5] [--out-dir profiles]

Each shape is depth D : log2 K; the defaults are D = 16 with 2^14 transfers and D = 24 with 2^13, whose 2 K writes
are the (K, D) of the updates benchmark (profiles/bench_rescue_merkle_updates.py), so both traces have n = 2^23 rows.
Per shape:
  * rollup kernel: ms_rescue_rollup alone (heap copy, transfers, trace and roots in device memory), timed by CUDA
    events after one warm-up, minimum of --reps calls, each from a fresh copy of the heap made outside the timed region.
    The call synchronises twice (its argument and balance checks), so the events span those too;
  * updates kernel: ms_rescue_merkle_updates on the same 2 K writes (the accounts and new leaves the rollup makes), in
    the same run and timed the same way: the part of the rollup kernel that hashes the paths;
  * rollup kernel split: torch.profiler's device time of one call, per kernel name: the balance resolution (the check,
    the radix sort by account, the gather, the segmented scan and the resolve), the updates part and the column fill.
    The resolution's and the updates' cub kernels share names, so resolution = the rollup call's kernels minus one
    updates call's, per name;
  * apply(): rollup.apply(device=...) wall time up to a device synchronise;
  * prove: GpuProver from the device trace, one warm-up, then --reps proofs; wall time, proof.timings per phase and the
    torch peak of the fastest;
  * verify: Stark.verify of the proof on the host;
  * the card name, power limit and SM clock limit are read in the same run (nvidia-smi, read-only query).
One JSON line per arm on stdout; writes <out-dir>/bench_rescue_rollup_2p23_h100.json (2p<log n> for other shapes)."""
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
from bench_rescue_merkle_updates import _events
from make_rescue_rollup_golden import accounts, transfers
from ministark_b200.examples import merkle as M
from ministark_b200.examples import rescue as R
from ministark_b200.examples import rollup as RL
from ministark_b200.prover import GpuProver

SEED = 5


def _profile(fn):
    """{kernel name: device seconds} of one call of fn under torch.profiler"""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if t:
            out[ev.key[:100]] = out.get(ev.key[:100], 0.0) + t / 1e6
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="16:14,24:13", help="comma-separated depth : log2 K pairs")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    shapes = [tuple(int(v) for v in s.split(":")) for s in args.shapes.split(",")]
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = dict(card(), options=list(vars(RL.OPTIONS).values()),
               timing="kernels: CUDA events; split: torch.profiler device time; apply(), prove, verify: wall clock up "
                      "to a device synchronise; seconds",
               shapes=[])
    for depth, log_k in shapes:
        K = 1 << log_k
        L = 1 << (depth - 1).bit_length()
        n = 32 * K * L
        log_n = n.bit_length() - 1
        shape = {"depth": depth, "K": K, "L": L, "log_n": log_n, "arms": []}
        res["shapes"].append(shape)

        def emit(a):
            shape["arms"].append(a)
            print(json.dumps(dict(a, card=res["card"], power_limit=res["power_limit"], depth=depth, K=K, log_n=log_n)),
                  flush=True)

        lv = accounts(depth, SEED)
        txs = transfers(lv, depth, K, SEED)
        nodes = M.tree(lv, device=0)
        dtx = torch.from_numpy(np.array(txs, dtype=np.uint64).view(np.int64)).to(dev)
        heap = torch.empty_like(nodes)
        out = torch.empty((23, n), dtype=torch.int64, device=dev)
        roots = torch.empty((K + 1, 4), dtype=torch.int64, device=dev)
        stream = torch.cuda.Stream(dev)
        with torch.cuda.stream(stream):                         # the context queues on this stream, and the events too
            ctx = R._context(dev)
        torch.cuda.synchronize()
        rollup = lambda: ctx.rescue_rollup(heap, depth, dtx, K, out, roots)
        r, rs = _events(rollup, args.reps, ctx, stream, before=lambda: heap.copy_(nodes))
        emit({"arm": "rollup_kernel", "kernel_s_min": r, "kernel_s_all": rs, "writes": 2 * K,
              "permutations": 4 * K * L})
        # the same 2 K writes for the updates kernel alone: accounts, and the new leaves as the rollup trace holds them
        heap.copy_(nodes)
        rollup()
        ctx.sync()
        w_idx = torch.from_numpy(np.array([a for s, d, _ in txs for a in (s, d)], dtype=np.uint64).view(np.int64)).to(dev)
        starts = torch.arange(0, n, 16 * L, device=dev)
        new_path = out[:8, starts + 8 * L].T.contiguous().cpu().numpy().view(np.uint64)     # new paths' first rows
        bits = (w_idx & 1).cpu().numpy().astype(bool)
        mont = np.where(bits[:, None], new_path[:, 4:8], new_path[:, :4])
        inv = pow(2**64, -1, RL.P)
        w_new = np.array([[int(v) * inv % RL.P for v in row] for row in mont], dtype=np.uint64)
        dnew = torch.from_numpy(w_new.view(np.int64)).to(dev)
        uout = torch.empty((15, n), dtype=torch.int64, device=dev)
        uroots = torch.empty((2 * K + 1, 4), dtype=torch.int64, device=dev)
        updates = lambda: ctx.rescue_merkle_updates(heap, depth, w_idx, dnew, 2 * K, uout, uroots)
        u, us = _events(updates, args.reps, ctx, stream, before=lambda: heap.copy_(nodes))
        heap.copy_(nodes)
        updates()
        ctx.sync()
        assert torch.equal(uout, out[:15]), "the updates kernel on the rollup's writes gives the rollup's columns 0..14"
        emit({"arm": "updates_kernel_same_writes", "kernel_s_min": u, "kernel_s_all": us, "writes": 2 * K})
        heap.copy_(nodes)
        whole = _profile(lambda: (rollup(), ctx.sync()))
        heap.copy_(nodes)
        upd = _profile(lambda: (updates(), ctx.sync()))
        fill = sum(t for k, t in whole.items() if "rollup_fill_kernel" in k)
        resolution = {k: t - upd.get(k, 0.0) for k, t in whole.items() if "rollup_fill_kernel" not in k}
        emit({"arm": "rollup_kernel_split", "device_s": {"balance_resolution": sum(resolution.values()),
                                                          "updates": sum(upd.values()), "column_fill": fill},
              "balance_resolution_by_kernel": resolution, "rollup_device_s_by_kernel": whole,
              "updates_device_s_by_kernel": upd,
              "resolution_over_updates_permutations": sum(resolution.values()) / sum(
                  t for k, t in upd.items() if "rescue_merkle_update_kernel" in k),
              "timing": "torch.profiler device time of one call, summed per kernel name"})
        del out, uout, heap, roots, uroots
        torch.cuda.empty_cache()
        times = []
        for _ in range(args.reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            trace, new_nodes, rts = RL.apply(nodes, depth, txs, device=0)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            del trace, new_nodes
        emit({"arm": "apply", "apply_s_min": min(times[1:]), "apply_s_all": times[1:]})
        trace, new_nodes, rts = RL.apply(nodes, depth, txs, device=0)
        assert rts[-1] == M.root(new_nodes)
        del new_nodes
        claim = RL.TransfersClaim(depth, rts[0], rts[-1], txs)
        p = GpuProver.shared(0)
        p.prove(claim, RL.OPTIONS, trace)
        runs = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            t0 = time.perf_counter()
            proof = p.prove(claim, RL.OPTIONS, trace)
            runs.append({"prove_s": time.perf_counter() - t0, "timings": proof.timings, "residency": p.last_residency,
                         "torch_peak_bytes": torch.cuda.max_memory_allocated(dev)})
        best = min(runs, key=lambda r: r["prove_s"])
        blob = proof.to_bytes()
        emit({"arm": "prove_1gpu", "prove_s_min": best["prove_s"], "prove_s_all": [r["prove_s"] for r in runs],
              "timings_of_min": best["timings"], "residency": best["residency"],
              "torch_peak_bytes": best["torch_peak_bytes"], "proof_bytes": len(blob)})
        t0 = time.perf_counter()
        claim.verify(blob, RL.SECURITY_LEVEL)
        emit({"arm": "verify", "verify_s": time.perf_counter() - t0})
        del trace, nodes, dtx
        torch.cuda.empty_cache()
    log_ns = sorted({s["log_n"] for s in res["shapes"]})
    name = f"bench_rescue_rollup_2p{'_'.join(map(str, log_ns))}_h100.json"
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, name), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
