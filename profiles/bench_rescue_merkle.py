#!/usr/bin/env python
"""examples/merkle: a Rescue-Prime Merkle tree and K authentication paths through it, proved against the root, with the
tree and the trace built on the GPU.

    profiles/bench_rescue_merkle.py [--shapes 16:15,24:14] [--reps 5] [--out-dir profiles]

Each shape is depth D : log2 K; the defaults are the two 2^22-row shapes (D = 16 with 2^15 paths, L = 16; D = 24 with
2^14 paths, L = 32, a 2^24-leaf tree).  Per shape:
  * tree: ms_rescue_merkle_tree on leaves already in device memory, timed by the host clock up to a device synchronise;
    minimum of --reps calls after one warm-up; reported as time and as permutations (2^D - 1 nodes) per second;
  * trace: ms_rescue_merkle_paths alone (heap and indices in device memory) and gen_trace(device=...) (index upload,
    the index check, kernel, leaf read-back), same timing;
  * prove: GpuProver from the device trace, one warm-up, then --reps proofs; wall time and proof.timings per phase;
  * verify: Stark.verify of the proof on the host;
  * the card name, power limit and SM clock limit are read in the same run (nvidia-smi, read-only query).
One JSON line per arm on stdout; writes <out-dir>/bench_rescue_merkle_2p22_h100.json (2p<log n> for other shapes)."""
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
from make_rescue_merkle_golden import indices, leaves
from ministark_b200.examples import merkle as M
from ministark_b200.examples import rescue as R
from ministark_b200.prover import GpuProver

SEED = 5


def _best(fn, reps, sync):
    fn()                                                        # warm-up
    times = []
    for _ in range(reps):
        sync()
        t0 = time.perf_counter()
        fn()
        sync()
        times.append(time.perf_counter() - t0)
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
    res = dict(card(), options=list(vars(M.OPTIONS).values()), timing="wall clock up to a device synchronise, seconds",
               shapes=[])
    for depth, log_k in shapes:
        K = 1 << log_k
        L = 1 << (depth - 1).bit_length()
        log_n = (8 * K * L).bit_length() - 1
        shape = {"depth": depth, "K": K, "L": L, "log_n": log_n, "arms": []}
        res["shapes"].append(shape)

        def emit(a):
            shape["arms"].append(a)
            print(json.dumps(dict(a, card=res["card"], power_limit=res["power_limit"], depth=depth, K=K, log_n=log_n)),
                  flush=True)

        ctx = R._context(dev)
        lv = torch.from_numpy(leaves(depth, SEED).view(np.int64)).to(dev)
        idx = indices(K, depth, SEED)
        nodes = torch.empty((2 << depth, 4), dtype=torch.int64, device=dev)
        t, ts = _best(lambda: ctx.rescue_merkle_tree(lv, depth, nodes), args.reps, ctx.sync)
        perms = (1 << depth) - 1
        emit({"arm": "tree", "kernel_s_min": t, "kernel_s_all": ts, "permutations": perms, "permutations_per_s": perms / t,
              "launches": max(depth - 6, 0) + 1})
        out = torch.empty((14, 8 * K * L), dtype=torch.int64, device=dev)
        didx = torch.from_numpy(idx.view(np.int64)).to(dev)
        k, ks = _best(lambda: ctx.rescue_merkle_paths(nodes, depth, didx, K, out), args.reps, ctx.sync)
        g, gs = _best(lambda: M.gen_trace(nodes, depth, idx, device=0), args.reps, torch.cuda.synchronize)
        emit({"arm": "trace", "kernel_s_min": k, "kernel_s_all": ks, "permutations": K * L,
              "permutations_per_s": K * L / k, "gen_trace_s_min": g, "gen_trace_s_all": gs})
        del out
        trace, lvs = M.gen_trace(nodes, depth, idx, device=0)
        claim = M.MerklePathsClaim(depth, M.root(nodes), lvs, idx)
        p = GpuProver.shared(0)
        p.prove(claim, M.OPTIONS, trace)
        runs = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            proof = p.prove(claim, M.OPTIONS, trace)
            runs.append({"prove_s": time.perf_counter() - t0, "timings": proof.timings, "residency": p.last_residency})
        best = min(runs, key=lambda r: r["prove_s"])
        blob = proof.to_bytes()
        emit({"arm": "prove_1gpu", "prove_s_min": best["prove_s"], "prove_s_all": [r["prove_s"] for r in runs],
              "timings_of_min": best["timings"], "residency": best["residency"], "proof_bytes": len(blob)})
        t0 = time.perf_counter()
        claim.verify(blob, M.SECURITY_LEVEL)
        emit({"arm": "verify", "verify_s": time.perf_counter() - t0})
        del trace, nodes, lv
        torch.cuda.empty_cache()
    log_ns = sorted({s["log_n"] for s in res["shapes"]})
    name = f"bench_rescue_merkle_2p{'_'.join(map(str, log_ns))}_h100.json"
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, name), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
