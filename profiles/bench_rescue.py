#!/usr/bin/env python
"""BASELINE config 5: the examples/rescue proof (K chains of L Rescue-Prime permutations), trace built on the GPU.

    profiles/bench_rescue.py [--log-k 10] [--log-l 9] [--reps 5] [--out-dir profiles]
    torchrun --nproc-per-node N profiles/bench_rescue.py ...        # the ShardedProver arm on N GPUs

  * trace: gen_trace(device=...) (allocation, kernel, digest read-back) and ms_rescue_chains alone, each timed by the
    host clock up to a device synchronise; minimum of --reps calls after one warm-up;
    reported as time per trace and as microseconds per permutation round along one chain (kernel time / (7 L): the
    chains run side by side);
  * prove: GpuProver from the device trace, one warm-up, then --reps proofs; wall time and proof.timings per phase;
  * verify: Stark.verify of the proof on the host;
  * under torchrun (WORLD_SIZE > 1): ShardedProver on every rank, bytes checked against rank 0's single-GPU proof;
  * the card name, power limit and SM clock limit are read in the same run (nvidia-smi, read-only query).
One JSON line per arm on stdout; rank 0 writes <out-dir>/bench_rescue_2p<log_n>[_<N>gpu]_h100.json."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from ministark_b200.examples import rescue as R
from ministark_b200.prover import GpuProver

SEED = [3141592653589793238, 2718281828459045235, 1618033988749894848, 1414213562373095048]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit, clock = (v.strip() for v in out.split(","))
        return {"card": name, "power_limit": limit, "max_sm_clock": clock}
    except Exception as e:
        return {"card": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def bench_trace(K, L, reps, device):
    R.gen_trace(SEED, K, L, device=device)                      # warm-up: module load, context
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        trace, digests = R.gen_trace(SEED, K, L, device=device)     # returns after its own synchronise
        times.append(time.perf_counter() - t0)
    ctx = R._context(torch.device("cuda", device))
    out = trace.base_columns()
    kern = []
    for _ in range(reps):
        ctx.sync()
        t0 = time.perf_counter()
        ctx.rescue_chains(SEED, K, L, out)
        ctx.sync()                                              # the context's stream: ends in a device synchronise
        kern.append(time.perf_counter() - t0)
    k = min(kern)
    return trace, digests, {"arm": "trace", "gen_trace_s_min": min(times), "kernel_s_min": k, "kernel_s_all": kern,
                            "us_per_round": k / (7 * L) * 1e6, "permutations": K * L}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-k", type=int, default=10)
    ap.add_argument("--log-l", type=int, default=9)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    K, L = 1 << args.log_k, 1 << args.log_l
    log_n = args.log_k + args.log_l + 3
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    torch.cuda.set_device(rank)
    res = dict(card(), K=K, L=L, log_n=log_n, options=list(vars(R.OPTIONS).values()),
               timing="wall clock up to a device synchronise, seconds", arms=[])

    def emit(arm):
        res["arms"].append(arm)
        if rank == 0:
            print(json.dumps(dict(arm, card=res["card"], power_limit=res["power_limit"], log_n=log_n)), flush=True)

    trace, digests, arm = bench_trace(K, L, args.reps, rank)
    emit(arm)
    claim = R.RescueChainsClaim(SEED, K, L, digests)
    if world == 1:
        p = GpuProver.shared(0)
        p.prove(claim, R.OPTIONS, trace)
        runs = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            proof = p.prove(claim, R.OPTIONS, trace)
            runs.append({"prove_s": time.perf_counter() - t0, "timings": proof.timings, "residency": p.last_residency})
        best = min(runs, key=lambda r: r["prove_s"])
        emit({"arm": "prove_1gpu", "prove_s_min": best["prove_s"], "prove_s_all": [r["prove_s"] for r in runs],
              "timings_of_min": best["timings"], "residency": best["residency"], "proof_bytes": len(proof.to_bytes())})
        blob = proof.to_bytes()
        t0 = time.perf_counter()
        claim.verify(blob, R.SECURITY_LEVEL)
        emit({"arm": "verify", "verify_s": time.perf_counter() - t0})
        name = f"bench_rescue_2p{log_n}_h100.json"
    else:
        import torch.distributed as dist
        from ministark_b200.prover_mgpu import ShardedProver
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        try:
            sp = ShardedProver(dist, rank)
            sp.prove(claim, R.OPTIONS, trace)
            times = []
            for _ in range(args.reps):
                torch.cuda.synchronize()
                dist.barrier()
                t0 = time.perf_counter()
                proof = sp.prove(claim, R.OPTIONS, trace)
                times.append(time.perf_counter() - t0)
            single = GpuProver(rank).prove(claim, R.OPTIONS, trace).to_bytes() if rank == 0 else None
            if rank == 0:
                assert proof.to_bytes() == single, "sharded proof differs from the single-GPU proof"
            emit({"arm": f"prove_sharded_{world}gpu", "prove_s_min": min(times), "prove_s_all": times,
                  "timings": proof.timings, "identical_to_single_gpu": True})
        finally:
            dist.destroy_process_group()
        name = f"bench_rescue_2p{log_n}_{world}gpu_h100.json"
    if rank == 0:
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, name), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
