#!/usr/bin/env python
"""examples/rescue's hash claim: K messages hashed by the Rescue-Prime sponge and proved, trace built on the GPU.

    profiles/bench_rescue_hash.py [--shapes 16:60,19:4] [--reps 5] [--out-dir profiles]
    torchrun --nproc-per-node N profiles/bench_rescue_hash.py ...       # the ShardedProver arm on N GPUs

Each shape is log2 K : message length in words; the defaults are the two 2^22-row shapes (2^16 messages of 60 words,
8 permutations each; 2^19 messages of 4 words, one permutation each).  Per shape:
  * trace: gen_hash_trace(device=...) (allocation, message upload, kernel, digest read-back) and ms_rescue_hash alone on
    messages already in device memory, each timed by the host clock up to a device synchronise; minimum of --reps calls
    after one warm-up; reported as time per trace and as permutations per second (K L permutations, filler included);
  * prove: GpuProver from the device trace, one warm-up, then --reps proofs; wall time and proof.timings per phase;
  * verify: Stark.verify of the proof on the host;
  * under torchrun (WORLD_SIZE > 1): ShardedProver on every rank, bytes checked against rank 0's single-GPU proof;
  * the card name, power limit and SM clock limit are read in the same run (nvidia-smi, read-only query).
One JSON line per arm on stdout; rank 0 writes <out-dir>/bench_rescue_hash_2p22[_<N>gpu]_h100.json (2p<log n> when a
shape is not 2^22 rows)."""
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
from make_rescue_hash_golden import messages
from ministark_b200.examples import rescue as R
from ministark_b200.prover import GpuProver


def bench_trace(msgs, reps, device):
    K, length = msgs.shape
    R.gen_hash_trace(msgs, device=device)                       # warm-up: module load, context
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        trace, digests = R.gen_hash_trace(msgs, device=device)  # returns after its own synchronise
        times.append(time.perf_counter() - t0)
    ctx = R._context(torch.device("cuda", device))
    out = trace.base_columns()
    dmsgs = torch.from_numpy(msgs.view(np.int64)).to(out.device)
    torch.cuda.synchronize()
    kern = []
    for _ in range(reps):
        ctx.sync()
        t0 = time.perf_counter()
        ctx.rescue_hash(dmsgs, K, length, out)
        ctx.sync()                                              # the context's stream: ends in a device synchronise
        kern.append(time.perf_counter() - t0)
    k = min(kern)
    L = out.shape[1] // (8 * K)
    return trace, digests, {"arm": "trace", "gen_hash_trace_s_min": min(times), "kernel_s_min": k, "kernel_s_all": kern,
                            "permutations": K * L, "permutations_per_s": K * L / k,
                            "message_blocks": K * (length // 8 + 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="16:60,19:4", help="comma-separated log2 K : length pairs")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    shapes = [tuple(int(v) for v in s.split(":")) for s in args.shapes.split(",")]
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    torch.cuda.set_device(rank)
    res = dict(card(), options=list(vars(R.OPTIONS).values()), timing="wall clock up to a device synchronise, seconds",
               shapes=[])
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        for log_k, length in shapes:
            K = 1 << log_k
            msgs = messages(K, length)
            trace, digests, arm = bench_trace(msgs, args.reps, rank)
            log_n = len(trace).bit_length() - 1
            shape = {"K": K, "length": length, "log_n": log_n, "arms": []}
            res["shapes"].append(shape)

            def emit(a):
                shape["arms"].append(a)
                if rank == 0:
                    print(json.dumps(dict(a, card=res["card"], power_limit=res["power_limit"], K=K, length=length,
                                          log_n=log_n)), flush=True)

            emit(arm)
            claim = R.RescueHashClaim(length, digests)
            if world == 1:
                p = GpuProver.shared(0)
                p.prove(claim, R.OPTIONS, trace)
                runs = []
                for _ in range(args.reps):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    proof = p.prove(claim, R.OPTIONS, trace)
                    runs.append({"prove_s": time.perf_counter() - t0, "timings": proof.timings,
                                 "residency": p.last_residency})
                best = min(runs, key=lambda r: r["prove_s"])
                emit({"arm": "prove_1gpu", "prove_s_min": best["prove_s"], "prove_s_all": [r["prove_s"] for r in runs],
                      "timings_of_min": best["timings"], "residency": best["residency"],
                      "proof_bytes": len(proof.to_bytes())})
                blob = proof.to_bytes()
                t0 = time.perf_counter()
                claim.verify(blob, R.SECURITY_LEVEL)
                emit({"arm": "verify", "verify_s": time.perf_counter() - t0})
            else:
                from ministark_b200.prover_mgpu import ShardedProver
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
            del trace
    finally:
        if dist is not None:
            dist.destroy_process_group()
    if rank == 0:
        log_ns = sorted({s["log_n"] for s in res["shapes"]})
        name = f"bench_rescue_hash_2p{'_'.join(map(str, log_ns))}{f'_{world}gpu' if world > 1 else ''}_h100.json"
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, name), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
