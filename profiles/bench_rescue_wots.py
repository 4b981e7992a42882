#!/usr/bin/env python
"""examples/wots: K Winternitz one-time signatures over Rescue-Prime, signed and proved valid in one proof, with the
signatures and the chain trace built on the GPU.

    profiles/bench_rescue_wots.py [--keys 489,490,978] [--reps 5] [--samples 3] [--out-dir profiles]

The defaults are the two counts whose 67 K chain blocks fill a power of two almost exactly, K = 489 (32,763 of 32,768
blocks, n = 2^22 rows) and K = 978 (65,526 of 65,536, n = 2^23), and the count just past the first of those
boundaries, K = 490 (32,830 chain blocks and 32,706 padding blocks, n = 2^23): the least aligned shape, where half the
trace is padding.  Keys, seeds and messages are SHAKE-256 words of a
fixed seed (tests/golden/make_rescue_wots_golden.py).  Per K:
  * sign kernel: ms_rescue_wots_sign alone (inputs and outputs in device memory), CUDA events after one warm-up, minimum
    of --reps calls.  It checks its words first and synchronises there, so the events span that too;
  * trace kernel: ms_rescue_wots_trace alone, timed the same way; it synchronises once more to check the roots before
    writing;
  * gen_trace(): wots.gen_trace(device=...) wall time up to a device synchronise;
  * prove: GpuProver from the device trace, one warm-up, then --reps proofs; wall time, proof.timings per phase and the
    torch peak of the fastest;
  * verify: Stark.verify of the proof on the host;
  * host verify: wots.verify of --samples signatures on the host with Python integers, per signature;
  * the card name, power limit and SM clock limit are read in the same run (nvidia-smi, read-only query).
One JSON line per arm on stdout; writes <out-dir>/bench_rescue_wots_2p<log n of the smallest K>_h100.json."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import torch

from bench_rescue import card
from bench_rescue_merkle_updates import _events
from make_rescue_wots_golden import keys, messages
from ministark_b200.examples import rescue as R
from ministark_b200.examples import wots as W
from ministark_b200.prover import GpuProver

SEED = 5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", default="489,490,978", help="comma-separated signature counts K")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--samples", type=int, default=3)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = dict(card(), options=list(vars(W.OPTIONS).values()),
               timing="kernels: CUDA events; gen_trace(), prove, verify: wall clock up to a device synchronise; host "
                      "verify: wall clock; seconds",
               shapes=[])
    for K in (int(v) for v in args.keys.split(",")):
        B = W._blocks(K)
        n = W.BLOCK * B
        log_n = n.bit_length() - 1
        shape = {"K": K, "blocks": B, "chain_blocks": W.CHAINS * K, "log_n": log_n, "arms": []}
        res["shapes"].append(shape)

        def emit(a):
            shape["arms"].append(a)
            print(json.dumps(dict(a, card=res["card"], power_limit=res["power_limit"], K=K, log_n=log_n)), flush=True)

        secrets, seeds = keys(K, SEED)
        msgs = messages(K, SEED)
        d_sec, d_seed, d_msg = (torch.from_numpy(a.view("int64")).to(dev) for a in (secrets, seeds, msgs))
        sigs = torch.empty((K, W.CHAINS, 4), dtype=torch.int64, device=dev)
        pks = torch.empty((K, W.PK), dtype=torch.int64, device=dev)
        out = torch.empty((W.NUM_BASE, n), dtype=torch.int64, device=dev)
        stream = torch.cuda.Stream(dev)
        with torch.cuda.stream(stream):                         # the context queues on this stream, and the events too
            ctx = R._context(dev)
        torch.cuda.synchronize()
        s, ss = _events(lambda: ctx.rescue_wots_sign(d_sec, d_seed, d_msg, K, sigs, pks), args.reps, ctx, stream)
        # sign: 67 K chain secrets and 15 steps each, then 67 K folds; verify: 15 chain slots and a fold per block
        emit({"arm": "sign_kernel", "kernel_s_min": s, "kernel_s_all": ss, "permutations": 17 * W.CHAINS * K})
        t, ts = _events(lambda: ctx.rescue_wots_trace(pks, d_msg, sigs, K, out), args.reps, ctx, stream)
        # the signatures' chain slots and folds run twice (ends and roots first, then the rows once every root
        # matched); the padding blocks' only in the write pass
        emit({"arm": "trace_kernel", "kernel_s_min": t, "kernel_s_all": ts, "permutations_in_trace": 16 * B,
              "permutations_computed": 16 * B + 16 * W.CHAINS * K})
        del out
        torch.cuda.empty_cache()
        times = []
        for _ in range(args.reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            trace = W.gen_trace(pks, msgs, sigs, device=0)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            del trace
        emit({"arm": "gen_trace", "gen_trace_s_min": min(times[1:]), "gen_trace_s_all": times[1:]})
        trace = W.gen_trace(pks, msgs, sigs, device=0)
        host_pks = [tuple(int(w) for w in r) for r in pks.cpu().numpy().view("uint64")]
        claim = W.SignaturesClaim(host_pks, msgs)
        p = GpuProver.shared(0)
        p.prove(claim, W.OPTIONS, trace)
        runs = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            t0 = time.perf_counter()
            proof = p.prove(claim, W.OPTIONS, trace)
            runs.append({"prove_s": time.perf_counter() - t0, "timings": proof.timings, "residency": p.last_residency,
                         "torch_peak_bytes": torch.cuda.max_memory_allocated(dev)})
        best = min(runs, key=lambda r: r["prove_s"])
        blob = proof.to_bytes()
        emit({"arm": "prove_1gpu", "prove_s_min": best["prove_s"], "prove_s_all": [r["prove_s"] for r in runs],
              "timings_of_min": best["timings"], "residency": best["residency"],
              "torch_peak_bytes": best["torch_peak_bytes"], "proof_bytes": len(blob)})
        t0 = time.perf_counter()
        claim.verify(blob, W.SECURITY_LEVEL)
        emit({"arm": "verify", "verify_s": time.perf_counter() - t0})
        host_sigs = sigs.cpu().numpy().view("uint64")
        times = []
        for k in range(min(args.samples, K)):
            t0 = time.perf_counter()
            assert W.verify(host_pks[k], msgs[k], host_sigs[k])
            times.append(time.perf_counter() - t0)
        emit({"arm": "host_verify_per_signature", "verify_s_mean": sum(times) / len(times), "verify_s_all": times})
        del trace, sigs, pks
        torch.cuda.empty_cache()
    name = f"bench_rescue_wots_2p{min(s['log_n'] for s in res['shapes'])}_h100.json"
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, name), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
