#!/usr/bin/env python
"""What filling a lookup's multiplicity column on the device costs (csrc/lookup.cu, ms_lookup_multiplicities), against
the host numpy route, and what share of a proof it takes.

    profiles/bench_lookup.py [--sizes 20 24] [--reps 10] [--out-dir profiles]

  * kernels: a W = 1, Q = 2 lookup (two value columns into a one-word table with duplicates) and examples/lookup's
    SquareLookupAirConfig lookup (W = 2, Q = 2, a selector), over random columns; ms_lookup_multiplicities timed with CUDA
    events, minimum of --reps calls after two warm-up calls;
  * in the same run, the host numpy route on the same (canonical) inputs: np.unique over the table and value tuples, the
    lowest table row of every tuple, np.bincount; its output words must equal the kernel's;
  * SquareLookupClaim proves from a device trace (SquareLookupClaim.gen_trace(n, device=0)), ProofOptions(16, 8, 4, 4, 8):
    one warm-up, then two proofs; timings["lookup_multiplicities"] beside the whole prove;
  * the card name and power limit are read in the same run (nvidia-smi, read-only query).
One JSON file per size: <out-dir>/bench_lookup_2p<log_n>_h100.json, and one JSON line per size on stdout."""
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
from ministark_b200.air import Lookup, ProofOptions
from ministark_b200.examples import lookup as L
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


def numpy_route(table, values, selectors):
    """table (W, n), values [(W, n)] canonical uint64, selectors [(n,)] or None -> n multiplicities (int64)"""
    W, n = table.shape
    allv = np.concatenate([table.T] + [v.T for v in values])
    uniq, inv = np.unique(allv[:, 0], return_inverse=True) if W == 1 else np.unique(allv, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    first = np.full(len(uniq), -1, dtype=np.int64)
    first[inv[:n][::-1]] = np.arange(n, dtype=np.int64)[::-1]
    counts = np.zeros(n, dtype=np.int64)
    for q in range(len(values)):
        hit = first[inv[n * (q + 1):n * (q + 2)]]
        on = hit >= 0 if selectors is None else (hit >= 0) & (selectors[q] == 1)
        counts += np.bincount(hit[on], minlength=n)
    return counts


def case(kind, log_n):
    n = 1 << log_n
    rng = np.random.default_rng(log_n)
    if kind == "W1_Q2":
        t = rng.integers(0, n // 4, size=n, dtype=np.uint64)
        canon = np.stack([t, t[rng.permutation(n)], t[rng.permutation(n)], np.zeros(n, dtype=np.uint64)])
        return Lookup((T(0),), ((T(1),), (T(2),)), 3, 4), canon, canon[[0]], [canon[[1]], canon[[2]]], None
    canon = L._square_columns(n, log_n).astype(np.uint64)
    return (L.SquareLookupAirConfig.lookups(n)[0], canon, canon[[0, 1]], [canon[[2, 4]], canon[[3, 5]]],
            [np.ones(n, dtype=np.uint64), canon[6]])


def bench_kernel(ctx, kind, log_n, reps):
    lk, canon, table, values, sel = case(kind, log_n)
    nbase, n = canon.shape
    base = torch.from_numpy(L._to_mont(canon).view(np.int64)).cuda()
    prog = E.compile_lookup_program(lk.table, lk.values, lk.selectors, nbase, log_n)
    W, Q = len(lk.table), len(lk.values)
    work = torch.empty(ctx.lookup_workspace_bytes(log_n, W, Q), dtype=torch.uint8, device="cuda")
    out = torch.empty(n, dtype=torch.int64, device="cuda")
    cols = [base[c] for c in range(nbase)]
    torch.cuda.synchronize()
    times = []
    for k in range(reps + 2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        missing, bad = ctx.lookup_multiplicities(prog, out, log_n, cols, W, Q, work)
        b.record()
        b.synchronize()
        if k >= 2:
            times.append(a.elapsed_time(b) / 1e3)
    assert not any(c for c, _ in missing) and not bad[0]
    t0 = time.perf_counter()
    counts = numpy_route(table, values, sel)
    t_np = time.perf_counter() - t0
    same = bool(np.array_equal(out.cpu().numpy().view(np.uint64), L._to_mont(counts.astype(np.uint64))))
    assert same, "the kernel and the numpy route disagree"
    return {"kernel_s_min": min(times), "kernel_s_all": times, "numpy_s": t_np, "identical_words": same,
            "workspace_bytes": work.numel(), "width": W, "tuples": Q}


def bench_prove(log_n):
    n = 1 << log_n
    opts = ProofOptions(16, 8, 4, 4, 8)
    trace = L.SquareLookupClaim.gen_trace(n, seed=1, device=0)
    p, claim = GpuProver.shared(0), L.SquareLookupClaim()
    p.prove(claim, opts, trace)
    runs = []
    for _ in range(2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        proof = p.prove(claim, opts, trace)
        wall = time.perf_counter() - t0
        runs.append({"prove_s": wall, "lookup_multiplicities_s": proof.timings["lookup_multiplicities"],
                     "timings": proof.timings, "residency": p.last_residency})
    return runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[20, 24])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    name, limit = card()
    ctx = ms.Context(0, stream=torch.cuda.current_stream().cuda_stream)
    for log_n in args.sizes:
        res = {"card": name, "power_limit": limit, "log_n": log_n, "timing": "kernels: CUDA events, seconds; prove: wall",
               "kernels": {k: bench_kernel(ctx, k, log_n, args.reps) for k in ("W1_Q2", "W2_Q2_square")},
               "square_prove": bench_prove(log_n)}
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, f"bench_lookup_2p{log_n}_h100.json"), "w") as f:
            json.dump(res, f, indent=1)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
