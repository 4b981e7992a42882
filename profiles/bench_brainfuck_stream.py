#!/usr/bin/env python
"""examples/brainfuck at 2^24 rows on one GPU: the streamed residency of GpuProver.  One JSON line on stdout.

    profiles/bench_brainfuck_stream.py [--burner A B C] [--compare-burner A B C] [--cpu] [--skip-compare]

  * cycle_burner(128, 128, 60) pads to 2^24 rows; ProofOptions(19, 16, 20, 16, 16), 17 Fp + 9 Fq3 columns;
  * one warm-up prove and two timed proves (host clock around a synchronised prove), per-phase times, the torch peak
    of device memory, the budget the residency was chosen against, the proof's SHA-256; the proof is checked by the
    restated verifier (oracle/stark_oracle.verify);
  * ms_lde_rows against ms_poly_eval at the query shape of that proof: every coefficient column of the three matrices
    (92 words per row) at 2 * 19 base-field points;
  * at the largest size where both residencies fit (cycle_burner(40, 40, 60) = 2^20 rows by default), resident against
    streamed prove time: what recomputing the coset blocks costs;
  * --cpu: the compiled CPU prover (oracle/cpu_prover) at the same size, in the same run (about 285 GB of host RAM at 2^24).
The card name and power limit are read in the same run (nvidia-smi, read-only query)."""
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
from ministark_b200.air import Air, ProofOptions
from ministark_b200.examples import brainfuck as bf
from ministark_b200.prover import GpuProver, peak_bytes

OPTS = (19, 16, 20, 16, 16)          # bf.OPTIONS


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (v.strip() for v in out.split(",", 1))
        return name, limit
    except Exception as e:          # the numbers still stand, but without their card they are incomplete
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def timed_proves(prover, claim, trace, reps=2):
    prover.prove(claim, bf.OPTIONS, trace)                                   # warm-up: AIR programs, plans, scratch
    runs = []
    for _ in range(reps):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t = time.perf_counter()
        proof = prover.prove(claim, bf.OPTIONS, trace)
        torch.cuda.synchronize()
        runs.append((time.perf_counter() - t, proof, torch.cuda.max_memory_allocated()))
    return runs


def estimates(claim, n):
    cfg, o = claim.AirConfig, bf.OPTIONS
    return peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, ms.FQ3,
                      Air(cfg, n, None, o).ce_blowup_factor, o.fri_folding_factor)


def kernel_compare(log_n, log_b, npoints=38, reps=3):
    """ms_lde_rows against ms_poly_eval over random coefficient matrices of the brainfuck shape"""
    ctx = ms.Context(0)
    n = 1 << log_n
    shapes = [(ms.FP, 17), (ms.FQ3, 9), (ms.FQ3, 16)]
    mats = []
    for k, (f, c) in enumerate(shapes):
        t = torch.empty((c, n * f), dtype=torch.int64, device="cuda")
        ctx.fill_random(t, t.numel(), 100 + k)
        mats.append((f, c, t))
    rng = np.random.default_rng(1)
    positions = [int(v) for v in rng.integers(0, n << log_b, size=npoints)]
    gN = ms.root_of_unity(log_n + log_b)
    brev = lambda v: int(format(v, f"0{log_n + log_b}b")[::-1], 2)
    xs = [ms.to_mont(7 * pow(ms.from_mont(gN), brev(p), ms.P)) for p in positions]
    pts = np.array([[x, 0, 0] for x in xs], dtype=np.uint64)

    def best(fn):
        fn()
        ts = []
        for _ in range(reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t)
        return min(ts), out

    t_rows, t_eval, same = 0.0, 0.0, True
    for f, c, t in mats:
        dt, rows = best(lambda: ctx.lde_rows(t, f, log_n, log_b, c, positions))
        t_rows += dt
        dt, ev = best(lambda: ctx.poly_eval(t, f, n, c, pts))
        t_eval += dt
        # the same values: poly_eval returns (col, point, 3) Fq3, lde_rows (point, col * f)
        same &= np.array_equal(rows.reshape(npoints, c, f), ev.transpose(1, 0, 2)[:, :, :f])
    del mats
    ctx.close()
    torch.cuda.empty_cache()
    return {"log_n": log_n, "points": npoints, "columns": "17 Fp + 9 Fq3 + 16 Fq3", "lde_rows_s": t_rows,
            "poly_eval_s": t_eval, "speedup": t_eval / t_rows, "values_equal": bool(same)}


def cpu_prove(a, b, c):
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "cpu_prover")
    ii, mi = bf.test_rng_fq3(2)
    t = time.perf_counter()
    r = json.loads(subprocess.run([exe, "bf", str(a), str(b), str(c)] + [str(v) for v in OPTS] +
                                  [str(v) for v in ii + mi], capture_output=True, text=True, check=True).stdout)
    r["wall_s"] = time.perf_counter() - t
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--burner", type=int, nargs=3, default=[128, 128, 60])
    ap.add_argument("--compare-burner", type=int, nargs=3, default=[40, 40, 60])
    ap.add_argument("--cpu", action="store_true", help="also run the compiled CPU prover at --burner (needs ~285 GB RAM at 2^24)")
    ap.add_argument("--skip-compare", action="store_true")
    args = ap.parse_args()
    name, power = card()
    res = {"bench": "brainfuck_stream", "gpu": name, "power_limit": power}

    a, b, c = args.burner
    src = bf.cycle_burner(a, b, c)
    t = time.perf_counter()
    trace, out = bf.simulate(src)
    res.update(program=f"cycle_burner({a},{b},{c})", rows=len(trace), cols="17 Fp + 9 Fq3", options=list(OPTS),
               simulate_s=time.perf_counter() - t)
    claim = bf.BrainfuckClaim(src, b"", out)
    prover = GpuProver(0)
    est = estimates(claim, len(trace))
    res["estimate_gib"] = {k: round(v / 2**30, 2) for k, v in est.items()}
    res["budget_gib"] = round(prover.memory_available() / 2**30, 2)
    runs = timed_proves(prover, claim, trace)
    res["residency"] = prover.last_residency
    res["prove_s"] = [round(r[0], 3) for r in runs]
    dt, proof, peak = min(runs, key=lambda r: r[0])
    res["torch_peak_gib"] = round(max(r[2] for r in runs) / 2**30, 2)
    res["phases_s"] = {k: round(v, 4) for k, v in proof.timings.items()}
    pb = proof.to_bytes()
    res["proof_bytes"] = len(pb)
    res["proof_sha256"] = hashlib.sha256(pb).hexdigest()
    res["same_bytes_every_run"] = len({r[1].to_bytes() for r in runs}) == 1
    del runs, proof
    t = time.perf_counter()
    from oracle import stark_oracle as SO
    SO.verify(claim, pb, bf.SECURITY_LEVEL, lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o)))
    res["verified"], res["verify_s"] = True, time.perf_counter() - t
    del prover
    torch.cuda.empty_cache()

    res["lde_rows_vs_poly_eval"] = kernel_compare(len(trace).bit_length() - 1, 4)

    if not args.skip_compare:
        a2, b2, c2 = args.compare_burner
        src2 = bf.cycle_burner(a2, b2, c2)
        trace2, out2 = bf.simulate(src2)
        claim2 = bf.BrainfuckClaim(src2, b"", out2)
        est2 = estimates(claim2, len(trace2))
        cmp = {"program": f"cycle_burner({a2},{b2},{c2})", "rows": len(trace2)}
        for label, budget in [("resident", None), ("streamed", (est2["streamed"] + est2["resident"]) // 2)]:
            p = GpuProver(0, memory_budget=budget)
            runs = timed_proves(p, claim2, trace2)
            cmp[label] = {"residency": p.last_residency, "prove_s": [round(r[0], 4) for r in runs],
                          "torch_peak_gib": round(max(r[2] for r in runs) / 2**30, 3),
                          "sha256": hashlib.sha256(runs[0][1].to_bytes()).hexdigest()}
            del p, runs
            torch.cuda.empty_cache()
        cmp["same_bytes"] = cmp["resident"]["sha256"] == cmp["streamed"]["sha256"]
        cmp["streamed_over_resident"] = round(min(cmp["streamed"]["prove_s"]) / min(cmp["resident"]["prove_s"]), 3)
        res["resident_vs_streamed"] = cmp

    if args.cpu:
        r = cpu_prove(a, b, c)
        res["cpu_prover"] = {k: r.get(k) for k in ("rows", "seconds", "verified", "threads", "wall_s")}
        res["speedup_vs_cpu"] = r["seconds"] / dt
    print(json.dumps(res))


if __name__ == "__main__":
    main()
