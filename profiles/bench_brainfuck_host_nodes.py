#!/usr/bin/env python
"""examples/brainfuck at 2^25 rows on one GPU: the streamed_host residency (Merkle node heaps in pinned host memory).
One JSON line on stdout.

    profiles/bench_brainfuck_host_nodes.py [--burner A B C] [--compare-burner A B C] [--host-reserve GIB]

  * cycle_burner(181, 181, 60) pads to 2^25 rows (its cycle count from ms_bf_run, its row count from the device trace);
    ProofOptions(19, 16, 20, 16, 16), 17 Fp + 9 Fq3 columns.  Resident and streamed do not fit an 80 GB card there;
    GpuProver gets a host budget of MemAvailable minus --host-reserve and picks streamed_host;
  * the Python prover: the first prove (which pins the node heaps) and one more, their phase times, the torch peak and
    the lowest free device memory (sampled every 5 ms) against the device estimate, the pinned bytes and the pinning time;
  * the command line (ministark_bf prove --host-memory): its prove time, residency, lowest free device memory and pinned
    bytes as it prints them; its proof part must equal the Python bytes, and both oracle/stark_oracle.verify and
    ministark_bf verify must accept it;
  * at 2^24 rows (cycle_burner(128, 128, 60)), streamed against streamed_host, alternating for --rounds rounds in the
    same process: prove times, and per phase the median with its range.  The commitments are where moving the node heaps
    to host memory costs; the other phases differ only by run-to-run noise.
If MemAvailable is below what the 2^25 run needs (the 48 GiB of heaps plus --host-reserve), the result says so and no time
is reported.  The card name and power limit are read in the same run (nvidia-smi, read-only query)."""
import argparse
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

import ministark_b200 as ms
from ministark_b200.air import Air, ProofOptions
from ministark_b200.examples import brainfuck as bf
from ministark_b200.prover import GpuProver, peak_bytes

CLI = os.path.join(ROOT, "ministark_b200", "ministark_bf")
GIB = 2**30


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (v.strip() for v in out.split(",", 1))
        return name, limit
    except Exception as e:          # the numbers still stand, but without their card they are incomplete
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def estimates(claim, n):
    cfg, o = claim.AirConfig, bf.OPTIONS
    return peak_bytes(n, o.lde_blowup_factor, cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, ms.FQ3,
                      Air(cfg, n, None, o).ce_blowup_factor, o.fri_folding_factor)


class LowestFree:
    """the lowest free device memory seen while the block runs, sampled every 5 ms on a thread"""

    def __enter__(self):
        self.low, self._stop = torch.cuda.mem_get_info(0)[0], threading.Event()
        self._t = threading.Thread(target=self._run)
        self._t.start()
        return self

    def _run(self):
        while not self._stop.wait(0.005):
            self.low = min(self.low, torch.cuda.mem_get_info(0)[0])

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()


def timed_prove(prover, claim, trace):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with LowestFree() as low:
        t = time.perf_counter()
        proof = prover.prove(claim, bf.OPTIONS, trace)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t
    return dt, proof, torch.cuda.max_memory_allocated() - base, low.low


def cli_prove(src, host_gib):
    d = tempfile.mkdtemp()
    path, dst = os.path.join(d, "p.bf"), os.path.join(d, "p.proof")
    with open(path, "w") as f:
        f.write(src)
    t = time.perf_counter()
    r = subprocess.run([CLI, "prove", path, "--dst", dst, "--host-memory", f"{host_gib:.2f}"], capture_output=True, text=True)
    wall = time.perf_counter() - t
    if r.returncode:
        return {"error": r.stderr.strip()}, None, path, dst
    grab = lambda pat: (re.search(pat, r.stdout) or [None, None])[1]
    out = {"wall_s": round(wall, 3), "prove_s": float(grab(r"Proof generated in: ([0-9.]+)s")),
           "trace_s": float(grab(r"execution trace .* in ([0-9.]+)s")), "residency": grab(r"Residency: (\S+)"),
           "pinned_bytes": int(grab(r"Pinned host memory: (\d+) bytes") or 0), "pin_s": float(grab(r"pinned in ([0-9.]+)s") or 0)}
    low = grab(r"Lowest free device memory between phases: (\d+) bytes")
    if low:
        out["lowest_free_gib"] = round(int(low) / GIB, 2)
    with open(dst, "rb") as f:
        blob = f.read()
    return out, blob, path, dst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--burner", type=int, nargs=3, default=[181, 181, 60])
    ap.add_argument("--compare-burner", type=int, nargs=3, default=[128, 128, 60])
    ap.add_argument("--host-reserve", type=float, default=8.0, help="GiB of MemAvailable left to the rest of the machine")
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds of the 2^24 comparison, after one warm-up round")
    args = ap.parse_args()
    name, power = card()
    res = {"bench": "brainfuck_host_nodes", "gpu": name, "power_limit": power}

    a, b, c = args.burner
    src = bf.cycle_burner(a, b, c)
    log, _ = ms.bf_run(bf.compile_program(src))
    t = time.perf_counter()
    trace, out = bf.simulate(src, device=0)
    torch.cuda.synchronize()
    n = len(trace)
    res.update(program=f"cycle_burner({a},{b},{c})", cycles=len(log) - 1, rows=n, cols="17 Fp + 9 Fq3",
               options=[19, 16, 20, 16, 16],
               device_trace_s=round(time.perf_counter() - t, 3))
    del log
    claim = bf.BrainfuckClaim(src, b"", out)
    est = estimates(claim, n)
    res["estimate_gib"] = {k: round(v / GIB, 2) for k, v in est.items()}
    avail = mem_available()
    res["host_mem_available_gib"] = round(avail / GIB, 2)
    host_budget = avail - int(args.host_reserve * GIB)
    if host_budget < est["host"]:
        res["skipped"] = (f"MemAvailable is {avail / GIB:.1f} GiB: the node heaps need {est['host'] / GIB:.1f} GiB plus "
                          f"{args.host_reserve} GiB left to the machine")
        print(json.dumps(res))
        return

    prover = GpuProver(0, host_memory_budget=host_budget)
    res["device_budget_gib"] = round(prover.memory_available() / GIB, 2)
    runs = []
    for k in range(2):
        if k:
            trace, _ = bf.simulate(src, device=0)        # the prover released the first trace's matrix
        runs.append(timed_prove(prover, claim, trace))
    res["residency"] = prover.last_residency
    res["pinned_bytes"] = prover.pinned_bytes
    res["pin_s"] = round(runs[0][1].timings.get("pin_host_memory", 0.0), 3)
    res["prove_s"] = {"first_with_pinning": round(runs[0][0], 3), "second": round(runs[1][0], 3)}
    res["phases_s"] = {k: round(v, 4) for k, v in runs[1][1].timings.items()}
    res["torch_peak_gib"] = round(max(r[2] for r in runs) / GIB, 2)
    res["lowest_free_gib"] = round(min(r[3] for r in runs) / GIB, 2)
    pb = runs[1][1].to_bytes()
    res["proof_sha256"] = hashlib.sha256(pb).hexdigest()
    res["same_bytes_every_run"] = runs[0][1].to_bytes() == pb
    del runs, trace
    prover.release_host_memory()                         # the command line pins its own heaps
    del prover
    torch.cuda.empty_cache()

    cli, blob, path, dst = cli_prove(src, host_budget / GIB)
    res["cli"] = cli
    if blob is not None:
        claim_b = claim.public_inputs_bytes(claim)
        res["cli"]["same_bytes_as_python"] = blob.startswith(claim_b) and blob[len(claim_b):] == pb
        ver = subprocess.run([CLI, "verify", path, "--proof", dst, "--output", out.decode()], capture_output=True, text=True)
        res["cli"]["cli_verify_accepts"] = ver.returncode == 0
    t = time.perf_counter()
    from oracle import stark_oracle as SO
    SO.verify(claim, pb, bf.SECURITY_LEVEL, lambda m, o: Air(claim.AirConfig, m, claim, ProofOptions(*o)))
    res["oracle_verified"], res["oracle_verify_s"] = True, round(time.perf_counter() - t, 2)

    # ---- 2^24: streamed against streamed_host, alternating
    a2, b2, c2 = args.compare_burner
    src2 = bf.cycle_burner(a2, b2, c2)
    trace2, out2 = bf.simulate(src2, device=0)
    claim2 = bf.BrainfuckClaim(src2, b"", out2)
    est2 = estimates(claim2, len(trace2))
    cmp = {"program": f"cycle_burner({a2},{b2},{c2})", "rows": len(trace2)}
    provers = {"streamed": GpuProver(0, memory_budget=(est2["streamed"] + est2["resident"]) // 2),
               "streamed_host": GpuProver(0, memory_budget=(est2["streamed_host"] + est2["streamed"]) // 2,
                                          host_memory_budget=est2["host"])}
    times = {k: [] for k in provers}
    phases = {k: [] for k in provers}
    digests = {k: set() for k in provers}
    for rnd in range(1 + args.rounds):                    # round 0 warms up (AIR programs, plans, pinning)
        for label, p in provers.items():
            trace2, _ = bf.simulate(src2, device=0)
            dt, proof, peak, low = timed_prove(p, claim2, trace2)
            assert p.last_residency == label
            digests[label].add(hashlib.sha256(proof.to_bytes()).hexdigest())
            if rnd:
                times[label].append(round(dt, 3))
                phases[label].append(proof.timings)
                cmp[label + "_torch_peak_gib"] = round(peak / GIB, 2)
    median = lambda v: sorted(v)[len(v) // 2]
    for label, runs in phases.items():                    # per phase: the median and the range over the timed rounds
        cmp[label + "_phases_s"] = {k: [round(median([t[k] for t in runs]), 4), round(min(t[k] for t in runs), 4),
                                        round(max(t[k] for t in runs), 4)] for k in runs[0]}
    cmp.update({k + "_prove_s": v for k, v in times.items()})
    cmp["same_bytes"] = len(digests["streamed"] | digests["streamed_host"]) == 1
    cmp["streamed_host_over_streamed"] = round(median(times["streamed_host"]) / median(times["streamed"]), 3)
    # the three commitments are the phases that write the heaps: their summed medians, per residency
    commits = ("base_trace_commitment", "extension_trace_commitment", "composition_trace_commitment")
    cmp["commitments_s"] = {k: round(sum(cmp[k + "_phases_s"][c][0] for c in commits), 4) for k in provers}
    res["streamed_vs_streamed_host_2p24"] = cmp
    print(json.dumps(res))


if __name__ == "__main__":
    main()
