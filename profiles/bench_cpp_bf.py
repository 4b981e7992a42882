#!/usr/bin/env python
"""The brainfuck command line (ministark_b200/ministark_bf: the C++ host layer, device trace + GpuProver) on one GPU.
One JSON line on stdout, also written to --out.

    profiles/bench_cpp_bf.py [--burner A B C] [--runs K] [--python] [--out FILE]

  * cycle_burner(40, 40, 60) pads to 2^20 rows, cycle_burner(128, 128, 60) to 2^24; ProofOptions(19, 16, 20, 16, 16);
  * K separate `prove` processes (each cold: context, NTT plans and scratch are built inside the timed prove): the trace
    and prove wall times the command line prints (host clock; the prover returns after its last device-to-host copy),
    the residency, the free device memory before the trace and the lowest ms_device_memory reading between the proof's
    phases, and the SHA-256 of the proof part of the file (the bytes after claim_bytes);
  * `verify` of the last file, timed;
  * --python: the Python prover (GpuProver on the device trace) at the same size in the same run: its first (cold) prove
    and two warm ones, its torch peak and its proof's SHA-256.
The card name and power limit are read in the same run (nvidia-smi, read-only query).  Other processes on the card
change its free memory, so the memory figures are readings, not a property of the prover alone."""
import argparse
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CLI = os.path.join(ROOT, "ministark_b200", "ministark_bf")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (v.strip() for v in out.split(",", 1))
        return name, limit
    except Exception as e:
        return "unknown", f"unknown ({e})"


def field(pattern, text, cast=float):
    m = re.search(pattern, text)
    if not m:
        raise RuntimeError(f"{pattern!r} not in the command line's output:\n{text}")
    return cast(m.group(1))


def cli_runs(source, runs, tmp):
    from ministark_b200.examples import brainfuck as bf
    src = os.path.join(tmp, "prog.bf")
    with open(src, "w") as f:
        f.write(source)
    out_runs = []
    for k in range(runs):
        dst = os.path.join(tmp, f"proof{k}.bin")
        t = time.perf_counter()
        r = subprocess.run([CLI, "prove", src, "--dst", dst], capture_output=True, text=True, timeout=1800)
        wall = time.perf_counter() - t
        if r.returncode:
            raise RuntimeError(r.stderr)
        output = b""
        claim = bf.BrainfuckClaim(source, b"", output)
        head = claim.public_inputs_bytes(claim)
        blob = open(dst, "rb").read()
        if not blob.startswith(head):
            raise RuntimeError("the file does not start with the claim")
        out_runs.append({
            "rows": field(r"rows=(\d+)", r.stdout, int),
            "trace_s": field(r"trace \(cols=17, rows=\d+\) in ([0-9.]+)s", r.stdout),
            "prove_s": field(r"Proof generated in: ([0-9.]+)s", r.stdout),
            "process_s": round(wall, 3),
            "residency": field(r"Residency: (\w+)", r.stdout, str),
            "free_before_gib": round(field(r"before the trace: (\d+) bytes", r.stdout, int) / 2**30, 2),
            "lowest_free_gib": round(field(r"between phases: (\d+) bytes", r.stdout, int) / 2**30, 2),
            "proof_part_bytes": len(blob) - len(head),
            "proof_part_sha256": hashlib.sha256(blob[len(head):]).hexdigest(),
        })
    t = time.perf_counter()
    v = subprocess.run([CLI, "verify", src, "--proof", dst, "--output", ""], capture_output=True, text=True, timeout=1800)
    verify = {"verified": v.returncode == 0, "verify_process_s": round(time.perf_counter() - t, 3),
              "message": (v.stdout + v.stderr).strip()}
    return out_runs, verify


def python_prover(source):
    import torch
    from ministark_b200.examples import brainfuck as bf
    from ministark_b200.prover import GpuProver
    trace, output = bf.simulate(source, device=0)
    claim = bf.BrainfuckClaim(source, b"", output)
    prover = GpuProver(0)
    torch.cuda.synchronize()
    t = time.perf_counter()
    prover.prove(claim, bf.OPTIONS, trace)          # cold, as every `prove` process is: evaluator programs, plans, scratch
    torch.cuda.synchronize()
    cold = round(time.perf_counter() - t, 3)
    times, peak, digests = [], 0, set()
    for _ in range(2):
        trace, _ = bf.simulate(source, device=0)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t = time.perf_counter()
        proof = prover.prove(claim, bf.OPTIONS, trace)
        torch.cuda.synchronize()
        times.append(round(time.perf_counter() - t, 3))
        peak = max(peak, torch.cuda.max_memory_allocated())
        digests.add(hashlib.sha256(proof.to_bytes()).hexdigest())
        del trace
    return {"cold_prove_s": cold, "prove_s": times, "residency": prover.last_residency, "torch_peak_gib": round(peak / 2**30, 2),
            "proof_sha256": sorted(digests)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--burner", type=int, nargs=3, default=[40, 40, 60])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--python", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    from ministark_b200.examples import brainfuck as bf
    if not os.path.exists(CLI):
        raise SystemExit(f"{CLI} is missing: run __graft_entry__.build() first")
    source = bf.cycle_burner(*a.burner)
    name, limit = card()
    with tempfile.TemporaryDirectory() as tmp:
        runs, verify = cli_runs(source, a.runs, tmp)
    res = {"bench": "cpp_bf_cli", "gpu": name, "power_limit": limit, "program": "cycle_burner(%d,%d,%d)" % tuple(a.burner),
           "rows": runs[0]["rows"], "options": [19, 16, 20, 16, 16], "runs": runs, **verify,
           "same_bytes_every_run": len({r["proof_part_sha256"] for r in runs}) == 1}
    if a.python:
        res["python_prover"] = python_prover(source)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
