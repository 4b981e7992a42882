#!/usr/bin/env python
"""What `GpuProver.prove(..., validate=True)` costs: the constraint check (csrc/check.cu) against the prove itself.

    profiles/bench_validate.py [--sizes 20 24] [--out-dir profiles]

  * examples/brainfuck cycle_burner(40, 40, 60) (2^20 rows, resident) and cycle_burner(128, 128, 60) (2^24 rows,
    streamed on an 80 GB card), ProofOptions(19, 16, 20, 16, 16): 48 constraints over 17 Fp + 9 Fq3 columns;
  * per size one warm-up prove with validation, then proves without and with validation, alternating, twice each; the
    check's time is the prover's timings["validate_constraints"] (host clock between two device synchronisations), the
    prove times are host clocks around synchronised proves; the proofs with and without validation must be identical;
  * the check kernel's registers, stack and spills from `nvcc -Xptxas -v` (compiled into a temporary directory);
  * the card name and power limit are read in the same run (nvidia-smi, read-only query).
One JSON file per size: <out-dir>/bench_validate_2p<log_n>_h100.json, and one JSON line per size on stdout."""
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
import torch

from ministark_b200.examples import brainfuck as bf
from ministark_b200.prover import GpuProver

BURNERS = {20: (40, 40, 60), 24: (128, 128, 60)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (v.strip() for v in out.split(",", 1))
        return name, limit
    except Exception as e:
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def kernel_resources():
    """ptxas' report for check_kernel (sm_90a), compiled outside the tree"""
    csrc = os.path.join(ROOT, "ministark_b200", "csrc")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        try:
            r = subprocess.run([nvcc, "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
                                "-c", os.path.join(csrc, "check.cu"), "-o", os.path.join(tmp, "check.o")],
                               capture_output=True, text=True, timeout=600)
        except Exception as e:
            return {"error": str(e)}
    lines = r.stderr.splitlines()
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln and "check_kernel" in ln:
            text = " ".join(lines[i:i + 4])
            num = lambda pat: int(m.group(1)) if (m := re.search(pat, text)) else None
            return {"registers": num(r"Used (\d+) registers"), "stack_bytes": num(r"(\d+) bytes stack frame"),
                    "spill_stores_bytes": num(r"(\d+) bytes spill stores"), "spill_loads_bytes": num(r"(\d+) bytes spill loads"),
                    "shared_bytes": num(r"(\d+) bytes smem") or 0}
    return {"error": "check_kernel not in the ptxas report", "stderr_tail": lines[-5:]}


def run(log_n, prover):
    a, b, c = BURNERS[log_n]
    t = time.perf_counter()
    src = bf.cycle_burner(a, b, c)
    trace, output = bf.simulate(src)
    sim = time.perf_counter() - t
    assert len(trace) == 1 << log_n, len(trace)
    claim = bf.BrainfuckClaim(src, b"", output)
    prover.prove(claim, bf.OPTIONS, trace, validate=True)                   # warm-up: programs, plans, scratch
    runs = {False: [], True: []}
    digests = set()
    for validate in (False, True, False, True):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t = time.perf_counter()
        proof = prover.prove(claim, bf.OPTIONS, trace, validate=validate)
        torch.cuda.synchronize()
        runs[validate].append({"prove_s": time.perf_counter() - t, "check_s": proof.timings.get("validate_constraints"),
                               "torch_peak_gib": torch.cuda.max_memory_allocated() / 2**30})
        digests.add(hashlib.sha256(proof.to_bytes()).hexdigest())
    assert len(digests) == 1, "validation changed the proof"
    checks = [r["check_s"] for r in runs[True]]
    plain = [r["prove_s"] for r in runs[False]]
    return {"program": f"cycle_burner({a},{b},{c})", "rows": len(trace), "log_n": log_n, "simulate_s": sim,
            "residency": prover.last_residency, "constraints": 48, "proof_sha256": digests.pop(),
            "without_validation": runs[False], "with_validation": runs[True],
            "check_s_min": min(checks), "prove_s_min": min(plain), "check_over_prove": min(checks) / min(plain)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[20, 24])
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_validate.py measures on a CUDA device; none is visible")
    name, limit = card()
    res_kernel = kernel_resources()
    os.makedirs(args.out_dir, exist_ok=True)
    for log_n in args.sizes:
        prover = GpuProver(0)
        res = {"card": name, "power_limit": limit, "check_kernel": res_kernel, **run(log_n, prover)}
        with open(os.path.join(args.out_dir, f"bench_validate_2p{log_n}_h100.json"), "w") as f:
            json.dump(res, f, indent=1)
        print(json.dumps(res), flush=True)
        del prover
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
