#!/usr/bin/env python
"""What building declared extension columns on the device costs (csrc/extension.cu, ms_extension_columns), against the
route it replaces and against the host callback.

    profiles/bench_extension.py [--sizes 20 24] [--reps 10] [--out-dir profiles]

  * declarations: examples/perm's two Fq3 running products (mul = alpha - a, alpha - b) and examples/lookup's LogUp running
    sum (add = m / (alpha - t) - 1 / (alpha - v)), over random base columns of 2^20 and 2^24 rows;
  * ms_extension_columns, one call building all K columns, timed with CUDA events after two warm-up calls;
  * in the same run, the A/B reference done here: one fused-evaluator launch per mul and per add expression into scratch
    columns (ms_eval_constraints_ptrs), then one ms_scan_affine per column; its output must equal the kernel's;
  * at 2^20 rows, end-to-end proves of examples/perm, ProofOptions(16, 8, 4, 4, 8): the host callback (PermClaim) against
    the declaration (PermDeclaredClaim), one warm-up each, then alternating, twice each; the proofs must be identical;
  * the new kernels' registers, stack and spills from `nvcc -Xptxas -v` (compiled into a temporary directory);
  * the card name and power limit are read in the same run (nvidia-smi, read-only query).
One JSON file per size: <out-dir>/bench_extension_2p<log_n>_h100.json, and one JSON line per size on stdout."""
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
import numpy as np
import torch

import ministark_b200 as ms
from ministark_b200 import expr as E
from ministark_b200.air import ProofOptions
from ministark_b200.examples import perm
from ministark_b200.prover import GpuProver

P = E.P
ALPHA = (0x1234567890ABCDEF % P, 0x0FEDCBA987654321 % P, 0x1111222233334444 % P)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (v.strip() for v in out.split(",", 1))
        return name, limit
    except Exception as e:
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def kernel_resources():
    """ptxas' report for the kernels of extension.cu (sm_90a), compiled outside the tree"""
    csrc = os.path.join(ROOT, "ministark_b200", "csrc")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        try:
            r = subprocess.run([nvcc, "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
                                "-c", os.path.join(csrc, "extension.cu"), "-o", os.path.join(tmp, "extension.o")],
                               capture_output=True, text=True, timeout=600)
        except Exception as e:
            return {"error": str(e)}
    lines, out = r.stderr.splitlines(), {}
    for i, ln in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S+)'", ln)
        if m and "ext_" in m.group(1):
            text = " ".join(lines[i:i + 4])
            num = lambda pat: int(x.group(1)) if (x := re.search(pat, text)) else None
            out[m.group(1)] = {"registers": num(r"Used (\d+) registers"), "stack_bytes": num(r"(\d+) bytes stack frame"),
                               "spill_stores_bytes": num(r"(\d+) bytes spill stores"),
                               "spill_loads_bytes": num(r"(\d+) bytes spill loads")}
    return out or {"error": "no extension kernel in the ptxas report", "stderr_tail": lines[-5:]}


def declarations(n):
    """name -> (base (3, n) Montgomery words, [(init, mul, add, inclusive)])"""
    rng = np.random.default_rng(n)
    small = lambda: rng.integers(0, min(n, 2**31), size=n, dtype=np.uint64) * np.uint64(2**64 % P)   # Montgomery, < 2^32
    al, T = E.Challenge(0), E.Trace
    return {
        "perm_2cols": (np.stack([small(), small(), small()]),
                       [(E.Constant(1), al - T(0), E.Constant(0), False), (E.Constant(1), al - T(1), E.Constant(0), False)]),
        "lookup_1col": (np.stack([small(), np.arange(n, dtype=np.uint64) * np.uint64(2**64 % P), small()]),
                        [(E.Constant(0), E.Constant(1), T(2) / (al - T(1)) - E.Constant(1) / (al - T(0)), False)]),
    }


def events_time(fn, reps, stream):
    """CUDA events on `stream`, the context's stream, around each of `reps` calls after two warm-up calls"""
    fn()
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) / 1e3)
    return times


def kernel_case(ctx, log_n, base_h, decl, reps):
    n = 1 << log_n
    base = torch.from_numpy(base_h.view(np.int64)).cuda()
    cols, isq = [base[c] for c in range(3)], [False] * 3
    K = len(decl)
    prog = E.compile_extension_program([d[1] for d in decl], [d[2] for d in decl], 3, log_n, 3).bind(challenges=[ALPHA])
    init = np.array([[ms.to_mont(w) for w in E.evaluate_at(d[0], 0, challenges=[ALPHA])] for d in decl], dtype=np.uint64)
    inclusive = [d[3] for d in decl]
    out = torch.empty((K, 3 * n), dtype=torch.int64, device="cuda")
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)          # the events below are recorded on the stream the kernels run on
    new = events_time(lambda: ctx.extension_columns(prog, out, log_n, cols, isq, ms.FQ3, init, inclusive), reps, stream)

    # the route it replaces: evaluator launches into 2K scratch columns, then one scan per column
    progs = [(E.compile_program(d[1], 3, symbolic=True).bind(challenges=[ALPHA]),
              E.compile_program(d[2], 3, symbolic=True).bind(challenges=[ALPHA])) for d in decl]
    mul, add = torch.empty((K, 3 * n), dtype=torch.int64, device="cuda"), torch.empty((K, 3 * n), dtype=torch.int64, device="cuda")
    ref = torch.empty((K, 3 * n), dtype=torch.int64, device="cuda")

    def old_route():
        for k, (pm, pa) in enumerate(progs):
            ctx.eval_constraints_ptrs(pm, mul[k], log_n, cols, isq, fq_field=ms.FQ3, offset=ms.ONE)
            ctx.eval_constraints_ptrs(pa, add[k], log_n, cols, isq, fq_field=ms.FQ3, offset=ms.ONE)
            ctx.scan_affine(ref[k], ms.FQ3, n, init[k], a=mul[k], a_field=ms.FQ3, b=add[k], b_field=ms.FQ3,
                            inclusive=inclusive[k])

    old = events_time(old_route, reps, stream)
    torch.cuda.synchronize()
    same = bool(torch.equal(out, ref))
    assert same, "ms_extension_columns differs from the evaluator + scan route"
    # algorithmic traffic: referenced base columns read twice, K Fq3 columns written (the old route also writes and reads
    # back 2K Fq3 scratch columns)
    nref = len({c for d in decl for e in d[1:3] for c, _ in _trace_leaves(e)})
    new_bytes = 2 * 8 * nref * n + 24 * K * n
    return {"columns": K, "base_columns_read": nref, "new_s": new, "new_s_min": min(new), "evaluator_plus_scan_s": old,
            "evaluator_plus_scan_s_min": min(old), "speedup_min_over_min": min(old) / min(new), "outputs_equal": same,
            "new_algorithmic_bytes": new_bytes, "new_gb_per_s_at_min": new_bytes / min(new) / 1e9}


def _trace_leaves(e):
    from ministark_b200.air import _leaves
    return _leaves(e, "trace")


def e2e_perm(log_n):
    n = 1 << log_n
    opts = ProofOptions(16, 8, 4, 4, 8)
    t = time.perf_counter()
    host = perm.gen_trace(n, seed=3)
    declared = perm.gen_trace(n, seed=3, extension=False)
    gen = time.perf_counter() - t
    prover = GpuProver(0)
    cases = {"host_callback": (perm.PermClaim(), host), "declared": (perm.PermDeclaredClaim(), declared)}
    for claim, trace in cases.values():
        prover.prove(claim, opts, trace)                                   # warm-up: programs, plans, scratch
    runs, digests = {k: [] for k in cases}, set()
    for name in ["host_callback", "declared"] * 2:
        claim, trace = cases[name]
        torch.cuda.synchronize()
        t = time.perf_counter()
        proof = prover.prove(claim, opts, trace)
        torch.cuda.synchronize()
        runs[name].append({"prove_s": time.perf_counter() - t,
                           "extension_trace_commitment_s": proof.timings["extension_trace_commitment"]})
        digests.add(hashlib.sha256(proof.to_bytes()).hexdigest())
    assert len(digests) == 1, "the declaration changed the proof"
    best = {k: min(r["prove_s"] for r in v) for k, v in runs.items()}
    return {"rows": n, "trace_generation_s": gen, "runs": runs, "prove_s_min": best,
            "host_over_declared": best["host_callback"] / best["declared"], "proof_sha256": digests.pop(),
            "residency": prover.last_residency}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[20, 24])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_extension.py measures on a CUDA device; none is visible")
    name, limit = card()
    res_kernel = kernel_resources()
    os.makedirs(args.out_dir, exist_ok=True)
    for log_n in args.sizes:
        ctx = ms.Context(0)
        res = {"card": name, "power_limit": limit, "kernels": res_kernel, "log_n": log_n, "timing": "CUDA events, seconds"}
        for key, (base, decl) in declarations(1 << log_n).items():
            res[key] = kernel_case(ctx, log_n, base, decl, args.reps)
        if log_n == 20:
            res["perm_prove_2p20"] = e2e_perm(20)
        with open(os.path.join(args.out_dir, f"bench_extension_2p{log_n}_h100.json"), "w") as f:
            json.dump(res, f, indent=1)
        print(json.dumps(res), flush=True)
        del ctx
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
