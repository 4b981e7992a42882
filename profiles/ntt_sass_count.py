#!/usr/bin/env python
"""Static SASS figures of the NTT networks, no GPU needed: csrc/ntt_tma.cu and a one-network probe kernel (load 16
words, dft_regs<4, INV>, store 16 words) are compiled for sm_90a with nvcc, with and without -DMS_DFT_REPAIR_EACH=1
(the networks that repair every butterfly), disassembled with cuobjdump, and counted by opcode class.  The kernels'
consumer loops run one tile per iteration, so the counts are per-thread instructions per tile; per element = / 16.

    python profiles/ntt_sass_count.py

Prints one markdown table row per kernel and build: ALU pipe (IADD3 LOP3 SHF SEL ISETP LEA VIADD), FMA pipe (IMAD*),
all instructions, and ptxas registers / spill stores."""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ministark_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ALU = ("IADD3", "LOP3", "SHF", "SEL", "ISETP", "LEA", "VIADD")
PROBE = r"""
#include "dft.cuh"
using namespace msntt;
template <bool INV> __global__ void probe_dft16(u64 *p) {
    u64 x[16];
    static_for<0, 16>([&](auto K) { x[K] = p[threadIdx.x + 256 * (int)K]; });
    dft_regs<4, INV>(x);
    static_for<0, 16>([&](auto K) { p[threadIdx.x + 256 * (int)K] = x[K]; });
}
template __global__ void probe_dft16<false>(u64 *);
template __global__ void probe_dft16<true>(u64 *);
"""


def compile_cubin(src, extra, tmp):
    out = os.path.join(tmp, os.path.basename(src) + ".cubin")
    r = subprocess.run([NVCC, "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin", "-I", CSRC,
                        "-I", os.path.join(CSRC, "build"), "-Xptxas", "-v", *extra, "-o", out, src],
                       capture_output=True, text=True, check=True)
    spills, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line) or re.search(r"Function properties for (\w+)", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and cur:
            spills[cur] = int(m.group(1))
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            spills[cur] = (spills.get(cur, 0), int(m.group(1)))
    return out, spills


def sass_counts(cubin):
    sass = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True, check=True).stdout
    per, cur = collections.defaultdict(collections.Counter), None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\w+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", line)
        if m and cur:
            per[cur][m.group(1).split(".")[0]] += 1
    return per


def short_name(mangled):
    """ntt_tma_kernel<TYPE, INV, BITREV, HAS_PRE, G> / ntt_tma_scatter_kernel<G> / probe_dft16<INV> from the mangled name"""
    m = re.search(r"(probe_dft16|ntt_tma_scatter_kernel|ntt_tma_kernel)I(.*?)EEv", mangled)
    if not m:
        return mangled
    args = [a.replace("Li", "").replace("Lb", "") for a in re.findall(r"L[ib]\d+", m.group(2))]
    return f"{m.group(1)}<{', '.join(args)}>"


def main():
    print("| build | kernel | ALU pipe | ALU / element | IMAD | all | registers | spill stores |")
    print("|---|---|---|---|---|---|---|---|")
    with tempfile.TemporaryDirectory() as tmp:
        probe = os.path.join(tmp, "probe.cu")
        with open(probe, "w") as f:
            f.write(PROBE)
        for label, extra in (("repair each butterfly (-DMS_DFT_REPAIR_EACH=1)", ["-DMS_DFT_REPAIR_EACH=1"]), ("96-bit limbs", [])):
            for src in (probe, os.path.join(CSRC, "ntt_tma.cu")):
                cubin, regs = compile_cubin(src, extra, tmp)
                per = sass_counts(cubin)
                for k in sorted(per):
                    ops = per[k]
                    alu = sum(v for op, v in ops.items() if op in ALU)
                    imad = sum(v for op, v in ops.items() if op.startswith("IMAD"))
                    sp, nr = regs.get(k, (0, None)) if isinstance(regs.get(k), tuple) else (regs.get(k, 0), None)
                    name = short_name(k)
                    print(f"| {label} | `{name}` | {alu} | {alu / 16:.1f} | {imad} | {sum(ops.values())} | {nr} | {sp} |")


if __name__ == "__main__":
    sys.exit(main())
