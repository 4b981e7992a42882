"""GPU: the "streamed_host" residency, whose Merkle node heaps live in pinned host memory (include/ministark_host_nodes.h,
ministark_b200/prover.py, include/ministark_prover.hpp, tools/bf_cli.cpp --host-memory).

  * ms_merkle_commit_block_sha256_host gives the local heaps and, with the top heap, the root of ms_merkle_commit_sha256,
    whose heap is the CPU oracle's;
  * it refuses pageable host memory and device memory with an error code;
  * the Python and C++ provers forced into streamed_host give the resident path's bytes on brainfuck at 2^16 and 2^20 rows,
    and the command line the recorded 2^20 proof;
  * the torch peak stays within the device estimate and the pinned bytes within the host estimate.
The same paths run on the CPU build in tests/test_host_nodes_cpu.py."""
import hashlib
import os
import subprocess

import numpy as np
import pytest
import torch

from ministark_b200 import FP, FQ3, Context, MsError
from ministark_b200.air import Air, ProofOptions
from ministark_b200.cosets import heap_location
from ministark_b200.examples import brainfuck as bf
from ministark_b200.prover import GpuProver, peak_bytes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_DIR = os.path.join(ROOT, "ministark_b200")
CLI = os.path.join(LIB_DIR, "ministark_bf")
BF_OPTS = (19, 16, 20, 16, 16)
P = 2**64 - 2**32 + 1
PROOF_SHA256_2P20 = "cbf317503bf28883d7a008838857a4b905063d8eb2e0bf03a5cd499aab87c4a1"


def _matrix(ncols, N, field, seed):
    rng = np.random.default_rng(seed)
    words = rng.integers(0, P, size=(ncols, N * field), dtype=np.uint64)
    return torch.from_numpy(words.view(np.int64)).cuda()


# five columns at every (log_N, log_b); the one-block (Fp 1, 7; Fq3 1, 3), constant-padding (Fp 8; Fq3 8 = 24 words)
# and multi-block (Fp 17) leaf shapes at 16 blocks of 256 rows.  The five-column cases keep the ids they had before the
# column count was a parameter.
_HOST_CASES = ([(field, 5, log_N, log_b) for log_N, log_b in [(12, 0), (12, 4), (14, 1), (16, 4), (16, 3)] for field in [FP, FQ3]]
               + [(FP, ncols, 12, 4) for ncols in (1, 7, 8, 17)] + [(FQ3, ncols, 12, 4) for ncols in (1, 3, 8)])


@pytest.mark.parametrize("field,ncols,log_N,log_b", _HOST_CASES,
                         ids=[f"{N}-{b}-{f}" + ("" if c == 5 else f"-{c}cols") for f, c, N, b in _HOST_CASES])
def test_block_host_heaps_equal_the_device_tree(orc, field, ncols, log_N, log_b):
    ctx = Context(0)
    N, beta = 1 << log_N, 1 << log_b
    log_n = log_N - log_b
    n = 1 << log_n
    mat = _matrix(ncols, N, field, seed=log_N * 10 + log_b + field)
    leaves, nodes = torch.empty((N, 4), dtype=torch.int64, device="cuda"), torch.empty((N, 4), dtype=torch.int64, device="cuda")
    root = ctx.merkle_commit(mat, field, N, ncols, leaves=leaves, nodes=nodes)
    want = nodes.cpu().numpy().view(np.uint8)
    assert np.array_equal(want, orc.merkle_nodes(orc.hash_rows(mat.cpu().numpy().view(np.uint64), field)))
    local = torch.full((beta, n, 32), 0xAB, dtype=torch.uint8).pin_memory()
    top = torch.zeros((2 * beta, 4), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()                # the context runs on its own stream
    for q in range(beta):
        ctx.merkle_commit_block_host(mat.data_ptr() + q * n * field * 8, field, log_n, ncols, local[q], top[beta + q], col_stride=N)
    if beta > 1:
        ctx.merkle_nodes(top[beta:], top, beta)
    ctx.sync()
    top = top.cpu().numpy().view(np.uint8)
    heaps = local.numpy()
    assert not heaps[:, 0].any()
    for i in range(1, N):
        b, j = heap_location(i, log_b)
        assert np.array_equal(top[j] if b is None else heaps[b, j], want[i]), (i, b, j)
    assert top[1].tobytes() == root
    ctx.close()


def test_pageable_and_device_subtrees_are_refused():
    ctx = Context(0)
    mat = _matrix(2, 1 << 10, FP, seed=1)
    root = torch.zeros(4, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    for buf, kind in [(np.zeros((1 << 10, 32), dtype=np.uint8), "pageable host"),
                      (torch.zeros((1 << 10, 32), dtype=torch.uint8, device="cuda"), "device")]:
        with pytest.raises(MsError, match=f"{kind} memory, not pinned host memory"):
            ctx.merkle_commit_block_host(mat, FP, 10, 2, buf, root)
    ctx.close()


def _bf_case(a, b, c):
    src = bf.cycle_burner(a, b, c)
    trace, output = bf.simulate(src, device=0)
    claim = bf.BrainfuckClaim(src, b"", output)
    n = len(trace)
    est = peak_bytes(n, 16, 17, 9, FQ3, Air(claim.AirConfig, n, None, ProofOptions(*BF_OPTS)).ce_blowup_factor, 16)
    return src, trace, claim, n, est


def _between(est):
    return (est["streamed_host"] + est["streamed"]) // 2


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("host_nodes_gpu") / "host_nodes_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "host_nodes_test.cpp"), "-o", exe,
                           "-L", LIB_DIR, "-lministark_b200", f"-Wl,-rpath,{LIB_DIR}"])

    def run(*args):
        out = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stderr
        return out.stdout
    return run


@pytest.mark.parametrize("burner,log_n", [((10, 10, 60), 16), ((40, 40, 60), 20)])
def test_streamed_host_python_and_cpp_equal_resident(driver, burner, log_n):
    src, trace, claim, n, est = _bf_case(*burner)
    assert n == 1 << log_n
    want = GpuProver.shared(0).prove(claim, ProofOptions(*BF_OPTS), trace).to_bytes()
    if log_n == 20:
        assert hashlib.sha256(want).hexdigest() == PROOF_SHA256_2P20
    p = GpuProver(0, memory_budget=_between(est), host_memory_budget=est["host"])
    trace, _ = bf.simulate(src, device=0)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    proof = p.prove(claim, ProofOptions(*BF_OPTS), trace, validate=log_n == 16)
    peak = torch.cuda.max_memory_allocated() - before
    assert p.last_residency == "streamed_host" and proof.to_bytes() == want
    assert peak <= est["streamed_host"], (peak, est)
    assert 0 < p.pinned_bytes <= est["host"] and "pin_host_memory" in proof.timings
    p.release_host_memory()
    which = "burner:%d:%d:%d" % burner
    residency, pinned, out, got = driver("bf", which, *BF_OPTS, _between(est), est["host"]).split()
    assert residency == "streamed_host" and 0 < int(pinned) <= est["host"] and bytes.fromhex(got) == want


def test_cli_host_memory_proves_the_recorded_2p20_proof(tmp_path):
    src = bf.cycle_burner(40, 40, 60)
    est = peak_bytes(1 << 20, 16, 17, 9, FQ3, 16, 16)
    path, dst = tmp_path / "b.bf", tmp_path / "b.proof"
    path.write_text(src)
    out = subprocess.run([CLI, "prove", str(path), "--dst", str(dst), "--memory-budget", f"{_between(est) / 2**30:.3f}",
                          "--host-memory", f"{est['host'] / 2**30 + 0.01:.3f}"], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    assert "Residency: streamed_host" in out.stdout and "Pinned host memory:" in out.stdout, out.stdout
    claim = bf.BrainfuckClaim(src, b"", b"")
    claim = claim.public_inputs_bytes(claim)
    blob = dst.read_bytes()
    assert blob.startswith(claim) and hashlib.sha256(blob[len(claim):]).hexdigest() == PROOF_SHA256_2P20
    ver = subprocess.run([CLI, "verify", str(path), "--proof", str(dst), "--output", ""], capture_output=True, text=True, timeout=900)
    assert ver.returncode == 0, ver.stderr
