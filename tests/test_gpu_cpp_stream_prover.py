"""GPU: the C++ prover's two residencies and its device-built brainfuck trace (include/ministark_prover.hpp,
tests/cpp/stream_prover_test.cpp) and the brainfuck command line (ministark_b200/ministark_bf, built by build() from
tools/bf_cli.cpp) on the product library.  The streamed and resident C++ proofs must equal the Python prover's bytes;
the command line must reproduce the recorded 2^20-row proof in both residencies, and refuse a proof that cannot fit
before it allocates anything.  The same binaries run on the CPU build in tests/test_cpp_stream_prover_cpu.py."""
import ctypes as C
import hashlib
import os
import subprocess

import pytest

from ministark_b200 import FP, FQ3
from ministark_b200.air import Air, ProofOptions
from ministark_b200.examples import brainfuck as bf
from ministark_b200.examples import fib
from ministark_b200.prover import GpuProver, _gib, peak_bytes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_DIR = os.path.join(ROOT, "ministark_b200")
CLI = os.path.join(LIB_DIR, "ministark_bf")
BF_OPTS = (19, 16, 20, 16, 16)
BURNER_2P20 = (40, 40, 60)
PROOF_SHA256_2P20 = "cbf317503bf28883d7a008838857a4b905063d8eb2e0bf03a5cd499aab87c4a1"


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("cpp_gpu") / "stream_prover_test")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "stream_prover_test.cpp"), "-o", exe,
                           "-L", LIB_DIR, "-lministark_b200", f"-Wl,-rpath,{LIB_DIR}"])

    def run(*args):
        out = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stderr
        return out.stdout
    return run


def _between(est):
    return (est["resident"] + est["streamed"]) // 2


def test_device_memory_entry_point():
    from ministark_b200 import _lib
    lib = _lib.load()
    h, free, total = C.c_void_p(), C.c_size_t(), C.c_size_t()
    assert lib.ms_ctx_create(0, C.byref(h)) == 0
    try:
        assert lib.ms_device_memory(h, C.byref(free), C.byref(total)) == 0
        assert 0 < free.value <= total.value and total.value > 16 << 30
        assert lib.ms_device_memory(h, None, None) == 0
    finally:
        lib.ms_ctx_destroy(h)


def test_fib_streamed_resident_and_python_proofs_identical(driver):
    log_rows, opts = 13, (32, 4, 8, 8, 64)
    trace, last = fib.gen_trace(8 << log_rows)
    claim = fib.FibClaim(last)
    n = 1 << log_rows
    est = peak_bytes(n, opts[1], 8, 0, FP, Air(claim.AirConfig, n, None, ProofOptions(*opts)).ce_blowup_factor, opts[3])
    want = GpuProver.shared(0).prove(claim, ProofOptions(*opts), trace).to_bytes()
    for budget, residency in [(0, "resident"), (_between(est), "streamed")]:
        got, proof = driver("fib", log_rows, *opts, budget).split()
        assert got == residency and bytes.fromhex(proof) == want


@pytest.mark.parametrize("which", ["hello", "burner:10:10:60"])
def test_brainfuck_streamed_resident_and_python_proofs_identical(driver, which):
    """hello_world and a cycle_burner of 2^16 rows, from the host trace and from the device trace"""
    src = bf.HELLO_WORLD if which == "hello" else bf.cycle_burner(10, 10, 60)
    trace, output = bf.simulate(src, device=0)
    n = len(trace)
    assert which == "hello" or n == 1 << 16
    claim = bf.BrainfuckClaim(src, b"", output)
    want = GpuProver.shared(0).prove(claim, ProofOptions(*BF_OPTS), trace).to_bytes()
    est = peak_bytes(n, 16, 17, 9, FQ3, Air(claim.AirConfig, n, None, ProofOptions(*BF_OPTS)).ce_blowup_factor, 16)
    for budget, residency in [(0, "resident"), (_between(est), "streamed")]:
        for kind in ("host", "device"):
            got, out, proof = driver("bf", which, *BF_OPTS, budget, kind).split()
            assert (got, out) == (residency, "out:" + output.hex()) and bytes.fromhex(proof) == want, (budget, kind)


def test_refusal_allocates_nothing(driver):
    est = peak_bytes(1 << 20, 16, 17, 9, FQ3, 16, 16)
    budget = est["streamed"] - 1
    for kind in ("host", "device"):
        assert driver("refuse", budget, kind).splitlines() == [
            f"the proof does not fit on the device: it needs about {_gib(est['resident'])} resident or "
            f"{_gib(est['streamed'])} streamed, and {_gib(budget)} is available", "extension built: 0", "allocations: 0"]


def _cli_prove(tmp_path, name, *extra):
    src, dst = tmp_path / f"{name}.bf", tmp_path / f"{name}.proof"
    src.write_text(bf.cycle_burner(*BURNER_2P20))
    out = subprocess.run([CLI, "prove", str(src), "--dst", str(dst)] + list(extra), capture_output=True, text=True, timeout=900)
    return out, src, dst


def test_cli_proves_the_recorded_2p20_proof_in_both_residencies(tmp_path):
    source = bf.cycle_burner(*BURNER_2P20)
    est = peak_bytes(1 << 20, 16, 17, 9, FQ3, 16, 16)
    between_gib = _between(est) / 2**30
    blobs = {}
    for name, extra, residency in [("default", [], "resident"), ("budget", ["--memory-budget", f"{between_gib:.3f}"], "streamed")]:
        out, src, dst = _cli_prove(tmp_path, name, *extra)
        assert out.returncode == 0, out.stderr
        assert "rows=1048576" in out.stdout and f"Residency: {residency}" in out.stdout, out.stdout
        assert 'Program output: ""' in out.stdout           # the burner prints nothing
        output = b""
        blob = dst.read_bytes()
        claim = bf.BrainfuckClaim(source, b"", output)
        claim = claim.public_inputs_bytes(claim)
        assert blob.startswith(claim)
        assert hashlib.sha256(blob[len(claim):]).hexdigest() == PROOF_SHA256_2P20
        blobs[name] = blob
        ver = subprocess.run([CLI, "verify", str(src), "--proof", str(dst), "--output", output.decode()], capture_output=True,
                             text=True, timeout=900)
        assert ver.returncode == 0 and "Proof verified in:" in ver.stdout, ver.stderr
    assert blobs["default"] == blobs["budget"]


def test_cli_refuses_a_proof_that_does_not_fit(tmp_path):
    out, _, dst = _cli_prove(tmp_path, "small", "--memory-budget", "1")
    assert out.returncode == 1 and "the proof does not fit on the device" in out.stderr and not dst.exists()
