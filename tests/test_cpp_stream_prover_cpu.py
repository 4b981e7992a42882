"""CPU-only: residency selection, the streamed residency and the device-built brainfuck trace of the C++ prover
(include/ministark_prover.hpp), and the brainfuck command line (tools/bf_cli.cpp), linked against the CPU build of the
ABI: the oracle's CPU ABI with the streamed residency, the constraint check, the brainfuck trace and ms_device_memory
(tests/cpp/device_cpu_abi.c), compiled into a temporary directory.

  * mshost::peak_bytes equals prover.peak_bytes, and the selection rules and the refusal are the Python prover's;
  * streamed proofs equal the CPU restatement of the reference prover (fib, brainfuck) and its verifier accepts them;
  * bf::simulate_device gives the host trace's proof bytes, bf::test_rng_fq3 the Python draws;
  * the command line writes claim_bytes ‖ proof and its verify refuses every tampered claim or proof."""
import os
import subprocess

import pytest

from ministark_b200 import FP, FQ3
from ministark_b200.air import Air, ProofOptions
from ministark_b200.examples import brainfuck as bf
from ministark_b200.examples import fib
from ministark_b200.prover import _gib, peak_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
BF_OPTS = (19, 16, 20, 16, 16)


@pytest.fixture(scope="module")
def cpu_lib(tmp_path_factory, orc):
    d = tmp_path_factory.mktemp("device_abi")
    subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-Wno-unused-function", "-shared", "-o", str(d / "libms_dev_cpu_abi.so"),
                           os.path.join(ROOT, "tests", "cpp", "device_cpu_abi.c")])
    return d


def _link(lib_dir, source, name):
    exe = lib_dir / name
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-I", INCLUDE, source, "-o", str(exe),
                           "-L", str(lib_dir), "-lms_dev_cpu_abi", f"-Wl,-rpath,{lib_dir}"])
    return str(exe)


@pytest.fixture(scope="module")
def driver(cpu_lib):
    exe = _link(cpu_lib, os.path.join(ROOT, "tests", "cpp", "stream_prover_test.cpp"), "stream_prover_test")

    def run(*args, ok=True):
        out = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=900)
        if ok:
            assert out.returncode == 0, out.stderr
        return out
    return run


@pytest.fixture(scope="module")
def cli(cpu_lib):
    return _link(cpu_lib, os.path.join(ROOT, "tools", "bf_cli.cpp"), "ministark_bf")


def _between(est):
    return (est["resident"] + est["streamed"]) // 2


def _fib_case(log_rows, opts):
    trace, last = fib.gen_trace(8 << log_rows)
    claim = fib.FibClaim(last)
    mk = lambda n, o: Air(claim.AirConfig, n, claim.get_public_inputs(), ProofOptions(*o))
    n = 1 << log_rows
    est = peak_bytes(n, opts[1], 8, 0, FP, mk(n, opts).ce_blowup_factor, opts[3])
    return trace, claim, mk, est


def _bf_case(src, opts=BF_OPTS):
    trace, out = bf.simulate(src)
    claim = bf.BrainfuckClaim(src, b"", out)
    mk = lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o))
    n = len(trace)
    est = peak_bytes(n, opts[1], 17, 9, FQ3, mk(n, opts).ce_blowup_factor, opts[3])
    return trace, out, claim, mk, est


# ---------------------------------------------------------------------------------------------- residency
@pytest.mark.parametrize("log_n", [3, 10, 20, 24])
@pytest.mark.parametrize("beta", [2, 16])
@pytest.mark.parametrize("nbase,next_,fq", [(8, 0, FP), (17, 9, FQ3), (3, 2, FQ3)])
@pytest.mark.parametrize("ce,ff", [(1, 2), (4, 8), (16, 16)])
def test_peak_bytes_equal_python(driver, log_n, beta, nbase, next_, fq, ce, ff):
    if ce > beta:
        pytest.skip("ce blow-up above the LDE blow-up")
    got = [int(v) for v in driver("peak", 1 << log_n, beta, nbase, next_, fq, ce, ff).stdout.split()]
    want = peak_bytes(1 << log_n, beta, nbase, next_, fq, ce, ff)
    assert got == [want["resident"], want["streamed"]]


@pytest.mark.parametrize("log_rows,opts", [(7, (16, 4, 4, 8, 16)), (13, (32, 4, 8, 8, 64))])
def test_fib_streamed_bytes_equal_cpu_restatement(driver, orc, log_rows, opts):
    from oracle import stark_oracle as SO
    trace, claim, mk, est = _fib_case(log_rows, opts)
    want = SO.cpu_prove(claim, opts, trace.base_columns(), mk)
    residency, proof = driver("fib", log_rows, *opts, _between(est)).stdout.split()
    assert residency == "streamed" and bytes.fromhex(proof) == want
    SO.verify(claim, bytes.fromhex(proof), 10, mk)


@pytest.mark.parametrize("kind", ["host", "device"])
def test_brainfuck_streamed_bytes_equal_cpu_restatement(driver, orc, kind):
    from oracle import stark_oracle as SO
    trace, out, claim, mk, est = _bf_case(bf.HELLO_WORLD)
    want = SO.cpu_prove(claim, BF_OPTS, trace.base_columns(), mk, ext_builder=trace.build_extension_columns)
    residency, output, proof = driver("bf", "hello", *BF_OPTS, _between(est), kind).stdout.split()
    assert residency == "streamed" and output == "out:" + out.hex() and bytes.fromhex(proof) == want
    SO.verify(claim, bytes.fromhex(proof), 96, mk)


def test_selection_rules(driver):
    """resident at or above its estimate (and with no budget, where the CPU build reports no device limit), streamed from
    its estimate up to below the resident one, refused below the streamed one with the Python prover's text"""
    _, _, _, est = _fib_case(7, (16, 4, 4, 8, 16))
    r, s = est["resident"], est["streamed"]
    for budget, want in [(0, "resident"), (r, "resident"), (r + 1, "resident"), (r - 1, "streamed"), (s, "streamed")]:
        assert driver("fib", 7, 16, 4, 4, 8, 16, budget).stdout.split()[0] == want, budget
    out = driver("fib", 7, 16, 4, 4, 8, 16, s - 1, ok=False)
    assert out.returncode == 1
    want = (f"the proof does not fit on the device: it needs about {_gib(r)} resident or {_gib(s)} streamed, "
            f"and {_gib(s - 1)} is available")
    assert out.stderr.strip() == "stream_prover_test: " + want


@pytest.mark.parametrize("kind", ["host", "device"])
def test_refusal_reads_no_trace_and_allocates_nothing(driver, kind):
    n = 1 << 20
    est = peak_bytes(n, 16, 17, 9, FQ3, 16, 16)
    budget = est["streamed"] - 1
    lines = driver("refuse", budget, kind).stdout.splitlines()
    assert lines == [f"the proof does not fit on the device: it needs about {_gib(est['resident'])} resident or "
                     f"{_gib(est['streamed'])} streamed, and {_gib(budget)} is available",
                     "extension built: 0", "allocations: 0"]


# ---------------------------------------------------------------------------------------------- brainfuck
def test_test_rng_fq3_equals_python(driver):
    got = [tuple(int(v) for v in line.split()) for line in driver("rng", 5).stdout.splitlines()]
    assert got == bf.test_rng_fq3(5)


@pytest.mark.parametrize("which,opts", [("hello", BF_OPTS), ("burner:4:4:4", (16, 16, 6, 8, 8)), ("burner:3:4:5", (8, 16, 4, 16, 16))])
def test_device_trace_proof_equals_host_trace_proof(driver, which, opts):
    src = bf.HELLO_WORLD if which == "hello" else bf.cycle_burner(*[int(v) for v in which.split(":")[1:]])
    *_, est = _bf_case(src, opts)
    for budget, residency in [(0, "resident"), (_between(est), "streamed")]:
        host = driver("bf", which, *opts, budget, "host").stdout.split()
        dev = driver("bf", which, *opts, budget, "device").stdout.split()
        assert host == dev and dev[0] == residency


# ---------------------------------------------------------------------------------------------- command line
def test_cli_round_trip_and_refusals(cli, orc, tmp_path):
    from oracle import stark_oracle as SO
    src_path, proof_path = tmp_path / "hello.bf", tmp_path / "hello.proof"
    src_path.write_text(bf.HELLO_WORLD)
    out = subprocess.run([cli, "prove", str(src_path), "--dst", str(proof_path)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    trace, output, claim, mk, _ = _bf_case(bf.HELLO_WORLD)
    assert f'Program output: "{output.decode()}"' in out.stdout and "Residency: resident" in out.stdout
    assert "Proof security (conjectured): 96bit" in out.stdout
    want = SO.cpu_prove(claim, BF_OPTS, trace.base_columns(), mk, ext_builder=trace.build_extension_columns)
    blob = proof_path.read_bytes()
    claim_part = claim.public_inputs_bytes(claim)
    assert blob == claim_part + want

    def verify(*extra, source=str(src_path), proof=str(proof_path), output=output.decode()):
        return subprocess.run([cli, "verify", source, "--proof", proof, "--output", output] + list(extra), capture_output=True,
                              text=True, timeout=900)

    ok = verify()
    assert ok.returncode == 0 and ok.stdout.startswith("Proof verified in:"), ok.stderr
    assert "different output" in verify(output="Hello World?\n").stderr
    assert "different input" in verify("--input", "x").stderr
    other = tmp_path / "other.bf"
    other.write_text(bf.HELLO_WORLD + ">")
    assert "different source code" in verify(source=str(other)).stderr
    flipped = bytearray(blob)
    flipped[len(claim_part) + (len(blob) - len(claim_part)) // 2] ^= 0x10
    bad = tmp_path / "flipped.proof"
    bad.write_bytes(bytes(flipped))
    r = verify(proof=str(bad))
    assert r.returncode == 1 and "verification failed" in r.stderr
    for cut in (10, len(claim_part) + 100):
        bad.write_bytes(blob[:cut])
        r = verify(proof=str(bad))
        assert r.returncode == 1 and "ministark_bf verify:" in r.stderr and ("truncated" in r.stderr or "verification failed" in r.stderr)
    r = verify(proof=str(tmp_path / "missing.proof"))
    assert r.returncode == 1 and "cannot read" in r.stderr


def test_device_header_is_bound_exported_and_separate(cpu_lib):
    import ctypes as C
    from ministark_b200 import _lib
    declared = _lib.header_symbols(_lib.DEVICE_HEADER_PATH)
    assert declared == sorted(_lib._DEVICE_SIGS) == ["ms_device_memory"]
    others = set(_lib.header_symbols()) | set(_lib.header_symbols(_lib.STREAM_HEADER_PATH)) | \
        set(_lib.header_symbols(_lib.BF_HEADER_PATH)) | set(_lib.header_symbols(_lib.CHECK_HEADER_PATH))
    assert not set(declared) & others
    product, cpu = C.CDLL(_lib.LIB_PATH), C.CDLL(str(cpu_lib / "libms_dev_cpu_abi.so"))
    assert all(hasattr(product, s) and hasattr(cpu, s) for s in declared)
    # the CPU build reports no device limit, so that off a GPU only an explicit budget limits a proof
    h, free, total = C.c_void_p(), C.c_size_t(), C.c_size_t()
    assert cpu.ms_ctx_create(0, C.byref(h)) == 0
    assert cpu.ms_device_memory(h, C.byref(free), C.byref(total)) == 0
    assert free.value == total.value == 2**64 - 1
    cpu.ms_ctx_destroy(h)
