"""CPU-only: the product's Python provers executed end to end without a GPU (harness: tests/cpu_device.py — the CPU
oracle's build of the C ABI underneath `ministark_b200._lib`, host tensors, no-op streams; the product has no such mode).

  * `GpuProver` (ministark_b200/prover.py): proof bytes == oracle/stark_oracle.cpu_prove for examples/fib, the Fq3
    permutation AIR and examples/brainfuck (extension columns through `build_extension_columns_device`);
  * `ShardedProver` (ministark_b200/prover_mgpu.py) over gloo, world size 2 and 4: every matrix sharded by LDE coset
    blocks, FRI layers by rows, Merkle paths assembled from their owners — the bytes must equal the single prover's;
    `validate=True` is refused before the trace is read.  This is the CPU cover of the N > 1 prover path (the NCCL run of the same code is tests/test_gpu_multi.py).
Every multi-process case runs in spawned workers that install the harness themselves; the pytest process never does."""
import os
import socket
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _make_case(which):
    from ministark_b200.examples import brainfuck as bf
    from ministark_b200.examples import fib, perm
    if which.startswith("fib"):
        _, log_rows, opts = which.split(":")
        trace, last = fib.gen_trace(8 << int(log_rows))
        return fib.FibClaim(last), tuple(int(v) for v in opts.split(",")), trace
    if which == "perm":
        return perm.PermClaim(), (16, 8, 4, 4, 8), perm.gen_trace(1 << 8, seed=3)
    src = bf.HELLO_WORLD if which == "brainfuck" else bf.cycle_burner(4, 4, 4)
    trace, output = bf.simulate(src)
    return bf.BrainfuckClaim(src, b"", output), ((19, 16, 20, 16, 16) if which == "brainfuck" else (16, 16, 6, 8, 8)), trace


def _cpu_restatement(which):
    from ministark_b200.air import Air, ProofOptions
    from oracle import stark_oracle as SO
    claim, opts, trace = _make_case(which)
    pub = claim if which in ("brainfuck", "burner") else claim.get_public_inputs()
    mk = lambda n, o: Air(claim.AirConfig, n, pub, ProofOptions(*o))
    ext = getattr(trace, "build_extension_columns", None)
    want = SO.cpu_prove(claim, opts, trace.base_columns(), mk, ext_builder=ext if claim.AirConfig.NUM_EXTENSION_COLUMNS else None)
    SO.verify(claim, want, 10, mk)
    return want


def _single_worker(which, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import cpu_device
    cpu_device.install()
    from ministark_b200.air import ProofOptions
    from ministark_b200.prover import GpuProver
    claim, opts, trace = _make_case(which)
    if which.startswith("fib"):         # the trace tiled from its period on the "device" (here: host memory), as a resident tensor
        from ministark_b200.examples import fib
        trace, _ = fib.gen_trace(8 * len(trace), device="cpu")
    p = GpuProver(0)
    first = p.prove(claim, ProofOptions(*opts), trace).to_bytes()
    q.put((first, p.prove(claim, ProofOptions(*opts), trace).to_bytes()))       # second proof: cached AIR programs re-bound


@pytest.mark.parametrize("which", ["fib:7:16,4,4,8,16", "fib:6:10,2,0,2,8", "fib:9:32,4,8,8,64", "fib:8:16,16,3,16,4", "perm", "brainfuck", "burner"])
def test_python_prover_bytes_equal_cpu_restatement(orc, which):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_single_worker, args=(which, q))
    p.start()
    first, second = q.get(timeout=600)
    p.join(timeout=60)
    assert p.exitcode == 0
    assert first == second == _cpu_restatement(which)


def _sharded_worker(rank, world, port, which, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.setdefault("OMP_NUM_THREADS", "2")           # `world` processes share the host cores (read when libgomp loads)
    import cpu_device
    cpu_device.install()
    import torch.distributed as dist
    from ministark_b200.air import ProofOptions
    from ministark_b200.prover_mgpu import ShardedProver
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        claim, opts, trace = _make_case(which)
        prover = ShardedProver(dist, rank)
        first = prover.prove(claim, ProofOptions(*opts), trace).to_bytes()
        second = prover.prove(claim, ProofOptions(*opts), trace).to_bytes()

        class Unread:
            """a witness whose columns must not be read: validate=True is refused before any work"""
            def __len__(self):
                return len(trace)

            def base_columns(self):
                raise AssertionError("the base columns were read")

        try:
            prover.prove(claim, ProofOptions(*opts), Unread(), validate=True)
            refusal = None
        except Exception as e:
            refusal = f"{type(e).__name__}: {e}"
        q.put((rank, first, second, refusal))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,which", [(2, "fib:7:16,4,4,8,16"), (2, "fib:10:32,4,8,8,64"), (2, "perm"), (2, "brainfuck"),
                                         (4, "fib:9:32,4,8,8,64"), (4, "brainfuck"), (2, "fib:6:10,2,0,2,8"), (8, "fib:8:16,8,3,4,8")])
def test_sharded_prover_over_gloo_bytes_equal_cpu_restatement(orc, world, which):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, port, which, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = [q.get(timeout=900) for _ in range(world)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    want = _cpu_restatement(which)
    for rank, first, second, refusal in got:        # every rank assembles the same proof, twice
        assert first == second == want, f"rank {rank}"
        assert refusal and refusal.startswith("ProvingError: ") and "sharded prover does not validate" in refusal, refusal


def _bad_input_worker(q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import cpu_device
    cpu_device.install()
    import numpy as np
    from ministark_b200.air import ProofOptions
    from ministark_b200.examples import fib
    from ministark_b200.prover import GpuProver, ProvingError
    trace, last = fib.gen_trace(8 << 6)
    cols = trace.base_columns().copy()
    cols[3, 17] ^= np.uint64(1)
    claim = fib.FibClaim(last)

    class Witness:
        def __init__(self, c):
            self.c = c

        def __len__(self):
            return self.c.shape[1]

        def base_columns(self):
            return self.c

        def build_extension_columns(self, challenges):
            return None

    p = GpuProver(0)
    bad = p.prove(claim, ProofOptions(10, 4, 0, 8, 4), Witness(cols)).to_bytes()
    try:
        p.prove(claim, ProofOptions(10, 4, 0, 8, 4), Witness(cols[:7]))
        shape_error = None
    except ProvingError as e:
        shape_error = str(e)
    q.put((bad, shape_error))


def test_python_prover_on_bad_inputs(orc):
    """the prover never checks the AIR (src/debug.rs is debug-only): a trace that violates it still yields a proof — the
    same bytes as the restated reference prover's — which the verifier refuses at the OOD consistency check
    (src/verifier.rs:84-86); a trace of the wrong shape is an error before any device work"""
    import numpy as np
    import torch.multiprocessing as mp
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.examples import fib
    from oracle import stark_oracle as SO
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_bad_input_worker, args=(q,))
    p.start()
    bad, shape_error = q.get(timeout=600)
    p.join(timeout=60)
    assert p.exitcode == 0
    trace, last = fib.gen_trace(8 << 6)
    cols = trace.base_columns().copy()
    cols[3, 17] ^= np.uint64(1)
    claim = fib.FibClaim(last)
    mk = lambda n, o: Air(claim.AirConfig, n, claim.get_public_inputs(), ProofOptions(*o))
    assert bad == SO.cpu_prove(claim, (10, 4, 0, 8, 4), cols, mk)
    with pytest.raises(SO.VerificationError, match="out-of-domain"):
        SO.verify(claim, bad, 10, mk)
    assert shape_error and "expected 8 base columns" in shape_error


def test_harness_is_not_reachable_from_the_product():
    """the loader the product uses opens only its own library; the harness lives under tests/ and is installed explicitly"""
    import inspect
    from ministark_b200 import _lib
    assert _lib.LIB_PATH.endswith("libministark_b200.so") and not getattr(_lib, "_cpu_device_installed", False)
    assert 'b"sm_90a" not in lib.ms_version()' in inspect.getsource(_lib.load)      # the loader insists on the CUDA build
    for dirpath, _, files in os.walk(os.path.join(ROOT, "ministark_b200")):
        for f in files:
            if f.endswith(".py"):
                assert "cpu_device" not in open(os.path.join(dirpath, f)).read(), f
