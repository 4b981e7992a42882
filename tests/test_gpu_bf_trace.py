"""GPU: the brainfuck execution trace built on the device (`simulate(..., device=0)`, include/ministark_bf.h).

  * the 17 base columns equal the host trace's bit for bit: the corpus, cycle_burner up to (40, 40, 60) (2^20 rows), a
    ~1000-cell tape walk, a program of more than 64 Ki instructions, one trace sized by its instruction table and one by
    its memory table, and 200 seeded random programs;
  * the helper columns and build_extension_columns_device equal the host trace's;
  * proofs from the device trace equal those from the host trace in both residencies, with validation, and the restated
    verifier accepts them; cycle_burner(40, 40, 60) reproduces the recorded proof;
  * after simulate returns only the (17, n) tensor is allocated; the VM's errors come before any allocation."""
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu

from test_bf_trace_cpu import ECHO, TAPE_WALK, _source, random_cases  # noqa: E402

LONG = "+-" * 40000 + "."                        # 80001 instructions: the ip histogram spans many blocks
INSTR_BOUND = "+" * 3000                         # L + P = 6001 rows against 3000 memory rows
MEM_BOUND = "+>" + "+" * 200 + "[-]" + "<+"      # cell 0 is touched at the first and the last cycle


def _both(src, inp=b""):
    from ministark_b200.examples import brainfuck as bf
    host, out_h = bf.simulate(src, inp)
    dev, out_d = bf.simulate(src, inp, device=0)
    assert out_d == out_h
    return host, dev


@pytest.mark.parametrize("src,inp", [(None, b""), (ECHO, b"hi"), ("burner:3,4,5", b""), ("burner:20,20,30", b""),
                                     ("burner:40,40,60", b""), (TAPE_WALK, b""), (LONG, b""), (INSTR_BOUND, b""),
                                     (MEM_BOUND, b"")])
def test_base_columns_equal_host_trace(src, inp):
    host, dev = _both(_source(src), inp)
    assert len(dev) == len(host)
    assert np.array_equal(dev.base_columns().cpu().numpy().view(np.uint64), host.base_columns())


def test_which_table_sets_n():
    from ministark_b200.examples import brainfuck as bf
    s = bf.simulate(INSTR_BOUND, device=0)[0].sizes
    assert s["instr_rows"] > s["mem_rows"] and s["n"] == 8192
    s = bf.simulate(MEM_BOUND, device=0)[0].sizes
    assert s["mem_rows"] > s["instr_rows"]
    assert s["n"] == 1 << (s["mem_rows"] - 1).bit_length()


def test_random_programs_equal_host_trace():
    bad = []
    for src, inp in random_cases(200, seed=2024):
        host, dev = _both(src, inp)
        if not np.array_equal(dev.base_columns().cpu().numpy().view(np.uint64), host.base_columns()):
            bad.append((src, inp))
    assert bad == []


@pytest.mark.parametrize("src", [None, "burner:20,20,30"])
def test_helper_and_extension_columns_equal_host_trace(src):
    import torch
    from ministark_b200 import Context
    host, dev = _both(_source(src))
    rng = np.random.default_rng(7)
    P = 2**64 - 2**32 + 1
    ch = [tuple(int(v) % P for v in rng.integers(0, 2**63, size=3)) for _ in range(11)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):            # the context and every tensor of the computation on one stream, as in a prover
        ctx = Context(0, stream=s.cuda_stream)
        base = dev.base_columns()
        aux = dev.helper_columns_device(ctx)
        want = host.build_extension_columns_device(ch, ctx, torch.from_numpy(host.base_columns().view(np.int64)).cuda())
        got = dev.build_extension_columns_device(ch, ctx, base)
        s.synchronize()
        assert np.array_equal(aux.cpu().numpy().view(np.uint64), host.helper_columns())
        assert torch.equal(got, want)


def test_matrix_is_complete_when_simulate_returns():
    """read on another stream at once, with nothing in between that waits for the device"""
    import torch
    from ministark_b200.examples import brainfuck as bf
    src = bf.cycle_burner(40, 40, 60)
    host, _ = bf.simulate(src)
    s = torch.cuda.Stream()
    dev, _ = bf.simulate(src, device=0)
    with torch.cuda.stream(s):
        copy = dev.base_columns().clone()
    s.synchronize()
    assert np.array_equal(copy.cpu().numpy().view(np.uint64), host.base_columns())


def _prove(trace, claim, opts, budget=None):
    from ministark_b200.air import ProofOptions
    from ministark_b200.prover import GpuProver
    p = GpuProver(0, memory_budget=budget)
    proof = p.prove(claim, ProofOptions(*opts), trace, validate=True).to_bytes()
    return proof, p.last_residency


@pytest.mark.parametrize("src", [None, "burner:20,20,30"])
def test_proofs_equal_host_trace_both_residencies(src):
    from ministark_b200 import FQ3
    from ministark_b200.air import Air, ProofOptions
    from ministark_b200.examples import brainfuck as bf
    from ministark_b200.prover import peak_bytes
    from oracle import stark_oracle as SO
    source = _source(src)
    host, dev = _both(source)
    _, out = bf.simulate(source)
    claim = bf.BrainfuckClaim(source, b"", out)
    opts = (19, 16, 20, 16, 16)
    o = ProofOptions(*opts)
    n = len(host)
    est = peak_bytes(n, 16, 17, 9, FQ3, Air(claim.AirConfig, n, None, o).ce_blowup_factor, 16)
    got = {}
    for residency, budget in [("resident", None), ("streamed", (est["streamed"] + est["resident"]) // 2)]:
        got[residency, "host"] = _prove(host, claim, opts, budget)
        got[residency, "device"] = _prove(dev, claim, opts, budget)      # the second proof of `dev` rebuilds its matrix
        assert got[residency, "device"] == got[residency, "host"] == (got[residency, "host"][0], residency)
    assert got["resident", "device"][0] == got["streamed", "device"][0]
    SO.verify(claim, got["resident", "device"][0], 10, lambda n, o: Air(claim.AirConfig, n, claim, ProofOptions(*o)))


def test_burner_40_40_60_reproduces_recorded_proof():
    from ministark_b200.examples import brainfuck as bf
    src = bf.cycle_burner(40, 40, 60)
    dev, out = bf.simulate(src, device=0)
    proof, residency = _prove(dev, bf.BrainfuckClaim(src, b"", out), (19, 16, 20, 16, 16))
    assert residency == "resident"
    assert hashlib.sha256(proof).hexdigest() == "cbf317503bf28883d7a008838857a4b905063d8eb2e0bf03a5cd499aab87c4a1"


def test_only_the_base_matrix_stays_allocated():
    import torch
    from ministark_b200.examples import brainfuck as bf
    live = lambda: torch.cuda.memory_stats(0)["allocation.all.current"]
    torch.cuda.synchronize()
    before, count = torch.cuda.memory_allocated(0), live()
    dev, _ = bf.simulate(bf.cycle_burner(20, 20, 30), device=0)
    # one live allocation, the (17, n) matrix; the allocator may book a cached block up to 1 MiB larger than asked
    assert live() - count == 1
    assert 0 <= torch.cuda.memory_allocated(0) - before - 17 * len(dev) * 8 <= 1 << 20
    del dev
    assert torch.cuda.memory_allocated(0) == before and live() == count


@pytest.mark.parametrize("src,inp,msg", [("<+", b"", "memory pointer leaves"), (",,", b"a", "input exhausted"),
                                         ("+[]", b"", "cycle cap")])
def test_errors_before_any_allocation(src, inp, msg):
    import torch
    import ministark_b200 as ms
    from ministark_b200.examples import brainfuck as bf
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(0)
    with pytest.raises(ms.MsError, match=msg):
        bf.simulate(src, inp, device=0, max_cycles=100_000)
    assert torch.cuda.memory_allocated(0) == before
