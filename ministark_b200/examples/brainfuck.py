"""examples/brainfuck (BrainSTARK): the reference's second example AIR — 17 base-field + 9 Fq3 extension columns.

    VM + base tables           examples/brainfuck/vm.rs:68-381
    column layout              examples/brainfuck/tables.rs:45-185
    extension columns          examples/brainfuck/trace.rs:70-279
    constraints                examples/brainfuck/constraints.rs, assembled in air.rs:77-135
    hints (evaluation terminals) examples/brainfuck/air.rs:34-75,138-164
    claim / coin / options     examples/brainfuck/main.rs:56-105

The constraints are the AIR's definition, so they are restated term by term (including the product — not sum — in
the processor table's memory-permutation transition, constraints.rs:214-224, which makes that constraint vacuous).
Values are canonical integers on the host; matrices are Montgomery words.  This is application-level host code: the
VM and the running products/evaluations are sequential scans in plain Python, good for the programs the reference
ships (hello_world pads to 2^11 rows).

Unverifiable restatement (SURVEY.md §8c): the two permutation initial values come from `ark_std::test_rng()` =
ChaCha12 (rand 0.8 StdRng) with ark-std's fixed seed; ChaCha12, the seed and `Fq3::rand` are restated from upstream
knowledge.  Soundness does not depend on them (any initial values verify); byte parity with the reference binary does.
"""
import numpy as np

from .. import expr as E
from ..air import AirConfig, ProofOptions, domain_generator
from ..prover import Stark, Trace

P = E.P
_R = 2**64
_RINV = pow(_R, -1, P)
OPTIONS = ProofOptions(19, 16, 20, 16, 16)          # main.rs:92-105, 96-bit security
SECURITY_LEVEL = 96

HELLO_WORLD = ("++++++++++[>+++++++>++++++++++>+++>+<<<<-]>++.>+.+++++++..+++.>++.<<+++++++++++++++.>.+++.------.--------.")


def cycle_burner(a, b, c):
    """a * b * (3c + 5) + O(a) cycles in three nested count-down loops; no cell ever exceeds max(a, b, c), so the
    u8 tape never wraps (a wrap would violate the MemVal transition constraints)."""
    assert max(a, b, c) < 256
    return "+" * a + "[>" + "+" * b + "[>" + "+" * c + "[-]<-]<-]"


OPCODES = [ord(c) for c in "><+-.,[]"]               # OpCode::VALUES order (vm.rs:23-33)
INC_PTR, DEC_PTR, INC, DEC, WRITE, READ, LOOP_BEGIN, LOOP_END = OPCODES

# ---- column indices (tables.rs): base 0..16, extension 17..25
CYCLE, IP, CURR_INSTR, NEXT_INSTR, MP, MEM_VAL, MEM_VAL_INV, DUMMY = range(8)          # processor
M_CYCLE, M_MP, M_MEM_VAL, M_DUMMY = range(8, 12)                                        # memory
I_IP, I_CURR_INSTR, I_NEXT_INSTR = range(12, 15)                                        # instruction
IN_VALUE, OUT_VALUE = 15, 16
P_INSTR_PERM, P_MEM_PERM, P_IN_EVAL, P_OUT_EVAL, M_PERM, I_PROC_PERM, I_PROG_EVAL, IN_EVAL, OUT_EVAL = range(17, 26)
# challenges / hints (tables.rs:11-42)
CH_A, CH_B, CH_C, CH_D, CH_E, CH_F, CH_ALPHA, CH_BETA, CH_GAMMA, CH_DELTA, CH_ETA = range(11)
H_INSTRUCTION, H_INPUT, H_INPUT_OFFSET, H_OUTPUT, H_OUTPUT_OFFSET = range(5)


# ---------------------------------------------------------------- VM (vm.rs)
def compile_program(source):
    program, stack = [], []
    for ch in source:
        if ch not in "><+-.,[]":
            continue
        program.append(ord(ch))
        if ch == "[":
            program.append(0)
            stack.append(len(program) - 1)
        elif ch == "]":
            last = stack.pop()
            program.append(last + 1)
            program[last] = len(program)
    return program


def simulate(source, input_bytes=b"", device=None, max_cycles=1 << 26):
    """returns (BrainfuckTrace, output bytes).
    device: run the VM natively (ms_bf_run) and build every table ON that device instead: returns
    (BrainfuckDeviceTrace, output bytes), whose base_columns() is the resident (17, n) tensor, identical word for word to
    the host trace's.  Raises MsError, before anything of the trace's size is allocated, when the memory pointer leaves
    the 1024-cell tape, the input runs out, or max_cycles cycles do not end the program."""
    if device is not None:
        return _simulate_device(source, input_bytes, device, max_cycles)
    program = compile_program(source)
    get = lambda i: program[i] if i < len(program) else 0
    tape = [0] * 1024
    cycle = ip = mp = mem_val = 0
    curr, nxt = program[0], get(1)
    inp = list(input_bytes)
    output, proc, instr, in_rows, out_rows = [], [], [], [], []
    for i in range(len(program)):
        instr.append([i, program[i], get(i + 1)])

    def push_state():
        proc.append([cycle, ip, curr, nxt, mp, mem_val, pow(mem_val, -1, P) if mem_val else 0, int(curr == 0)])
        instr.append([ip, curr, nxt])

    while ip < len(program):
        push_state()
        if curr == LOOP_BEGIN:
            ip = program[ip + 1] if mem_val == 0 else ip + 2
        elif curr == LOOP_END:
            ip = program[ip + 1] if mem_val != 0 else ip + 2
        elif curr == DEC_PTR:
            ip, mp = ip + 1, mp - 1
        elif curr == INC_PTR:
            ip, mp = ip + 1, mp + 1
        elif curr == INC:
            ip, tape[mp] = ip + 1, (tape[mp] + 1) & 0xFF
        elif curr == DEC:
            ip, tape[mp] = ip + 1, (tape[mp] - 1) & 0xFF
        elif curr == WRITE:
            ip += 1
            output.append(tape[mp])
            out_rows.append([tape[mp]])
        elif curr == READ:
            ip += 1
            tape[mp] = inp.pop(0)
            in_rows.append([tape[mp]])
        else:
            raise ValueError(f"unrecognized instruction at ip:{ip}")
        cycle += 1
        curr, nxt, mem_val = get(ip), get(ip + 1), tape[mp]
    push_state()
    instr.sort(key=lambda r: r[0])                       # stable, like sort_by_key
    # derive_memory_rows (vm.rs:338-381)
    mem = [[r[CYCLE], r[MP], r[MEM_VAL], 0] for r in proc if r[CURR_INSTR] != 0]
    mem.sort(key=lambda r: (r[1], r[0]))
    # dummy rows so that the cycle count never jumps within one address (the reference inserts them one at a time)
    filled = []
    for k, c in enumerate(mem):
        filled.append(c)
        if k + 1 < len(mem) and c[1] == mem[k + 1][1]:
            filled.extend([cy, c[1], c[2], 1] for cy in range(c[0] + 1, mem[k + 1][0]))
    mem = filled
    longest = max(len(proc), len(mem), len(instr), len(in_rows), len(out_rows))
    n = longest if longest & (longest - 1) == 0 else 1 << longest.bit_length()
    while len(proc) < n:
        l = proc[-1]
        proc.append([l[CYCLE] + 1, l[IP], 0, 0, l[MP], l[MEM_VAL], l[MEM_VAL_INV], 1])
    while len(mem) < n:
        l = mem[-1]
        mem.append([l[0] + 1, l[1], l[2], 1])
    last_ip = instr[-1][0]
    while len(instr) < n:
        instr.append([last_ip, 0, 0])
    in_rows += [[0]] * (n - len(in_rows))
    out_rows += [[0]] * (n - len(out_rows))
    rows = [p + m + i_ + a + b for p, m, i_, a, b in zip(proc, mem, instr, in_rows, out_rows)]
    return BrainfuckTrace(rows), bytes(output)


# ---------------------------------------------------------------- ChaCha12 test_rng (restated, see module docstring)
def _chacha_core(st, rounds):
    w = list(st)
    rot = lambda v, r: ((v << r) | (v >> (32 - r))) & 0xFFFFFFFF

    def qr(a, b, c, d):
        w[a] = (w[a] + w[b]) & 0xFFFFFFFF; w[d] = rot(w[d] ^ w[a], 16)
        w[c] = (w[c] + w[d]) & 0xFFFFFFFF; w[b] = rot(w[b] ^ w[c], 12)
        w[a] = (w[a] + w[b]) & 0xFFFFFFFF; w[d] = rot(w[d] ^ w[a], 8)
        w[c] = (w[c] + w[d]) & 0xFFFFFFFF; w[b] = rot(w[b] ^ w[c], 7)

    for _ in range(rounds // 2):
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
    return [(a + b) & 0xFFFFFFFF for a, b in zip(w, st)]


def _chacha_block(key_words, counter, rounds=12):
    """rand_chacha layout: 64-bit block counter in words 12-13, stream id 0 in words 14-15"""
    return _chacha_core([0x61707865, 0x3320646E, 0x79622D32, 0x6B206574] + list(key_words)
                        + [counter & 0xFFFFFFFF, counter >> 32, 0, 0], rounds)


def test_rng_fq3(count):
    """`count` Fq3 draws from ark_std::test_rng()"""
    seed = bytes([1, 0, 0, 0, 23, 0, 0, 0, 200, 1, 0, 0, 210, 30, 0, 0] + [0] * 16)
    key = [int.from_bytes(seed[4 * i:4 * i + 4], "little") for i in range(8)]
    words, ctr, out = [], 0, []

    def next_u64():
        nonlocal words, ctr
        if len(words) < 2:
            words += _chacha_block(key, ctr)
            ctr += 1
        lo, hi = words[0], words[1]
        words = words[2:]
        return (hi << 32) | lo

    def fp():
        while True:
            w = next_u64()
            if w < P:
                return w * _RINV % P
    return [(fp(), fp(), fp()) for _ in range(count)]


# ---------------------------------------------------------------- trace
def _sub_scaled(acc, ch, v):
    """acc - ch * v for Fq3 acc, ch and base-field v"""
    return tuple((a - c * v) % P for a, c in zip(acc, ch))


class BrainfuckTrace(Trace):
    def __init__(self, rows):
        self.rows = rows
        # every entry is a small integer except MemValInv = 1 / mem_val with mem_val < 256: Montgomery words are
        # v * (2^64 mod p) = v * (2^32 - 1) (no reduction needed below 2^32) and a 256-entry table of inverses
        ints = np.array([[0 if c == MEM_VAL_INV else v for c, v in enumerate(r)] for r in rows], dtype=np.uint64).T
        self.int_cols = np.ascontiguousarray(ints).astype(np.int64)
        base = np.ascontiguousarray(ints * np.uint64(0xFFFFFFFF))
        inv_lut = np.array([0] + [pow(v, -1, P) * _R % P for v in range(1, 256)], dtype=np.uint64)
        base[MEM_VAL_INV] = inv_lut[ints[MEM_VAL]]
        super().__init__(base, self._extension)

    def helper_columns(self):
        """0/1 row conditions (and the values they gate) that look at neighbouring rows or at opcodes — functions of the
        base trace only, computed once with vectorised numpy; Montgomery words (v * (2^32 - 1) needs no reduction)"""
        if getattr(self, "_aux", None) is None:
            col = lambda c: self.int_cols[c]
            n = len(self.rows)
            ci, mv = col(CURR_INSTR), col(MEM_VAL)
            nxt_mv = np.concatenate([mv[1:], mv[:1]])
            iip, ici = col(I_IP), col(I_CURR_INSTR)
            prev_ip = np.concatenate([[-1], iip[:-1]])
            aux = np.stack([
                ci != 0,                                               # 0 processor row is not padding
                ci == READ, (ci == READ) * nxt_mv,                     # 1, 2
                ci == WRITE, (ci == WRITE) * nxt_mv,                   # 3, 4
                col(M_DUMMY) == 0,                                     # 5 memory row is real
                (ici != 0) & (np.arange(n) > 0) & (iip == prev_ip),    # 6 instruction permutation advances
                iip != prev_ip,                                        # 7 program evaluation advances
            ]).astype(np.uint64)
            self._aux = aux * np.uint64(0xFFFFFFFF)
        return self._aux

    def build_extension_columns_device(self, challenges, ctx, base_dev):
        import torch
        d_aux = torch.from_numpy(self.helper_columns().view(np.int64)).to(base_dev.device)
        return _device_extension(len(self.rows), d_aux, [tuple(c) for c in challenges], ctx, base_dev)

    def _extension(self, ch):
        """gen_*_ext_matrix (trace.rs:108-279): running products / evaluations, row by row"""
        rows, n = self.rows, len(self.rows)
        instr_initial, mem_initial = test_rng_fq3(2)
        mul, add = E.q_mul, E.q_add
        lift = lambda v: (v % P, 0, 0)
        ext = [[None] * 9 for _ in range(n)]
        # processor table
        ipp, mpp, ie, oe = instr_initial, mem_initial, (0, 0, 0), (0, 0, 0)
        for r in range(n):
            row = rows[r]
            ext[r][0], ext[r][1] = ipp, mpp
            if row[CURR_INSTR] != 0:
                ipp = mul(ipp, _sub_scaled(_sub_scaled(_sub_scaled(ch[CH_ALPHA], ch[CH_A], row[IP]), ch[CH_B], row[CURR_INSTR]),
                                            ch[CH_C], row[NEXT_INSTR]))
                mpp = mul(mpp, _sub_scaled(_sub_scaled(_sub_scaled(ch[CH_BETA], ch[CH_D], row[CYCLE]), ch[CH_E], row[MP]),
                                            ch[CH_F], row[MEM_VAL]))
            ext[r][2], ext[r][3] = ie, oe
            if row[CURR_INSTR] == READ:
                ie = add(mul(ie, ch[CH_GAMMA]), lift(rows[r + 1][MEM_VAL]))
            elif row[CURR_INSTR] == WRITE:
                oe = add(mul(oe, ch[CH_DELTA]), lift(rows[r + 1][MEM_VAL]))
        # memory table
        perm = mem_initial
        for r in range(n):
            row = rows[r]
            ext[r][4] = perm
            if row[M_DUMMY] == 0:
                perm = mul(perm, _sub_scaled(_sub_scaled(_sub_scaled(ch[CH_BETA], ch[CH_D], row[M_CYCLE]), ch[CH_E], row[M_MP]),
                                              ch[CH_F], row[M_MEM_VAL]))
        # instruction table
        perm, ev, prev_addr = instr_initial, (0, 0, 0), P - 1
        for r in range(n):
            row = rows[r]
            if row[I_CURR_INSTR] != 0 and r > 0 and row[I_IP] == rows[r - 1][I_IP]:
                perm = mul(perm, _sub_scaled(_sub_scaled(_sub_scaled(ch[CH_ALPHA], ch[CH_A], row[I_IP]), ch[CH_B], row[I_CURR_INSTR]),
                                              ch[CH_C], row[I_NEXT_INSTR]))
            ext[r][5] = perm
            if row[I_IP] != prev_addr:
                ev = mul(ch[CH_ETA], ev)
                for c, col in ((CH_A, I_IP), (CH_B, I_CURR_INSTR), (CH_C, I_NEXT_INSTR)):
                    ev = tuple((e + k * row[col]) % P for e, k in zip(ev, ch[c]))
            ext[r][6] = ev
            prev_addr = row[I_IP]
        # input / output tables
        for slot, col, c in ((7, IN_VALUE, CH_GAMMA), (8, OUT_VALUE, CH_DELTA)):
            ev = (0, 0, 0)
            for r in range(n):
                ev = add(mul(ev, ch[c]), lift(rows[r][col]))
                ext[r][slot] = ev
        out = np.empty((9, 3 * n), dtype=np.uint64)
        for c in range(9):
            out[c] = [w * _R % P for r in range(n) for w in ext[r][c]]
        return out


# ---------------------------------------------------------------- the trace built on the device (include/ministark_bf.h)
_CONTEXTS = {}


def _torch_device(device):
    import torch
    dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def _context(dev):
    """one context per device for building traces, queued on torch's current stream when that is a stream of its own (a
    handle of 0, the legacy default stream, leaves the context on its own non-blocking stream: callers sync it)"""
    import torch
    from .. import Context
    key = (dev.type, dev.index)
    if key not in _CONTEXTS:
        _CONTEXTS[key] = Context(dev.index or 0)
    ctx = _CONTEXTS[key]
    if dev.type == "cuda":
        ctx.set_stream(torch.cuda.current_stream(dev).cuda_stream)
    return ctx


def _device_tables(program, log, dev):
    """the (17, n) base matrix on `dev` from the program (uint32 words) and the run's records: the table lengths first
    (one device-to-host sync), then the fill.  The uploaded log and the workspace are freed before it returns, and the
    matrix is complete: a prover may read it on another stream."""
    import torch
    ctx = _context(dev)
    d_prog = torch.from_numpy(program.view(np.int32)).to(dev)
    d_log = torch.from_numpy(log.view(np.int64)).to(dev)
    sizes = ctx.bf_trace_sizes(d_prog, program.size, d_log, log.size)
    base = torch.empty((17, sizes["n"]), dtype=torch.int64, device=dev)
    work = torch.empty(sizes["work_bytes"], dtype=torch.uint8, device=dev)
    if base.is_cuda:                    # the context's stream may not be torch's: torch's own work on this memory is done
        torch.cuda.current_stream(dev).synchronize()
    ctx.bf_trace_fill(d_prog, program.size, d_log, log.size, sizes, work, base)
    ctx.sync()                          # the fill is done before its inputs go back to the allocator and base is handed over
    del work, d_log, d_prog
    return base, sizes


def _simulate_device(source, input_bytes, device, max_cycles):
    from .. import bf_run
    program = np.array(compile_program(source), dtype=np.uint32)
    log, output = bf_run(program, input_bytes, max_cycles)
    return BrainfuckDeviceTrace(program, log, _torch_device(device)), output


class BrainfuckDeviceTrace(Trace):
    """The trace of one run with its base columns resident on a device, built from the run's records (ms_bf_run) by
    ms_bf_trace_sizes / ms_bf_trace_fill; equal word for word to `BrainfuckTrace(rows).base_columns()`.

    The host keeps only the program and the records (8 bytes per processor row).  A prover that no longer needs the
    natural-order matrix (GpuProver, once the extension columns are built) calls release_base_columns(), so that the
    proof's peak device memory is what it is for a host trace; base_columns() rebuilds the matrix from the records when
    asked again."""

    def __init__(self, program, log, device):
        self.program, self.log, self.device = program, log, device
        base, self.sizes = _device_tables(program, log, device)
        super().__init__(base)
        self.n = self.sizes["n"]

    def __len__(self):
        return self.n

    def base_columns(self):
        if self._base is None:
            self._base, _ = _device_tables(self.program, self.log, self.device)
        return self._base

    def helper_columns_device(self, ctx, base_dev=None):
        """BrainfuckTrace.helper_columns() computed on the device from the base matrix: an (8, n) int64 tensor, written on
        ctx's stream (not synchronised)"""
        import torch
        base = self.base_columns() if base_dev is None else base_dev
        aux = torch.empty((8, self.n), dtype=torch.int64, device=base.device)
        ctx.bf_helper_columns(base, self.n, aux)
        return aux

    def release_base_columns(self):
        """drop the trace's reference to the base matrix (other references keep it alive until they go)"""
        self._base = None

    def build_extension_columns_device(self, challenges, ctx, base_dev):
        return _device_extension(self.n, self.helper_columns_device(ctx, base_dev), [tuple(c) for c in challenges], ctx,
                                 base_dev)

    def to_host(self):
        """the same trace as a host BrainfuckTrace (downloads the base matrix and decodes it; slow at large n)"""
        words = self.base_columns().cpu().numpy().view(np.uint64)
        rows = (words // np.uint64(0xFFFFFFFF)).T.tolist()          # every value but MemValInv is below 2^32
        for r in rows:
            r[MEM_VAL_INV] = pow(r[MEM_VAL], -1, P) if r[MEM_VAL] else 0
        return BrainfuckTrace(rows)

    def build_extension_columns(self, challenges):
        return self.to_host()._extension(challenges)


_FACTOR_PROGRAMS = {}


def _device_extension(n, d_aux, ch, ctx, base_dev):
    """The nine extension columns of `BrainfuckTrace._extension`, built on the device: every column is
    x_0 = init, x_(i+1) = x_i * a_i + b_i  with per-row multipliers / addends that are pointwise expressions of the
    base row (evaluated by the fused evaluator over the resident trace) — then one parallel scan (ms_scan_affine).
    Row conditions that look at neighbouring rows or at opcodes are the eight 0/1 helper columns `d_aux` (device, (8, n)):
    computed from the integer rows on the host for a host trace, by ms_bf_helper_columns for a device trace."""
    import torch
    from .. import FP, FQ3, ONE
    log_n = n.bit_length() - 1
    NB = 17
    AUX = lambda k: E.Trace(NB + k, 0)
    T, CH = (lambda c: E.Trace(c, 0)), E.Challenge
    one = E.Constant(1)
    instr_fp = lambda ip, c, nx: CH(CH_ALPHA) - CH(CH_A) * ip - CH(CH_B) * c - CH(CH_C) * nx
    mem_fp = lambda cy, mp, v: CH(CH_BETA) - CH(CH_D) * cy - CH(CH_E) * mp - CH(CH_F) * v
    gated = lambda mask, factor: one + mask * (factor - one)                      # factor where mask = 1, else 1
    cols = [base_dev[c] for c in range(NB)] + [d_aux[k] for k in range(d_aux.shape[0])]
    is_q = [False] * len(cols)
    sz = 3 * n

    def evaluate(expr):
        out = torch.empty(sz, dtype=torch.int64, device=base_dev.device)
        prog = _FACTOR_PROGRAMS.get(id(expr))               # the factor expressions do not depend on the proof: compiled once
        if prog is None:                                    # (hash-consed Expr nodes live as long as the process)
            prog = _FACTOR_PROGRAMS[id(expr)] = E.compile_program(expr, len(cols), symbolic=True)
        ctx.eval_constraints_ptrs(prog.bind(challenges=ch), out, log_n, cols, is_q, fq_field=FQ3, offset=ONE)
        return out

    mont3 = lambda v: np.array([c * _R % P for c in v], dtype=np.uint64)
    instr_initial, mem_initial = test_rng_fq3(2)
    zero3 = np.zeros(3, dtype=np.uint64)
    ext = torch.empty((9, sz), dtype=torch.int64, device=base_dev.device)
    scan = lambda k, init, **kw: ctx.scan_affine(ext[k], FQ3, n, init, **kw)
    scan(0, mont3(instr_initial), a=evaluate(gated(AUX(0), instr_fp(T(IP), T(CURR_INSTR), T(NEXT_INSTR)))), a_field=FQ3)
    scan(1, mont3(mem_initial), a=evaluate(gated(AUX(0), mem_fp(T(CYCLE), T(MP), T(MEM_VAL)))), a_field=FQ3)
    scan(2, zero3, a=evaluate(gated(AUX(1), CH(CH_GAMMA))), a_field=FQ3, b=d_aux[2], b_field=FP)
    scan(3, zero3, a=evaluate(gated(AUX(3), CH(CH_DELTA))), a_field=FQ3, b=d_aux[4], b_field=FP)
    scan(4, mont3(mem_initial), a=evaluate(gated(AUX(5), mem_fp(T(M_CYCLE), T(M_MP), T(M_MEM_VAL)))), a_field=FQ3)
    scan(5, mont3(instr_initial), a=evaluate(gated(AUX(6), instr_fp(T(I_IP), T(I_CURR_INSTR), T(I_NEXT_INSTR)))), a_field=FQ3,
         inclusive=True)
    scan(6, zero3, a=evaluate(gated(AUX(7), CH(CH_ETA))), a_field=FQ3,
         b=evaluate(AUX(7) * (CH(CH_A) * T(I_IP) + CH(CH_B) * T(I_CURR_INSTR) + CH(CH_C) * T(I_NEXT_INSTR))), b_field=FQ3, inclusive=True)
    scan(7, zero3, a_const=mont3(ch[CH_GAMMA]), b=base_dev[IN_VALUE], b_field=FP, inclusive=True)
    scan(8, zero3, a_const=mont3(ch[CH_DELTA]), b=base_dev[OUT_VALUE], b_field=FP, inclusive=True)
    return ext


# ---------------------------------------------------------------- constraints (constraints.rs)
def _c(v):
    return E.Constant(v)


def _instr_zerofier(instr):
    prod = None
    for op in OPCODES:
        t = instr - _c(op)
        prod = t if prod is None else prod * t
    return prod


def _if_not_instr(which, ind):
    prod = None
    for op in OPCODES:
        if op != which:
            t = ind - _c(op)
            prod = t if prod is None else prod * t
    return prod


def _if_instr(which, ind):
    return ind - _c(which)


def _constraint_sets():
    T, CH, H = E.Trace, E.Challenge, E.Hint
    cur, nx = (lambda c: T(c, 0)), (lambda c: T(c, 1))
    one = _c(1)
    two = one + one
    # --- ProcessorBaseColumn
    proc_boundary = [cur(CYCLE), cur(IP), cur(MP), cur(MEM_VAL), cur(MEM_VAL_INV), cur(DUMMY)]
    mem_val_is_zero = cur(MEM_VAL) * cur(MEM_VAL_INV) - one
    acc = [None, None, None]
    ip_step = nx(IP) - cur(IP) - one
    same_mp, same_val = nx(MP) - cur(MP), nx(MEM_VAL) - cur(MEM_VAL)
    per_instr = {
        INC_PTR: (ip_step, nx(MP) - cur(MP) - one, None),
        DEC_PTR: (ip_step, nx(MP) - cur(MP) + one, None),
        INC: (ip_step, same_mp, nx(MEM_VAL) - cur(MEM_VAL) - one),
        DEC: (ip_step, same_mp, nx(MEM_VAL) - cur(MEM_VAL) + one),
        WRITE: (ip_step, same_mp, None),
        READ: (ip_step, same_mp, same_val),
        LOOP_BEGIN: (cur(MEM_VAL) * (nx(IP) - cur(IP) - two) + mem_val_is_zero * (nx(IP) - cur(NEXT_INSTR)), same_mp, same_val),
        LOOP_END: (mem_val_is_zero * (nx(IP) - cur(IP) - two) + cur(MEM_VAL) * (nx(IP) - cur(NEXT_INSTR)), same_mp, same_val),
    }
    for op in OPCODES:
        deselector = _if_not_instr(op, cur(CURR_INSTR))
        for k in range(3):
            rhs = per_instr[op][k]
            if rhs is not None:
                term = deselector * rhs * cur(CURR_INSTR)
                acc[k] = term if acc[k] is None else acc[k] + term
    proc_transition = acc + [
        nx(CYCLE) - cur(CYCLE) - one,
        cur(MEM_VAL) * mem_val_is_zero,
        cur(MEM_VAL_INV) * mem_val_is_zero,
        (nx(DUMMY) - one) * nx(DUMMY),
        _instr_zerofier(cur(CURR_INSTR)) * (cur(DUMMY) - one) + cur(CURR_INSTR) * cur(DUMMY),
    ]
    # --- ProcessorExtensionColumn
    pext_boundary = [cur(P_IN_EVAL), cur(P_OUT_EVAL)]
    instr_fp = lambda ip, ci, ni: CH(CH_ALPHA) - CH(CH_A) * ip - CH(CH_B) * ci - CH(CH_C) * ni
    mem_fp = lambda cy, mp, mv: CH(CH_BETA) - CH(CH_D) * cy - CH(CH_E) * mp - CH(CH_F) * mv
    i_fp = instr_fp(cur(I_IP), cur(I_CURR_INSTR), cur(I_NEXT_INSTR))
    p_fp = instr_fp(cur(IP), cur(CURR_INSTR), cur(NEXT_INSTR))
    m_fp = mem_fp(cur(M_CYCLE), cur(M_MP), cur(M_MEM_VAL))
    pm_fp = mem_fp(cur(CYCLE), cur(MP), cur(MEM_VAL))
    pext_terminal = [
        cur(I_CURR_INSTR) * (cur(DUMMY) - one) * (cur(I_PROC_PERM) * i_fp - cur(P_INSTR_PERM) * p_fp)
        + _instr_zerofier(cur(I_CURR_INSTR)) * (cur(DUMMY) - one) * (cur(I_PROC_PERM) - cur(P_INSTR_PERM) * p_fp)
        + cur(I_CURR_INSTR) * cur(DUMMY) * (cur(I_PROC_PERM) * i_fp - cur(P_INSTR_PERM))
        + _instr_zerofier(cur(I_CURR_INSTR)) * cur(DUMMY) * (cur(I_PROC_PERM) - cur(P_INSTR_PERM)),
        (cur(M_DUMMY) - one) * (cur(DUMMY) - one) * (cur(M_PERM) * m_fp - cur(P_MEM_PERM) * pm_fp)
        + cur(M_DUMMY) * (cur(DUMMY) - one) * (cur(M_PERM) - cur(P_MEM_PERM) * pm_fp)
        + (cur(M_DUMMY) - one) * cur(DUMMY) * (cur(M_PERM) * m_fp - cur(P_MEM_PERM))
        + cur(M_DUMMY) * cur(DUMMY) * (cur(M_PERM) - cur(P_MEM_PERM)),
        cur(P_IN_EVAL) - H(H_INPUT),
        cur(P_OUT_EVAL) - H(H_OUTPUT),
    ]
    pext_transition = [
        cur(CURR_INSTR) * (cur(P_INSTR_PERM) * p_fp - nx(P_INSTR_PERM)) + cur(DUMMY) * (cur(P_INSTR_PERM) - nx(P_INSTR_PERM)),
        cur(CURR_INSTR) * (cur(P_MEM_PERM) * pm_fp - nx(P_MEM_PERM)) * cur(DUMMY) * (cur(P_MEM_PERM) - nx(P_MEM_PERM)),
        cur(CURR_INSTR) * _if_not_instr(READ, cur(CURR_INSTR)) * (nx(P_IN_EVAL) - CH(CH_GAMMA) * cur(P_IN_EVAL) - nx(MEM_VAL))
        + _if_instr(READ, cur(CURR_INSTR)) * (nx(P_IN_EVAL) - cur(P_IN_EVAL)),
        cur(CURR_INSTR) * _if_not_instr(WRITE, cur(CURR_INSTR)) * (nx(P_OUT_EVAL) - cur(P_OUT_EVAL) * CH(CH_DELTA) - cur(MEM_VAL))
        + _if_instr(WRITE, cur(CURR_INSTR)) * (nx(P_OUT_EVAL) - cur(P_OUT_EVAL)),
    ]
    # --- Memory
    mem_boundary = [cur(M_CYCLE), cur(M_MP), cur(M_MEM_VAL)]
    dmp = nx(M_MP) - cur(M_MP)
    mem_transition = [
        (dmp - one) * dmp,
        dmp * nx(M_MEM_VAL),
        (nx(M_DUMMY) - one) * nx(M_DUMMY),
        dmp * cur(M_DUMMY),
        (nx(M_MEM_VAL) - cur(M_MEM_VAL)) * cur(M_DUMMY),
        (dmp - one) * (nx(M_CYCLE) - cur(M_CYCLE) - one),
    ]
    mext_transition = [(nx(M_PERM) - cur(M_PERM) * m_fp) * (cur(M_DUMMY) - one) + (nx(M_PERM) - cur(M_PERM)) * cur(M_DUMMY)]
    # --- Instruction
    instr_boundary = [cur(I_IP)]
    dip = nx(I_IP) - cur(I_IP)
    instr_transition = [
        (dip - one) * dip,
        (dip - one) * (nx(I_CURR_INSTR) - cur(I_CURR_INSTR)),
        (dip - one) * (nx(I_NEXT_INSTR) - cur(I_NEXT_INSTR)),
    ]
    iext_boundary = [cur(I_PROG_EVAL) - CH(CH_A) * cur(I_IP) - CH(CH_B) * cur(I_CURR_INSTR) - CH(CH_C) * cur(I_NEXT_INSTR)]
    iext_terminal = [cur(I_PROG_EVAL) - H(H_INSTRUCTION)]
    next_fp = instr_fp(nx(I_IP), nx(I_CURR_INSTR), nx(I_NEXT_INSTR))
    iext_transition = [
        cur(I_CURR_INSTR) * (cur(I_IP) - nx(I_IP) + one) * (nx(I_PROC_PERM) - cur(I_PROC_PERM) * next_fp)
        + _instr_zerofier(cur(I_CURR_INSTR)) * (nx(I_PROC_PERM) - cur(I_PROC_PERM))
        + (cur(I_IP) - nx(I_IP)) * (cur(I_PROC_PERM) - nx(I_PROC_PERM)),
        (dip - one) * (nx(I_PROG_EVAL) - cur(I_PROG_EVAL))
        + dip * (nx(I_PROG_EVAL) - cur(I_PROG_EVAL) * CH(CH_ETA) - CH(CH_A) * nx(I_IP) - CH(CH_B) * nx(I_CURR_INSTR)
                 - CH(CH_C) * nx(I_NEXT_INSTR)),
    ]
    # --- Input / Output
    in_boundary, out_boundary = [cur(IN_EVAL) - cur(IN_VALUE)], [cur(OUT_EVAL) - cur(OUT_VALUE)]
    in_terminal = [cur(IN_EVAL) - H(H_INPUT) * H(H_INPUT_OFFSET)]
    out_terminal = [cur(OUT_EVAL) - H(H_OUTPUT) * H(H_OUTPUT_OFFSET)]
    in_transition = [cur(IN_EVAL) * CH(CH_GAMMA) + nx(IN_VALUE) - nx(IN_EVAL)]
    out_transition = [cur(OUT_EVAL) * CH(CH_DELTA) + nx(OUT_VALUE) - nx(OUT_EVAL)]
    transition = (proc_transition + pext_transition + mem_transition + mext_transition + instr_transition + iext_transition
                  + in_transition + out_transition)
    boundary = proc_boundary + pext_boundary + mem_boundary + instr_boundary + iext_boundary + in_boundary + out_boundary
    terminal = pext_terminal + iext_terminal + in_terminal + out_terminal
    return transition, boundary, terminal


class BrainfuckAirConfig(AirConfig):
    NUM_BASE_COLUMNS = 17
    NUM_EXTENSION_COLUMNS = 9
    FQ_IS_FP = False

    @staticmethod
    def constraints(trace_len):
        g = domain_generator(trace_len.bit_length() - 1)
        x, one = E.X(), _c(1)
        first, last = _c(1), _c(pow(g, trace_len - 1, P))
        transition, boundary, terminal = _constraint_sets()
        but_last = (x - last) / (x ** trace_len - one)
        return ([c * but_last for c in transition] + [c / (x - first) for c in boundary] + [c / (x - last) for c in terminal])

    @staticmethod
    def gen_hints(trace_len, claim, challenges):
        """air.rs:34-75"""
        ch = [tuple(c) for c in challenges]

        def io_terminal(symbols, challenge):
            if trace_len < len(symbols):        # a verifier handed a forged trace length: the offset would be negative
                raise ValueError(f"trace length {trace_len} is shorter than the {len(symbols)} input / output symbols")
            acc = (0, 0, 0)
            for s in symbols:
                acc = E.q_add(E.q_mul(challenge, acc), (s, 0, 0))
            return acc, E.q_pow(challenge, trace_len - len(symbols))

        in_arg, in_off = io_terminal(claim.input, ch[CH_GAMMA])
        out_arg, out_off = io_terminal(claim.output, ch[CH_DELTA])
        program = compile_program(claim.source_code) + [0]
        acc = (0, 0, 0)
        for ip, curr in enumerate(program):
            nxt = program[ip + 1] if ip + 1 < len(program) else 0
            acc = E.q_mul(acc, ch[CH_ETA])
            for c, v in ((CH_A, ip), (CH_B, curr), (CH_C, nxt)):
                acc = tuple((a + k * v) % P for a, k in zip(acc, ch[c]))
        return [acc, in_arg, in_off, out_arg, out_off]


class BrainfuckClaim(Stark):
    AirConfig = BrainfuckAirConfig

    def __init__(self, source_code, input_bytes, output_bytes):
        self.source_code, self.input, self.output = source_code, bytes(input_bytes), bytes(output_bytes)

    def get_public_inputs(self):
        return self

    def public_inputs_bytes(self, claim):
        """derived CanonicalSerialize of {source_code: String, input: Vec<u8>, output: Vec<u8>}: u64 length + bytes each"""
        vec = lambda b: len(b).to_bytes(8, "little") + b
        return vec(claim.source_code.encode()) + vec(claim.input) + vec(claim.output)
