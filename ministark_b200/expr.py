"""expr.py — symbolic constraint expressions and their compilation to the fused evaluator program.

Host-side mirror of the reference's input format for constraint evaluation:
    Expr<AlgebraicItem<FieldVariant<Fp, Fq>>>        src/expression.rs:31-39, src/constraints.rs:21-28
with leaves  X | Constant | Challenge(i) | Hint(i) | Trace(column, row offset)  and nodes
Neg | Add | Mul | Div | Pow(usize), and  Periodic(coeffs, interval_size)  (src/constraints.rs:107-146): the polynomial
with these coefficients in  y = x^(trace_len / interval_size), i.e. a column that repeats every interval_size rows.

The reference evaluates this DAG either with one GPU dispatch + barrier + full HBM round trip per
node (eval_gpu.rs, disabled: src/air.rs:104-117) or on the CPU in 512-element chunks
(eval_cpu.rs:76-150).  Here `compile_program` flattens the DAG once (hash-consed = the effect
of reuse_shared_nodes, src/expression.rs:186-357; constant sub-expressions folded on the host;
registers reused by liveness) into a linear typed program that ONE kernel (csrc/eval.cu) runs per
evaluation point with all temporaries on chip.
"""
import numpy as np

P = 2**64 - 2**32 + 1
_R = 2**64
_RINV = pow(_R, -1, P)

FP, FQ = 0, 1  # value types: base field / extension ("Fq" is Fq3, or Fp itself when the AIR has Fq = Fp)

# opcodes (must match csrc/eval.cuh).  OP_DIV and OP_CHECK occur only in checked programs (compile_check_program,
# csrc/check.cu): OP_DIV is Constraint::check's division, OP_CHECK k, r marks constraint k failed where register r is None
OP_X, OP_CONST, OP_TRACE, OP_NEG, OP_ADD, OP_SUB, OP_MUL, OP_INV, OP_POW, OP_STORE, OP_PERIODIC, OP_DIV, OP_CHECK = range(13)
MAX_REGS = 48


# ---- canonical-integer extension arithmetic for host-side constant folding (X^3 = 2)
def _q(v):
    return (v % P, 0, 0) if isinstance(v, int) else tuple(int(x) % P for x in v)


def q_add(a, b):
    return tuple((x + y) % P for x, y in zip(a, b))


def q_neg(a):
    return tuple((-x) % P for x in a)


def q_mul(a, b):
    pr = [0] * 5
    for i in range(3):
        for j in range(3):
            pr[i + j] += a[i] * b[j]
    return ((pr[0] + 2 * pr[3]) % P, (pr[1] + 2 * pr[4]) % P, pr[2] % P)


def q_pow(a, e):
    if e < 0:
        raise ValueError(f"negative exponent {e}")
    r = (1, 0, 0)
    while e:
        if e & 1:
            r = q_mul(r, a)
        a = q_mul(a, a)
        e >>= 1
    return r


def q_inv(a):
    return q_pow(a, P**3 - 2)


class Expr:
    """Immutable, hash-consed expression node.  Build with X(), Constant(), Challenge(), Hint(),
    Trace() and the operators + - * / ** and unary -."""
    _pool = {}
    __slots__ = ("kind", "args", "_key")

    def __new__(cls, kind, *args):
        key = (kind,) + tuple(a._key if isinstance(a, Expr) else a for a in args)
        node = cls._pool.get(key)
        if node is None:
            node = object.__new__(cls)
            node.kind, node.args = kind, args
            node._key = id(node)
            cls._pool[key] = node
        return node

    @staticmethod
    def _lift(v):
        return v if isinstance(v, Expr) else Constant(v)

    def __add__(self, o):
        return Expr("add", self, Expr._lift(o))

    __radd__ = __add__

    def __sub__(self, o):
        return Expr("add", self, Expr("neg", Expr._lift(o)))   # a - b = a + (-b), as the reference's Sub impl

    def __rsub__(self, o):
        return Expr._lift(o) - self

    def __mul__(self, o):
        return Expr("mul", self, Expr._lift(o))

    __rmul__ = __mul__

    def __truediv__(self, o):
        return Expr("div", self, Expr._lift(o))

    def __neg__(self):
        return Expr("neg", self)

    def __pow__(self, e):
        return Expr("pow", self, int(e))

    def to_tuple(self, memo=None):
        """plain nested-tuple form (shared nodes stay shared) — the exchange format the tests hand
        to the CPU oracle's evaluator."""
        memo = {} if memo is None else memo
        if id(self) not in memo:
            memo[id(self)] = (self.kind,) + tuple(a.to_tuple(memo) if isinstance(a, Expr) else a for a in self.args)
        return memo[id(self)]


def X():
    return Expr("x")


def Constant(v, ext=False):
    """canonical integer (base field) or 3-tuple of canonical integers (extension)"""
    if isinstance(v, (tuple, list)):
        return Expr("const", tuple(int(x) % P for x in v), True)
    return Expr("const", (int(v) % P, 0, 0), bool(ext))


def Challenge(i):
    return Expr("chal", int(i))


def Hint(i):
    return Expr("hint", int(i))


def Trace(col, offset=0):
    return Expr("trace", int(col), int(offset))


def Periodic(coeffs, interval_size):
    """PeriodicColumn::new (src/constraints.rs:107-126): coefficients (canonical ints, or 3-tuples for extension
    elements) of a polynomial in x^(trace_len / interval_size); both lengths are powers of two, len(coeffs) <= interval"""
    coeffs = tuple(tuple(int(x) % P for x in c) if isinstance(c, (tuple, list)) else int(c) % P for c in coeffs)
    n, m = len(coeffs), int(interval_size)
    if n == 0 or n & (n - 1) or m & (m - 1) or n > m:
        raise ValueError("periodic column: lengths must be powers of two with len(coeffs) <= interval_size")
    return Expr("periodic", coeffs, m)


def evaluate_at(expr, x, trace=None, challenges=(), hints=(), ccoefs=(), trace_len=None):
    """the value of `expr` at ONE point, on the host: Expr::graph_eval with the leaves of the verifier's out-of-domain
    check (src/verifier.rs:207-229).  x: the point; trace: {(column, offset): value}; challenges / hints / ccoefs: the
    values of Challenge(i) / Hint(i) / CompositionCoeff(i); Periodic(coeffs, interval) is its polynomial at
    x^(trace_len / interval).  Values are canonical ints or 3-tuples; the result is a 3-tuple.  A zero denominator raises
    ZeroDivisionError."""
    post, seen, stack = [], set(), [(expr, False)]
    while stack:                       # iterative post-order (DAGs can be deep)
        node, done = stack.pop()
        if done:
            post.append(node)
            continue
        if id(node) in seen:
            continue
        seen.add(id(node))
        stack.append((node, True))
        stack.extend((a, False) for a in node.args if isinstance(a, Expr) and id(a) not in seen)
    x = _q(x)
    val = {}
    for nd in post:
        k, a = nd.kind, nd.args
        if k == "x":
            v = x
        elif k == "const":
            v = a[0]
        elif k in _SYMBOLIC:
            v = _q({"chal": challenges, "hint": hints, "ccoef": ccoefs}[k][a[0]])
        elif k == "trace":
            v = _q(trace[(a[0], a[1])])
        elif k == "periodic":
            y = q_pow(x, trace_len // a[1])
            v = (0, 0, 0)
            for c in reversed(a[0]):
                v = q_add(q_mul(v, y), _q(c))
        elif k == "neg":
            v = q_neg(val[id(a[0])])
        elif k == "add":
            v = q_add(val[id(a[0])], val[id(a[1])])
        elif k == "mul":
            v = q_mul(val[id(a[0])], val[id(a[1])])
        elif k in ("div", "inv"):
            d = val[id(a[-1])]
            if not any(d):
                raise ZeroDivisionError(f"zero denominator in a {k} node")
            v = q_inv(d) if k == "inv" else q_mul(val[id(a[0])], q_inv(d))
        elif k == "pow":
            v = q_pow(val[id(a[0])], a[1])
        else:
            raise ValueError(f"unsupported node {k}")
        val[id(nd)] = v
    return val[id(expr)]


class Program:
    def __init__(self, code, consts, nregs, out_is_q, bindings=(), periodic=()):
        self.code = np.ascontiguousarray(code, dtype=np.uint32).reshape(-1, 4)
        self.consts = np.ascontiguousarray(consts, dtype=np.uint64).reshape(-1, 3)
        self.nregs, self.out_is_q = nregs, out_is_q
        self.bindings = list(bindings)          # (constant slot, "chal" | "hint" | "ccoef", index): filled by bind()
        # periodic columns: (column slot in the evaluator's column table, coeffs, interval_size, is_ext, log2 of the
        # table length = interval_size * lde_step); the tables are built by periodic_tables() and appended to the columns
        self.periodic = list(periodic)

    def bind(self, challenges=(), hints=(), ccoefs=()):
        """a copy of this program whose symbolic constants hold this proof's verifier randomness.  The instruction
        stream — and with it the run-time specialised kernel (csrc/eval_jit.cu keys on the code only) — is shared by
        every proof of the same AIR and trace length; only this small table changes."""
        src = {"chal": challenges, "hint": hints, "ccoef": ccoefs}
        consts = self.consts.copy()
        for slot, kind, idx in self.bindings:
            consts[slot] = [c * _R % P for c in _q(src[kind][idx])]
        return Program(self.code, consts, self.nregs, self.out_is_q, periodic=self.periodic)

    def __len__(self):
        return self.code.shape[0]


_SYMBOLIC = ("chal", "hint", "ccoef")


def periodic_tables(ctx, program, log_n, lde_step, offset_canonical=7):
    """eval_periodic_column (src/eval_cpu.rs:234-256) for every periodic column of `program`, on the device: the
    coefficients zero-padded to interval_size * lde_step, transformed over the coset  offset^(n / interval) * <g>  —
    natural order; the evaluator indexes the table with (point index mod table length).  Returns a list of
    (device pointer, is_ext); the caller appends them to the column list in program.periodic order and keeps the
    pointers alive until the evaluation has run (ctx.free them afterwards)."""
    import ctypes as C
    out = []
    n = 1 << log_n
    for _, coeffs, interval, is_q, log_len in program.periodic:
        lanes = 3 if is_q else 1
        length = 1 << log_len
        host = np.zeros(length * lanes, dtype=np.uint64)
        for k, c in enumerate(coeffs):
            v = c if isinstance(c, tuple) else (c, 0, 0)
            for w in range(lanes):
                host[k * lanes + w] = v[w] * _R % P
        off = pow(offset_canonical, n // interval, P) * _R % P
        ctx.ntt_batch(host, lanes, log_len, 1, offset=off)          # host buffer: staged through the device
        ptr = ctx.alloc_device(host.nbytes)
        ctx._ck(ctx.lib.ms_copy(ctx.h, ptr, host.ctypes.data, host.nbytes))
        out.append((ptr, is_q))
    return out


def _batch_inverses(root, num_base_cols):
    """Montgomery's trick inside one evaluation point: the inverses 1/d_1 .. 1/d_k of the program (operands that vary with
    the point and contain no inverse themselves, grouped by field) become ONE inversion of d_1 ... d_k and 3(k - 1)
    multiplications.  An inversion is a ~72-multiplication Fermat chain, so the three denominators of a composition
    constraint ((x - t_0), (x^n - 1), (x - t_(n-1))) or of the DEEP polynomial cost one chain instead of three.
    Only denominators that are functions of the point alone (x, constants, periodic columns) are batched — a denominator
    that reads a trace cell keeps its own inversion.  Valid when no batched operand vanishes on the evaluation domain:
    true for zerofier denominators over the LDE coset, which is disjoint from the trace domain, and (as for the
    reference's own formulas) for x - z with z out of domain; with a zero operand EVERY inverse of the batch would come
    out 0 where the reference's batch inversion skips zeros (src/eval_cpu.rs:280-295), so generic user expressions keep
    their independent inversions (the default)."""
    post, seen, stack = [], set(), [(root, False)]
    while stack:
        node, done = stack.pop()
        if done:
            post.append(node)
            continue
        if id(node) in seen:
            continue
        seen.add(id(node))
        stack.append((node, True))
        stack.extend((a, False) for a in node.args if isinstance(a, Expr) and id(a) not in seen)
    has_inv, varies, reads_trace, typ = {}, {}, {}, {}
    for nd in post:
        kids = [a for a in nd.args if isinstance(a, Expr)]
        has_inv[id(nd)] = nd.kind == "inv" or any(has_inv[id(k)] for k in kids)
        varies[id(nd)] = nd.kind in ("x", "trace", "periodic") or any(varies[id(k)] for k in kids)
        reads_trace[id(nd)] = nd.kind == "trace" or any(reads_trace[id(k)] for k in kids)
        if nd.kind == "const":
            typ[id(nd)] = FQ if nd.args[1] else FP
        elif nd.kind in _SYMBOLIC or nd.kind in ("chal", "hint"):
            typ[id(nd)] = FQ
        elif nd.kind == "x":
            typ[id(nd)] = FP
        elif nd.kind == "trace":
            typ[id(nd)] = FP if nd.args[0] < num_base_cols else FQ
        elif nd.kind == "periodic":
            typ[id(nd)] = FQ if any(isinstance(c, tuple) for c in nd.args[0]) else FP
        else:
            typ[id(nd)] = max(typ[id(k)] for k in kids)
    groups = {}
    for nd in post:
        if nd.kind == "inv" and varies[id(nd.args[0])] and not has_inv[id(nd.args[0])] and not reads_trace[id(nd.args[0])]:
            groups.setdefault(typ[id(nd)], []).append(nd)
    repl = {}
    for members in groups.values():
        if len(members) < 2:
            continue
        ds = [m.args[0] for m in members]
        prefix = [ds[0]]
        for d in ds[1:]:
            prefix.append(Expr("mul", prefix[-1], d))
        inv = Expr("inv", prefix[-1])
        for i in range(len(ds) - 1, 0, -1):
            repl[id(members[i])] = Expr("mul", inv, prefix[i - 1])
            inv = Expr("mul", inv, ds[i])
        repl[id(members[0])] = inv
    if not repl:
        return root
    rebuilt = {}
    for nd in post:
        if id(nd) in repl:
            rebuilt[id(nd)] = repl[id(nd)]
        else:
            rebuilt[id(nd)] = Expr(nd.kind, *[rebuilt[id(a)] if isinstance(a, Expr) else a for a in nd.args])
    return rebuilt[id(root)]


def _rewrite(roots, trace_len):
    """the evaluator's form of the DAG under `roots` (one memo for all of them, so shared nodes stay shared): a / b becomes
    a * inv(b) with inv(b) hash-consed, so a denominator shared by many constraints (the zerofier X^n - 1) is inverted
    once per point instead of once per Div node; with trace_len, degree adjustments x^(a n + b) become (x^n)^a * x^b"""
    rewritten = {}

    def rewrite(e):
        stack = [e]
        while stack:
            node = stack[-1]
            if id(node) in rewritten:
                stack.pop()
                continue
            kids = [a for a in node.args if isinstance(a, Expr)]
            todo = [a for a in kids if id(a) not in rewritten]
            if todo:
                stack.extend(todo)
                continue
            args = tuple(rewritten[id(a)] if isinstance(a, Expr) else a for a in node.args)
            if node.kind == "div":
                rewritten[id(node)] = Expr("mul", args[0], Expr("inv", args[1]))
            elif node.kind == "pow" and args[0].kind == "x" and trace_len and args[1] >= 2 * trace_len and args[1] % trace_len < 64:
                # degree adjustments are x^(a n + b) with a < ce_blowup and a small b (src/air.rs:50-82): computed as
                # (x^n)^a * x^b they share the log2(n) squarings of x^n — which the zerofier needs anyway — instead of
                # paying ~1.5 log2(a n) multiplications each
                a_, b_ = divmod(args[1], trace_len)
                v = Expr("pow", Expr("pow", args[0], trace_len), a_) if a_ > 1 else Expr("pow", args[0], trace_len)
                if b_:
                    v = Expr("mul", v, Expr("pow", args[0], b_) if b_ > 1 else args[0])
                rewritten[id(node)] = v
            else:
                rewritten[id(node)] = Expr(node.kind, *args)
            stack.pop()
        return rewritten[id(e)]

    return [rewrite(e) for e in roots]


def compile_program(expr, num_base_cols, challenges=(), hints=(), lde_step=1, log_ce=None, fold_pow0=True, symbolic=False,
                    num_cols=None, max_live_leaves=None, batch_inverses=False):
    """Flatten `expr` into the evaluator's linear program.

    batch_inverses: see _batch_inverses — for programs whose denominators cannot vanish on the evaluation domain (the
    AIR composition and DEEP programs built by air.py).

    max_live_leaves: keep at most this many leaf values (trace cells, constants, x) in registers; beyond it the least
    recently used one is dropped and loaded again at its next use.  A sum that names every column twice (the grouped
    DEEP expression, deep.py) then runs in a dozen registers instead of one per column.

    num_cols: total number of trace columns (base + extension); periodic tables take the column slots after them
    (required when the expression has Periodic leaves).

    symbolic=True keeps Challenge / Hint / CompositionCoeff leaves as run-time constants (Program.bind fills them in)
    instead of folding their values into the program: compile once per AIR, bind per proof.

    challenges / hints: extension elements as 3-tuples (or ints) of canonical integers, substituted
    as constants exactly like eval_cpu.rs:116-118.  Trace(col, off) with col < num_base_cols reads a
    base-field column, otherwise extension column col - num_base_cols; the row shift is
    lde_step * off (eval_cpu.rs:119-123).  The result is always stored as an Fq element.
    """
    trace_len = (1 << log_ce) // lde_step if log_ce is not None and lde_step >= 1 else 0
    expr = _rewrite([expr], trace_len)[0]
    if batch_inverses:
        expr = _batch_inverses(expr, num_base_cols)
    code, consts, nregs, typ, bindings, periodic = _lower(
        [expr], lambda k, r, t: [OP_STORE | (t << 8), 0, r, 0], num_base_cols, challenges, hints, lde_step, log_ce, symbolic,
        num_cols, max_live_leaves)
    return Program(code, consts, nregs, typ[id(expr)] == FQ, bindings, periodic)


def compile_extension_program(muls, adds, num_base_cols, log_n, num_cols):
    """Flatten the row maps of K declared extension columns (air.RunningColumn) into ONE evaluator program for
    csrc/extension.cu: mul_k is stored to slot 2k and add_k to slot 2k + 1, subexpressions shared between them are computed
    once per row.  Trace(col, off) reads column[(i + off) mod 2^log_n] of the natural-order trace; X is g_n^i; periodic
    tables come from periodic_tables(ctx, program, log_n, 1, offset_canonical=1).  Challenges and hints stay symbolic
    (Program.bind).  Division is a * inv(b), and the inverse of zero is zero, on the device and in host folding alike."""
    roots = _rewrite([Expr._lift(r) for pair in zip(muls, adds) for r in pair], 0)
    code, consts, nregs, _, bindings, periodic = _lower(
        roots, lambda k, r, t: [OP_STORE | (t << 8), k, r, 0], num_base_cols, (), (), 1, log_n, True, num_cols, None)
    return Program(code, consts, nregs, True, bindings, periodic)


def lookup_slots(width, ntuples):
    """the output slots of a lookup program: the table words 0..W-1, then per value tuple q its selector at
    W + q (W + 1) and its words right after it"""
    return width + ntuples * (width + 1)


def compile_lookup_program(table, values, selectors, num_base_cols, log_n):
    """Flatten one lookup (air.Lookup) into ONE evaluator program for csrc/lookup.cu: table word k is stored to slot k,
    value tuple q's selector (Constant 1 without selectors) to slot W + q (W + 1) and its word k to the slot k + 1 after
    that.  Every expression is over the base field: Trace(col, off) reads column[(i + off) mod 2^log_n] of the
    natural-order trace, X is g_n^i, periodic tables come from periodic_tables(ctx, program, log_n, 1,
    offset_canonical=1).  With no value tuples it stores a permutation's W source words (air.Permutation,
    csrc/permutation.cu)."""
    W = len(table)
    roots = [Expr._lift(t) for t in table]
    for q, v in enumerate(values):
        roots.append(Constant(1) if selectors is None else Expr._lift(selectors[q]))
        roots += [Expr._lift(w) for w in v]
    assert len(roots) == lookup_slots(W, len(values))
    roots = _rewrite(roots, 0)
    code, consts, nregs, _, bindings, periodic = _lower(
        roots, lambda k, r, t: [OP_STORE | (t << 8), k, r, 0], num_base_cols, (), (), 1, log_n, True, num_base_cols, None)
    return Program(code, consts, nregs, False, bindings, periodic)


def compile_check_program(constraints, num_base_cols, log_n, num_cols, symbolic=True, challenges=(), hints=()):
    """Flatten every constraint into ONE checked program for csrc/check.cu, which runs Constraint::check
    (src/constraints.rs:168-249) at every row of the trace domain of size 2^log_n: values carry a None flag, Div is the
    checked division (OP_DIV) and root k ends with OP_CHECK k.  Subexpressions shared by several constraints (x^n - 1,
    a transition term) are hash-consed and computed once per row.

    Unlike compile_program: no a/b -> a * inv(b) rewrite and no batched inverses (a vanishing denominator is exactly
    what the check looks for), and a division whose denominator folds to zero on the host is left to the kernel, so
    host folding gives the kernel's Option result.  Trace(col, off) reads column[(i + off) mod 2^log_n]; periodic
    tables come from periodic_tables(ctx, program, log_n, 1, offset_canonical=1)."""
    roots = list(constraints)
    code, consts, nregs, _, bindings, periodic = _lower(
        roots, lambda k, r, t: [OP_CHECK, 0, r, k], num_base_cols, challenges, hints, 1, log_n, symbolic, num_cols, None)
    return Program(code, consts, nregs, False, bindings, periodic)


def _lower(roots, finish, num_base_cols, challenges, hints, lde_step, log_ce, symbolic, num_cols, max_live_leaves):
    """post-order, constant folding, typing and register allocation of the DAG under `roots`; finish(k, register, type)
    gives the instruction that consumes root k right after it is computed.  Returns (code, consts, nregs, typ,
    bindings, periodic)."""
    order, seen = [], set()

    def visit(e):                      # iterative post-order (DAGs can be deep)
        # Sethi-Ullman flavoured order: the operand with the larger subtree is evaluated first, so a long
        # left-deep sum of constraint terms keeps one accumulator live instead of every term
        size, st = {}, [(e, False)]
        while st:
            node, done = st.pop()
            if done:
                size[id(node)] = 1 + sum(size[id(a)] for a in node.args if isinstance(a, Expr))
                continue
            if id(node) in size:
                continue
            size[id(node)] = 0
            st.append((node, True))
            st.extend((a, False) for a in node.args if isinstance(a, Expr) and id(a) not in size)
        stack = [(e, False)]
        while stack:
            node, done = stack.pop()
            if id(node) in seen and not done:
                continue
            if done:
                order.append(node)
                continue
            seen.add(id(node))
            stack.append((node, True))
            kids = [a for a in node.args if isinstance(a, Expr) and id(a) not in seen]
            kids.sort(key=lambda a: size[id(a)])          # popped last-in first-out: largest subtree first
            for a in kids:
                stack.append((a, False))

    for e in roots:
        visit(e)
    # constant folding + typing
    cval, typ = {}, {}
    for nd in order:
        k, a = nd.kind, nd.args
        if k == "const":
            cval[id(nd)] = a[0]
            typ[id(nd)] = FQ if a[1] else FP
        elif k in _SYMBOLIC and symbolic:
            typ[id(nd)] = FQ
        elif k == "chal":
            cval[id(nd)] = _q(challenges[a[0]])
            typ[id(nd)] = FQ
        elif k == "hint":
            cval[id(nd)] = _q(hints[a[0]])
            typ[id(nd)] = FQ
        elif k == "x":
            typ[id(nd)] = FP
        elif k == "trace":
            typ[id(nd)] = FP if a[0] < num_base_cols else FQ
        elif k == "periodic":
            typ[id(nd)] = FQ if any(isinstance(c, tuple) for c in a[0]) else FP
        else:
            kids = [x for x in a if isinstance(x, Expr)]
            typ[id(nd)] = max(typ[id(x)] for x in kids)
            if all(id(x) in cval for x in kids):
                v = [cval[id(x)] for x in kids]
                if k == "neg":
                    cval[id(nd)] = q_neg(v[0])
                elif k == "add":
                    cval[id(nd)] = q_add(v[0], v[1])
                elif k == "mul":
                    cval[id(nd)] = q_mul(v[0], v[1])
                elif k == "inv":
                    cval[id(nd)] = q_inv(v[0])
                elif k == "pow":
                    cval[id(nd)] = q_pow(v[0], a[1])
                elif k == "div" and any(v[1]):
                    cval[id(nd)] = q_mul(v[0], q_inv(v[1]))     # a zero denominator is left to the checked kernel
    root_of = {}
    for i, e in enumerate(roots):
        root_of.setdefault(id(e), []).append(i)
    # last use (for register reuse), skipping folded nodes
    live_nodes = [nd for nd in order if id(nd) not in cval or id(nd) in root_of]
    last_use = {}
    for idx, nd in enumerate(live_nodes):
        for x in nd.args:
            if isinstance(x, Expr):
                last_use[id(x)] = idx
    consts, const_idx = [], {}

    def const_slot(v):
        if v not in const_idx:
            const_idx[v] = len(consts)
            consts.append([x * _R % P for x in v])      # Montgomery words
        return const_idx[v]

    code, reg_of, free, nregs = [], {}, [], 0
    # Leaves (x, trace loads, constants) are rematerialisable: when the register file is full the least recently used
    # one is dropped and simply loaded again at its next use (large AIRs such as examples/brainfuck touch ~50 distinct
    # trace cells from dozens of constraints).  Interior temporaries are never evicted.
    leaf_regs, pinned, touch = {}, set(), {}

    bindings, sym_slot = [], {}
    periodic, periodic_slot = [], {}

    def is_leaf(x):
        return id(x) in cval or x.kind in ("x", "trace", "periodic") or x.kind in _SYMBOLIC

    def alloc():
        nonlocal nregs
        if free:
            return free.pop()
        if nregs < MAX_REGS:
            nregs += 1
            return nregs - 1
        victims = [k for k in leaf_regs if k not in pinned]
        if not victims:
            raise ValueError(f"expression needs more than {MAX_REGS} live temporaries")
        k = min(victims, key=lambda v: touch.get(v, -1))
        del leaf_regs[k]
        return reg_of.pop(k)

    def emit_leaf(x):
        if max_live_leaves is not None:
            while len(leaf_regs) >= max_live_leaves:
                victims = [k for k in leaf_regs if k not in pinned]
                if not victims:
                    break
                k = min(victims, key=lambda v: touch.get(v, -1))
                del leaf_regs[k]
                free.append(reg_of.pop(k))
        r = alloc()
        if id(x) in cval:
            code.append([OP_CONST | (typ[id(x)] << 8), r, const_slot(cval[id(x)]), 0])
        elif x.kind in _SYMBOLIC:
            key = (x.kind, x.args[0])
            if key not in sym_slot:
                sym_slot[key] = len(consts)
                consts.append([0, 0, 0])
                bindings.append((sym_slot[key], x.kind, x.args[0]))
            code.append([OP_CONST | (FQ << 8), r, sym_slot[key], 0])
        elif x.kind == "x":
            code.append([OP_X, r, 0, 0])
        elif x.kind == "periodic":
            coeffs, interval = x.args
            if num_cols is None:
                raise ValueError("compile_program: num_cols is needed to place the periodic tables")
            if id(x) not in periodic_slot:
                log_len = (interval * lde_step).bit_length() - 1
                if log_ce is not None and log_len > log_ce:
                    raise ValueError("periodic column interval exceeds the trace length")
                periodic_slot[id(x)] = num_cols + len(periodic)
                periodic.append((periodic_slot[id(x)], coeffs, interval, typ[id(x)] == FQ, log_len))
            slot = periodic_slot[id(x)]
            code.append([OP_PERIODIC | (typ[id(x)] << 8), r, slot, periodic[slot - num_cols][4]])
        else:
            col, off = x.args
            shift = lde_step * off
            if log_ce is not None:
                shift %= (1 << log_ce)
            code.append([OP_TRACE | (int(col >= num_base_cols) << 8), r, col, shift & 0xFFFFFFFF])
        reg_of[id(x)] = r
        leaf_regs[id(x)] = x
        return r

    def operand(x):
        """register holding node x (materialising constants and evicted leaves on demand); pins it for this instruction"""
        r = reg_of[id(x)] if id(x) in reg_of else emit_leaf(x)
        pinned.add(id(x))
        touch[id(x)] = len(code)
        return r

    def release(x, idx):
        if last_use.get(id(x)) == idx and id(x) in reg_of:
            free.append(reg_of.pop(id(x)))
            leaf_regs.pop(id(x), None)

    def finish_roots(nd, idx):
        for i in root_of.get(id(nd), ()):
            code.append(finish(i, reg_of[id(nd)], typ[id(nd)]))
        if last_use.get(id(nd), -1) <= idx and id(nd) in reg_of:     # no later consumer: the register is free again
            free.append(reg_of.pop(id(nd)))
            leaf_regs.pop(id(nd), None)

    for idx, nd in enumerate(live_nodes):
        k, a = nd.kind, nd.args
        pinned.clear()
        if is_leaf(nd):
            if id(nd) in root_of:     # a root that is itself a leaf / constant
                operand(nd)
                finish_roots(nd, idx)
            continue                  # loaded lazily at first use
        if k == "neg":
            ra = operand(a[0])
            release(a[0], idx)
            r = alloc()
            code.append([OP_NEG | (typ[id(a[0])] << 8), r, ra, 0])
        elif k in ("add", "mul", "div"):
            ra, rb = operand(a[0]), operand(a[1])
            release(a[0], idx)
            release(a[1], idx)
            r = alloc()
            op = {"add": OP_ADD, "mul": OP_MUL, "div": OP_DIV}[k]
            code.append([op | (typ[id(a[0])] << 8) | (typ[id(a[1])] << 9), r, ra, rb])
        elif k == "inv":
            ra = operand(a[0])
            release(a[0], idx)
            r = alloc()
            code.append([OP_INV | (typ[id(a[0])] << 8), r, ra, 0])
        elif k == "pow":
            ra = operand(a[0])
            release(a[0], idx)
            r = alloc()
            if a[1] >= 2**32:
                raise ValueError("exponent too large")
            code.append([OP_POW | (typ[id(a[0])] << 8), r, ra, a[1]])
        else:
            raise ValueError(f"unsupported node {k}")
        reg_of[id(nd)] = r
        if id(nd) in root_of:
            finish_roots(nd, idx)
    return (np.array(code, dtype=np.uint32), np.array(consts if consts else [[0, 0, 0]], dtype=np.uint64), max(nregs, 1), typ,
            bindings, periodic)
