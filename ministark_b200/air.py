"""air.py — host-side mirror of the reference's AIR description for the prover driver (prover.py).

    ProofOptions                      src/lib.rs:86-132
    AirConfig / Air                   src/air.rs:26-247
    constraint degree bookkeeping     src/constraints.rs:131-146,325-347,404-455
    composition constraint            src/air.rs:50-82

Constraints are `ministark_b200.expr.Expr` DAGs over the leaves X | Constant | Challenge(i) | Hint(i) |
Trace(column, offset) | Periodic(coeffs, interval_size) plus, inside the
composition constraint only, CompositionCoeff(i) — the verifier randomness that is substituted as
constants once the channel has produced it (src/air.rs:96-101).

Extension columns may be declared the same way (AirConfig.extension_columns, RunningColumn): the prover then builds them
on the device from the base trace instead of calling a host builder.  So may LogUp lookups (AirConfig.lookups, Lookup) and
sorted-copy permutation arguments (AirConfig.permutations, Permutation), whose constraints the package generates.

This module is pure bookkeeping (a few hundred DAG nodes): no field data is touched here.
"""
from dataclasses import dataclass

from . import expr as E

P = E.P
TWO_ADIC_ROOT = pow(7, (P - 1) >> 32, P)        # arkworks' 2^32-th root of unity for Goldilocks (SURVEY.md §8c)
GENERATOR = 7                                    # Fp::GENERATOR, the LDE coset offset (src/air.rs:42-44)


def domain_generator(log_n):
    """Radix2EvaluationDomain::group_gen for size 2^log_n"""
    return pow(TWO_ADIC_ROOT, 1 << (32 - log_n), P)


@dataclass(frozen=True)
class ProofOptions:
    num_queries: int
    lde_blowup_factor: int
    grinding_factor: int
    fri_folding_factor: int
    fri_max_remainder_coeffs: int

    def __post_init__(self):
        # the reference's const asserts, src/lib.rs:109-114
        assert 1 <= self.num_queries <= 128
        b = self.lde_blowup_factor
        assert 1 <= b <= 128 and b & (b - 1) == 0
        assert self.grinding_factor <= 50
        assert self.fri_folding_factor in (2, 4, 8, 16)          # src/fri.rs:185-192

    def to_bytes(self):
        """derived CanonicalSerialize: the five u8 fields in declaration order"""
        return bytes([self.num_queries, self.lde_blowup_factor, self.grinding_factor, self.fri_folding_factor,
                      self.fri_max_remainder_coeffs])

    # FriOptions (src/fri.rs:30-69)
    def fri_num_layers(self, domain_size):
        k = 0
        while domain_size > self.fri_max_remainder_coeffs * self.lde_blowup_factor:
            domain_size //= self.fri_folding_factor
            k += 1
        return k

    def fri_remainder_size(self, domain_size):
        while domain_size > self.fri_max_remainder_coeffs * self.lde_blowup_factor:
            domain_size //= self.fri_folding_factor
        return domain_size


def CompositionCoeff(i):
    return E.Expr("ccoef", int(i))


def _ceil_power_of_two(v):
    """src/utils.rs:76-82 (0 is not a power of two and 0usize.next_power_of_two() == 1)"""
    if v == 0:
        return 1
    return v if v & (v - 1) == 0 else 1 << v.bit_length()


def degree(expr, trace_degree):
    """(numerator degree, denominator degree) by the reference's rules (src/constraints.rs:404-455): Add takes the
    cross-multiplied maximum and ADDS the denominators, Neg is the identity, Mul/Div/Pow as for rational functions."""
    memo = {}
    order, seen = [], set()
    stack = [(expr, False)]
    while stack:
        node, done = stack.pop()
        if done:
            order.append(node)
            continue
        if id(node) in seen:
            continue
        seen.add(id(node))
        stack.append((node, True))
        for a in node.args:
            if isinstance(a, E.Expr) and id(a) not in seen:
                stack.append((a, False))
    for nd in order:
        k, a = nd.kind, nd.args
        if k in ("const", "chal", "hint", "ccoef"):
            d = (0, 0)
        elif k == "trace":
            d = (trace_degree, 0)
        elif k == "x":
            d = (1, 0)
        elif k == "periodic":
            # PeriodicColumn::degree (src/constraints.rs:131-138): (len(coeffs) - 1) * (trace_len / interval_size)
            d = ((len(a[0]) - 1) * ((trace_degree + 1) // a[1]), 0)
        elif k == "neg":
            d = memo[id(a[0])]
        elif k == "add":
            (an, ad), (bn, bd) = memo[id(a[0])], memo[id(a[1])]
            d = (max(an + bd, bn + ad), ad + bd)
        elif k == "mul":
            (an, ad), (bn, bd) = memo[id(a[0])], memo[id(a[1])]
            d = (an + bn, ad + bd)
        elif k == "div":
            (an, ad), (bn, bd) = memo[id(a[0])], memo[id(a[1])]
            d = (an + bd, ad + bn)
        elif k == "pow":
            n, dd = memo[id(a[0])]
            d = (n * a[1], dd * a[1])
        else:
            raise ValueError(f"unsupported node {k}")
        memo[id(nd)] = d
    return memo[id(expr)]


def blowup_factor(expr, trace_len):
    """Constraint::blowup_factor (src/constraints.rs:142-146,340-347)"""
    trace_degree = trace_len - 1
    num, den = degree(expr, trace_degree)
    deg = max(num - den, 0)                                    # saturating_sub
    return _ceil_power_of_two(deg) // trace_degree


def _leaves(expr, kind):
    out, seen, stack = set(), set(), [expr]
    while stack:
        node = stack.pop()
        if id(node) in seen:
            continue
        seen.add(id(node))
        if node.kind == kind:
            out.add(node.args)
        stack.extend(a for a in node.args if isinstance(a, E.Expr))
    return out


MAX_DECLARED_COLUMNS = 8                         # csrc/extension.cu builds at most this many columns in one pass


@dataclass(frozen=True)
class RunningColumn:
    """One declared extension column: x_0 = init, x_(i+1) = x_i * mul(i) + add(i) over the trace domain, a running
    product (add = 0), running evaluation (mul = a challenge) or running sum (mul = 1).  Row i holds x_i, or x_(i+1) when
    `inclusive`.  Values are in Fq (Fq3, or Fp when FQ_IS_FP).

    mul / add: Exprs (or field values) over Constant, Challenge, Hint, X, Periodic and Trace(c, offset) of a BASE column
    c, any offset; the row index wraps mod n as in constraint evaluation on the trace domain, and X at row i is g_n^i.
    Division is allowed, and a zero denominator gives 0 (the inverse of zero is zero), so a LogUp-style
    add = m / (alpha - t) - 1 / (alpha - v) can be declared.  init: an Expr (or field value) over Constant, Challenge and
    Hint only, evaluated on the host."""
    init: object
    mul: object = 1
    add: object = 0
    inclusive: bool = False


def _as_expr(v):
    if isinstance(v, E.Expr):
        return v
    return E.Constant(tuple(v)) if isinstance(v, (tuple, list)) else E.Constant(v)


MAX_LOOKUP_WIDTH = 4                             # csrc/lookup.cu: at most this many words per tuple
MAX_LOOKUP_TUPLES = 4                            # and this many value tuples per lookup


@dataclass(frozen=True)
class Lookup:
    """One LogUp lookup (AirConfig.lookups): at every row i where selectors[q](i) == 1 (every row without selectors), the
    tuple values[q] at row i is a row of the table, the tuple `table` at row j for j = 0..n-1.  Every row of `table` is a
    table entry; pad a short table by repeating a real entry.

    table: W Exprs (or Fp values), values: Q tuples of W Exprs, selectors: None or Q Exprs, 1 <= W, Q <= 4.  They read
    Constant (Fp), X, Periodic and Trace(c, offset) of a base column c at any offset (the row index wraps mod n); never a
    challenge, a hint, an extension column or a multiplicity column, since the multiplicities are filled before the base
    trace is committed.

    multiplicity: a base column the prover writes: row j holds the number of (row, value tuple) pairs that look up the
    table tuple at row j; a tuple that occurs more than once in the table counts at its lowest row only, the others get 0.
    running_sum: an extension column the package declares and constrains.  AirConfig.extension_columns returns None at
    its position.

    Challenges: with c0 the number of challenges the AIR's own constraints draw, lookup l (in declaration order) takes the
    next index as alpha_l, and one more as beta_l only when W > 1.  Tuples are compressed as t_0 + beta t_1 + beta^2 t_2 +
    ..., and d_0 = alpha - (table tuple), d_q = alpha - (value tuple q).  The running sum is s_0 = 0,
    s_(i+1) = s_i + m_i / d_0 - sum_q sigma_q / d_q (sigma_q: the selector, 1 without one), and three constraints are
    appended after the AIR's own, per lookup: s_0 = 0, the step with its denominators cleared on every row but the last,
    and the whole sum being zero at the last row.

    Soundness: the multiplicity fill is untrusted prover work; the generated constraints are what make a proof a proof of
    the lookup.  The package does not constrain a selector to {0, 1}: if it is a witness column, the AIR must.  With
    FQ_IS_FP = True alpha is drawn from the 64-bit base field, and the argument's soundness error is about (Q + 1) n / p."""
    table: tuple
    values: tuple
    multiplicity: int
    running_sum: int
    selectors: tuple = None


MAX_PERMUTATION_WIDTH = 4                        # csrc/permutation.cu: at most this many words per tuple


@dataclass(frozen=True)
class Permutation:
    """One sorted-copy permutation argument (AirConfig.permutations): the target columns hold the source tuples of every
    row, sorted.  It is how a read/write memory is proven: the accesses in execution order are the source, the same
    accesses sorted by (address, clock) the target, and the AIR's own constraints check the sorted table row by row.

    source: W Exprs (or Fp values), 1 <= W <= 4.  They read Constant (Fp), X, Periodic and Trace(c, offset) of a base
    column c at any offset (the row index wraps mod n); never a challenge, a hint, an extension column, a permutation's
    target column or a lookup's multiplicity column, since the targets are filled before the base trace is committed.

    target: W distinct base columns the prover writes: row j of target[k] holds word k of the j-th source tuple in
    ascending lexicographic order of the canonical integers, word 0 first.  Equal tuples keep their row order (the sort
    is stable), so an AIR that wants "by address, then clock" orders its tuple that way.  The targets are filled before
    the lookups' multiplicities, so a lookup may read them.
    running_product: an extension column the package declares and constrains.  AirConfig.extension_columns returns
    None at its position.

    Challenges: after the AIR's own and the lookups', permutation p (in declaration order) takes the next index as
    alpha_p, and one more as beta_p only when W > 1.  Tuples are compressed as c(t) = t_0 + beta t_1 + beta^2 t_2 + ....
    The running product is z_0 = 1, z_(i+1) = z_i (alpha - c(source_i)) / (alpha - c(target_i)), and three constraints are
    appended after the lookups', per permutation: z_0 = 1; on every row but the last, the step with its denominator
    cleared, z_(i+1) (alpha - c(target_i)) - z_i (alpha - c(source_i)); at the last row,
    z_(n-1) (alpha - c(source_(n-1))) - (alpha - c(target_(n-1))).

    Soundness: the fill is untrusted prover work, and the generated constraints prove only that the target rows are a
    permutation of the source rows.  That the target is SORTED is not proven by the package: an AIR that relies on the
    order must constrain it itself, for example with a range-check Lookup on the differences of its keys.  The
    argument's error is at most about W n / |Fq| (Schwartz-Zippel in alpha and beta): with FQ_IS_FP = True and
    n = 2^24 rows, about 2^-38."""
    source: tuple
    target: tuple
    running_product: int


class AirConfig:
    """Subclass and override, as with the reference's trait (src/air.rs:26-48).  Field values handed to and
    returned by the hooks are canonical integers (Fp) or 3-tuples of canonical integers (Fq3)."""
    NUM_BASE_COLUMNS = 0
    NUM_EXTENSION_COLUMNS = 0
    FQ_IS_FP = True              # type Fq = Fp (examples/fib) vs. Fq = Fq3 (examples/brainfuck)

    @staticmethod
    def constraints(trace_len):
        raise NotImplementedError

    @staticmethod
    def gen_hints(trace_len, public_inputs, challenges):
        return []

    @staticmethod
    def domain_offset():
        return GENERATOR

    @staticmethod
    def extension_columns(trace_len):
        """None (the trace builds its own extension columns), or one RunningColumn per extension column, in column
        order: the prover then builds them on the device from the base trace whenever the trace brings no builder of its
        own.  A declaration adds no constraint: the AIR's constraints must still enforce every declared column.  With
        lookups or permutations: None at every lookup's running-sum and every permutation's running-product position (the
        package declares those columns), or None as a whole when every extension column is one of them."""
        return None

    @staticmethod
    def lookups(trace_len):
        """the AIR's LogUp lookups (Lookup), in declaration order.  The package generates their constraints and
        running-sum columns, and the prover fills their multiplicity columns on the device."""
        return []

    @staticmethod
    def permutations(trace_len):
        """the AIR's sorted-copy permutation arguments (Permutation), in declaration order.  The package generates their
        constraints and running-product columns, and the prover fills their target columns on the device."""
        return []


class Air:
    """Air::new (src/air.rs:142-160): constraints, the composition constraint and the ce blow-up factor."""

    def __init__(self, config, trace_len, public_inputs, options):
        assert trace_len & (trace_len - 1) == 0
        self.config, self.trace_len, self.public_inputs, self.options = config, trace_len, public_inputs, options
        self.log_n = trace_len.bit_length() - 1
        self.constraints = list(config.constraints(trace_len))
        hook = getattr(config, "lookups", None)
        self.lookups = self._lookups(list(hook(trace_len)) if hook is not None else [])
        hook = getattr(config, "permutations", None)
        self.permutations = self._permutations(list(hook(trace_len)) if hook is not None else [])
        self.constraints += self._lookup_constraints() + self._permutation_constraints()
        # AirConfig::composition_constraint (src/air.rs:50-82)
        ce_blowup = max(blowup_factor(c, trace_len) for c in self.constraints)
        composition_degree = trace_len * ce_blowup - 1
        trace_degree = trace_len - 1
        x = E.X()
        total = None
        for i, c in enumerate(self.constraints):
            num, den = degree(c, trace_degree)
            evaluation_degree = num - den
            assert evaluation_degree <= composition_degree
            adj = composition_degree - evaluation_degree
            term = c * (x ** adj * CompositionCoeff(2 * i) + CompositionCoeff(2 * i + 1))
            total = term if total is None else total + term
        self.composition_constraint = total
        self.ce_blowup_factor = blowup_factor(total, trace_len)
        assert self.ce_blowup_factor <= options.lde_blowup_factor
        hook = getattr(config, "extension_columns", None)
        self.extension_declaration = self._declaration(self._merge_generated(hook(trace_len) if hook is not None else None))

    def _lookups(self, decl):
        """AirConfig.lookups checked against the AIR: Lookups with Expr fields, or ValueError.  Also assigns each lookup its
        challenges (self.lookup_challenges: (alpha index, beta index or None))"""
        cfg = self.config
        nbase, next_ = cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS
        idx = [a[0] for c in self.constraints for a in _leaves(c, "chal")]
        chal = max(idx) + 1 if idx else 0
        out, self.lookup_challenges = [], []
        mults, sums = {}, {}
        for l, lk in enumerate(decl):
            if not isinstance(lk, Lookup):
                raise ValueError(f"lookup {l}: expected a Lookup, got {type(lk).__name__}")
            m, s = lk.multiplicity, lk.running_sum
            if not 0 <= m < nbase:
                raise ValueError(f"lookup {l}: multiplicity column {m} is not a base column (0..{nbase - 1})")
            if m in mults:
                raise ValueError(f"lookup {l}: multiplicity column {m} is also lookup {mults[m]}'s")
            if not nbase <= s < nbase + next_:
                raise ValueError(f"lookup {l}: running-sum column {s} is not an extension column ({nbase}..{nbase + next_ - 1})")
            if s in sums:
                raise ValueError(f"lookup {l}: running-sum column {s} is also lookup {sums[s]}'s")
            mults[m], sums[s] = l, l
            table, values = tuple(lk.table), tuple(tuple(v) for v in lk.values)
            W, Q = len(table), len(values)
            if not 1 <= W <= MAX_LOOKUP_WIDTH:
                raise ValueError(f"lookup {l}: table tuples of width {W}; 1 to {MAX_LOOKUP_WIDTH} are supported")
            if not 1 <= Q <= MAX_LOOKUP_TUPLES:
                raise ValueError(f"lookup {l}: {Q} value tuples; 1 to {MAX_LOOKUP_TUPLES} are supported")
            for q, v in enumerate(values):
                if len(v) != W:
                    raise ValueError(f"lookup {l}: value tuple {q} has width {len(v)}, the table {W}")
            sel = None if lk.selectors is None else tuple(lk.selectors)
            if sel is not None and len(sel) != Q:
                raise ValueError(f"lookup {l}: {len(sel)} selectors for {Q} value tuples")
            out.append(Lookup(tuple(_as_expr(t) for t in table), tuple(tuple(_as_expr(w) for w in v) for v in values), m, s,
                              None if sel is None else tuple(_as_expr(e) for e in sel)))
            self.lookup_challenges.append((chal, chal + 1 if W > 1 else None))
            chal += 2 if W > 1 else 1
        self._next_challenge = chal
        for l, lk in enumerate(out):
            named = [(f"table[{k}]", e) for k, e in enumerate(lk.table)]
            named += [(f"values[{q}][{k}]", e) for q, v in enumerate(lk.values) for k, e in enumerate(v)]
            named += [(f"selectors[{q}]", e) for q, e in enumerate(lk.selectors or ())]
            for name, e in named:
                for kind, what in (("chal", "a challenge"), ("hint", "a hint"), ("ccoef", "a composition coefficient")):
                    if _leaves(e, kind):
                        raise ValueError(f"lookup {l}: {name} reads {what}")
                if any(ext for _, ext in _leaves(e, "const")):
                    raise ValueError(f"lookup {l}: {name} reads an extension-field constant")
                for col, off in sorted(_leaves(e, "trace")):
                    if col in mults:
                        raise ValueError(f"lookup {l}: {name} reads Trace({col}, {off}), the multiplicity column of lookup "
                                         f"{mults[col]}")
                    if not 0 <= col < nbase:
                        raise ValueError(f"lookup {l}: {name} reads Trace({col}, {off}), which is not a base column "
                                         f"(0..{nbase - 1})")
        return out

    def _permutations(self, decl):
        """AirConfig.permutations checked against the AIR and its lookups: Permutations with Expr sources, or ValueError.
        Also assigns each permutation its challenges (self.permutation_challenges: (alpha index, beta index or None)),
        after the lookups'"""
        cfg = self.config
        nbase, next_ = cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS
        mults = {lk.multiplicity: l for l, lk in enumerate(self.lookups)}
        sums = {lk.running_sum: l for l, lk in enumerate(self.lookups)}
        chal = self._next_challenge
        out, self.permutation_challenges = [], []
        targets, products = {}, {}
        for p, pm in enumerate(decl):
            if not isinstance(pm, Permutation):
                raise ValueError(f"permutation {p}: expected a Permutation, got {type(pm).__name__}")
            source, target = tuple(pm.source), tuple(int(t) for t in pm.target)
            W = len(source)
            if not 1 <= W <= MAX_PERMUTATION_WIDTH:
                raise ValueError(f"permutation {p}: source tuples of width {W}; 1 to {MAX_PERMUTATION_WIDTH} are supported")
            if len(target) != W:
                raise ValueError(f"permutation {p}: {len(target)} target columns for source tuples of width {W}")
            for t in target:
                if not 0 <= t < nbase:
                    raise ValueError(f"permutation {p}: target column {t} is not a base column (0..{nbase - 1})")
                if t in targets:
                    who = "repeated" if targets[t] == p else f"also permutation {targets[t]}'s"
                    raise ValueError(f"permutation {p}: target column {t} is {who}")
                if t in mults:
                    raise ValueError(f"permutation {p}: target column {t} is the multiplicity column of lookup {mults[t]}")
                targets[t] = p
            z = pm.running_product
            if not nbase <= z < nbase + next_:
                raise ValueError(f"permutation {p}: running-product column {z} is not an extension column "
                                 f"({nbase}..{nbase + next_ - 1})")
            if z in sums:
                raise ValueError(f"permutation {p}: running-product column {z} is lookup {sums[z]}'s running sum")
            if z in products:
                raise ValueError(f"permutation {p}: running-product column {z} is also permutation {products[z]}'s")
            products[z] = p
            out.append(Permutation(tuple(_as_expr(e) for e in source), target, z))
            self.permutation_challenges.append((chal, chal + 1 if W > 1 else None))
            chal += 2 if W > 1 else 1
        for p, pm in enumerate(out):
            for k, e in enumerate(pm.source):
                for kind, what in (("chal", "a challenge"), ("hint", "a hint"), ("ccoef", "a composition coefficient")):
                    if _leaves(e, kind):
                        raise ValueError(f"permutation {p}: source[{k}] reads {what}")
                if any(ext for _, ext in _leaves(e, "const")):
                    raise ValueError(f"permutation {p}: source[{k}] reads an extension-field constant")
                for col, off in sorted(_leaves(e, "trace")):
                    if col in targets:
                        raise ValueError(f"permutation {p}: source[{k}] reads Trace({col}, {off}), a target column of "
                                         f"permutation {targets[col]}")
                    if col in mults:
                        raise ValueError(f"permutation {p}: source[{k}] reads Trace({col}, {off}), the multiplicity column "
                                         f"of lookup {mults[col]}")
                    if not 0 <= col < nbase:
                        raise ValueError(f"permutation {p}: source[{k}] reads Trace({col}, {off}), which is not a base "
                                         f"column (0..{nbase - 1})")
        return out

    @staticmethod
    def _compressed(beta, tup):
        """t_0 + beta t_1 + beta^2 t_2 + ... with beta = Challenge(beta)"""
        acc = tup[0]
        bpow = None
        for t in tup[1:]:
            bpow = E.Challenge(beta) if bpow is None else bpow * E.Challenge(beta)
            acc = acc + bpow * t
        return acc

    def _lookup_denominators(self, l):
        lk = self.lookups[l]
        a, b = self.lookup_challenges[l]
        alpha = E.Challenge(a)
        return [alpha - self._compressed(b, lk.table)] + [alpha - self._compressed(b, v) for v in lk.values]

    def _permutation_denominators(self, p):
        """(alpha - c(source), alpha - c(target)) of permutation p"""
        pm = self.permutations[p]
        a, b = self.permutation_challenges[p]
        alpha = E.Challenge(a)
        return alpha - self._compressed(b, pm.source), alpha - self._compressed(b, [E.Trace(t, 0) for t in pm.target])

    def _lookup_constraints(self):
        """the three constraints of every lookup (Lookup), appended after the AIR's own.  With Q = 1, W = 1 and no selectors
        they are, node for node, the LogUp constraints examples/lookup.py's LookupAirConfig writes by hand."""
        n = self.trace_len
        g = domain_generator(self.log_n)
        x, one = E.X(), E.Constant(1)
        first, last = E.Constant(1), E.Constant(pow(g, n - 1, P))
        but_last = (x - last) / (x ** n - one)
        out = []
        for l, lk in enumerate(self.lookups):
            d = self._lookup_denominators(l)
            Q = len(lk.values)
            m, s, s1 = E.Trace(lk.multiplicity, 0), E.Trace(lk.running_sum, 0), E.Trace(lk.running_sum, 1)
            num = m
            for dq in d[1:]:
                num = num * dq
            for q in range(1, Q + 1):
                term = None
                for r in range(Q + 1):
                    if r != q:
                        term = d[r] if term is None else term * d[r]
                if lk.selectors is not None:
                    term = lk.selectors[q - 1] * term
                num = num - term
            step, total = s1 - s, s
            for dq in d:
                step, total = step * dq, total * dq
            out += [s / (x - first), (step - num) * but_last, (total + num) / (x - last)]
        return out

    def _permutation_constraints(self):
        """the three constraints of every permutation (Permutation), appended after the lookups'.  They are, node for node,
        the ones examples/memory.py's MemoryAirConfig writes by hand."""
        n = self.trace_len
        g = domain_generator(self.log_n)
        x, one = E.X(), E.Constant(1)
        first, last = E.Constant(1), E.Constant(pow(g, n - 1, P))
        but_last = (x - last) / (x ** n - one)
        out = []
        for p, pm in enumerate(self.permutations):
            ds, dt = self._permutation_denominators(p)
            z, z1 = E.Trace(pm.running_product, 0), E.Trace(pm.running_product, 1)
            out += [(z - one) / (x - first), (z1 * dt - z * ds) * but_last, (z * ds - dt) / (x - last)]
        return out

    def _merge_generated(self, decl):
        """the user's extension_columns with every lookup's running sum (RunningColumn(init=0, add=m / d_0 -
        sum_q sigma_q / d_q)) and every permutation's running product (RunningColumn(init=1, mul=(alpha - c(source)) /
        (alpha - c(target)))) put in its place, or ValueError"""
        if not self.lookups and not self.permutations:
            return decl
        cfg = self.config
        nbase, next_ = cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS
        pos = {lk.running_sum - nbase: (f"lookup {l}'s running sum", l) for l, lk in enumerate(self.lookups)}
        ppos = {pm.running_product - nbase: (f"permutation {p}'s running product", p) for p, pm in enumerate(self.permutations)}
        if decl is None:
            if len(pos) + len(ppos) != next_:
                raise ValueError(f"extension_columns returned None, but only {len(pos) + len(ppos)} of the {next_} extension "
                                 f"columns are lookup running sums or permutation running products")
            decl = [None] * next_
        decl = list(decl)
        if len(decl) != next_:
            raise ValueError(f"extension_columns declares {len(decl)} columns but NUM_EXTENSION_COLUMNS is {next_}")
        for k, col in enumerate(decl):
            if (k in pos or k in ppos) and col is not None:
                raise ValueError(f"extension column {nbase + k}: {(pos.get(k) or ppos[k])[0]} is declared by the package; "
                                 f"extension_columns must return None there")
            if k not in pos and k not in ppos and not isinstance(col, RunningColumn):
                raise ValueError(f"extension column {nbase + k}: expected a RunningColumn, got {type(col).__name__}")
        for k, (_, l) in pos.items():
            lk, d = self.lookups[l], self._lookup_denominators(l)
            add = E.Trace(lk.multiplicity, 0) / d[0]
            for q, dq in enumerate(d[1:]):
                add = add - (E.Constant(1) if lk.selectors is None else lk.selectors[q]) / dq
            decl[k] = RunningColumn(init=0, add=add)
        for k, (_, p) in ppos.items():
            ds, dt = self._permutation_denominators(p)
            decl[k] = RunningColumn(init=1, mul=ds / dt)
        return decl

    def _declaration(self, decl):
        """AirConfig.extension_columns checked against the AIR: RunningColumns with Expr fields, or ValueError"""
        if decl is None:
            return None
        cfg = self.config
        decl = list(decl)
        if len(decl) != cfg.NUM_EXTENSION_COLUMNS:
            raise ValueError(f"extension_columns declares {len(decl)} columns but NUM_EXTENSION_COLUMNS is "
                             f"{cfg.NUM_EXTENSION_COLUMNS}")
        if len(decl) > MAX_DECLARED_COLUMNS:
            raise ValueError(f"extension_columns declares {len(decl)} columns; at most {MAX_DECLARED_COLUMNS} can be built")
        nchal = self.num_challenges()
        out = []
        for k, col in enumerate(decl):
            c = cfg.NUM_BASE_COLUMNS + k
            if not isinstance(col, RunningColumn):
                raise ValueError(f"extension column {c}: expected a RunningColumn, got {type(col).__name__}")
            col = RunningColumn(_as_expr(col.init), _as_expr(col.mul), _as_expr(col.add), bool(col.inclusive))
            for name in ("init", "mul", "add"):
                e = getattr(col, name)
                for kind in ("ccoef",) + (("trace", "x", "periodic") if name == "init" else ()):
                    if _leaves(e, kind):
                        what = {"ccoef": "a composition coefficient", "trace": "the trace", "x": "X",
                                "periodic": "a periodic column"}[kind]
                        raise ValueError(f"extension column {c}: {name} reads {what}")
                for col_idx, off in sorted(_leaves(e, "trace")):
                    if not 0 <= col_idx < cfg.NUM_BASE_COLUMNS:
                        raise ValueError(f"extension column {c}: {name} reads Trace({col_idx}, {off}), which is not a base "
                                         f"column (0..{cfg.NUM_BASE_COLUMNS - 1})")
                for (i,) in sorted(_leaves(e, "chal")):
                    if i >= nchal:
                        raise ValueError(f"extension column {c}: {name} reads Challenge({i}), but the constraints make the "
                                         f"channel draw {nchal} challenges")
            out.append(col)
        return out

    def lde_blowup_factor(self):
        return self.options.lde_blowup_factor

    # ---- compiled evaluator programs, shared by every proof of this AIR and trace length (the verifier randomness
    # enters through Program.bind, not through the instruction stream)
    def composition_program(self):
        if getattr(self, "_composition_program", None) is None:
            cfg = self.config
            log_ce = self.log_n + self.ce_blowup_factor.bit_length() - 1
            self._composition_program = E.compile_program(self.composition_constraint, cfg.NUM_BASE_COLUMNS,
                                                          lde_step=self.ce_blowup_factor, log_ce=log_ce, symbolic=True,
                                                          batch_inverses=True)   # zerofier denominators: never 0 on the LDE coset
        return self._composition_program

    def deep_program(self):
        if getattr(self, "_deep_program", None) is None:
            from . import deep
            cfg = self.config
            log_N = self.log_n + self.options.lde_blowup_factor.bit_length() - 1
            expr, keys = deep.deep_expression_symbolic(self.trace_arguments(), cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS,
                                                       self.ce_blowup_factor)
            self._deep_program = (E.compile_program(expr, cfg.NUM_BASE_COLUMNS, log_ce=log_N, symbolic=True, max_live_leaves=8,
                                                    batch_inverses=True), keys)
        return self._deep_program

    def check_program(self):
        """every constraint as one checked program over the trace domain (csrc/check.cu; challenges and hints are bound
        per proof), for the prover's optional constraint validation (ministark_b200/validate.py)"""
        if getattr(self, "_check_program", None) is None:
            cfg = self.config
            self._check_program = E.compile_check_program(self.constraints, cfg.NUM_BASE_COLUMNS, self.log_n,
                                                          cfg.NUM_BASE_COLUMNS + cfg.NUM_EXTENSION_COLUMNS)
        return self._check_program

    def extension_program(self):
        """the declared extension columns' row maps as one evaluator program (csrc/extension.cu; challenges and hints are
        bound per proof), or None without a declaration"""
        if getattr(self, "_extension_program", None) is None and self.extension_declaration:
            d = self.extension_declaration
            self._extension_program = E.compile_extension_program([c.mul for c in d], [c.add for c in d],
                                                                  self.config.NUM_BASE_COLUMNS, self.log_n,
                                                                  self.config.NUM_BASE_COLUMNS)
        return getattr(self, "_extension_program", None)

    def lookup_programs(self):
        """one evaluator program per lookup, for its multiplicity fill (csrc/lookup.cu, expr.compile_lookup_program)"""
        if getattr(self, "_lookup_programs", None) is None:
            nbase = self.config.NUM_BASE_COLUMNS
            self._lookup_programs = [E.compile_lookup_program(lk.table, lk.values, lk.selectors, nbase, self.log_n)
                                     for lk in self.lookups]
        return self._lookup_programs

    def permutation_programs(self):
        """one evaluator program per permutation, storing its source words, for its target fill (csrc/permutation.cu;
        expr.compile_lookup_program with no value tuples)"""
        if getattr(self, "_permutation_programs", None) is None:
            nbase = self.config.NUM_BASE_COLUMNS
            self._permutation_programs = [E.compile_lookup_program(pm.source, (), None, nbase, self.log_n)
                                          for pm in self.permutations]
        return self._permutation_programs

    # the three walks below depend on the constraints only: done once per Air (the provers copy a cached Air per proof,
    # and each walk of the brainfuck AIR costs ~0.5 ms of a 10 ms proof)
    def num_challenges(self):
        if getattr(self, "_num_challenges", None) is None:
            idx = [a[0] for c in self.constraints for a in _leaves(c, "chal")]
            self._num_challenges = max(idx) + 1 if idx else 0
        return self._num_challenges

    def num_composition_constraint_coeffs(self):
        if getattr(self, "_num_ccoefs", None) is None:
            idx = [a[0] for a in _leaves(self.composition_constraint, "ccoef")]
            self._num_ccoefs = max(idx) + 1 if idx else 0
        return self._num_ccoefs

    def gen_hints(self, challenges):
        return self.config.gen_hints(self.trace_len, self.public_inputs, challenges)

    def trace_arguments(self):
        """BTreeSet<(column, offset)> — sorted by column, then signed offset (src/air.rs:240-246)"""
        if getattr(self, "_trace_arguments", None) is None:
            args = set()
            for c in self.constraints:
                args |= _leaves(c, "trace")
            self._trace_arguments = sorted(args)
        return list(self._trace_arguments)

    def substitute_composition_coeffs(self, coeffs):
        """the map_leaves of AirConfig::eval_constraint (src/air.rs:96-101): CompositionCoeff(i) -> Constant"""
        memo = {}

        def sub(e):
            stack = [e]
            while stack:
                node = stack[-1]
                if id(node) in memo:
                    stack.pop()
                    continue
                todo = [a for a in node.args if isinstance(a, E.Expr) and id(a) not in memo]
                if todo:
                    stack.extend(todo)
                    continue
                if node.kind == "ccoef":
                    v = coeffs[node.args[0]]
                    memo[id(node)] = E.Constant(v) if isinstance(v, (tuple, list)) else E.Constant(v, ext=True)
                else:
                    memo[id(node)] = E.Expr(node.kind, *[memo[id(a)] if isinstance(a, E.Expr) else a for a in node.args])
                stack.pop()
            return memo[id(e)]

        return sub(self.composition_constraint)
