"""validate.py — the reference's unfinished default_validate_constraints (src/debug.rs:10-128), on the device.

The reference's debug builds call Stark::validate_constraints (src/stark.rs:65-75) right after the extension trace
commitment (src/prover.rs:74-75); its body is a TODO whose intended algorithm is left as a comment: warn about trace
columns, challenges and hints no constraint uses, evaluate every constraint at every row of the trace domain with
Constraint::check (src/constraints.rs:168-249: division by zero with a non-zero numerator gives None) and report the
first constraint that is None somewhere, with its row and the values of x, of each Trace(col, offset), each challenge and
each hint in it.  Without the check an invalid trace still proves (every committed polynomial is low degree by
construction) and only the verifier's out-of-domain check rejects it, naming nothing.

Here every constraint is checked at every row in one kernel pass over the natural-order trace the prover already holds
(csrc/check.cu, `Context.check_constraints`), and every failing constraint is reported with its first failing row and
the number of failing rows.  The cells named in the report are gathered from the resident columns; no column is copied
to the host.
"""
import warnings
from dataclasses import dataclass

from . import FP, FQ3
from . import expr as E
from .air import _leaves, domain_generator
from .prover import ProvingError

P = E.P
_RINV = pow(2**64, -1, P)
_NONE = 2**64 - 1


@dataclass(frozen=True)
class Violation:
    """constraint `constraint` is None (src/constraints.rs:168-249) at `count` rows of the trace domain, the lowest being
    `first_row`; `values`: (label, value) of x and of every Trace / Challenge / Hint leaf of the constraint at that row,
    as canonical integers (3-tuples for Fq3), sorted by label and deduplicated"""
    constraint: int
    first_row: int
    count: int
    values: tuple

    def message(self):
        """the reference's report (src/debug.rs), with the number of failing rows"""
        vals = "\n".join(f"{label} = {value}" for label, value in self.values)
        return (f"Constraint {self.constraint} does not evaluate to a low degree polynomial. Divide by zero occurs at row "
                f"{self.first_row} ({self.count} failing rows).\n\nExpression values:\n{vals}")


def _unused_warnings(air, num_challenges, num_hints):
    cfg = air.config
    cols, chals, hints = set(), set(), set()
    for c in air.constraints:
        cols |= {a[0] for a in _leaves(c, "trace")}
        chals |= {a[0] for a in _leaves(c, "chal")}
        hints |= {a[0] for a in _leaves(c, "hint")}
    for i in range(cfg.NUM_BASE_COLUMNS + cfg.NUM_EXTENSION_COLUMNS):
        if i not in cols:
            warnings.warn(f"no constraints for execution trace column {i}", stacklevel=3)
    for i in range(num_challenges):
        if i not in chals:
            warnings.warn(f"challenge at index {i} never used", stacklevel=3)
    for i in range(num_hints):
        if i not in hints:
            warnings.warn(f"hint at index {i} never used", stacklevel=3)


def validate_constraints(ctx, air, challenges, hints, base, ext):
    """Check every constraint of `air` at every row of the trace domain.  base: (NUM_BASE_COLUMNS, n) natural-order
    base columns, ext: None or (NUM_EXTENSION_COLUMNS, n * fq) extension columns, both device buffers (torch tensors);
    challenges / hints: canonical integers or 3-tuples.  Emits the reference's three warnings (unused column, challenge,
    hint) through `warnings.warn` and returns the list of `Violation`s, by constraint index (empty: the trace
    satisfies the AIR)."""
    cfg = air.config
    fq = FP if cfg.FQ_IS_FP else FQ3
    log_n, n = air.log_n, air.trace_len
    nbase, next_ = cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS
    _unused_warnings(air, len(challenges), len(hints))
    prog = air.check_program().bind(challenges=challenges, hints=hints)
    cols = [base[c] for c in range(nbase)] + ([ext[c] for c in range(next_)] if next_ else [])
    tables = E.periodic_tables(ctx, prog, log_n, 1, offset_canonical=1)
    try:
        first, count = ctx.check_constraints(prog, cols + [p for p, _ in tables], [False] * nbase + [True] * next_ +
                                             [q for _, q in tables], fq, log_n, len(air.constraints))
    finally:
        for p, _ in tables:
            ctx.free(p)
    failing = [k for k in range(len(air.constraints)) if int(first[k]) != _NONE]
    if not failing:
        return []

    # the cells the reports name: every row any failing constraint reads at its first failing row, gathered in one call
    # per matrix
    leaves = {k: sorted(_leaves(air.constraints[k], "trace")) for k in failing}
    rows = sorted({(int(first[k]) + off) % n for k in failing for _, off in leaves[k]})
    where = {r: j for j, r in enumerate(rows)}
    brows = ctx.gather_rows(base, FP, n, nbase, rows) if rows and nbase else None
    erows = ctx.gather_rows(ext, fq, n, next_, rows) if rows and next_ else None

    def canon(words):
        v = tuple(int(w) * _RINV % P for w in words)
        return v[0] if len(v) == 1 else v

    def field_value(v):
        v = E._q(v)
        return v if fq == FQ3 else v[0]

    g = domain_generator(log_n)
    out = []
    for k in failing:
        row = int(first[k])
        vals = {"x": pow(g, row, P)}
        for col, off in leaves[k]:
            j = where[(row + off) % n]
            cell = brows[j, col:col + 1] if col < nbase else erows[j, (col - nbase) * fq:(col - nbase + 1) * fq]
            vals[f"Trace(col={col:0>3}, offset={off:0>3})"] = canon(cell)
        for (i,) in _leaves(air.constraints[k], "chal"):
            vals[f"Challenge({i})"] = field_value(challenges[i])
        for (i,) in _leaves(air.constraints[k], "hint"):
            vals[f"Hint({i})"] = field_value(hints[i])
        out.append(Violation(k, row, int(count[k]), tuple(sorted(vals.items()))))
    return out


class ConstraintViolation(ProvingError):
    """the trace does not satisfy its AIR: `violations` lists every failing constraint; the message is the reference's
    report for the lowest failing constraint index"""

    def __init__(self, violations):
        self.violations = list(violations)
        super().__init__(self.violations[0].message())
