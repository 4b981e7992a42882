"""verifier.py — default_verify (src/verifier.rs:27-183): checks a Proof against a Stark's claim on the host.

Same order of coin reseeds and draws as the reference's verifier, and so as the prover (prover.py):

    security level                 Proof::security_level_bits (src/proof.rs:126-147)
    base / extension / composition commitments, challenges, hints, composition coefficients, z
    out-of-domain consistency      ood_constraint_evaluation (src/verifier.rs:207-229) against Horner over the
                                   composition trace's out-of-domain values
    DEEP coefficients, FRI alphas  Stark.gen_deep_coeffs; FriVerifier::new (src/fri.rs:293-352)
    proof of work, query positions
    trace rows                     MatrixMerkleTree::verify_rows (src/merkle.rs:209-281, 364-386) on three trees
    DEEP evaluations               deep_composition_evaluations (src/verifier.rs:231-297)
    FRI                            verify_generic and verify_remainder (src/fri.rs:354-512)

A proof has a few dozen queries at most, so the work is a few hundred SHA-256 compressions (hashlib), one evaluation of
the composition constraint at z and an ff-point interpolation per FRI layer and query, all in Python integers.

Every refusal is a VerificationError whose `kind` is the reference's variant (src/verifier.rs:187-202,
src/fri.rs:253-270), or one of EXTRA_KINDS for proofs the reference has no variant for.  Two groups of proofs get those:

  * proofs on which the reference panics or reads past a slice: a trace length that is not a power of two or that the
    AIR cannot take (its hints or constraints refuse it), too few out-of-domain values, query rows or FRI layers, a
    zero denominator;
  * malformed proofs the reference accepts, refused here on purpose: surplus execution-trace out-of-domain values (the
    reference zips them away), surplus FRI layers (it reads only as many as the options give) and an extension trace
    commitment for an AIR without extension columns, or none for one with them (it then reads the extension rows
    unchecked).  No honest prover emits these.
"""
from collections import deque
from dataclasses import dataclass

from . import expr as E
from .air import Air, GENERATOR, domain_generator
from .channel import hash_elements, merge
from .cosets import brev
from .deep import ood_points

P = E.P

# kinds with no variant in the reference (the module docstring lists the proofs that get them)
EXTRA_KINDS = ("InvalidTraceLength", "InvalidAir", "ExtensionTraceMismatch", "OodEvaluationCountMismatch",
               "TraceQueryCountMismatch", "FriLayerCountMismatch", "FriLayerQueryCountMismatch", "ZeroDenominator")


class VerificationError(Exception):
    """a proof the verifier refuses.  kind: the reference's VerificationError variant (or one of EXTRA_KINDS);
    layer: the FRI layer of LayerCommitmentInvalid / InvalidDegreeRespectingProjection / CodewordTruncation;
    degree: the expected degree of RemainderDegreeMismatch"""

    def __init__(self, kind, message, layer=None, degree=None):
        super().__init__(f"{kind}: {message}")
        self.kind, self.layer, self.degree = kind, layer, degree


@dataclass
class VerifierChannelArtifacts:
    """src/channel.rs: the verifier randomness of an accepted proof.  Elements as the prover draws them: canonical ints
    when Fq = Fp, 3-tuples otherwise"""
    air_challenges: list
    air_hints: list
    fri_alphas: list
    query_positions: list


def _scale(a, s):
    return tuple(c * s % P for c in a)


def _horner(coeffs, x):
    acc = (0, 0, 0)
    for c in reversed(coeffs):
        acc = E.q_add(E.q_mul(acc, x), c)
    return acc


def _inv(a):
    if not any(a):
        raise VerificationError("ZeroDenominator", "a DEEP denominator x - z g^k is zero")
    return E.q_inv(a)


def _merkle_verify(root, view, indices):
    """MerkleTreeImpl::verify (src/merkle.rs:209-281); False where the reference errs or panics"""
    height = view.height
    if height > 63:                            # 1 << height overflows the reference's usize
        return False
    n = 1 << height
    if any(i >= n for i in indices):
        return False
    indices = sorted(set(indices))
    siblings, nodes = deque(view.sibling_leaves), deque(view.nodes)
    leaf_q = deque(zip(indices, view.initial_leaves))
    node_q = deque()
    while leaf_q:
        index, leaf = leaf_q.popleft()
        node_index = (n + index) >> 1
        if leaf_q and leaf_q[0][0] == index ^ 1:
            node_q.append((node_index, merge(leaf, leaf_q.popleft()[1])))
            continue
        if not siblings:
            return False
        sib = siblings.popleft()
        node_q.append((node_index, merge(leaf, sib) if index % 2 == 0 else merge(sib, leaf)))
    if siblings:
        return False
    while node_q:
        index, h = node_q.popleft()
        if index < 2:                           # the root (index 0: a height-0 view, which the reference cannot take)
            return index == 1 and not node_q and h == root
        if node_q and node_q[0][0] == index ^ 1:
            node_q.append((index >> 1, merge(h, node_q.popleft()[1])))
            continue
        if not nodes:
            return False
        sib = nodes.popleft()
        node_q.append((index >> 1, merge(h, sib) if index % 2 == 0 else merge(sib, h)))
    return True


def _verify_rows(root, row_ids, rows, view):
    """MatrixMerkleTree::verify_rows (src/merkle.rs:364-386): the leaves are the hashes of the rows, sorted by id"""
    if view is None:
        return False
    instances = sorted(dict(zip(row_ids, rows)).items())
    if view.initial_leaves != [hash_elements(row) for _, row in instances]:
        return False
    return _merkle_verify(root, view, [i for i, _ in instances])


def _chunks(values, k):
    return [values[i:i + k] for i in range(0, len(values), k)]


def verify(stark, proof, required_security_bits):
    """default_verify: returns the VerifierChannelArtifacts of an accepted proof, raises VerificationError otherwise.
    stark: the claim (its AirConfig and get_public_inputs()); proof: a Proof (Proof.from_bytes reads the wire format)."""
    cfg = stark.AirConfig
    fq_is_fp = cfg.FQ_IS_FP
    lift = E._q
    if proof.security_level_bits(fq_is_fp) < required_security_bits:
        raise VerificationError("InvalidProofSecurity", "proof params do not satisfy security requirements")

    options, n = proof.options, proof.trace_len
    beta, ff = options.lde_blowup_factor, options.fri_folding_factor
    log_n, log_b = n.bit_length() - 1, beta.bit_length() - 1
    if n < 2 or n & (n - 1) or log_n + log_b > 32:
        raise VerificationError("InvalidTraceLength", f"trace length {n} is not a power of two whose LDE domain "
                                f"(blowup {beta}) has at most 2^32 points")
    try:
        air = Air(cfg, n, stark.get_public_inputs(), options)
    except (ValueError, AssertionError, ArithmeticError) as e:    # e.g. Air::new's assert ce blow-up <= LDE blow-up
        raise VerificationError("InvalidAir", f"the AIR cannot be built for trace length {n} and {options}") from e
    nbase, next_, ce_blowup = cfg.NUM_BASE_COLUMNS, cfg.NUM_EXTENSION_COLUMNS, air.ce_blowup_factor
    if (proof.extension_trace_commitment is None) != (next_ == 0):
        raise VerificationError("ExtensionTraceMismatch", f"the AIR has {next_} extension columns and the proof "
                                f"{'no' if proof.extension_trace_commitment is None else 'an'} extension trace commitment")
    public_coin = stark.gen_public_coin(air)

    public_coin.reseed_with_digest(proof.base_trace_commitment)
    air_challenges = [public_coin.draw() for _ in range(air.num_challenges())]
    try:
        air_hints = air.gen_hints(air_challenges)
    except (ValueError, AssertionError, ArithmeticError) as e:      # e.g. brainfuck: a trace shorter than its output
        raise VerificationError("InvalidAir", f"the AIR's hints cannot be built for trace length {n}: {e}") from e
    if proof.extension_trace_commitment is not None:
        public_coin.reseed_with_digest(proof.extension_trace_commitment)
    composition_coeffs = [public_coin.draw() for _ in range(air.num_composition_constraint_coeffs())]
    public_coin.reseed_with_digest(proof.composition_trace_commitment)

    z = public_coin.draw()
    trace_oods, comp_oods = proof.execution_trace_ood_evals, proof.composition_trace_ood_evals
    public_coin.reseed_with_field_elements(list(trace_oods) + list(comp_oods))
    trace_arguments = air.trace_arguments()
    if len(trace_oods) != len(trace_arguments) or len(comp_oods) != ce_blowup:
        raise VerificationError("OodEvaluationCountMismatch", f"{len(trace_oods)} execution trace and {len(comp_oods)} "
                                f"composition trace out-of-domain values, the AIR has {len(trace_arguments)} and {ce_blowup}")
    zq = lift(z)
    ood_map = dict(zip(trace_arguments, (lift(v) for v in trace_oods)))
    comp_oods = [lift(v) for v in comp_oods]
    try:
        calculated = E.evaluate_at(air.composition_constraint, zq, ood_map, air_challenges, air_hints, composition_coeffs,
                                   trace_len=n)
    except ZeroDivisionError as e:
        raise VerificationError("ZeroDenominator", "the composition constraint has a zero denominator at z") from e
    if calculated != _horner(comp_oods, zq):
        raise VerificationError("InconsistentOodConstraintEvaluations",
                                "constraint evaluations at the out-of-domain point are inconsistent")

    ex_alphas, co_alphas, (d_alpha, d_beta) = stark.gen_deep_coeffs(public_coin, air)

    # FriVerifier::new: max_poly_degree = trace_len - 1, so the FRI domain is the LDE domain
    layers = proof.fri_proof.layers
    N = n * beta
    fri_alphas, codeword_len = [], N
    for i, layer in enumerate(layers):
        public_coin.reseed_with_digest(layer.commitment)
        fri_alphas.append(public_coin.draw())
        if i != len(layers) - 1 and codeword_len % ff:
            raise VerificationError("CodewordTruncation", f"{codeword_len} can't be divided by {ff} (layer {i})", layer=i)
        codeword_len //= ff
    public_coin.reseed_with_field_elements(proof.fri_proof.remainder_coeffs)

    if options.grinding_factor:
        if not public_coin.verify_proof_of_work(options.grinding_factor, proof.pow_nonce):
            raise VerificationError("FriProofOfWork", "insufficient proof of work on fri commitments")
        public_coin.reseed_with_int(proof.pow_nonce)

    positions = public_coin.draw_queries(options.num_queries, N)

    q = proof.trace_queries
    base_rows = _chunks(q.base_trace_values, nbase)
    ext_rows = _chunks(q.extension_trace_values, next_) if next_ else []
    comp_rows = _chunks(q.composition_trace_values, ce_blowup)
    k = len(positions)
    if (len(q.base_trace_values) != k * nbase or len(q.extension_trace_values) != k * next_
            or len(q.composition_trace_values) != k * ce_blowup):
        raise VerificationError("TraceQueryCountMismatch", f"the trace queries do not hold one row per query position "
                                f"({k} positions)")
    if not _verify_rows(proof.base_trace_commitment, positions, base_rows, q.base_trace_proof):
        raise VerificationError("BaseTraceQueryDoesNotMatchCommitment", "query does not resolve to the base trace commitment")
    if next_ and not _verify_rows(proof.extension_trace_commitment, positions, ext_rows, q.extension_trace_proof):
        raise VerificationError("ExtensionTraceQueryDoesNotMatchCommitment",
                                "query does not resolve to the extension trace commitment")
    if not _verify_rows(proof.composition_trace_commitment, positions, comp_rows, q.composition_trace_proof):
        raise VerificationError("CompositionTraceQueryDoesNotMatchCommitment",
                                "query does not resolve to the composition trace commitment")

    # deep_composition_evaluations.  The terms of the trace arguments with the same offset share the denominator
    # x - z g^offset, so their numerators are summed first: one inversion per offset and query
    g_lde = domain_generator(log_n + log_b)
    z_points, z_n = ood_points(zq, log_n, [off for _, off in trace_arguments], ce_blowup)
    by_offset = {}
    for j, (col, off) in enumerate(trace_arguments):
        by_offset.setdefault(off, (z_points[off], []))[1].append((col, lift(ex_alphas[j]), ood_map[(col, off)]))
    co_alphas = [lift(a) for a in co_alphas]
    d_alpha, d_beta = lift(d_alpha), lift(d_beta)
    deep_evals = []
    for i, pos in enumerate(positions):
        x = GENERATOR * pow(g_lde, brev(pos, log_n + log_b), P) % P
        row = [(v, 0, 0) for v in base_rows[i]] + ([lift(v) for v in ext_rows[i]] if next_ else [])
        ev = (0, 0, 0)
        for z_shift, terms in by_offset.values():
            num = (0, 0, 0)
            for col, alpha, ood in terms:
                num = E.q_add(num, E.q_mul(alpha, E.q_add(row[col], E.q_neg(ood))))
            ev = E.q_add(ev, E.q_mul(num, _inv(E.q_add((x, 0, 0), E.q_neg(z_shift)))))
        num = (0, 0, 0)
        for alpha, value, ood in zip(co_alphas, comp_rows[i], comp_oods):
            num = E.q_add(num, E.q_mul(alpha, E.q_add(lift(value), E.q_neg(ood))))
        ev = E.q_add(ev, E.q_mul(num, _inv(E.q_add((x, 0, 0), E.q_neg(z_n)))))
        deep_evals.append(E.q_mul(ev, E.q_add(d_alpha, _scale(d_beta, x))))

    _verify_fri(proof.fri_proof, options, [lift(a) for a in fri_alphas], positions, deep_evals, N, g_lde)
    return VerifierChannelArtifacts(air_challenges, air_hints, fri_alphas, positions)


def _verify_fri(fri_proof, options, alphas, positions, evaluations, domain_size, domain_gen):
    """FriVerifier::verify / verify_generic / verify_remainder.  The folding domain has offset 1: layer points are
    powers of the domain generator"""
    if len(positions) != len(evaluations):
        raise VerificationError("NumPositionEvaluationMismatch",
                                "the number of query positions does not match the number of evaluations")
    ff, beta = options.fri_folding_factor, options.lde_blowup_factor
    layers = fri_proof.layers
    num_layers = options.fri_num_layers(domain_size)
    if num_layers != len(layers):
        raise VerificationError("FriLayerCountMismatch", f"{len(layers)} FRI layers, the options give {num_layers}")
    w_inv = pow(domain_generator(ff.bit_length() - 1), -1, P)
    w_inv_pow = [pow(w_inv, k, P) for k in range(ff)]
    log_ff = ff.bit_length() - 1
    nat_order = [brev(t, log_ff) for t in range(ff)]
    for i, (layer, alpha) in enumerate(zip(layers, alphas)):
        folded = sorted(set(p // ff for p in positions))
        if len(layer.flattenend_rows) != len(folded) * ff:
            raise VerificationError("FriLayerQueryCountMismatch", f"layer {i} holds {len(layer.flattenend_rows)} values "
                                    f"for {len(folded)} rows of {ff}", layer=i)
        rows = _chunks(layer.flattenend_rows, ff)
        if not _verify_rows(layer.commitment, folded, rows, layer.merkle_proof):
            raise VerificationError("LayerCommitmentInvalid", f"queries do not resolve to their commitment in layer {i}",
                                    layer=i)
        rows = [[E._q(v) for v in row] for row in rows]
        row_of = {p: row for p, row in zip(folded, rows)}
        if evaluations != [row_of[p // ff][p % ff] for p in positions]:
            raise VerificationError("InvalidDegreeRespectingProjection",
                                    f"degree respecting projection is invalid for layer {i}", layer=i)
        # each row: the bit-reversed evaluations over the coset offset * <w>, w of order ff; interpolate, evaluate at alpha.
        # The 1/ff of the inverse transform cancels against the reference's "* N"
        evaluations = []
        for p, row in zip(folded, rows):
            offset_inv = pow(pow(domain_gen, brev(p, domain_size.bit_length() - 1 - log_ff), P), -1, P)
            nat = [row[t] for t in nat_order]
            coeffs, s = [], 1
            for j in range(ff):
                acc = (0, 0, 0)
                for t in range(ff):
                    acc = E.q_add(acc, _scale(nat[t], w_inv_pow[j * t % ff]))
                coeffs.append(_scale(acc, s))
                s = s * offset_inv % P
            evaluations.append(_horner(coeffs, alpha))
        positions = folded
        domain_gen = pow(domain_gen, ff, P)
        domain_size //= ff

    # verify_remainder
    remainder = [E._q(c) for c in fri_proof.remainder_coeffs]
    degree = len(remainder) - 1
    while degree > 0 and not any(remainder[degree]):
        degree -= 1
    expected_degree = domain_size // beta - 1
    if degree > expected_degree:
        raise VerificationError("RemainderDegreeMismatch", f"remainder is not a degree {expected_degree} polynomial",
                                degree=expected_degree)
    for p, want in zip(positions, evaluations):
        if _horner(remainder, (pow(domain_gen, brev(p, domain_size.bit_length() - 1), P), 0, 0)) != want:
            raise VerificationError("RemainderCommitmentInvalid", "remainder is invalid")
