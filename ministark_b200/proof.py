"""proof.py — Proof, Queries, FriProof, LayerProof, MerkleView and their wire format.

Mirrors src/proof.rs:43-66, src/trace.rs:37-66, src/fri.rs:71-125, src/merkle.rs:71-80.  The byte layout is
ark-serialize's (compressed mode): struct fields in declaration order; integers little-endian (usize as u64);
Vec<T> = u64 length + items; Option<T> = one tag byte (0 / 1) + item; a digest = the 32-byte slice, i.e. u64
length 32 + bytes (SerdeOutput delegates to the byte slice, src/utils.rs:552-560); an Fp = 8-byte LE canonical
integer; an Fq3 = c0 ‖ c1 ‖ c2.  (ark-serialize itself is not under /root/reference: SURVEY.md §8c lists these
conventions as restated from upstream.)

Field elements inside a Proof are canonical integers (Fp) or 3-tuples (Fq3).

`Proof.from_bytes` reads the same layout back.  Anything that is not exactly one serialized Proof — truncated input,
trailing bytes, a digest length other than 32, an Option tag other than 0 or 1, a field element >= p, or options that
ProofOptions refuses — raises ProofFormatError, whose message names the field.
"""
from dataclasses import dataclass, field
from typing import List, Optional

from .air import ProofOptions
from .channel import P, serialize_element


class ProofFormatError(ValueError):
    """bytes that are not a serialized Proof"""


class _Reader:
    def __init__(self, data):
        self.b, self.i = bytes(data), 0

    def take(self, k, what):
        if k > len(self.b) - self.i:
            raise ProofFormatError(f"{what}: truncated (needs {k} bytes at offset {self.i}, {len(self.b) - self.i} left)")
        v = self.b[self.i:self.i + k]
        self.i += k
        return v

    def u64(self, what):
        return int.from_bytes(self.take(8, what), "little")

    def digest(self, what):
        k = self.u64(what)
        if k != 32:
            raise ProofFormatError(f"{what}: digest length {k}, not 32")
        return self.take(32, what)

    def element(self, what, lanes):
        """lanes 1: a canonical int; lanes 3: a 3-tuple"""
        v = [int.from_bytes(self.take(8, what), "little") for _ in range(lanes)]
        if any(c >= P for c in v):
            raise ProofFormatError(f"{what}: {max(v)} is not a canonical field element (>= p)")
        return v[0] if lanes == 1 else tuple(v)

    def vec(self, what, item, min_item_bytes):
        k = self.u64(what)
        if k * min_item_bytes > len(self.b) - self.i:          # refused before anything is allocated for the items
            raise ProofFormatError(f"{what}: truncated (length {k}, {len(self.b) - self.i} bytes left)")
        return [item(f"{what}[{j}]") for j in range(k)]

    def option(self, what, item):
        tag = self.take(1, what)[0]
        if tag not in (0, 1):
            raise ProofFormatError(f"{what}: Option tag {tag}, not 0 or 1")
        return item(what) if tag else None

    def view(self, what):
        d = lambda w: self.digest(w)
        return MerkleView(self.vec(f"{what}.nodes", d, 40), self.vec(f"{what}.initial_leaves", d, 40),
                          self.vec(f"{what}.sibling_leaves", d, 40), int.from_bytes(self.take(4, f"{what}.height"), "little"))


def _options(raw):
    """ProofOptions from its five bytes, refusing what its constructor asserts against (src/lib.rs:109-114)"""
    nq, blowup, grinding, ff, max_rem = raw
    if not 1 <= nq <= 128:
        raise ProofFormatError(f"options.num_queries: {nq} is not in 1..=128")
    if not 1 <= blowup <= 128 or blowup & (blowup - 1):
        raise ProofFormatError(f"options.lde_blowup_factor: {blowup} is not a power of two in 1..=128")
    if grinding > 50:
        raise ProofFormatError(f"options.grinding_factor: {grinding} is more than 50")
    if ff not in (2, 4, 8, 16):
        raise ProofFormatError(f"options.fri_folding_factor: {ff} is not 2, 4, 8 or 16")
    return ProofOptions(nq, blowup, grinding, ff, max_rem)


def _u64(v):
    return int(v).to_bytes(8, "little")


def _vec(items, enc):
    return _u64(len(items)) + b"".join(enc(x) for x in items)


def _digest(d):
    return _u64(32) + bytes(d)


@dataclass
class MerkleView:
    nodes: List[bytes]
    initial_leaves: List[bytes]
    sibling_leaves: List[bytes]
    height: int

    def to_bytes(self):
        return (_vec(self.nodes, _digest) + _vec(self.initial_leaves, _digest) + _vec(self.sibling_leaves, _digest)
                + int(self.height).to_bytes(4, "little"))


@dataclass
class LayerProof:
    flattenend_rows: list            # (sic) src/fri.rs:101
    merkle_proof: MerkleView
    commitment: bytes

    def to_bytes(self):
        return _vec(self.flattenend_rows, serialize_element) + self.merkle_proof.to_bytes() + _digest(self.commitment)


@dataclass
class FriProof:
    layers: List[LayerProof]
    remainder_coeffs: list

    def to_bytes(self):
        return _vec(self.layers, LayerProof.to_bytes) + _vec(self.remainder_coeffs, serialize_element)


@dataclass
class Queries:
    base_trace_values: list
    extension_trace_values: list
    composition_trace_values: list
    base_trace_proof: MerkleView
    extension_trace_proof: Optional[MerkleView]
    composition_trace_proof: MerkleView

    def to_bytes(self):
        ext = b"\x00" if self.extension_trace_proof is None else b"\x01" + self.extension_trace_proof.to_bytes()
        return (_vec(self.base_trace_values, serialize_element) + _vec(self.extension_trace_values, serialize_element)
                + _vec(self.composition_trace_values, serialize_element) + self.base_trace_proof.to_bytes() + ext
                + self.composition_trace_proof.to_bytes())


@dataclass
class Proof:
    options: ProofOptions
    trace_len: int
    base_trace_commitment: bytes
    extension_trace_commitment: Optional[bytes]
    composition_trace_commitment: bytes
    fri_proof: FriProof
    pow_nonce: int
    trace_queries: Queries
    execution_trace_ood_evals: list
    composition_trace_ood_evals: list
    timings: dict = field(default_factory=dict, compare=False)      # per-phase wall clock, like the reference's println!s

    def to_bytes(self):
        ext = (b"\x00" if self.extension_trace_commitment is None
               else b"\x01" + _digest(self.extension_trace_commitment))
        return (self.options.to_bytes() + _u64(self.trace_len) + _digest(self.base_trace_commitment) + ext
                + _digest(self.composition_trace_commitment) + self.fri_proof.to_bytes() + _u64(self.pow_nonce)
                + self.trace_queries.to_bytes() + _vec(self.execution_trace_ood_evals, serialize_element)
                + _vec(self.composition_trace_ood_evals, serialize_element))

    @classmethod
    def from_bytes(cls, data, fq_is_fp):
        """the inverse of to_bytes (CanonicalDeserialize, src/proof.rs:80-122).  fq_is_fp: the AIR's Fq is Fp (Fq values
        are canonical ints) rather than Fq3 (3-tuples); base trace values are always ints.  Raises ProofFormatError."""
        r = _Reader(data)
        fq_lanes = 1 if fq_is_fp else 3
        fq = lambda w: r.element(w, fq_lanes)
        fp = lambda w: r.element(w, 1)
        options = _options(r.take(5, "options"))
        trace_len = r.u64("trace_len")
        base_root = r.digest("base_trace_commitment")
        ext_root = r.option("extension_trace_commitment", r.digest)
        comp_root = r.digest("composition_trace_commitment")
        layer = lambda w: LayerProof(r.vec(f"{w}.flattenend_rows", fq, 8 * fq_lanes), r.view(f"{w}.merkle_proof"),
                                     r.digest(f"{w}.commitment"))
        fri = FriProof(r.vec("fri_proof.layers", layer, 8 + 3 * 8 + 4 + 40),
                       r.vec("fri_proof.remainder_coeffs", fq, 8 * fq_lanes))
        pow_nonce = r.u64("pow_nonce")
        queries = Queries(r.vec("trace_queries.base_trace_values", fp, 8),
                          r.vec("trace_queries.extension_trace_values", fq, 8 * fq_lanes),
                          r.vec("trace_queries.composition_trace_values", fq, 8 * fq_lanes),
                          r.view("trace_queries.base_trace_proof"),
                          r.option("trace_queries.extension_trace_proof", r.view),
                          r.view("trace_queries.composition_trace_proof"))
        trace_oods = r.vec("execution_trace_ood_evals", fq, 8 * fq_lanes)
        comp_oods = r.vec("composition_trace_ood_evals", fq, 8 * fq_lanes)
        if r.i != len(r.b):
            raise ProofFormatError(f"composition_trace_ood_evals: {len(r.b) - r.i} trailing bytes after the proof")
        return cls(options, trace_len, base_root, ext_root, comp_root, fri, pow_nonce, queries, trace_oods, comp_oods)

    def security_level_bits(self, fq_is_fp=None):
        """Proof::security_level_bits (src/proof.rs:126-147): the least of the field security (bits of Fq less
        log2 of the LDE domain size), the FRI query security (log2(blowup) per query plus the grinding bits) and the 128
        bits of SHA-256's collision resistance (Merkle trees and public coin).  fq_is_fp=None: Fq is read off the
        proof's elements (Fq3 values are 3-tuples)."""
        if fq_is_fp is None:
            fq_vals = self.composition_trace_ood_evals + self.execution_trace_ood_evals + self.fri_proof.remainder_coeffs
            if not fq_vals:
                raise ValueError("the proof holds no Fq value to tell Fp from Fq3: pass fq_is_fp")
            fq_is_fp = not isinstance(fq_vals[0], (tuple, list))
        o = self.options
        lde_domain_size = self.trace_len * o.lde_blowup_factor
        field_security = (64 if fq_is_fp else 192) - (lde_domain_size.bit_length() - 1)
        fri_query_security = (o.lde_blowup_factor.bit_length() - 1) * o.num_queries + o.grinding_factor
        return min(field_security, fri_query_security, 128)
