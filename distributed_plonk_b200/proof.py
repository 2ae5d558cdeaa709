"""The verifying key and the proof of the resident prover as a PLONK verifier sees them (jf-plonk's VerifyingKey and Proof,
dispatcher2.rs:699-710), and the conversions from the library's raw forms: 144-byte normalised Jacobian points
(Montgomery Fq) to affine canonical (x, y), raw Montgomery Fr to canonical Python ints."""
from __future__ import annotations

import struct
from dataclasses import dataclass

import numpy as np

from .transcript import R_MOD

FQ_MOD = 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB
_FQ_R = (1 << 384) % FQ_MOD
_FQ_RINV = pow(_FQ_R, -1, FQ_MOD)
_FR_R = (1 << 256) % R_MOD
_FR_RINV = pow(_FR_R, -1, R_MOD)


def fr_to_int(a) -> int:
    """raw Montgomery Fr (np.uint64[4]) -> canonical int"""
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return int.from_bytes(a.tobytes(), "little") * _FR_RINV % R_MOD


def fr_from_int(v: int) -> np.ndarray:
    """canonical int -> raw Montgomery Fr (np.uint64[4])"""
    return np.frombuffer((v % R_MOD * _FR_R % R_MOD).to_bytes(32, "little"), dtype=np.uint64).copy()


def point_from_jacobian(raw) -> tuple | None:
    """144-byte Jacobian (X, Y, Z in Montgomery Fq) -> affine canonical (x, y), or None for the identity (Z = 0)"""
    b = np.ascontiguousarray(raw, dtype=np.uint8).tobytes()
    X, Y, Z = (int.from_bytes(b[i:i + 48], "little") * _FQ_RINV % FQ_MOD for i in (0, 48, 96))
    if Z == 0:
        return None
    zi = pow(Z, -1, FQ_MOD)
    zi2 = zi * zi % FQ_MOD
    return X * zi2 % FQ_MOD, Y * zi2 * zi % FQ_MOD


def _fq_raw(v: int) -> bytes:
    return (int(v) % FQ_MOD * _FQ_R % FQ_MOD).to_bytes(48, "little")


def _fq_from_raw(b: bytes) -> int:
    return int.from_bytes(b, "little") * _FQ_RINV % FQ_MOD


def point_to_raw(pt) -> bytes:
    """affine canonical (x, y) or None -> raw ark GroupAffine<G1> (104 B: x, y Montgomery, infinity flag, padding);
    the identity is (0, 1, true)"""
    if pt is None:
        return _fq_raw(0) + _fq_raw(1) + b"\x01" + bytes(7)
    return _fq_raw(pt[0]) + _fq_raw(pt[1]) + bytes(8)


def point_from_raw(raw) -> tuple | None:
    """the inverse of point_to_raw"""
    b = np.ascontiguousarray(raw, dtype=np.uint8).tobytes()
    return None if b[96] else (_fq_from_raw(b[0:48]), _fq_from_raw(b[48:96]))


def g2_to_raw(q) -> bytes:
    """G2 point ((x.c0, x.c1), (y.c0, y.c1)) canonical ints, or None -> raw ark GroupAffine<G2> (200 B: x.c0, x.c1, y.c0,
    y.c1 Montgomery, infinity flag, padding); the identity is (0, 1, true)"""
    if q is None:
        return _fq_raw(0) * 2 + _fq_raw(1) + _fq_raw(0) + b"\x01" + bytes(7)
    (x0, x1), (y0, y1) = q
    return b"".join(_fq_raw(v) for v in (x0, x1, y0, y1)) + bytes(8)


def g2_from_raw(raw) -> tuple | None:
    """the inverse of g2_to_raw"""
    b = np.ascontiguousarray(raw, dtype=np.uint8).tobytes()
    if b[192]:
        return None
    v = [_fq_from_raw(b[48 * i:48 * (i + 1)]) for i in range(4)]
    return (v[0], v[1]), (v[2], v[3])


def g1_compress(pt) -> bytes:
    """ark-serialize 0.3 compressed point (48 B): x little-endian, bit 7 of the last byte set when y > -y, bit 6 for
    the identity - the format dp_init_compressed reads"""
    if pt is None:
        return bytes(47) + bytes([1 << 6])
    x, y = pt
    b = bytearray(int(x).to_bytes(48, "little"))
    if y > FQ_MOD - y:
        b[47] |= 1 << 7
    return bytes(b)


def g2_compress(q) -> bytes:
    """ark-serialize 0.3 compressed G2 point (96 B): x.c0 then x.c1, 48 little-endian bytes each; bit 7 of the last byte
    set when y > -y (Fq2 ordered by c1 first, then c0), bit 6 for the identity - the format dp_g2_decompress reads"""
    if q is None:
        return bytes(95) + bytes([1 << 6])
    (x0, x1), (y0, y1) = q
    b = bytearray(int(x0).to_bytes(48, "little") + int(x1).to_bytes(48, "little"))
    if (y1, y0) > ((-y1) % FQ_MOD, (-y0) % FQ_MOD):
        b[95] |= 1 << 7
    return bytes(b)


_DECOMPRESS_WHY = {1: "a coordinate is not below p", 2: "both flag bits set", 3: "not a point of the curve", 4: "not in the r-torsion subgroup"}
N_K, N_SELECTORS, N_SIGMAS = 5, 13, 5


def decompress_points(ctx, encodings, what: str) -> list:
    """compressed G1 points (48 B each) -> affine (x, y) or None, decoded and checked to lie in the r-torsion subgroup on the
    GPU (dp_g1_decompress); ValueError naming the first rejected point"""
    from ._binding import DP_E_ARG, DpError
    try:
        raw = ctx.g1_decompress(np.frombuffer(b"".join(encodings), dtype=np.uint8).reshape(len(encodings), 48), check_subgroup=True)
    except DpError as e:
        if e.code != DP_E_ARG:
            raise
        raise ValueError(f"point {e.index} of {what}: {_DECOMPRESS_WHY.get(e.why, e.msg)}") from e
    return [point_from_raw(r) for r in raw]


class _Reader:
    """the bytes of an ark-serialize record, taken front to back; ValueError when they run out or are left over"""

    def __init__(self, b, what: str):
        self.b, self.off, self.what = bytes(b), 0, what

    def take(self, k: int) -> bytes:
        if self.off + k > len(self.b):
            raise ValueError(f"truncated {self.what}: {len(self.b)} bytes")
        self.off += k
        return self.b[self.off - k:self.off]

    def u64(self) -> int:
        return struct.unpack("<Q", self.take(8))[0]

    def vec(self, expected: int, size: int, name: str) -> list:
        n = self.u64()
        if n != expected:
            raise ValueError(f"{self.what}: {name} has {n} entries, expected {expected}")
        return [self.take(size) for _ in range(n)]

    def end(self):
        if self.off != len(self.b):
            raise ValueError(f"{len(self.b) - self.off} trailing bytes after the {self.what}")


@dataclass
class VerifyingKey:
    """what a verifier needs of a circuit: the gate-domain size n, the number of public inputs, the coset representatives
    k[5] (ints), the 13 selector and 5 sigma commitments (affine (x, y) or None)"""
    n: int
    num_inputs: int
    k: list
    selector_comms: list
    sigma_comms: list

    def to_bytes(self) -> bytes:
        """The fields in the order above under ark-serialize 0.3 conventions: n and num_inputs as u64 LE, each vector a
        u64 LE length then its items, k as 32 canonical bytes each, points compressed (48 B).  1064 bytes.  This is this
        library's own record: jf-plonk's VerifyingKey lists different fields from version to version."""
        vec = lambda items, enc: struct.pack("<Q", len(items)) + b"".join(enc(x) for x in items)
        return (struct.pack("<QQ", self.n, self.num_inputs) + vec(self.k, lambda v: int(v).to_bytes(32, "little"))
                + vec(self.selector_comms, g1_compress) + vec(self.sigma_comms, g1_compress))

    @classmethod
    def from_bytes(cls, ctx, b) -> "VerifyingKey":
        """The inverse of to_bytes.  The 18 points are decompressed and checked to lie in the r-torsion subgroup on the GPU
        (dp_g1_decompress; ctx needs no init).  ValueError on a truncated input, trailing bytes, vector lengths other than
        5 / 13 / 5, a k >= r, n not a power of two (or above 2^32, the field's largest domain), num_inputs > n, or a rejected point."""
        r = _Reader(b, "verifying key")
        n, num_inputs = r.u64(), r.u64()
        k = [int.from_bytes(v, "little") for v in r.vec(N_K, 32, "k")]
        comp = r.vec(N_SELECTORS, 48, "selector_comms") + r.vec(N_SIGMAS, 48, "sigma_comms")
        r.end()
        if n == 0 or n & (n - 1) or n > 1 << 32:
            raise ValueError(f"verifying key: n = {n} is not a power of two up to 2^32")
        if num_inputs > n:
            raise ValueError(f"verifying key: {num_inputs} public inputs exceed n = {n}")
        for i, v in enumerate(k):
            if v >= R_MOD:
                raise ValueError(f"verifying key: k[{i}] is not below r")
        p = decompress_points(ctx, comp, "the verifying key")
        return cls(n, num_inputs, k, p[:N_SELECTORS], p[N_SELECTORS:])


@dataclass
class Proof:
    """jf-plonk's Proof: points affine (x, y) or None, evaluations canonical ints"""
    wires_poly_comms: list
    prod_perm_poly_comm: tuple | None
    split_quot_poly_comms: list
    opening_proof: tuple | None
    shifted_opening_proof: tuple | None
    wires_evals: list
    wire_sigma_evals: list
    perm_next_eval: int

    @classmethod
    def from_raw(cls, commitments, evals) -> "Proof":
        """from what ResidentProver.prove returns: 13 commitments (144 B: 5 wires, z, 5 quotient chunks, the two opening
        proofs) and 10 evaluations (raw Fr: 5 wires, 4 sigmas, z at zeta * omega)"""
        p = [point_from_jacobian(c) for c in commitments]
        e = [fr_to_int(v) for v in evals]
        assert len(p) == 13 and len(e) == 10
        return cls(p[0:5], p[5], p[6:11], p[11], p[12], e[0:5], e[5:9], e[9])

    def commitments(self) -> list:
        """the 13 points in the order of from_raw"""
        return list(self.wires_poly_comms) + [self.prod_perm_poly_comm] + list(self.split_quot_poly_comms) + [self.opening_proof, self.shifted_opening_proof]

    def evaluations(self) -> list:
        return list(self.wires_evals) + list(self.wire_sigma_evals) + [self.perm_next_eval]

    def to_bytes(self) -> bytes:
        """ark-serialize 0.3 CanonicalSerialize of jf-plonk's Proof: each Vec a u64 LE length, then its items; points
        compressed (48 B), field elements 32 canonical bytes.  976 bytes"""
        vec = lambda items, enc: struct.pack("<Q", len(items)) + b"".join(enc(x) for x in items)
        fr = lambda v: int(v).to_bytes(32, "little")
        return (vec(self.wires_poly_comms, g1_compress) + g1_compress(self.prod_perm_poly_comm) + vec(self.split_quot_poly_comms, g1_compress)
                + g1_compress(self.opening_proof) + g1_compress(self.shifted_opening_proof)
                + vec(self.wires_evals, fr) + vec(self.wire_sigma_evals, fr) + fr(self.perm_next_eval))


@dataclass
class ProofEvaluations:
    """one instance's evaluations in a BatchProof: 5 wires and 4 sigmas at zeta, z at zeta * omega (canonical ints)"""
    wires_evals: list
    wire_sigma_evals: list
    perm_next_eval: int

    def evaluations(self) -> list:
        return list(self.wires_evals) + list(self.wire_sigma_evals) + [self.perm_next_eval]


@dataclass
class BatchProof:
    """k instances of one circuit proved together (ResidentProver.prove_batch, DESIGN.md 3.11): per instance its 5 wire
    commitments, its permutation-product commitment and its evaluations; shared, the 5 quotient-chunk commitments of the
    folded quotient and the two opening proofs.  Points affine (x, y) or None, evaluations canonical ints."""
    wires_poly_comms_vec: list
    prod_perm_poly_comms_vec: list
    poly_evals_vec: list
    split_quot_poly_comms: list
    opening_proof: tuple | None
    shifted_opening_proof: tuple | None

    def __len__(self) -> int:
        return len(self.wires_poly_comms_vec)

    @classmethod
    def from_raw(cls, k: int, commitments, evals) -> "BatchProof":
        """from what the batch rounds return: 6k + 7 commitments (144 B: 5k wires, k z, 5 quotient chunks, the two opening
        proofs) and 10k evaluations (raw Fr: per instance 5 wires, 4 sigmas, z at zeta * omega)"""
        p = [point_from_jacobian(c) for c in commitments]
        e = [fr_to_int(v) for v in evals]
        assert len(p) == 6 * k + 7 and len(e) == 10 * k
        q = 6 * k
        return cls([p[5 * i:5 * i + 5] for i in range(k)], p[5 * k:6 * k],
                   [ProofEvaluations(e[10 * i:10 * i + 5], e[10 * i + 5:10 * i + 9], e[10 * i + 9]) for i in range(k)],
                   p[q:q + 5], p[q + 5], p[q + 6])

    def instance(self, i: int) -> Proof:
        """instance i's share as a Proof, with the shared quotient and openings (a batch of one is exactly that Proof)"""
        e = self.poly_evals_vec[i]
        return Proof(list(self.wires_poly_comms_vec[i]), self.prod_perm_poly_comms_vec[i], list(self.split_quot_poly_comms),
                     self.opening_proof, self.shifted_opening_proof, list(e.wires_evals), list(e.wire_sigma_evals), e.perm_next_eval)

    def to_bytes(self) -> bytes:
        """ark-serialize 0.3 conventions, as Proof.to_bytes: wires_poly_comms_vec (Vec of Vecs of 5 points),
        prod_perm_poly_comms_vec, poly_evals_vec (Vec of records: Vec of 5 wire evals, Vec of 4 sigma evals, perm_next_eval),
        split_quot_poly_comms, opening_proof, shifted_opening_proof.  368 + 632 k bytes.  This library's own record: byte
        parity with jf-plonk's BatchProof is not claimed."""
        vec = lambda items, enc: struct.pack("<Q", len(items)) + b"".join(enc(x) for x in items)
        fr = lambda v: int(v).to_bytes(32, "little")
        ev = lambda e: vec(e.wires_evals, fr) + vec(e.wire_sigma_evals, fr) + fr(e.perm_next_eval)
        return (vec(self.wires_poly_comms_vec, lambda ws: vec(ws, g1_compress)) + vec(self.prod_perm_poly_comms_vec, g1_compress)
                + vec(self.poly_evals_vec, ev) + vec(self.split_quot_poly_comms, g1_compress)
                + g1_compress(self.opening_proof) + g1_compress(self.shifted_opening_proof))
