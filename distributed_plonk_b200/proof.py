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


@dataclass
class VerifyingKey:
    """what a verifier needs of a circuit: the gate-domain size n, the number of public inputs, the coset representatives
    k[5] (ints), the 13 selector and 5 sigma commitments (affine (x, y) or None)"""
    n: int
    num_inputs: int
    k: list
    selector_comms: list
    sigma_comms: list


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
