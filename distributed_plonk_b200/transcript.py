"""The Fiat-Shamir transcript of the resident prover: Keccak-f[1600], the subset of Strobe-128 that merlin 3.0.0 uses,
merlin's Transcript, and PlonkTranscript, which feeds merlin byte for byte what the reference prover's
FakeStandardTranscript feeds it (dispatcher2.rs:44-154) - so the challenges beta, gamma, alpha, zeta, v are the ones a
jf-plonk verifier re-derives from (verifying key, public inputs, proof).

Host work on a few kilobytes per proof, hashed sequentially: pure Python, 64-bit lanes as Python ints.  The merlin and
Strobe details are restated from memory of merlin 3.0.0 / keccak 0.1.2 (the versions the reference's Cargo.lock pins);
rust/dump_fixtures.rs writes the records that pin them to the crate (DESIGN.md 3.6, 5).
"""
from __future__ import annotations

import struct

R_MOD = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001   # BLS12-381 scalar field
FR_SIZE_IN_BITS = 255

# ------------------------------------------------------------------ Keccak-f[1600] on 25 lanes, lane (x, y) at x + 5y
_RC = (0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B, 0x0000000080000001,
       0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088, 0x0000000080008009, 0x000000008000000A,
       0x000000008000808B, 0x800000000000008B, 0x8000000000008089, 0x8000000000008003, 0x8000000000008002, 0x8000000000000080,
       0x000000000000800A, 0x800000008000000A, 0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008)
_ROT = (0, 1, 62, 28, 27,  36, 44, 6, 55, 20,  3, 10, 43, 25, 39,  41, 45, 15, 21, 8,  18, 2, 61, 56, 14)   # rho offset of lane x + 5y
# rho and pi together: lane x + 5y, rotated by _ROT, moves to lane y + 5 ((2x + 3y) mod 5)
_RHO_PI = tuple((i, (i // 5) + 5 * ((2 * (i % 5) + 3 * (i // 5)) % 5), _ROT[i]) for i in range(25))
_M64 = (1 << 64) - 1


def f1600(a: list) -> None:
    """the Keccak-f[1600] permutation, 24 rounds, in place on a list of 25 lanes"""
    b = [0] * 25
    for rc in _RC:
        c0 = a[0] ^ a[5] ^ a[10] ^ a[15] ^ a[20]
        c1 = a[1] ^ a[6] ^ a[11] ^ a[16] ^ a[21]
        c2 = a[2] ^ a[7] ^ a[12] ^ a[17] ^ a[22]
        c3 = a[3] ^ a[8] ^ a[13] ^ a[18] ^ a[23]
        c4 = a[4] ^ a[9] ^ a[14] ^ a[19] ^ a[24]
        d = (c4 ^ (((c1 << 1) | (c1 >> 63)) & _M64), c0 ^ (((c2 << 1) | (c2 >> 63)) & _M64), c1 ^ (((c3 << 1) | (c3 >> 63)) & _M64),
             c2 ^ (((c4 << 1) | (c4 >> 63)) & _M64), c3 ^ (((c0 << 1) | (c0 >> 63)) & _M64))
        for src, dst, r in _RHO_PI:
            v = a[src] ^ d[src % 5]
            b[dst] = ((v << r) | (v >> (64 - r))) & _M64
        for y in (0, 5, 10, 15, 20):
            b0, b1, b2, b3, b4 = b[y], b[y + 1], b[y + 2], b[y + 3], b[y + 4]
            a[y] = b0 ^ (~b1 & b2)
            a[y + 1] = b1 ^ (~b2 & b3)
            a[y + 2] = b2 ^ (~b3 & b4)
            a[y + 3] = b3 ^ (~b4 & b0)
            a[y + 4] = b4 ^ (~b0 & b1)
        a[0] ^= rc


def keccak_f(state: bytearray) -> None:
    """f1600 on a 200-byte state (lanes little-endian)"""
    lanes = list(struct.unpack("<25Q", state))
    f1600(lanes)
    state[:] = struct.pack("<25Q", *lanes)


# ------------------------------------------------------------------ Strobe-128, the operations merlin uses
STROBE_R = 166
FLAG_I, FLAG_A, FLAG_C, FLAG_T, FLAG_M, FLAG_K = 1, 2, 4, 8, 16, 32


class Strobe128:
    def __init__(self, protocol_label: bytes | None):
        """protocol_label None: an empty object for clone()"""
        if protocol_label is None:
            return
        st = bytearray(200)
        st[0:6] = bytes([1, STROBE_R + 2, 1, 0, 1, 96])
        st[6:18] = b"STROBEv1.0.2"
        keccak_f(st)
        self.st, self.pos, self.pos_begin, self.cur_flags = st, 0, 0, 0
        self.meta_ad(protocol_label, False)

    def clone(self) -> "Strobe128":
        s = Strobe128(None)
        s.st, s.pos, s.pos_begin, s.cur_flags = bytearray(self.st), self.pos, self.pos_begin, self.cur_flags
        return s

    def _run_f(self):
        st = self.st
        st[self.pos] ^= self.pos_begin
        st[self.pos + 1] ^= 0x04
        st[STROBE_R + 1] ^= 0x80
        keccak_f(st)
        self.pos = self.pos_begin = 0

    def _absorb(self, data):
        i, n, st = 0, len(data), self.st
        while i < n:                                          # whole runs up to the rate at a time
            k = min(n - i, STROBE_R - self.pos)
            p = self.pos
            st[p:p + k] = (int.from_bytes(st[p:p + k], "little") ^ int.from_bytes(data[i:i + k], "little")).to_bytes(k, "little")
            self.pos += k
            i += k
            if self.pos == STROBE_R:
                self._run_f()

    def _squeeze(self, k: int) -> bytes:
        out = bytearray()
        while len(out) < k:
            m = min(k - len(out), STROBE_R - self.pos)
            p = self.pos
            out += self.st[p:p + m]
            self.st[p:p + m] = bytes(m)
            self.pos += m
            if self.pos == STROBE_R:
                self._run_f()
        return bytes(out)

    def _begin_op(self, flags: int, more: bool):
        if more:
            assert self.cur_flags == flags, "an operation continued with other flags"
            return
        assert not flags & FLAG_T, "the T flag is not supported"
        old_begin = self.pos_begin
        self.pos_begin = self.pos + 1
        self.cur_flags = flags
        self._absorb(bytes([old_begin, flags]))
        if flags & (FLAG_C | FLAG_K) and self.pos != 0:
            self._run_f()

    def meta_ad(self, data: bytes, more: bool):
        self._begin_op(FLAG_M | FLAG_A, more)
        self._absorb(data)

    def ad(self, data: bytes, more: bool):
        self._begin_op(FLAG_A, more)
        self._absorb(data)

    def prf(self, k: int, more: bool) -> bytes:
        self._begin_op(FLAG_I | FLAG_A | FLAG_C, more)
        return self._squeeze(k)


# ------------------------------------------------------------------ merlin
class Transcript:
    """merlin::Transcript: Transcript(label), append_message, challenge_bytes, clone"""

    def __init__(self, label: bytes | None):
        if label is None:
            return
        self.strobe = Strobe128(b"Merlin v1.0")
        self.append_message(b"dom-sep", label)

    def clone(self) -> "Transcript":
        t = Transcript(None)
        t.strobe = self.strobe.clone()
        return t

    def append_message(self, label: bytes, message: bytes):
        self.strobe.meta_ad(label, False)
        self.strobe.meta_ad(struct.pack("<I", len(message)), True)
        self.strobe.ad(message, False)

    def challenge_bytes(self, label: bytes, k: int) -> bytes:
        self.strobe.meta_ad(label, False)
        self.strobe.meta_ad(struct.pack("<I", k), True)
        return self.strobe.prf(k, False)


# ------------------------------------------------------------------ the PLONK transcript
FQ_BYTES = 48


def fr_bytes(v: int) -> bytes:
    """ark-ff 0.3 `to_bytes!` of an Fr: 32 canonical little-endian bytes"""
    return int(v).to_bytes(32, "little")


def g1_bytes(pt) -> bytes:
    """ark-ec 0.3 GroupAffine ToBytes of a commitment: x, y (48 canonical LE bytes each), the infinity flag (1 byte).
    pt = (x, y) Python ints, or None for the identity, which is (0, 1, true)"""
    if pt is None:
        return bytes(FQ_BYTES) + (1).to_bytes(FQ_BYTES, "little") + b"\x01"
    return int(pt[0]).to_bytes(FQ_BYTES, "little") + int(pt[1]).to_bytes(FQ_BYTES, "little") + b"\x00"


class PlonkTranscript:
    """FakeStandardTranscript (dispatcher2.rs:44-154) over merlin.  Field elements are canonical Python ints, points are
    affine (x, y) ints or None.  `transcript` may be any object with merlin's append_message / challenge_bytes"""

    def __init__(self, transcript=None):
        self.t = Transcript(b"PlonkProof") if transcript is None else transcript

    def clone(self) -> "PlonkTranscript":
        return PlonkTranscript(self.t.clone())

    def append_vk(self, vk):
        """the verifying-key half of append_vk_and_pub_input: the same for every proof of a circuit"""
        m = self.t.append_message
        m(b"field size in bits", struct.pack("<Q", FR_SIZE_IN_BITS))
        m(b"domain size", struct.pack("<Q", vk.n))
        m(b"input size", struct.pack("<Q", vk.num_inputs))
        for k in vk.k:
            m(b"wire subsets separators", fr_bytes(k))
        for c in vk.selector_comms:
            m(b"selector commitments", g1_bytes(c))
        for c in vk.sigma_comms:
            m(b"sigma commitments", g1_bytes(c))

    def append_pub_input(self, pub_input):
        for v in pub_input:
            self.t.append_message(b"public input", fr_bytes(v))

    def append_vk_and_pub_input(self, vk, pub_input):
        self.append_vk(vk)
        self.append_pub_input(pub_input)

    def append_commitments(self, label: bytes, comms):
        for c in comms:
            self.t.append_message(label, g1_bytes(c))

    def append_commitment(self, label: bytes, comm):
        self.t.append_message(label, g1_bytes(comm))

    def append_proof_evaluations(self, wires_evals, wire_sigma_evals, perm_next_eval):
        for v in wires_evals:
            self.t.append_message(b"wire_evals", fr_bytes(v))
        for v in wire_sigma_evals:
            self.t.append_message(b"wire_sigma_evals", fr_bytes(v))
        self.t.append_message(b"perm_next_eval", fr_bytes(perm_next_eval))

    def get_and_append_challenge(self, label: bytes) -> int:
        """64 squeezed bytes read little-endian mod r (ark-ff 0.3 from_le_bytes_mod_order), appended under the same label"""
        c = int.from_bytes(self.t.challenge_bytes(label, 64), "little") % R_MOD
        self.t.append_message(label, fr_bytes(c))
        return c
