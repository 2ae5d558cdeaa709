"""A restatement of the PLONK verifier for the tests: its own Keccak-f[1600] / Strobe-128 / merlin transcription (byte
arrays, written apart from the package's lane-based one in distributed_plonk_b200/transcript.py), the challenges jf-plonk's
verifier derives from (verifying key, public inputs, proof) - beta, gamma, alpha, zeta, v, then u after the two opening
proofs - and the batch check with the pairing replaced by the known trapdoor tau of a test SRS, as check_kzg_opening does.

TEST INFRASTRUCTURE ONLY: the product never imports it.  vk and proof are read by attribute (the package's VerifyingKey
and Proof, or what proof_from_bytes decodes); points are affine (x, y) ints or None, field elements canonical ints."""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

from oracle.py import bls12_381 as B

R = B.FR_MOD


# ------------------------------------------------------------------ Keccak-f[1600], textbook form on a 200-byte array
def _rc_bit(t: int) -> int:
    """the LFSR x^8 + x^6 + x^5 + x^4 + 1 of the Keccak reference"""
    if t % 255 == 0:
        return 1
    r = 1
    for _ in range(t % 255):
        r <<= 1
        if r & 0x100:
            r ^= 0x171
    return r & 1


ROUND_CONSTANTS = [sum(_rc_bit(j + 7 * i) << ((1 << j) - 1) for j in range(7)) for i in range(24)]
RHO = [[0] * 5 for _ in range(5)]
_x, _y = 1, 0
for _t in range(24):
    RHO[_x][_y] = (_t + 1) * (_t + 2) // 2 % 64
    _x, _y = _y, (2 * _x + 3 * _y) % 5


def _rot(v: int, r: int) -> int:
    return ((v << r) | (v >> (64 - r))) & 0xFFFFFFFFFFFFFFFF if r else v


def keccak_f(st: bytearray) -> None:
    A = [[int.from_bytes(st[8 * (x + 5 * y):8 * (x + 5 * y) + 8], "little") for y in range(5)] for x in range(5)]
    for rnd in range(24):
        C = [A[x][0] ^ A[x][1] ^ A[x][2] ^ A[x][3] ^ A[x][4] for x in range(5)]
        D = [C[(x - 1) % 5] ^ _rot(C[(x + 1) % 5], 1) for x in range(5)]
        A = [[A[x][y] ^ D[x] for y in range(5)] for x in range(5)]
        Bm = [[0] * 5 for _ in range(5)]
        for x in range(5):
            for y in range(5):
                Bm[y][(2 * x + 3 * y) % 5] = _rot(A[x][y], RHO[x][y])
        A = [[Bm[x][y] ^ ((~Bm[(x + 1) % 5][y]) & Bm[(x + 2) % 5][y]) for y in range(5)] for x in range(5)]
        A[0][0] ^= ROUND_CONSTANTS[rnd]
    for x in range(5):
        for y in range(5):
            st[8 * (x + 5 * y):8 * (x + 5 * y) + 8] = A[x][y].to_bytes(8, "little")


# ------------------------------------------------------------------ Strobe-128 / merlin, byte by byte as merlin's strobe.rs
STROBE_R = 166
I_, A_, C_, T_, M_, K_ = 1, 2, 4, 8, 16, 32


class Strobe:
    def __init__(self, label: bytes):
        self.st = bytearray(200)
        self.st[0:6] = bytes([1, STROBE_R + 2, 1, 0, 1, 96])
        self.st[6:18] = b"STROBEv1.0.2"
        keccak_f(self.st)
        self.pos = self.pos_begin = self.cur_flags = 0
        self.meta_ad(label, False)

    def copy(self):
        s = object.__new__(Strobe)
        s.st, s.pos, s.pos_begin, s.cur_flags = bytearray(self.st), self.pos, self.pos_begin, self.cur_flags
        return s

    def run_f(self):
        self.st[self.pos] ^= self.pos_begin
        self.st[self.pos + 1] ^= 0x04
        self.st[STROBE_R + 1] ^= 0x80
        keccak_f(self.st)
        self.pos = 0
        self.pos_begin = 0

    def absorb(self, data):
        for byte in data:
            self.st[self.pos] ^= byte
            self.pos += 1
            if self.pos == STROBE_R:
                self.run_f()

    def squeeze(self, k):
        out = bytearray(k)
        for i in range(k):
            out[i] = self.st[self.pos]
            self.st[self.pos] = 0
            self.pos += 1
            if self.pos == STROBE_R:
                self.run_f()
        return bytes(out)

    def begin_op(self, flags, more):
        if more:
            assert self.cur_flags == flags
            return
        old_begin = self.pos_begin
        self.pos_begin = self.pos + 1
        self.cur_flags = flags
        self.absorb([old_begin, flags])
        if (flags & (C_ | K_)) != 0 and self.pos != 0:
            self.run_f()

    def meta_ad(self, data, more):
        self.begin_op(M_ | A_, more)
        self.absorb(data)

    def ad(self, data, more):
        self.begin_op(A_, more)
        self.absorb(data)

    def prf(self, k, more):
        self.begin_op(I_ | A_ | C_, more)
        return self.squeeze(k)


class Merlin:
    def __init__(self, label: bytes):
        self.s = Strobe(b"Merlin v1.0")
        self.append_message(b"dom-sep", label)

    def clone(self):
        m = object.__new__(Merlin)
        m.s = self.s.copy()
        return m

    def append_message(self, label: bytes, message: bytes):
        self.s.meta_ad(label, False)
        self.s.meta_ad(len(message).to_bytes(4, "little"), True)
        self.s.ad(message, False)

    def challenge_bytes(self, label: bytes, k: int) -> bytes:
        self.s.meta_ad(label, False)
        self.s.meta_ad(k.to_bytes(4, "little"), True)
        return self.s.prf(k, False)


# ------------------------------------------------------------------ jf-plonk's verifier transcript
def _fr(v):
    return (int(v) % R).to_bytes(32, "little")


def _pt(p):
    if p is None:
        return (0).to_bytes(48, "little") + (1).to_bytes(48, "little") + b"\x01"
    return p[0].to_bytes(48, "little") + p[1].to_bytes(48, "little") + b"\x00"


def _challenge(t: Merlin, label: bytes) -> int:
    c = int.from_bytes(t.challenge_bytes(label, 64), "little") % R
    t.append_message(label, _fr(c))
    return c


def challenges(vk, pub_input, proof) -> dict:
    """beta, gamma, alpha, zeta, v, u as jf-plonk's verifier derives them"""
    t = Merlin(b"PlonkProof")
    t.append_message(b"field size in bits", (255).to_bytes(8, "little"))
    t.append_message(b"domain size", vk.n.to_bytes(8, "little"))
    t.append_message(b"input size", vk.num_inputs.to_bytes(8, "little"))
    for k in vk.k:
        t.append_message(b"wire subsets separators", _fr(k))
    for c in vk.selector_comms:
        t.append_message(b"selector commitments", _pt(c))
    for c in vk.sigma_comms:
        t.append_message(b"sigma commitments", _pt(c))
    for v in pub_input:
        t.append_message(b"public input", _fr(v))
    ch = {}
    for c in proof.wires_poly_comms:
        t.append_message(b"witness_poly_comms", _pt(c))
    ch["beta"], ch["gamma"] = _challenge(t, b"beta"), _challenge(t, b"gamma")
    t.append_message(b"perm_poly_comms", _pt(proof.prod_perm_poly_comm))
    ch["alpha"] = _challenge(t, b"alpha")
    for c in proof.split_quot_poly_comms:
        t.append_message(b"quot_poly_comms", _pt(c))
    ch["zeta"] = _challenge(t, b"zeta")
    for v in proof.wires_evals:
        t.append_message(b"wire_evals", _fr(v))
    for v in proof.wire_sigma_evals:
        t.append_message(b"wire_sigma_evals", _fr(v))
    t.append_message(b"perm_next_eval", _fr(proof.perm_next_eval))
    ch["v"] = _challenge(t, b"v")
    t.append_message(b"open_proof", _pt(proof.opening_proof))
    t.append_message(b"shifted_open_proof", _pt(proof.shifted_opening_proof))
    ch["u"] = _challenge(t, b"u")
    return ch


# ------------------------------------------------------------------ the batch check with the trapdoor
def _aff104(p) -> np.ndarray:
    return np.frombuffer(B.g1_affine_to_bytes(p), dtype=np.uint8).copy()


def _k(v: int) -> np.ndarray:
    return np.frombuffer((v % R).to_bytes(32, "little"), dtype=np.uint64).copy()


def verify(orc, vk, pub_input, proof, tau: int) -> bool:
    """tau * (W + u W') == zeta W + u zeta omega W' + F - E, F and E as in jf-plonk's batch verification"""
    ch = challenges(vk, pub_input, proof)
    be, ga, al, ze, v, u = (ch[k] for k in ("beta", "gamma", "alpha", "zeta", "v", "u"))
    n = vk.n
    om = B.Domain(n).group_gen
    inv = lambda x: pow(x % R, -1, R)
    zh = (pow(ze, n, R) - 1) % R
    l1 = zh * inv(n * (ze - 1)) % R
    pi = sum(p * pow(om, i, R) * zh * inv(n * (ze - pow(om, i, R))) for i, p in enumerate(pub_input)) % R
    w, s, zw = list(proof.wires_evals), list(proof.wire_sigma_evals), proof.perm_next_eval
    prod_s = 1
    for wi, si in zip(w[:4], s):
        prod_s = prod_s * (wi + be * si + ga) % R
    r0 = (pi - al * al * l1 - al * zw * (w[4] + ga) * prod_s) % R
    a, b, c, d, e = w
    ab, cd = a * b % R, c * d % R
    sel = [a, b, c, d, ab, cd, pow(a, 5, R), pow(b, 5, R), pow(c, 5, R), pow(d, 5, R), -e, 1, ab * cd * e]
    cz = al
    for wi, ki in zip(w, vk.k):
        cz = cz * (wi + be * ki * ze + ga) % R
    cz = (cz + al * al * l1) % R
    cs = -al * be * zw * prod_s
    zn2 = pow(ze, n + 2, R)
    quot = [-zh * pow(zn2, j, R) for j in range(5)]
    vs = [pow(v, i, R) for i in range(10)]
    points = list(vk.selector_comms) + [proof.prod_perm_poly_comm, vk.sigma_comms[4]] + list(proof.split_quot_poly_comms) \
        + list(proof.wires_poly_comms) + list(vk.sigma_comms[:4])
    scalars = sel + [cz + u, cs] + quot + vs[1:6] + vs[6:10]
    bases = np.stack([_aff104(p) for p in points])
    sc = np.stack([np.frombuffer(B.fr_to_mont_bytes(x % R), dtype=np.uint64) for x in scalars])
    F = orc.commit(bases, sc)
    e_sc = (-r0 + sum(vs[1 + i] * w[i] for i in range(5)) + sum(vs[6 + i] * s[i] for i in range(4)) + u * zw) % R
    gen = orc.g1_generator()
    J = lambda aff: orc.affine_to_jacobian(aff)
    W, Ws = _aff104(proof.opening_proof), _aff104(proof.shifted_opening_proof)
    rhs = orc.g1_add(F, J(orc.g1_mul(gen, _k(-e_sc))))
    rhs = orc.g1_add(rhs, J(orc.g1_mul(W, _k(ze))))
    rhs = orc.g1_add(rhs, J(orc.g1_mul(Ws, _k(u * ze * om))))
    lhs = orc.g1_add(J(orc.g1_mul(W, _k(tau))), J(orc.g1_mul(Ws, _k(tau * u))))
    return bool(np.array_equal(orc.normalize(lhs), orc.normalize(rhs)))


# ------------------------------------------------------------------ the proof's bytes
def proof_from_bytes(b: bytes):
    """ark-serialize 0.3 CanonicalDeserialize of jf-plonk's Proof (976 B here); raises ValueError on a bad encoding"""
    off = [0]

    def take(k):
        out = b[off[0]:off[0] + k]
        if len(out) != k:
            raise ValueError("short proof")
        off[0] += k
        return out

    pt = lambda: B.g1_decompress(take(48))
    fr = lambda: int.from_bytes(take(32), "little")
    vec = lambda f: [f() for _ in range(int.from_bytes(take(8), "little"))]
    p = SimpleNamespace(wires_poly_comms=vec(pt), prod_perm_poly_comm=pt(), split_quot_poly_comms=vec(pt), opening_proof=pt(),
                        shifted_opening_proof=pt(), wires_evals=vec(fr), wire_sigma_evals=vec(fr), perm_next_eval=fr())
    if off[0] != len(b):
        raise ValueError("trailing bytes")
    return p
