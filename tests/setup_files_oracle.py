"""Plain-Python counterparts of the setup-file kernels, for tests/test_setup_files.py: the Fq2 square root, the compressed
G2 encoding, a twist point outside the r-torsion, and the ChaCha20 block function behind dp_srs_check's scalars.

TEST INFRASTRUCTURE ONLY, next to tests/pairing_oracle.py (whose Fq2 and G2 arithmetic it uses).  Written apart from
csrc/pairing.cuh: the square root here is the exponentiation in Fq2 for p = 3 mod 4 (a^((p - 3) / 4), then one more
exponentiation by (p - 1) / 2 unless the first already shows a = -(x0)^2), not the kernel's norm method, and every root
is checked by squaring."""
from __future__ import annotations

import struct

from tests import pairing_oracle as po

P = po.P


def f2_pow(a, e: int):
    acc = (1, 0)
    for bit in bin(e)[2:]:
        acc = po.f2_mul(acc, acc)
        if bit == "1":
            acc = po.f2_mul(acc, a)
    return acc


def f2_sqrt(a):
    """a square root of a in Fq2, or None when a is not a square"""
    if a == (0, 0):
        return (0, 0)
    a1 = f2_pow(a, (P - 3) // 4)
    x0 = po.f2_mul(a1, a)
    alpha = po.f2_mul(a1, x0)                       # a^((p - 1) / 2)
    if alpha == (P - 1, 0):
        x = po.f2_mul((0, 1), x0)
    else:
        x = po.f2_mul(f2_pow(po.f2_add(alpha, (1, 0)), (P - 1) // 2), x0)
    return x if po.f2_mul(x, x) == a else None


def f2_larger_than_neg(y) -> bool:
    """y > -y with Fq2 ordered by c1 first, then c0"""
    return (y[1], y[0]) > ((-y[1]) % P, (-y[0]) % P)


def g2_compress(q) -> bytes:
    if q is None:
        return bytes(95) + b"\x40"
    (x0, x1), y = q
    b = bytearray(x0.to_bytes(48, "little") + x1.to_bytes(48, "little"))
    if f2_larger_than_neg(y):
        b[95] |= 0x80
    return bytes(b)


def g2_decompress(b: bytes, check_subgroup: bool = True):
    """(point, 0) or (None, why) with the library's reason codes 1..4; the identity is (None, 0)"""
    positive, infinity = bool(b[95] & 0x80), bool(b[95] & 0x40)
    if positive and infinity:
        return None, 2
    if infinity:
        return None, 0
    x = (int.from_bytes(b[:48], "little"), int.from_bytes(b[48:95] + bytes([b[95] & 0x3F]), "little"))
    if x[0] >= P or x[1] >= P:
        return None, 1
    y = f2_sqrt(po.f2_add(po.f2_mul(po.f2_mul(x, x), x), po.G2_B))
    if y is None:
        return None, 3
    if f2_larger_than_neg(y) != positive:
        y = ((-y[0]) % P, (-y[1]) % P)
    q = (x, y)
    if check_subgroup and po.g2_mul(q, po.R) is not None:
        return None, 4
    return q, 0


def twist_point_outside_subgroup():
    """the first x = (k, 0) with a point on the twist; without cofactor clearing it is outside the r-torsion (the twist's
    group order is r times a cofactor of about 2^508)"""
    for k in range(1, 1000):
        x = (k, 0)
        y = f2_sqrt(po.f2_add(po.f2_mul(po.f2_mul(x, x), x), po.G2_B))
        if y is not None and po.g2_mul((x, y), po.R) is not None:
            return (x, y)
    raise AssertionError("no twist point found")


# ------------------------------------------------------------------ ChaCha20 (RFC 8439 section 2.3)
def chacha20_block(key: bytes, counter: int, nonce: bytes) -> bytes:
    s = list(struct.unpack("<4I", b"expand 32-byte k")) + list(struct.unpack("<8I", key)) + [counter] + list(struct.unpack("<3I", nonce))
    x = s[:]
    rotl = lambda v, c: ((v << c) | (v >> (32 - c))) & 0xFFFFFFFF

    def quarter(a, b, c, d):
        x[a] = (x[a] + x[b]) & 0xFFFFFFFF; x[d] = rotl(x[d] ^ x[a], 16)
        x[c] = (x[c] + x[d]) & 0xFFFFFFFF; x[b] = rotl(x[b] ^ x[c], 12)
        x[a] = (x[a] + x[b]) & 0xFFFFFFFF; x[d] = rotl(x[d] ^ x[a], 8)
        x[c] = (x[c] + x[d]) & 0xFFFFFFFF; x[b] = rotl(x[b] ^ x[c], 7)

    for _ in range(10):
        quarter(0, 4, 8, 12); quarter(1, 5, 9, 13); quarter(2, 6, 10, 14); quarter(3, 7, 11, 15)
        quarter(0, 5, 10, 15); quarter(1, 6, 11, 12); quarter(2, 7, 8, 13); quarter(3, 4, 9, 14)
    return struct.pack("<16I", *((a + b) & 0xFFFFFFFF for a, b in zip(x, s)))


def srs_check_scalars(seed: bytes, n: int) -> list:
    """rho_0 .. rho_(n-2) as dp_srs_check draws them: 128 bits each, four per ChaCha20 block with counter i div 4 and an
    all-zero nonce"""
    out = []
    for i in range(n - 1):
        blk = chacha20_block(seed, i // 4, bytes(12))
        out.append(int.from_bytes(blk[16 * (i % 4):16 * (i % 4) + 16], "little"))
    return out
