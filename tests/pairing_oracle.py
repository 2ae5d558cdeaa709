"""The BLS12-381 pairing in plain Python integers, by definition, for the tests of dp_multi_pairing / dp_srs_open_key.

TEST INFRASTRUCTURE ONLY: the product never imports it.  Written apart from csrc/pairing.cuh: Fq12 here is the polynomial
ring Fq[w]/(w^12 - 2 w^6 + 2) (w^6 = xi = u + 1, so u = w^6 - 1 and u^2 = -1), G2 uses the textbook affine chord-and-
tangent formulas on the twist, the Miller loop evaluates each line in Fq12 at P on the untwisted point
psi(Q) = (x w^-2, y w^-3) without any division (every line is scaled by a factor of a proper subfield, which the final
exponentiation kills), and the final exponentiation is a plain pow.  The library's value is the cube of the textbook
reduced pairing (DESIGN.md section 3.8), so `pairing` raises to 3 (p^12 - 1) / r as well.  A pairing takes about a
second here: the tests use it for a handful of values."""
from __future__ import annotations

from oracle.py import bls12_381 as B

P = B.FQ_MOD
R = B.FR_MOD
X_ABS = 0xD201000000010000            # the BLS parameter is x = -X_ABS
FINAL_EXP_POWER = 3                   # the library's e = (f^((p^12 - 1) / r))^3
FINAL_EXP = FINAL_EXP_POWER * (P ** 12 - 1) // R

# ------------------------------------------------------------------ Fq2 = Fq[u]/(u^2 + 1), pairs (c0, c1)
def f2_add(a, b):
    return ((a[0] + b[0]) % P, (a[1] + b[1]) % P)


def f2_sub(a, b):
    return ((a[0] - b[0]) % P, (a[1] - b[1]) % P)


def f2_mul(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def f2_inv(a):
    t = pow(a[0] * a[0] + a[1] * a[1], -1, P)
    return (a[0] * t % P, -a[1] * t % P)


def f2_scale(a, k: int):
    return (a[0] * k % P, a[1] * k % P)


# ------------------------------------------------------------------ G2: y^2 = x^3 + 4 (u + 1), affine, None = infinity
G2_B = (4, 4)
G2_GEN = ((0x024AA2B2F08F0A91260805272DC51051C6E47AD4FA403B02B4510B647AE3D1770BAC0326A805BBEFD48056C8C121BDB8,
           0x13E02B6052719F607DACD3A088274F65596BD0D09920B61AB5DA61BBDC7F5049334CF11213945D57E5AC7D055D042B7E),
          (0x0CE5D527727D6E118CC9CDC6DA2E351AADFD9BAA8CBDD3A76D429A695160D12C923AC9CC3BACA289E193548608B82801,
           0x0606C4A02EA734CC32ACD2B02BC28B99CB3E287E85A763AF267492AB572E99AB3F370D275CEC1DA1AAA9075FF05F79BE))


def g2_on_twist(q) -> bool:
    if q is None:
        return True
    x, y = q
    return f2_mul(y, y) == f2_add(f2_mul(f2_mul(x, x), x), G2_B)


def g2_neg(q):
    return None if q is None else (q[0], ((-q[1][0]) % P, (-q[1][1]) % P))


def g2_add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    (x1, y1), (x2, y2) = a, b
    if x1 == x2:
        if f2_add(y1, y2) == (0, 0):
            return None
        lam = f2_mul(f2_scale(f2_mul(x1, x1), 3), f2_inv(f2_scale(y1, 2)))
    else:
        lam = f2_mul(f2_sub(y2, y1), f2_inv(f2_sub(x2, x1)))
    x3 = f2_sub(f2_sub(f2_mul(lam, lam), x1), x2)
    return (x3, f2_sub(f2_mul(lam, f2_sub(x1, x3)), y1))


def g2_mul(q, k: int):
    acc, add = None, q
    while k:
        if k & 1:
            acc = g2_add(acc, add)
        add = g2_add(add, add)
        k >>= 1
    return acc


def g2_to_bytes(q) -> bytes:
    """raw ark 0.3 GroupAffine<g2::Parameters> (200 B): x.c0, x.c1, y.c0, y.c1 Montgomery, infinity flag, padding;
    the identity is (0, 1, true)"""
    if q is None:
        return B.fq_to_mont_bytes(0) * 2 + B.fq_to_mont_bytes(1) + B.fq_to_mont_bytes(0) + b"\x01" + bytes(7)
    (x0, x1), (y0, y1) = q
    return b"".join(B.fq_to_mont_bytes(v) for v in (x0, x1, y0, y1)) + bytes(8)


def g2_from_bytes(b: bytes):
    if b[192]:
        return None
    v = [B.fq_from_mont_bytes(b[48 * i:48 * (i + 1)]) for i in range(4)]
    return ((v[0], v[1]), (v[2], v[3]))


# ------------------------------------------------------------------ Fq12 = Fq[w]/(w^12 - 2 w^6 + 2), 12 coefficients
ONE = [1] + [0] * 11


def f12_mul(a, b):
    t = [0] * 23
    for i, ai in enumerate(a):
        if ai:
            for j, bj in enumerate(b):
                t[i + j] += ai * bj
    for k in range(22, 11, -1):       # w^k = w^(k-12) (2 w^6 - 2)
        c = t[k]
        t[k - 6] += 2 * c
        t[k - 12] -= 2 * c
    return [v % P for v in t[:12]]


def f12_pow(a, e: int):
    acc = ONE
    for bit in bin(e)[2:]:
        acc = f12_mul(acc, acc)
        if bit == "1":
            acc = f12_mul(acc, a)
    return acc


def f12_sub(a, b):
    return [(x - y) % P for x, y in zip(a, b)]


def f12_from_fq2(a):
    """a0 + a1 u = (a0 - a1) + a1 w^6"""
    z = [0] * 12
    z[0], z[6] = (a[0] - a[1]) % P, a[1] % P
    return z


def f12_from_fq(a: int):
    return [a % P] + [0] * 11


W_INV = [0] * 12                      # w (w^11 - 2 w^5) = w^12 - 2 w^6 = -2
W_INV[5], W_INV[11] = 1, (-pow(2, -1, P)) % P
W_INV2 = f12_mul(W_INV, W_INV)
W_INV3 = f12_mul(W_INV2, W_INV)


def untwist(q):
    """psi: E'(Fq2) -> E(Fq12), (x, y) -> (x w^-2, y w^-3)"""
    return f12_mul(f12_from_fq2(q[0]), W_INV2), f12_mul(f12_from_fq2(q[1]), W_INV3)


def to_tower_bytes(f) -> bytes:
    """the library's layout: c0.b0.c0, c0.b0.c1, c0.b1.c0, ..., c1.b2.c1 (Fq12 = Fq6 + Fq6 w, Fq6 = Fq2 (1, v, v^2),
    v = w^2), each a Montgomery Fq; the coefficient of w^e, e < 6, is (a + b u) with b = f[e + 6], a = f[e] + b"""
    out = [0] * 12
    for e in range(6):
        b = f[e + 6]
        i, j = e % 2, e // 2
        out[6 * i + 2 * j], out[6 * i + 2 * j + 1] = (f[e] + b) % P, b
    return b"".join(B.fq_to_mont_bytes(v) for v in out)


def from_tower_bytes(raw: bytes):
    v = [B.fq_from_mont_bytes(raw[48 * k:48 * (k + 1)]) for k in range(12)]
    f = [0] * 12
    for i in range(2):
        for j in range(3):
            a, b = v[6 * i + 2 * j], v[6 * i + 2 * j + 1]
            e = 2 * j + i
            f[e] = (f[e] + a - b) % P
            f[e + 6] = (f[e + 6] + b) % P
    return f


# ------------------------------------------------------------------ the pairing
def _line(t, s, p):
    """the line through psi(t) and psi(s) (the tangent when t == s), evaluated at p in E(Fq), times its denominator"""
    xt, yt = untwist(t)
    xp, yp = f12_from_fq(p[0]), f12_from_fq(p[1])
    if t == s:                        # (yp - yt) 2 yt - 3 xt^2 (xp - xt)
        return f12_sub(f12_mul(f12_sub(yp, yt), [2 * c for c in yt]), f12_mul([3 * c for c in f12_mul(xt, xt)], f12_sub(xp, xt)))
    xs, ys = untwist(s)               # (yp - yt)(xs - xt) - (ys - yt)(xp - xt)
    return f12_sub(f12_mul(f12_sub(yp, yt), f12_sub(xs, xt)), f12_mul(f12_sub(ys, yt), f12_sub(xp, xt)))


def miller_abs_x(p, q):
    """f_{|x|,Q}(P) up to subfield factors; p = (x, y) ints in E(Fq), q on the twist, both finite"""
    t, f = q, ONE
    for bit in bin(X_ABS)[3:]:
        f = f12_mul(f12_mul(f, f), _line(t, t, p))
        t = g2_add(t, t)
        if bit == "1":
            f = f12_mul(f, _line(t, q, p))
            t = g2_add(t, q)
    return f


def multi_pairing(pairs):
    """prod e(P_i, Q_i) as the library defines it: the Miller values f_{|x|} multiplied, then raised to
    -3 (p^12 - 1) / r (x < 0: f_x = 1 / f_{|x|} up to a vertical line)"""
    f = ONE
    for p, q in pairs:
        if p is not None and q is not None:
            f = f12_mul(f, miller_abs_x(p, q))
    return f12_pow(f, (P ** 12 - 1) - FINAL_EXP)


def pairing(p, q):
    return multi_pairing([(p, q)])
