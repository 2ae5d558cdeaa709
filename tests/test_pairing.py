"""dp_multi_pairing, dp_srs_open_key, dp_msm_points and dp_g1_decompress on the kernel-logic emulator: the pairing oracle
(tests/pairing_oracle.py) checks itself; the library equals it byte for byte; bilinearity and inverses on more samples
with the library alone; every argument error and rejection reason."""
import ctypes as C
import random

import numpy as np
import pytest

from distributed_plonk_b200._binding import Context, DpError
from oracle.py import bls12_381 as B
from tests import pairing_oracle as po

R, P = po.R, po.P
G, H = B.G1_GEN, po.G2_GEN
ONE = po.to_tower_bytes(po.ONE)


def g1raw(pts) -> np.ndarray:
    return np.frombuffer(b"".join(B.g1_affine_to_bytes(p) for p in pts), dtype=np.uint8).reshape(-1, 104)


def g2raw(qs) -> np.ndarray:
    return np.frombuffer(b"".join(po.g2_to_bytes(q) for q in qs), dtype=np.uint8).reshape(-1, 200)


def f2_sqrt(a):
    """a square root in Fq2 (p = 3 mod 4), or None"""
    a1 = _f2_pow(a, (P - 3) // 4)
    alpha = po.f2_mul(po.f2_mul(a1, a1), a)
    x0 = po.f2_mul(a1, a)
    if alpha == (P - 1, 0):
        x = po.f2_mul((0, 1), x0)
    else:
        x = po.f2_mul(_f2_pow(po.f2_add((1, 0), alpha), (P - 1) // 2), x0)
    return x if po.f2_mul(x, x) == a else None


def _f2_pow(a, e):
    acc = (1, 0)
    for bit in bin(e)[2:]:
        acc = po.f2_mul(acc, acc)
        if bit == "1":
            acc = po.f2_mul(acc, a)
    return acc


def twist_point_outside_g2():
    """a point of the twist E'(Fq2) that is not in the r-torsion (the cofactor is huge: almost every point)"""
    for x0 in range(1, 50):
        x = (x0, 1)
        y = f2_sqrt(po.f2_add(po.f2_mul(po.f2_mul(x, x), x), po.G2_B))
        if y is not None and po.g2_mul((x, y), R) is not None:
            return (x, y)
    raise AssertionError("no twist point found")


@pytest.fixture(scope="module")
def ctx(emul_lib):
    c = Context(emul_lib, 0, 0, 1)          # never initialised: a verifier holds no G1 SRS
    yield c
    c.close()


# ------------------------------------------------------------------ the oracle checks itself
def test_oracle_self_checks():
    assert po.g2_on_twist(H) and po.g2_mul(H, R) is None and po.g2_mul(H, R - 1) == po.g2_neg(H)
    x = -po.X_ABS
    assert R == x ** 4 - x ** 2 + 1 and P == (x - 1) ** 2 * R // 3 + x
    # the hard part the library's final exponentiation uses: 3 (p^4 - p^2 + 1) / r
    assert 3 * (P ** 4 - P ** 2 + 1) // R == (x - 1) ** 2 * (x + P) * (x ** 2 + P ** 2 - 1) + 3
    assert (P ** 4 - P ** 2 + 1) % R == 0 and (P ** 12 - 1) % R == 0
    e = po.pairing(G, H)
    assert e != po.ONE and po.f12_pow(e, R) == po.ONE
    rng = random.Random(16000)
    a, b = rng.randrange(1, R), rng.randrange(1, R)
    assert po.pairing(B.g1_mul(G, a), po.g2_mul(H, b)) == po.f12_pow(e, a * b % R)
    assert po.from_tower_bytes(po.to_tower_bytes(e)) == e


# ------------------------------------------------------------------ library against the oracle
def test_multi_pairing_matches_the_oracle(ctx):
    rng = random.Random(16100)
    pts = [B.g1_mul(G, rng.randrange(1, R)) for _ in range(3)]
    qs = [po.g2_mul(H, rng.randrange(1, R)) for _ in range(3)]
    for pairs in ([(pts[0], qs[0])], [(pts[0], qs[0]), (pts[1], qs[1])], [(pts[0], qs[0]), (None, qs[1]), (pts[2], qs[2])],
                  [(pts[1], None), (pts[2], qs[0])]):
        got = ctx.multi_pairing(g1raw([p for p, _ in pairs]), g2raw([q for _, q in pairs]))
        assert got.tobytes() == po.to_tower_bytes(po.multi_pairing(pairs)), f"k = {len(pairs)}"
    assert ctx.multi_pairing(g1raw([]), g2raw([])).tobytes() == ONE
    assert ctx.multi_pairing(g1raw([None]), g2raw([H])).tobytes() == ONE


@pytest.mark.parametrize("tau", [1, R - 1, 0x3A5F0C1E2D4B6978A1B2C3D4E5F60718293A4B5C6D7E8F90A1B2C3D4E5F6071])
def test_open_key_matches_the_oracle(ctx, tau):
    got = ctx.srs_open_key(tau)
    assert got[0].tobytes() == po.g2_to_bytes(H)
    assert got[1].tobytes() == po.g2_to_bytes(po.g2_mul(H, tau))


@pytest.mark.parametrize("n", [0, 1, 2, 31, 300])
def test_msm_points_matches_the_oracle_without_init(orc, ctx, n):
    bases = orc.gen_bases(16200 + n, n, 64, True) if n else np.zeros((0, 104), dtype=np.uint8)
    sc = orc.gen_fr(16300 + n, n, False) if n else np.zeros((0, 4), dtype=np.uint64)
    if n >= 2:
        sc[1] = 0                                    # a zero scalar
        bases[-1] = np.frombuffer(B.g1_affine_to_bytes(None), dtype=np.uint8)   # an infinity point
    got = ctx.msm_points(bases, sc)
    if n == 0:
        assert B.g1_jacobian_from_bytes(got.tobytes()) is None
        return
    assert np.array_equal(orc.normalize(got), orc.normalize(orc.msm(bases, sc)))


# ------------------------------------------------------------------ the library alone, more samples
def test_bilinearity_and_inverses(ctx):
    rng = random.Random(16400)
    for _ in range(3):
        a, b = rng.randrange(1, R), rng.randrange(1, R)
        p, q = B.g1_mul(G, rng.randrange(1, R)), po.g2_mul(H, rng.randrange(1, R))
        e = lambda pairs: ctx.multi_pairing(g1raw([x for x, _ in pairs]), g2raw([y for _, y in pairs])).tobytes()
        ap, bp, aq, bq = B.g1_mul(p, a), B.g1_mul(p, b), po.g2_mul(q, a), po.g2_mul(q, b)
        assert e([(B.g1_mul(p, (a + b) % R), q)]) == e([(ap, q), (bp, q)])          # linear in the first argument
        assert e([(p, po.g2_mul(q, (a + b) % R))]) == e([(p, aq), (p, bq)])         # ... and in the second
        assert e([(ap, q)]) == e([(p, aq)])
        assert e([(B.g1_neg(p), q)]) == e([(p, po.g2_neg(q))])
        assert e([(p, q), (B.g1_neg(p), q)]) == ONE and e([(p, q), (p, po.g2_neg(q))]) == ONE
        assert e([(p, q)]) != ONE


# ------------------------------------------------------------------ argument errors and rejections
def test_argument_errors(emul_lib, ctx):
    L, h = emul_lib, ctx.h
    out = np.zeros(1024, dtype=np.uint8)
    g1, g2 = g1raw([G]), g2raw([H])
    assert L.dp_multi_pairing(None, g1.ctypes.data, g2.ctypes.data, 1, out.ctypes.data) == -1
    assert L.dp_multi_pairing(h, None, g2.ctypes.data, 1, out.ctypes.data) == -1
    assert L.dp_multi_pairing(h, g1.ctypes.data, None, 1, out.ctypes.data) == -1
    assert L.dp_multi_pairing(h, g1.ctypes.data, g2.ctypes.data, 1, None) == -1
    tau = (5).to_bytes(32, "little")
    assert L.dp_srs_open_key(None, tau, out.ctypes.data) == -1
    assert L.dp_srs_open_key(h, None, out.ctypes.data) == -1
    assert L.dp_srs_open_key(h, tau, None) == -1
    sc = np.zeros((1, 4), dtype=np.uint64)
    assert L.dp_msm_points(None, g1.ctypes.data, sc.ctypes.data, 1, out.ctypes.data) == -1
    assert L.dp_msm_points(h, None, sc.ctypes.data, 1, out.ctypes.data) == -1
    assert L.dp_msm_points(h, g1.ctypes.data, None, 1, out.ctypes.data) == -1
    assert L.dp_msm_points(h, g1.ctypes.data, sc.ctypes.data, 1, None) == -1
    c48 = np.zeros(48, dtype=np.uint8)
    assert L.dp_g1_decompress(None, c48.ctypes.data, 1, 1, out.ctypes.data, None, None) == -1
    assert L.dp_g1_decompress(h, None, 1, 1, out.ctypes.data, None, None) == -1
    assert L.dp_g1_decompress(h, c48.ctypes.data, 1, 1, None, None, None) == -1
    assert L.dp_g1_decompress(h, None, 0, 1, None, None, None) == 0
    assert not out.any()
    for bad, word in ((0, "zero"), (R, "canonical"), ((1 << 256) - 1, "canonical")):
        with pytest.raises(DpError) as e:
            ctx.srs_open_key(bad)
        assert e.value.code == -1 and word in str(e.value)


def test_multi_pairing_rejects_bad_points(ctx):
    q_off = (H[0], po.f2_add(H[1], (1, 0)))                             # not on the twist
    q_out = twist_point_outside_g2()                                     # on the twist, not in the r-torsion
    p_off = (G[0], (G[1] + 1) % P)
    not_fq = bytearray(B.g1_affine_to_bytes(G))
    not_fq[0:48] = P.to_bytes(48, "little")                              # a coordinate >= p
    g2_not_fq = bytearray(po.g2_to_bytes(H))
    g2_not_fq[48:96] = ((1 << 384) - 1).to_bytes(48, "little")
    cases = [
        (g1raw([G, p_off]), g2raw([H, H]), "pair 1", "not on the curve"),
        (np.frombuffer(bytes(not_fq), np.uint8)[None], g2raw([H]), "pair 0", "G1 coordinate"),
        (g1raw([G, G, G]), g2raw([H, H, q_off]), "pair 2", "not on the twist"),
        (g1raw([G, G]), g2raw([q_out, H]), "pair 0", "r-torsion"),
        (g1raw([G]), np.frombuffer(bytes(g2_not_fq), np.uint8)[None], "pair 0", "G2 coordinate"),
    ]
    for g1, g2, where, word in cases:
        with pytest.raises(DpError) as e:
            ctx.multi_pairing(g1, g2)
        assert e.value.code == -1 and where in str(e.value) and word in str(e.value), str(e.value)
    assert po.g2_on_twist(q_out)                                         # no cofactor clearing: rejected as it is


def test_g1_decompress_and_every_reason_code(orc, ctx):
    pts = orc.gen_bases(16500, 40, 40, True)
    comp = orc.g1_compress(pts)
    assert np.array_equal(ctx.g1_decompress(comp), pts)
    assert np.array_equal(ctx.g1_decompress(comp, check_subgroup=False), pts)
    not_sq = next(x for x in range(1, 100) if pow((x ** 3 + 4) % P, (P - 1) // 2, P) != 1)
    outside = orc.g1_point_outside_subgroup()
    for why, enc in ((1, P.to_bytes(48, "little")), (2, bytes(47) + b"\xc0"), (3, not_sq.to_bytes(48, "little")),
                     (4, outside.tobytes())):
        bad = comp.copy()
        bad[7] = np.frombuffer(enc, dtype=np.uint8)
        bad[9] = np.frombuffer(enc, dtype=np.uint8)
        with pytest.raises(DpError) as e:
            ctx.g1_decompress(bad)
        assert (e.value.code, e.value.index, e.value.why) == (-1, 7, why), str(e.value)
    bad = comp.copy()
    bad[3] = outside
    got = ctx.g1_decompress(bad, check_subgroup=False)                  # on the curve: accepted without the check
    assert np.array_equal(got[3], orc.g1_decompress(outside[None], False)[0][0])
    idx, why = C.c_size_t(), C.c_int()
    out = np.zeros((40, 104), dtype=np.uint8)
    assert ctx.lib.dp_g1_decompress(ctx.h, comp.ctypes.data, 40, 1, out.ctypes.data, C.byref(idx), C.byref(why)) == 0
    assert (idx.value, why.value) == (40, 0) and np.array_equal(out, pts)
