"""The setup ceremony on the kernel-logic emulator: dp_srs_update against dp_srs_powers_of_tau of the product tau s (byte
for byte, G1 and G2), against the plain double-and-add of dp_debug_srs_update_plain and the oracle's g1_mul, the
endomorphism constants and the scalar split, the argument errors, a library-drawn s, and the whole ceremony through
files: ceremony_start, three contributions, load_ceremony_srs, a proof over the final SRS verified by a party that holds
three byte strings, and every refusal of load_ceremony_srs and contribution_from_bytes."""
import random
import struct

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import DP_E_ARG, DP_E_STATE, Context, DpError
from distributed_plonk_b200.proof import FQ_MOD, g2_from_raw, point_from_raw
from distributed_plonk_b200.srs import (G1_GEN, G2_GEN, Contribution, ceremony_start, contribute, contribution_from_bytes,
                                        load_ceremony_srs, load_srs, open_key, save_srs, universal_setup)
from distributed_plonk_b200.transcript import R_MOD
from distributed_plonk_b200.verifier import verify_bytes
from tests import pairing_oracle as po
from tests import setup_files_oracle as so
from tests import test_circuit as tc

TAU = 0x2B1E4A1D6F3C0E5A7B9D8C6E4F2A1B3C5D7E9F0A1B2C3D4E5F6A7B8C9D0E1F2
LAMBDA = 0xAC45A4010001A40200000000FFFFFFFF
BETA = 0x1A0111EA397FE699EC02408663D4DE85AA0D857D89759AD4897D29650FB85F9B409427EB4F49FFFD8BFD00000000AAAC


def scalar(k: int) -> np.ndarray:
    return np.frombuffer(int(k).to_bytes(32, "little"), dtype=np.uint64)


def setup_ctx(lib, n: int, tau: int = TAU):
    c = Context(lib, 0, 0, 1)
    universal_setup(c, torch, n - 1, 32, 256, tau=tau, device="cpu")
    return c


def bases_and_msm(c, n):
    """the context's bases and an MSM over them: what an update must leave as it was"""
    sc = np.stack([scalar(k) for k in range(3, 3 + n)])
    return c.get_bases(0, n), c.msm(0, n, sc)


# ------------------------------------------------------------------ the endomorphism split
def test_glv_constants():
    assert LAMBDA * LAMBDA + LAMBDA + 1 == R_MOD
    assert pow(BETA, 3, FQ_MOD) == 1 and BETA != 1
    x = -0xD201000000010000
    assert LAMBDA == x * x - 1


def test_phi_of_g_is_lambda_g(orc):
    g = orc.g1_generator()
    lam_g = point_from_raw(orc.g1_mul(g, scalar(LAMBDA)))
    assert lam_g == (G1_GEN[0] * BETA % FQ_MOD, G1_GEN[1])


def split(k: int):
    """the kernel's split: k2 = floor(k / lambda), k1 = k mod lambda"""
    return k % LAMBDA, k // LAMBDA


@pytest.mark.parametrize("k", [0, 1, LAMBDA - 1, LAMBDA, LAMBDA + 1, LAMBDA * LAMBDA + LAMBDA, 0x1234567890ABCDEF << 180])
def test_split_recombines_and_fits_128_bits(k):
    k1, k2 = split(k)
    assert k1 + LAMBDA * k2 == k and 0 <= k1 < LAMBDA and 0 <= k2 <= LAMBDA + 1 < 1 << 128
    rng = random.Random(k)
    for _ in range(20):
        k = rng.randrange(R_MOD)
        k1, k2 = split(k)
        assert k1 + LAMBDA * k2 == k and k2 < 1 << 128


# ------------------------------------------------------------------ dp_srs_update against the generator
@pytest.mark.parametrize("n", [2, 35, 131, (1 << 10) + 3])
def test_update_equals_the_srs_of_tau_s(emul_lib, n):
    c = setup_ctx(emul_lib, n)
    g2 = c.srs_open_key(TAU)
    before = bases_and_msm(c, n)
    rng = random.Random(n)
    for s in [1, 2, R_MOD - 1, rng.randrange(1, R_MOD)] if n <= 131 else [rng.randrange(1, R_MOD)]:
        pts, g2_out = c.srs_update(g2, n, s)
        assert np.array_equal(pts, c.g1_compress(c.srs_powers_of_tau(TAU * s % R_MOD, n))), s
        assert np.array_equal(g2_out[0], c.srs_open_key(s)[1]) and np.array_equal(g2_out[1], c.srs_open_key(TAU * s % R_MOD)[1])
        if n <= 35:
            plain, plain_g2 = c.srs_update(g2, n, s, plain=True)
            assert np.array_equal(plain, pts) and np.array_equal(plain_g2, g2_out)
    after = bases_and_msm(c, n)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    c.close()


@pytest.mark.parametrize("s", [1, LAMBDA - 1, LAMBDA, LAMBDA + 1, R_MOD - 1, 0x5EED << 200])
def test_scalar_split_edges_against_the_oracle(orc, emul_lib, s):
    """N = 2: Q_1 = s P_1, so s itself is the scalar the kernel splits; the oracle's double-and-add is independent of it"""
    c = setup_ctx(emul_lib, 2)
    pts, _ = c.srs_update(c.srs_open_key(TAU), 2, s)
    p1 = c.get_bases(1, 1)
    assert pts[0].tobytes() == orc.g1_compress(orc.g1_generator().reshape(1, 104)).tobytes()
    assert pts[1].tobytes() == orc.g1_compress(orc.g1_mul(p1[0], scalar(s)).reshape(1, 104)).tobytes()
    c.close()


def test_a_few_points_against_the_oracle(orc, emul_lib):
    n, s = 70, 0x0DDC0FFEE0DDC0FFEE
    c = setup_ctx(emul_lib, n)
    pts, _ = c.srs_update(c.srs_open_key(TAU), n, s)
    bases = c.get_bases(0, n)
    for i in (0, 1, 2, 33, 69):
        want = orc.g1_compress(orc.g1_mul(bases[i], scalar(pow(s, i, R_MOD))).reshape(1, 104))
        assert pts[i].tobytes() == want.tobytes(), i
    c.close()


def test_two_updates_compose(emul_lib):
    n, s1, s2 = 37, 0xA11CE, 0xB0B << 64
    a = setup_ctx(emul_lib, n)
    pts1, g2_1 = a.srs_update(a.srs_open_key(TAU), n, s1)
    b = Context(emul_lib, 0, 0, 1)
    b.init_compressed(pts1, 32, 256)
    pts2, g2_2 = b.srs_update(np.stack([a.srs_open_key(TAU)[0], g2_1[1]]), n, s2)      # h, tau s1 h: the new file's G2 half
    t = TAU * s1 * s2 % R_MOD
    assert np.array_equal(pts2, a.g1_compress(a.srs_powers_of_tau(t, n)))
    assert np.array_equal(g2_2[1], a.srs_open_key(t)[1])
    a.close()
    b.close()


def test_errors_leave_the_context_as_it_was(emul_lib):
    n = 35
    c = setup_ctx(emul_lib, n)
    g2 = c.srs_open_key(TAU)
    before = bases_and_msm(c, n)
    for s in (0, R_MOD, (1 << 256) - 1):
        with pytest.raises(DpError) as e:
            c.srs_update(g2, n, s)
        assert e.value.code == DP_E_ARG
    out48, out400 = np.zeros((n, 48), dtype=np.uint8), np.zeros((2, 200), dtype=np.uint8)
    for args in ((None, g2.ctypes.data, None, out400.ctypes.data), (None, None, out48.ctypes.data, out400.ctypes.data),
                 (None, g2.ctypes.data, out48.ctypes.data, None)):
        assert c.lib.dp_srs_update(c.h, *args) == DP_E_ARG
    assert c.lib.dp_srs_update(None, None, g2.ctypes.data, out48.ctypes.data, out400.ctypes.data) == DP_E_ARG
    outside = np.frombuffer(po.g2_to_bytes(so.twist_point_outside_subgroup()), dtype=np.uint8)
    off_twist = np.frombuffer(po.g2_to_bytes(((1, 0), (1, 0))), dtype=np.uint8)
    for bad, word in ((outside, "r-torsion"), (off_twist, "twist")):
        for at in (0, 1):
            q = g2.copy()
            q[at] = bad
            with pytest.raises(DpError, match=word) as e:
                c.srs_update(q, n, 5)
            assert e.value.code == DP_E_ARG
    after = bases_and_msm(c, n)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    c.close()
    fresh = Context(emul_lib, 0, 0, 1)
    with pytest.raises(DpError) as e:
        fresh.srs_update(g2, 2, 5)
    assert e.value.code == DP_E_STATE
    fresh.init(np.zeros((0, 104), dtype=np.uint8), 32, 256)
    with pytest.raises(DpError) as e:
        fresh.srs_update(g2, 0, 5, out48=np.zeros((0, 48), dtype=np.uint8))
    assert e.value.code == DP_E_STATE
    fresh.close()


def test_library_drawn_s_gives_different_files_that_both_verify(emul_lib):
    n = 35
    c = setup_ctx(emul_lib, n)
    g2 = c.srs_open_key(TAU)
    (a, ga), (b, gb) = c.srs_update(g2, n), c.srs_update(g2, n)
    assert not np.array_equal(a, b) and not np.array_equal(ga, gb)
    for pts, g in ((a, ga), (b, gb)):
        v = Context(emul_lib, 0, 0, 1)
        v.init_compressed(pts, 32, 256)
        assert v.srs_check(np.stack([g2[0], g[1]]))
        v.close()
    c.close()


# ------------------------------------------------------------------ the ceremony through files
N_CEREMONY_LOG = 6


@pytest.fixture(scope="module")
def ceremony(emul_lib, tmp_path_factory):
    """ceremony_start, then three contributions in three contexts: the file paths and the receipts"""
    d = tmp_path_factory.mktemp("ceremony")
    n = 1 << N_CEREMONY_LOG
    paths = [d / f"srs{j}.bin" for j in range(4)]
    ceremony_start(paths[0], n + 3)
    receipts = []
    for j in range(3):
        c = Context(emul_lib, 0, 0, 1)
        receipts.append(contribute(c, paths[j], paths[j + 1], n, 8 * n))
        c.close()
    return paths, receipts


def test_ceremony_start_is_the_srs_of_tau_1(emul_lib, tmp_path):
    path = tmp_path / "start.bin"
    ceremony_start(path, 5)
    c = setup_ctx(emul_lib, 5, tau=1)
    save_srs(c, tmp_path / "tau1.bin", open_key(c, 1))
    assert path.read_bytes() == (tmp_path / "tau1.bin").read_bytes()
    c.close()
    with pytest.raises(ValueError):
        ceremony_start(path, 1)


def test_contribute_writes_the_srs_of_tau_s(emul_lib, tmp_path):
    n, s = 35, 0xC0FFEE
    start = tmp_path / "a.bin"
    ceremony_start(start, n)
    c = Context(emul_lib, 0, 0, 1)
    r = contribute(c, start, tmp_path / "b.bin", 32, 256, secret=s)
    ref = setup_ctx(emul_lib, n, tau=s)
    save_srs(ref, tmp_path / "ref.bin", open_key(ref, s))
    assert (tmp_path / "b.bin").read_bytes() == (tmp_path / "ref.bin").read_bytes()
    assert r == Contribution(G1_GEN, point_from_raw(ref.get_bases(1, 1)[0]), po.g2_mul(G2_GEN, s))
    assert len(r.to_bytes()) == 192 and contribution_from_bytes(c, r.to_bytes()) == r
    ref.close()
    one = tmp_path / "one.bin"
    one.write_bytes(struct.pack("<Q", 1) + (tmp_path / "a.bin").read_bytes()[8:56] + (tmp_path / "a.bin").read_bytes()[-192:])
    with pytest.raises(ValueError, match="at least 2 points"):
        contribute(c, one, tmp_path / "c.bin", 32, 256)
    c.close()


def test_ceremony_then_prove_and_verify(orc, emul_lib, ceremony):
    paths, receipts = ceremony
    n = 1 << N_CEREMONY_LOG
    assert len({p.read_bytes() for p in paths}) == 4
    b = Context(emul_lib, 0, 0, 1)
    key = load_ceremony_srs(b, paths[3], receipts, n, 8 * n)
    assert key.h == G2_GEN
    pr, _, (_, _, witness, _) = tc.prover_from_circuit(orc, b, N_CEREMONY_LOG, 20100, "cpu")
    proof, pub = pr.prove_circuit(tc.witness_host(witness, "cpu"))
    vk_bytes, proof_bytes = pr.verifying_key().to_bytes(), proof.to_bytes()
    del pr
    b.close()
    v = Context(emul_lib, 0, 0, 1)
    assert verify_bytes(v, vk_bytes, key.to_bytes(), pub, proof_bytes)
    flipped = bytearray(proof_bytes)
    flipped[len(proof_bytes) - 10 * 32 - 8] ^= 1
    assert not verify_bytes(v, vk_bytes, key.to_bytes(), pub, bytes(flipped))
    v.close()


def test_ceremony_refusals(orc, emul_lib, ceremony, tmp_path):
    paths, receipts = ceremony
    n = 1 << N_CEREMONY_LOG
    final = paths[3].read_bytes()
    r0, r1, r2 = receipts
    other_pk = po.g2_mul(G2_GEN, 0x5151)

    def at(i):
        return 8 + 48 * i

    replaced = tmp_path / "replaced.bin"
    g5 = orc.g1_compress(orc.g1_mul(orc.g1_generator(), scalar(5)).reshape(1, 104)).tobytes()
    replaced.write_bytes(final[:at(9)] + g5 + final[at(10):])
    unrelated = tmp_path / "unrelated.bin"
    u = setup_ctx(emul_lib, n + 3, tau=0x7777)
    save_srs(u, unrelated, open_key(u, 0x7777))
    made_up = Contribution(G1_GEN, point_from_raw(u.get_bases(1, 1)[0]), po.g2_mul(G2_GEN, 0x7778))
    u.close()
    changed_h = tmp_path / "changed_h.bin"                      # h' = 2h, beta h' = tau 2h: consistent, but not the start's h
    c = Context(emul_lib, 0, 0, 1)
    load_srs(c, paths[3], n, 8 * n)
    blob = bytearray(final)
    two_h = po.g2_mul(G2_GEN, 2)
    beta_h = g2_from_raw(c.g2_decompress(np.frombuffer(final[-96:], dtype=np.uint8).reshape(1, 96))[0])
    blob[-192:] = so.g2_compress(two_h) + so.g2_compress(po.g2_add(beta_h, beta_h))
    changed_h.write_bytes(bytes(blob))
    cases = [
        ("a pubkey of another s", paths[3], [r0, Contribution(r1.old, r1.new, other_pk), r2], "contribution 1 fails"),
        ("an identity pubkey", paths[3], [r0, r1, Contribution(r2.old, r2.new, None)], "contribution 2: pubkey .* identity"),
        ("two receipts swapped", paths[3], [r1, r0, r2], "contribution 0 does not start"),
        ("a broken link", paths[3], [r0, r2], "contribution 1 does not start"),
        ("a missing last receipt", paths[3], [r0, r1], "not P_1"),
        ("one point replaced", replaced, receipts, "consecutive powers"),
        ("an unrelated tau with a made-up receipt", unrelated, [made_up], "contribution 0 fails"),
        ("a changed h", changed_h, receipts, "standard G2 generator"),
        ("an empty chain", paths[3], [], "empty"),
    ]
    for name, path, chain, word in cases:
        with pytest.raises(ValueError, match=word):
            load_ceremony_srs(c, path, chain, n, 8 * n)
            pytest.fail(name)
        with pytest.raises(DpError):                            # no bases are left, as after a failed load_srs check
            c.get_bases(0, 1)
    assert load_ceremony_srs(c, paths[3], receipts, n, 8 * n).h == G2_GEN
    good = r1.to_bytes()
    for data, word in ((good[:-1], "truncated"), (good + b"\x00", "trailing"),
                       (good[:96] + so.g2_compress(None), "identity"),
                       (good[:96] + so.g2_compress(so.twist_point_outside_subgroup()), "r-torsion"),
                       (FQ_MOD.to_bytes(48, "little") + good[48:], "point 0")):
        with pytest.raises(ValueError, match=word):
            contribution_from_bytes(c, data)
    c.close()
