"""Setup files on the kernel-logic emulator: dp_g1_compress / dp_get_bases_compressed / dp_g2_compress / dp_g2_decompress
against the Python oracles (tests/setup_files_oracle.py, oracle/py), every rejection code of the G2 decoder, dp_srs_check
on the SRS of universal_setup and on six ways of spoiling it, its two MSM results against the oracle's MSM over the
Python ChaCha20 scalars (which the RFC 8439 test vector pins), the save_srs / load_srs round trip, a prover and a verifier
in separate contexts that never see tau, and the malformed files."""
import random
import struct

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import DP_E_STATE, Context, DpError
from distributed_plonk_b200.proof import FQ_MOD, VerifyingKey, g2_compress, g2_to_raw
from distributed_plonk_b200.srs import OpenKey, load_srs, open_key, open_key_from_bytes, save_srs, universal_setup
from distributed_plonk_b200.transcript import R_MOD
from distributed_plonk_b200.verifier import verify_bytes
from tests import pairing_oracle as po
from tests import setup_files_oracle as so
from tests import test_circuit as tc
from tests import test_proof as tp

TAU = 0x3C6EF372FE94F82BA54FF53A5F1D36F1510E527FADE682D19B05688C2B3E6C1F
SEED = bytes(range(32))


def scalar(k: int) -> np.ndarray:
    return np.frombuffer(int(k).to_bytes(32, "little"), dtype=np.uint64)


def uninitialised(ctx) -> bool:
    try:
        ctx.get_bases(0, 0)
    except DpError as e:
        return e.code == DP_E_STATE
    return False


@pytest.fixture(scope="module")
def ctx(emul_lib):
    c = Context(emul_lib, 0, 0, 1)               # never initialised
    yield c
    c.close()


# ------------------------------------------------------------------ the oracles themselves
def test_chacha20_block_is_rfc_8439_section_2_3_2():
    key, nonce = bytes(range(32)), bytes.fromhex("000000090000004a00000000")
    want = bytes.fromhex("10f1e7e4d13b5915500fdd1fa32071c4c7d1f4c733c068030422aa9ac3d46c4e"
                         "d2826446079faa0914c2d705d98b02a2b5129cd1de164eb9cbd083e8a2503c4e")
    assert so.chacha20_block(key, 1, nonce) == want


def test_fq2_square_root_oracle():
    rng = random.Random(18000)
    squares = 0
    for _ in range(20):
        a = (rng.randrange(FQ_MOD), rng.randrange(FQ_MOD))
        s = so.f2_sqrt(po.f2_mul(a, a))
        assert s in (a, ((-a[0]) % FQ_MOD, (-a[1]) % FQ_MOD))
        squares += so.f2_sqrt(a) is not None
    assert 0 < squares < 20
    assert so.g2_decompress(so.g2_compress(po.G2_GEN)) == (po.G2_GEN, 0)


# ------------------------------------------------------------------ G1
def test_g1_compress_matches_the_oracle_and_round_trips(orc, ctx):
    bases = orc.gen_bases(18100, 300, 300, True)
    bases[7] = ctx.g1_decompress(np.frombuffer(bytes(47) + b"\x40", dtype=np.uint8).reshape(1, 48))[0]      # the identity
    comp = ctx.g1_compress(bases)
    assert np.array_equal(comp, orc.g1_compress(bases))
    signs = {int(c[47]) >> 7 for c in comp if not c[47] & 0x40}
    assert signs == {0, 1} and comp[7].tobytes() == bytes(47) + b"\x40"
    assert np.array_equal(ctx.g1_decompress(comp), bases)
    assert ctx.g1_compress(np.zeros((0, 104), dtype=np.uint8)).shape == (0, 48)


def test_get_bases_compressed(orc, emul_lib):
    bases = orc.gen_bases(18200, 70, 70, True)
    c = Context(emul_lib, 0, 0, 1)
    with pytest.raises(DpError) as e:
        c.get_bases_compressed(0, 1)
    assert e.value.code == DP_E_STATE
    c.init(bases, 16, 128)
    want = orc.g1_compress(bases)
    assert np.array_equal(c.get_bases_compressed(0, 70), want)
    assert np.array_equal(c.get_bases_compressed(13, 40), want[13:53])
    assert c.get_bases_compressed(70, 0).shape == (0, 48)
    with pytest.raises(DpError):
        c.get_bases_compressed(31, 40)
    c.close()


# ------------------------------------------------------------------ G2
def g2_points():
    rng = random.Random(18300)
    return [po.G2_GEN, None] + [po.g2_mul(po.G2_GEN, rng.randrange(1, R_MOD)) for _ in range(6)]


def test_g2_compress_and_decompress_match_the_oracle(ctx):
    pts = g2_points()
    raw = np.frombuffer(b"".join(po.g2_to_bytes(q) for q in pts), dtype=np.uint8).reshape(-1, 200)
    comp = ctx.g2_compress(raw)
    for q, c in zip(pts, comp):
        assert c.tobytes() == so.g2_compress(q) == g2_compress(q)
        assert so.g2_decompress(c.tobytes()) == (q, 0)
    assert {int(c[95]) >> 6 for c in comp} == {0, 1, 2}          # both signs and the identity
    assert np.array_equal(ctx.g2_decompress(comp), raw)
    assert np.array_equal(ctx.g2_decompress(comp, check_subgroup=False), raw)
    # a root with c1 = 0 and one with c0 = 0 exercise the second key of the order and the a1 = 0 branch of the root
    for x in ((k, 0) for k in range(1, 40)):
        y = so.f2_sqrt(po.f2_add(po.f2_mul(po.f2_mul(x, x), x), po.G2_B))
        if y is not None:
            for q in ((x, y), po.g2_neg((x, y))):
                enc = np.frombuffer(so.g2_compress(q), dtype=np.uint8).reshape(1, 96)
                assert ctx.g2_decompress(enc, check_subgroup=False)[0].tobytes() == po.g2_to_bytes(q)


def test_g2_decompress_rejection_codes(ctx):
    good = [so.g2_compress(q) for q in g2_points()[:5]]
    not_square = next((k, 0) for k in range(1, 100) if so.f2_sqrt(po.f2_add(po.f2_mul(po.f2_mul((k, 0), (k, 0)), (k, 0)), po.G2_B)) is None)
    outside = so.twist_point_outside_subgroup()
    both = bytearray(good[0])
    both[95] |= 0xC0
    cases = [
        (1, FQ_MOD.to_bytes(48, "little") + good[0][48:]),
        (1, good[0][:48] + (FQ_MOD + 1).to_bytes(48, "little")),
        (2, bytes(both)),
        (3, so.g2_compress((not_square, (0, 1)))),
        (4, so.g2_compress(outside)),
    ]
    for at, (why, enc) in enumerate(cases):
        assert so.g2_decompress(enc)[1] == why
        batch = good[:at] + [enc] + good[at:]
        with pytest.raises(DpError) as e:
            ctx.g2_decompress(np.frombuffer(b"".join(batch), dtype=np.uint8).reshape(-1, 96))
        assert (e.value.index, e.value.why) == (at, why), (at, why, str(e.value))
    enc = np.frombuffer(so.g2_compress(outside), dtype=np.uint8).reshape(1, 96)
    assert ctx.g2_decompress(enc, check_subgroup=False)[0].tobytes() == po.g2_to_bytes(outside)
    # two bad points: the first is reported
    with pytest.raises(DpError) as e:
        ctx.g2_decompress(np.frombuffer(good[0] + cases[3][1] + cases[2][1], dtype=np.uint8).reshape(-1, 96))
    assert (e.value.index, e.value.why) == (1, 3)


# ------------------------------------------------------------------ dp_srs_check
N_SRS = 35


@pytest.fixture(scope="module")
def srs(orc, emul_lib):
    """a context over universal_setup(TAU) with N_SRS bases, its raw bases and its raw G2 pair"""
    c = Context(emul_lib, 0, 0, 1)
    universal_setup(c, torch, N_SRS - 1, 32, 256, tau=TAU, device="cpu")
    yield c, c.get_bases(0, N_SRS), c.srs_open_key(TAU)
    c.close()


def test_srs_check_accepts_the_setup_and_its_msms_match_the_oracle(orc, srs):
    c, bases, g2 = srs
    assert c.srs_check(g2, SEED)
    last = c.last_srs_check()
    rho = np.concatenate([scalar(r) for r in so.srs_check_scalars(SEED, N_SRS)]).reshape(-1, 4)
    assert np.array_equal(orc.normalize(last["A"]), orc.normalize(orc.msm(bases[:-1], rho)))
    assert np.array_equal(orc.normalize(last["B"]), orc.normalize(orc.msm(bases[1:], rho)))
    assert c.srs_check(g2)                                       # the library draws the seed
    assert not np.array_equal(c.last_srs_check()["A"], last["A"])
    assert np.array_equal(c.get_bases(0, N_SRS), bases)          # the context is as it was
    assert not c.srs_check(c.srs_open_key(TAU + 1), SEED)         # beta h of another tau
    with pytest.raises(ValueError):
        c.srs_check(g2, b"short")


def test_srs_check_refuses_a_spoiled_srs(orc, emul_lib, srs, ctx):
    _, bases, g2 = srs
    with pytest.raises(DpError) as e:
        ctx.srs_check(g2, SEED)
    assert e.value.code == DP_E_STATE
    other = orc.g1_mul(orc.g1_generator(), scalar(0xDEADBEEF))     # a subgroup point that is no power of tau
    spoiled = {}
    for at in (1, N_SRS // 2, N_SRS - 1):
        b = bases.copy()
        b[at] = other
        spoiled[f"replaced at {at}"] = b
    b = bases.copy()
    b[[10, 11]] = b[[11, 10]]
    spoiled["swapped"] = b
    spoiled["2g, 2 tau g, ..."] = np.stack([orc.g1_mul(p, scalar(2)) for p in bases])
    c = Context(emul_lib, 0, 0, 1)
    for name, b in spoiled.items():
        c.init(b, 32, 256)
        assert not c.srs_check(g2, SEED), name
    c.init(bases[:1], 32, 256)                                    # one base: only the generator test
    assert c.srs_check(g2, SEED)
    c.init(bases[1:2], 32, 256)
    assert not c.srs_check(g2, SEED)
    c.close()


# ------------------------------------------------------------------ files
def test_save_load_round_trip(emul_lib, srs, tmp_path):
    a, bases, _ = srs
    key = open_key(a, TAU)
    path = tmp_path / "srs.bin"
    assert save_srs(a, path, key) == N_SRS
    blob = path.read_bytes()
    assert len(blob) == 8 + 48 * N_SRS + 192 and struct.unpack("<Q", blob[:8])[0] == N_SRS
    assert blob[-192:] == so.g2_compress(po.G2_GEN) + so.g2_compress(po.g2_mul(po.G2_GEN, TAU))
    b = Context(emul_lib, 0, 0, 1)
    assert load_srs(b, path, 32, 256) == key
    assert np.array_equal(b.get_bases(0, N_SRS), bases)
    assert open_key_from_bytes(b, key.to_bytes()) == key and len(key.to_bytes()) == 240
    b.close()


def test_prover_and_verifier_in_separate_contexts_never_see_tau(orc, emul_lib, tmp_path):
    log_n, seed = 6, 18400
    n = 1 << log_n
    path = tmp_path / "srs.bin"
    # 1. the setup party
    a = Context(emul_lib, 0, 0, 1)
    universal_setup(a, torch, n + 2, n, 8 * n, tau=TAU, device="cpu")
    open_key_bytes = open_key(a, TAU).to_bytes()
    other_key_bytes = open_key(a, TAU + 1).to_bytes()
    save_srs(a, path, open_key(a, TAU))
    a.close()
    # 2. the prover: the SRS file only
    b = Context(emul_lib, 0, 0, 1)
    load_srs(b, path, n, 8 * n)
    pr, _, (_, _, witness, _) = tc.prover_from_circuit(orc, b, log_n, seed, "cpu")
    proof, pub = pr.prove_circuit(tc.witness_host(witness, "cpu"))
    vk = pr.verifying_key()
    vk_bytes, proof_bytes = vk.to_bytes(), proof.to_bytes()
    b.close()
    # 3. the verifier: three byte strings, a context that is never initialised
    c = Context(emul_lib, 0, 0, 1)
    assert len(vk_bytes) == 1064 and VerifyingKey.from_bytes(c, vk_bytes) == vk
    assert verify_bytes(c, vk_bytes, open_key_bytes, pub, proof_bytes)
    # 4. tampering
    ev0 = len(proof_bytes) - 10 * 32 - 8 - 8                      # the first of the ten evaluations
    flipped = bytearray(proof_bytes)
    flipped[ev0 + 8] ^= 1
    assert not verify_bytes(c, vk_bytes, open_key_bytes, pub, bytes(flipped))
    bad_vk = VerifyingKey(vk.n, vk.num_inputs, vk.k, vk.selector_comms[:3] + [tp.another_point(vk.selector_comms[3])] + vk.selector_comms[4:],
                          vk.sigma_comms)
    assert not verify_bytes(c, bad_vk.to_bytes(), open_key_bytes, pub, proof_bytes)
    assert not verify_bytes(c, vk_bytes, other_key_bytes, pub, proof_bytes)
    assert not verify_bytes(c, vk_bytes, open_key_bytes, [(pub[0] + 1) % R_MOD] + pub[1:], proof_bytes)
    assert uninitialised(c)
    c.close()


def test_malformed_files(orc, emul_lib, srs, tmp_path):
    a, bases, _ = srs
    key = open_key(a, TAU)
    good = tmp_path / "good.bin"
    save_srs(a, good, key)
    blob = good.read_bytes()

    def at(i):
        return 8 + 48 * i

    other = orc.g1_compress(orc.g1_mul(orc.g1_generator(), scalar(0xDEADBEEF)).reshape(1, 104)).tobytes()
    cases = {
        "truncated": (blob[:-1], "truncated"),
        "header only": (blob[:5], "truncated"),
        "trailing byte": (blob + b"\x00", "over-long"),
        "count + 1": (struct.pack("<Q", N_SRS + 1) + blob[8:], "truncated"),
        "count - 1": (struct.pack("<Q", N_SRS - 1) + blob[8:], "over-long"),
        "count 0": (struct.pack("<Q", 0) + blob[8:], "count"),
        "count 2^32 + 1": (struct.pack("<Q", (1 << 32) + 1) + blob[8:], "count"),
        "x >= p": (blob[:at(5)] + FQ_MOD.to_bytes(48, "little") + blob[at(6):], "point 5 rejected"),
        "outside the subgroup": (blob[:at(9)] + orc.g1_point_outside_subgroup().tobytes() + blob[at(10):], "point 9 rejected"),
        "h flags": (blob[:-97] + bytes([blob[-97] | 0xC0]) + blob[-96:], "h of the SRS file"),
        "one wrong point": (blob[:at(7)] + other + blob[at(8):], "consecutive powers"),
        "beta_h of another tau": (blob[:-96] + so.g2_compress(po.g2_mul(po.G2_GEN, TAU + 1)), "consecutive powers"),
    }
    c = Context(emul_lib, 0, 0, 1)
    for name, (data, word) in cases.items():
        path = tmp_path / "bad.bin"
        path.write_bytes(data)
        with pytest.raises(ValueError, match=word):
            load_srs(c, path, 32, 256)
            pytest.fail(name)
        if word == "consecutive powers":
            with pytest.raises(DpError):                          # the refused points are gone
                c.get_bases(0, 1)
        else:
            assert uninitialised(c), name
    # the wrong point passes when the consistency check is switched off: the subgroup check alone does not see it
    path.write_bytes(cases["one wrong point"][0])
    load_srs(c, path, 32, 256, check=False)
    assert not uninitialised(c)
    c.close()

    v = Context(emul_lib, 0, 0, 1)
    g = key.g
    vk = VerifyingKey(64, 3, [1, 2, 3, 4, 5], [g] * 13, [g] * 5)
    enc = vk.to_bytes()
    assert VerifyingKey.from_bytes(v, enc) == vk
    twelve = enc[:16 + 8 + 5 * 32] + struct.pack("<Q", 12) + enc[16 + 8 + 5 * 32 + 8 + 48:]
    bad_vks = {
        "12 selector commitments": twelve,
        "trailing": enc + b"\x00",
        "truncated": enc[:-1],
        "n not a power of two": struct.pack("<Q", 65) + enc[8:],
        "num_inputs > n": enc[:8] + struct.pack("<Q", 65) + enc[16:],
        "k >= r": enc[:24] + R_MOD.to_bytes(32, "little") + enc[56:],
        "a commitment with x >= p": enc[:-48] + FQ_MOD.to_bytes(48, "little"),
    }
    for name, data in bad_vks.items():
        with pytest.raises(ValueError):
            VerifyingKey.from_bytes(v, data)
            pytest.fail(name)
    ok_bytes = key.to_bytes()
    for data in (ok_bytes + b"\x00", ok_bytes[:-1], ok_bytes[:47] + b"\xc0" + ok_bytes[48:], ok_bytes[:-1] + bytes([ok_bytes[-1] | 0xC0])):
        with pytest.raises(ValueError):
            open_key_from_bytes(v, data)
    assert isinstance(open_key_from_bytes(v, ok_bytes), OpenKey) and uninitialised(v)
    v.close()
