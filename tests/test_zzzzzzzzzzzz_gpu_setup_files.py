"""Setup files on the GPU: a setup party, a prover that loads the SRS file and a verifier that holds three byte strings, in
separate contexts, at 2^16 gates, with the tampered variants; dp_g1_compress at 2^20 points against the oracle and back
through dp_g1_decompress; the G2 decoder's rejection codes; and one save / load / check of a 2^22 + 3-point SRS, also with
one point replaced (tests/test_setup_files.py on the emulator)."""
import os
import random

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import DP_E_STATE, Context, DpError
from distributed_plonk_b200.proof import VerifyingKey
from distributed_plonk_b200.srs import load_srs, open_key, save_srs, universal_setup
from distributed_plonk_b200.transcript import R_MOD
from distributed_plonk_b200.verifier import verify_bytes
from tests import pairing_oracle as po
from tests import setup_files_oracle as so
from tests import test_proof as tp

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
DEV = "cpu" if DRY else "cuda"
TAU = 0x1F83D9ABFB41BD6B5BE0CD19137E2179A54FF53A5F1D36F1510E527FADE682D1


def test_separate_setup_prover_and_verifier_at_2p16(orc, gpu_lib, tmp_path):
    log_n = 6 if DRY else 16
    n, seed = 1 << log_n, 19000
    path = tmp_path / "srs.bin"
    a = Context(gpu_lib, 0, 0, 1)
    universal_setup(a, torch, n + 2, n, 8 * n, tau=TAU, device=DEV)
    key = open_key(a, TAU)
    other_key_bytes = open_key(a, TAU + 1).to_bytes()
    assert save_srs(a, path, key) == n + 3
    bases = a.get_bases(0, n + 3)
    a.close()

    b = Context(gpu_lib, 0, 0, 1)
    assert load_srs(b, path, n, 8 * n) == key
    assert np.array_equal(b.get_bases(0, n + 3), bases)
    pr, _, (_, _, witness, _) = tp.tc.prover_from_circuit(orc, b, log_n, seed, DEV)
    proof, pub = pr.prove_circuit(tp.tc.witness_host(witness, DEV))
    vk = pr.verifying_key()
    vk_bytes, proof_bytes = vk.to_bytes(), proof.to_bytes()
    del pr
    b.close()

    c = Context(gpu_lib, 0, 0, 1)                                    # never initialised, never sees tau
    assert VerifyingKey.from_bytes(c, vk_bytes) == vk
    assert verify_bytes(c, vk_bytes, key.to_bytes(), pub, proof_bytes)
    flipped = bytearray(proof_bytes)
    flipped[len(proof_bytes) - 10 * 32 - 8] ^= 1                     # inside the first evaluation
    assert not verify_bytes(c, vk_bytes, key.to_bytes(), pub, bytes(flipped))
    bad_vk = VerifyingKey(vk.n, vk.num_inputs, vk.k, vk.selector_comms, vk.sigma_comms[:2] + [tp.another_point(vk.sigma_comms[2])] + vk.sigma_comms[3:])
    assert not verify_bytes(c, bad_vk.to_bytes(), key.to_bytes(), pub, proof_bytes)
    assert not verify_bytes(c, vk_bytes, other_key_bytes, pub, proof_bytes)
    assert not verify_bytes(c, vk_bytes, key.to_bytes(), [(pub[0] + 1) % R_MOD] + pub[1:], proof_bytes)
    with pytest.raises(DpError) as e:
        c.get_bases(0, 0)
    assert e.value.code == DP_E_STATE
    c.close()


def test_g1_compress_at_2p20(orc, gpu_lib):
    n = 1 << (8 if DRY else 20)
    c = Context(gpu_lib, 0, 0, 1)
    bases = c.gen_bases(19100, n)
    comp = c.g1_compress(bases)
    rng = random.Random(19101)
    idx = sorted({0, n - 1, *(rng.randrange(n) for _ in range(64))})
    assert np.array_equal(comp[idx], orc.g1_compress(bases[idx]))
    assert {int(v) >> 7 for v in comp[:, 47]} == {0, 1}
    assert np.array_equal(c.g1_decompress(comp, check_subgroup=False), bases)
    c.close()


def test_g2_round_trip_and_rejection_codes(gpu_lib):
    rng = random.Random(19200)
    c = Context(gpu_lib, 0, 0, 1)
    pts = [po.G2_GEN, None] + [po.g2_mul(po.G2_GEN, rng.randrange(1, R_MOD)) for _ in range(4)]
    raw = np.frombuffer(b"".join(po.g2_to_bytes(q) for q in pts), dtype=np.uint8).reshape(-1, 200)
    comp = c.g2_compress(raw)
    assert [v.tobytes() for v in comp] == [so.g2_compress(q) for q in pts]
    assert np.array_equal(c.g2_decompress(comp), raw)
    good = so.g2_compress(po.G2_GEN)
    not_square = next((k, 0) for k in range(1, 100) if so.f2_sqrt(po.f2_add(po.f2_mul(po.f2_mul((k, 0), (k, 0)), (k, 0)), po.G2_B)) is None)
    cases = [(1, po.P.to_bytes(48, "little") + good[48:]), (2, good[:95] + bytes([good[95] | 0xC0])),
             (3, so.g2_compress((not_square, (0, 1)))), (4, so.g2_compress(so.twist_point_outside_subgroup()))]
    for at, (why, enc) in enumerate(cases):
        batch = [good] * at + [enc] + [good] * (4 - at)
        with pytest.raises(DpError) as e:
            c.g2_decompress(np.frombuffer(b"".join(batch), dtype=np.uint8).reshape(-1, 96))
        assert (e.value.index, e.value.why) == (at, why)
    c.close()


def test_save_load_check_at_2p22_plus_3(orc, gpu_lib, tmp_path):
    log_n = 5 if DRY else 22
    n = (1 << log_n) + 3
    path = tmp_path / "srs.bin"
    a = Context(gpu_lib, 0, 0, 1)
    universal_setup(a, torch, n - 1, 1 << log_n, 8 << log_n, tau=TAU, device=DEV)
    key = open_key(a, TAU)
    assert a.srs_check(a.srs_open_key(TAU), bytes(32))
    assert save_srs(a, path, key) == n and os.path.getsize(path) == 8 + 48 * n + 192
    idx = [0, 1, n // 2, n - 1]
    want = [a.get_bases(i, 1) for i in idx]
    a.close()
    b = Context(gpu_lib, 0, 0, 1)
    assert load_srs(b, path, 1 << log_n, 8 << log_n) == key
    assert all(np.array_equal(b.get_bases(i, 1), w) for i, w in zip(idx, want))
    # one point in the middle replaced by another point of the subgroup: only the consistency check sees it
    with open(path, "r+b") as f:
        f.seek(8 + 48 * (n // 2))
        f.write(orc.g1_compress(orc.g1_generator().reshape(1, 104)).tobytes())
    with pytest.raises(ValueError, match="consecutive powers"):
        load_srs(b, path, 1 << log_n, 8 << log_n)
    b.close()
