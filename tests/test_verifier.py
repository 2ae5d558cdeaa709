"""verifier.verify / batch_verify / proof_from_bytes on the kernel-logic emulator, over universal_setup(TAU) and
open_key(TAU): proofs of tests/test_circuit.py's satisfied circuits (log_n = 6 and 7, blinded) are accepted without the
trapdoor; on every tampering tests/test_proof.check_rejections builds the pairing verifier and the trapdoor check
(tests/plonk_verifier.verify) agree - both reject; a wrong open key is rejected; the proof bytes decode back and every
malformed encoding is a ValueError; batch_verify accepts proofs of two circuits and rejects a corrupted one at every
position."""
import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context
from distributed_plonk_b200.proof import FQ_MOD, Proof
from distributed_plonk_b200.srs import open_key, universal_setup
from distributed_plonk_b200.transcript import R_MOD
from distributed_plonk_b200.verifier import batch_verify, proof_from_bytes, verify
from tests import plonk_verifier as pv
from tests import test_circuit as tc
from tests import test_proof as tp

TAU = 0x1D2C3B4A5968778695A4B3C2D1E0F0E1D2C3B4A5968778695A4B3C2D1E0F1234


class Setup:
    """a context over universal_setup(TAU), a prover of one satisfied circuit, its verifying key and the open key"""

    def __init__(self, orc, lib, log_n, seed):
        n = 1 << log_n
        self.ctx = Context(lib, 0, 0, 1)
        universal_setup(self.ctx, torch, n + 2, n, 8 * n, tau=TAU, device="cpu")
        self.pr, _, (_, _, self.witness, _) = tc.prover_from_circuit(orc, self.ctx, log_n, seed, "cpu")
        self.vk = self.pr.verifying_key()
        self.seed = seed

    def prove(self):
        return self.pr.prove_circuit(tc.witness_host(self.witness, "cpu"))


@pytest.fixture(scope="module")
def s6(orc, emul_lib):
    s = Setup(orc, emul_lib, 6, 15000)
    yield s
    s.ctx.close()


@pytest.fixture(scope="module")
def s7(orc, emul_lib):
    s = Setup(orc, emul_lib, 7, 15100)
    yield s
    s.ctx.close()


@pytest.fixture(scope="module")
def ok(s6):
    return open_key(s6.ctx, TAU)


def test_open_key_is_the_setup_of_tau(s6, ok):
    from tests import pairing_oracle as po
    assert ok.h == po.G2_GEN and ok.beta_h == po.g2_mul(po.G2_GEN, TAU)
    assert ok.g == pv.B.G1_GEN


def test_verify_accepts_and_a_wrong_open_key_rejects(orc, s6, ok):
    proof, pub = s6.prove()
    assert pv.verify(orc, s6.vk, pub, proof, TAU)
    assert verify(s6.ctx, s6.vk, ok, pub, proof)
    timings = {}
    assert verify(s6.ctx, s6.vk, ok, pub, proof, timings)
    assert set(timings) == {"transcript_scalars_ms", "msm_ms", "pairing_ms"}
    assert not verify(s6.ctx, s6.vk, open_key(s6.ctx, TAU + 1), pub, proof)


def test_agrees_with_the_trapdoor_check_on_every_tampering(orc, s6, ok, monkeypatch):
    """check_rejections asserts that tests/plonk_verifier.verify rejects each tampered proof; wrapped, every one of its
    calls is also put to the pairing verifier, which must give the same answer"""
    trapdoor = pv.verify
    calls = []

    def both(orc_, vk, pub, proof, tau):
        want = trapdoor(orc_, vk, pub, proof, tau)
        got = verify(s6.ctx, vk, ok, pub, proof)
        assert got == want, f"pairing verifier {got}, trapdoor check {want} (call {len(calls)})"
        calls.append(want)
        return want

    monkeypatch.setattr(pv, "verify", both)
    tp.check_rejections(orc, s6.pr, s6.witness, TAU, "cpu", s6.seed + 1)
    assert calls[0] is True and calls.count(False) == len(calls) - 1 and len(calls) >= 27


def test_argument_errors(s6, ok):
    proof, pub = s6.prove()
    with pytest.raises(ValueError):
        verify(s6.ctx, s6.vk, ok, pub[:-1], proof)
    with pytest.raises(ValueError):
        verify(s6.ctx, s6.vk, ok, pub + [1], proof)
    with pytest.raises(ValueError):
        verify(s6.ctx, s6.vk, ok, [R_MOD] + pub[1:], proof)
    bad = Proof(proof.wires_poly_comms[:4], proof.prod_perm_poly_comm, proof.split_quot_poly_comms, proof.opening_proof,
                proof.shifted_opening_proof, proof.wires_evals, proof.wire_sigma_evals, proof.perm_next_eval)
    with pytest.raises(ValueError):
        verify(s6.ctx, s6.vk, ok, pub, bad)
    with pytest.raises(ValueError):
        batch_verify(s6.ctx, ok, [])
    assert verify(s6.ctx, s6.vk, ok, [(pub[0] + 1) % R_MOD] + pub[1:], proof) is False


def test_proof_bytes_round_trip_and_malformed_encodings(orc, s6, ok):
    proof, pub = s6.prove()
    b = proof.to_bytes()
    back = proof_from_bytes(s6.ctx, b)
    assert back == proof
    assert verify(s6.ctx, s6.vk, ok, pub, back)

    def at(i):                        # offset of commitment i (0..12) in the encoding
        return 8 + 48 * i + (8 if i >= 6 else 0)

    def patched(off, new):
        return b[:off] + new + b[off + len(new):]

    fr0 = 8 + 5 * 48 + 48 + 8 + 5 * 48 + 2 * 48 + 8     # first evaluation
    not_sq = next(x for x in range(1, 100) if pow((x ** 3 + 4) % FQ_MOD, (FQ_MOD - 1) // 2, FQ_MOD) != 1)
    cases = {
        "truncated": b[:-1],
        "empty": b"",
        "trailing": b + b"\x00",
        "wires length 4": patched(0, (4).to_bytes(8, "little")),
        "quotient length 6": patched(8 + 6 * 48, (6).to_bytes(8, "little")),
        "wire evals length 4": patched(fr0 - 8, (4).to_bytes(8, "little")),
        "sigma evals length 5": patched(fr0 + 5 * 32, (5).to_bytes(8, "little")),
        "x >= p": patched(at(3), FQ_MOD.to_bytes(48, "little")),
        "both flags": patched(at(6) + 47, bytes([b[at(6) + 47] | 0xC0])),
        "no such point": patched(at(12), not_sq.to_bytes(48, "little")),
        "outside the subgroup": patched(at(11), orc.g1_point_outside_subgroup().tobytes()),
        "evaluation = r": patched(fr0 + 32 * 2, R_MOD.to_bytes(32, "little")),
        "last evaluation >= r": patched(len(b) - 32, ((1 << 256) - 1).to_bytes(32, "little")),
    }
    for name, enc in cases.items():
        with pytest.raises(ValueError):
            proof_from_bytes(s6.ctx, enc)
            pytest.fail(name)


def test_batch_verify_two_circuits(s6, s7, ok):
    items = []
    for s in (s6, s7, s6, s7):
        proof, pub = s.prove()
        items.append((s.vk, pub, proof))
    assert batch_verify(s6.ctx, ok, items)
    assert batch_verify(s6.ctx, ok, items[:1]) == verify(s6.ctx, items[0][0], ok, items[0][1], items[0][2]) is True
    for j in range(len(items)):
        vk, pub, proof = items[j]
        bad = Proof(proof.wires_poly_comms, proof.prod_perm_poly_comm, proof.split_quot_poly_comms, proof.opening_proof,
                    proof.shifted_opening_proof, proof.wires_evals, proof.wire_sigma_evals, (proof.perm_next_eval + 1) % R_MOD)
        corrupted = items[:j] + [(vk, pub, bad)] + items[j + 1:]
        assert not batch_verify(s6.ctx, ok, corrupted), f"accepted a batch with proof {j} corrupted"
        assert batch_verify(s6.ctx, ok, [(vk, pub, bad)]) == verify(s6.ctx, vk, ok, pub, bad) is False
    # a proof of one circuit checked against the other circuit's key
    assert not batch_verify(s6.ctx, ok, [items[0], (s7.vk, items[0][1], items[0][2])])
