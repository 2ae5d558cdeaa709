"""The verifier on the GPU: dp_multi_pairing and dp_srs_open_key equal the pairing oracle on two pairs; dp_msm_points at
2^16 points equals the oracle's MSM; universal_setup -> load_circuit -> prove_circuit at 2^16 gates, in both round-3
layouts, accepted by verify without the trapdoor and rejected when tampered; a batch_verify of 8 proofs
(tests/test_pairing.py and tests/test_verifier.py on the emulator)."""
import os
import random

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context
from distributed_plonk_b200.proof import Proof
from distributed_plonk_b200.srs import open_key, universal_setup
from distributed_plonk_b200.transcript import R_MOD
from distributed_plonk_b200.verifier import batch_verify, proof_from_bytes, verify
from oracle.py import bls12_381 as B
from tests import pairing_oracle as po
from tests import test_proof as tp

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
DEV = "cpu" if DRY else "cuda"
TAU = 0x6A09E667F3BCC908B2FB1366EA957D3E3ADEC17512775099DA2F590B0667322A


def test_pairing_and_open_key_match_the_oracle(gpu_lib):
    rng = random.Random(17000)
    c = Context(gpu_lib, 0, 0, 1)
    pairs = [(B.g1_mul(B.G1_GEN, rng.randrange(1, R_MOD)), po.g2_mul(po.G2_GEN, rng.randrange(1, R_MOD))) for _ in range(2)]
    g1 = np.frombuffer(b"".join(B.g1_affine_to_bytes(p) for p, _ in pairs), dtype=np.uint8).reshape(2, 104)
    g2 = np.frombuffer(b"".join(po.g2_to_bytes(q) for _, q in pairs), dtype=np.uint8).reshape(2, 200)
    assert c.multi_pairing(g1, g2).tobytes() == po.to_tower_bytes(po.multi_pairing(pairs))
    ok = c.srs_open_key(TAU)
    assert ok[0].tobytes() == po.g2_to_bytes(po.G2_GEN) and ok[1].tobytes() == po.g2_to_bytes(po.g2_mul(po.G2_GEN, TAU))
    c.close()


def test_msm_points_at_2p16(orc, gpu_lib):
    n = 1 << (8 if DRY else 16)
    c = Context(gpu_lib, 0, 0, 1)                   # no dp_init
    bases = orc.gen_bases(17100, n, n, True)
    sc = orc.gen_fr(17101, n, False)
    sc[5] = 0
    assert np.array_equal(orc.normalize(c.msm_points(bases, sc)), orc.normalize(orc.msm(bases, sc)))
    c.close()


@pytest.mark.parametrize("quotient", ["whole", "sliced"])
def test_proofs_at_2p16_verify_without_the_trapdoor(orc, gpu_lib, quotient):
    log_n = 6 if DRY else 16
    n, seed = 1 << log_n, 17200
    c = Context(gpu_lib, 0, 0, 1)
    universal_setup(c, torch, n + 2, n, 8 * n, tau=TAU, device=DEV)
    ok = open_key(c, TAU)
    pr, vk, (_, _, witness, _) = tp.tc.prover_from_circuit(orc, c, log_n, seed, DEV, quotient)
    wit = tp.tc.witness_host(witness, DEV)
    proof, pub = pr.prove_circuit(wit)
    assert verify(c, pr.verifying_key(), ok, pub, proof), f"2^{log_n}, {quotient}"
    assert verify(c, pr.verifying_key(), ok, pub, proof_from_bytes(c, proof.to_bytes()))
    com, ev = proof.commitments(), proof.evaluations()
    ev[3] = (ev[3] + 1) % R_MOD
    assert not verify(c, pr.verifying_key(), ok, pub, Proof(com[0:5], com[5], com[6:11], com[11], com[12], ev[0:5], ev[5:9], ev[9]))
    com = proof.commitments()
    com[8] = tp.another_point(com[8])
    assert not verify(c, pr.verifying_key(), ok, pub, Proof(com[0:5], com[5], com[6:11], com[11], com[12], *[proof.evaluations()[i:j] for i, j in ((0, 5), (5, 9))], proof.perm_next_eval))
    assert not verify(c, pr.verifying_key(), ok, [(pub[0] + 1) % R_MOD] + pub[1:], proof)
    if quotient == "whole":
        items = []
        for _ in range(8):
            p, pb = pr.prove_circuit(wit)
            items.append((pr.verifying_key(), pb, p))
        assert batch_verify(c, ok, items)
        vk_, pb, p = items[5]
        bad = Proof(p.wires_poly_comms, p.prod_perm_poly_comm, p.split_quot_poly_comms, p.opening_proof, p.shifted_opening_proof,
                    p.wires_evals, p.wire_sigma_evals, (p.perm_next_eval + 1) % R_MOD)
        assert not batch_verify(c, ok, items[:5] + [(vk_, pb, bad)] + items[6:])
    c.close()
