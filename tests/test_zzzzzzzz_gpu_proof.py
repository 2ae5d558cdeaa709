"""ResidentProver.prove_circuit on the GPU, over SRSs with a known trapdoor at 2^12 and 2^16 gates: proofs blinded with
scalars the library draws verify in both round-3 layouts; prove_circuit equals prove_witness on the challenges it
derived; tampered proofs are rejected (tests/test_proof.py on the emulator)."""
import os

import pytest

from tests import test_proof as tp

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
DEV = "cpu" if DRY else "cuda"


@pytest.mark.parametrize("log_n", [12, 16])
@pytest.mark.parametrize("quotient", ["whole", "sliced"])
def test_prove_circuit_verifies(orc, gpu_lib, quotient, log_n):
    if DRY:
        log_n = 6 if log_n == 12 else 7
    seed = 12000 + log_n
    c, pr, witness, tau = tp.setup(orc, gpu_lib, log_n, seed, DEV, quotient)
    vk = pr.verifying_key()
    wit = tp.tc.witness_host(witness, DEV)
    (p1, pub1), (p2, pub2) = pr.prove_circuit(wit), pr.prove_circuit(wit)       # blinded, library-drawn scalars
    assert p1 != p2
    assert tp.pv.verify(orc, vk, pub1, p1, tau) and tp.pv.verify(orc, vk, pub2, p2, tau), f"2^{log_n}, {quotient}"
    tp.check_equals_prove_witness(orc, pr, witness, tau, DEV, seed)
    c.close()


def test_tampered_proofs_are_rejected_at_2p12(orc, gpu_lib):
    log_n = 6 if DRY else 12
    c, pr, witness, tau = tp.setup(orc, gpu_lib, log_n, 12100, DEV)
    tp.check_rejections(orc, pr, witness, tau, DEV, 12100, every=False)
    c.close()
