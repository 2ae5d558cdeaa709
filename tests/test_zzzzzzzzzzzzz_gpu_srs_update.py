"""The setup ceremony on the GPU: dp_srs_update byte for byte against dp_srs_powers_of_tau of tau s at 2^20 + 3 points
(across the SRS_CHUNK boundary) and at 2^24 + 3, written once to host and once to device memory, and a three-contribution
ceremony through files at 2^16 + 3 points followed by a 2^16-gate proof that a party holding three byte strings accepts
(tests/test_srs_update.py on the emulator)."""
import os

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context
from distributed_plonk_b200.srs import ceremony_start, contribute, load_ceremony_srs, universal_setup
from distributed_plonk_b200.transcript import R_MOD
from distributed_plonk_b200.verifier import verify_bytes
from tests import test_proof as tp

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
DEV = "cpu" if DRY else "cuda"
TAU = 0x0F1E2D3C4B5A69788796A5B4C3D2E1F00112233445566778899AABBCCDDEEFF
S = 0x243F6A8885A308D313198A2E03707344A4093822299F31D0082EFA98EC4E6C89


def free_bytes() -> int:
    return (1 << 40) if DRY else torch.cuda.mem_get_info()[0]


@pytest.mark.parametrize("log_n", [20, 24])
def test_update_equals_the_srs_of_tau_s(gpu_lib, log_n):
    if DRY:
        log_n = {20: 6, 24: 7}[log_n]
    n = (1 << log_n) + 3
    # the context's bases and MSM table, the reference's 104-byte points, and three 48-byte outputs
    need = n * (104 + 3 * 48) + (24 << 30 if log_n == 24 else 0)
    if free_bytes() < need:
        pytest.skip(f"2^{log_n} + 3 points need about {need >> 30} GiB of device memory, {free_bytes() >> 30} GiB are free")
    c = Context(gpu_lib, 0, 0, 1)
    universal_setup(c, torch, n - 1, 1 << min(log_n, 20), 8 << min(log_n, 20), tau=TAU, device=DEV)
    g2 = c.srs_open_key(TAU)
    t = TAU * S % R_MOD
    ref = torch.empty((n, 104), dtype=torch.uint8, device=DEV)
    c.srs_powers_of_tau_into(t, n, ref.data_ptr())
    want = torch.empty((n, 48), dtype=torch.uint8, device=DEV)
    c._ck(c.lib.dp_g1_compress(c.h, ref.data_ptr(), n, want.data_ptr()))
    del ref
    dev = torch.empty((n, 48), dtype=torch.uint8, device=DEV)
    _, g2_dev = c.srs_update(g2, n, S, out48=dev.data_ptr())
    assert torch.equal(dev, want)
    del dev
    host, g2_host = c.srs_update(g2, n, S)
    assert np.array_equal(host, want.cpu().numpy())
    assert np.array_equal(g2_dev, g2_host)
    assert np.array_equal(g2_host[0], c.srs_open_key(S)[1]) and np.array_equal(g2_host[1], c.srs_open_key(t)[1])
    del want, host
    c.close()
    if not DRY:
        torch.cuda.empty_cache()


def test_three_contributions_then_prove_and_verify_at_2p16(orc, gpu_lib, tmp_path):
    log_n = 6 if DRY else 16
    n, seed = 1 << log_n, 20200
    paths = [tmp_path / f"srs{j}.bin" for j in range(4)]
    ceremony_start(paths[0], n + 3)
    receipts = []
    for j in range(3):
        c = Context(gpu_lib, 0, 0, 1)
        receipts.append(contribute(c, paths[j], paths[j + 1], n, 8 * n))
        c.close()
    b = Context(gpu_lib, 0, 0, 1)
    key = load_ceremony_srs(b, paths[3], receipts, n, 8 * n)
    with pytest.raises(ValueError, match="does not start"):
        load_ceremony_srs(b, paths[3], receipts[1:], n, 8 * n)
    key = load_ceremony_srs(b, paths[3], receipts, n, 8 * n)
    pr, _, (_, _, witness, _) = tp.tc.prover_from_circuit(orc, b, log_n, seed, DEV)
    proof, pub = pr.prove_circuit(tp.tc.witness_host(witness, DEV))
    vk_bytes, proof_bytes = pr.verifying_key().to_bytes(), proof.to_bytes()
    del pr
    b.close()
    v = Context(gpu_lib, 0, 0, 1)                                    # never initialised, never sees a secret
    assert verify_bytes(v, vk_bytes, key.to_bytes(), pub, proof_bytes)
    flipped = bytearray(proof_bytes)
    flipped[len(proof_bytes) - 10 * 32 - 8] ^= 1                     # inside the first evaluation
    assert not verify_bytes(v, vk_bytes, key.to_bytes(), pub, bytes(flipped))
    v.close()
