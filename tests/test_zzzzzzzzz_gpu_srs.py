"""dp_srs_powers_of_tau on the GPU: byte equality with the oracle's [tau^i] G at 2^12 + 3 and 2^16 + 3 points; at
2^22 + 3 every point at once through the KZG identity commit(p) = p(tau) G plus 64 sampled points (the ends, both sides of
every launch chunk, random ones); and universal_setup -> load_circuit -> prove_circuit at 2^16 gates, in both round-3
layouts, accepted by the verifier, with tampered proofs rejected (tests/test_srs.py on the emulator)."""
import os

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context
from distributed_plonk_b200.srs import universal_setup
from distributed_plonk_b200.transcript import R_MOD
from tests import test_proof as tp

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
DEV = "cpu" if DRY else "cuda"
CHUNK = 1 << 20                 # SRS_CHUNK (csrc/srs.cuh): points per kernel launch
TAU = 0x5EED5EED0123456789ABCDEF0FEDCBA9876543210C0FFEE1234ABCD5678EF01


def u256(v: int) -> np.ndarray:
    return np.frombuffer(int(v).to_bytes(32, "little"), dtype=np.uint64).copy()


def sample_indices(n: int, seed: int, count: int = 64) -> list:
    idx = {0, 1, n - 1}
    for b in range(CHUNK, n, CHUNK):
        idx |= {b - 1, b, b + 1}
    rng = np.random.default_rng(seed)
    while len(idx) < count:
        idx.add(int(rng.integers(0, n)))
    return sorted(i for i in idx if 0 <= i < n)


def check_device_srs(orc, ctx, tau: int, n: int, device: str, seed: int) -> dict:
    """n points into a device buffer, dp_init from it (device to device), then: the library's commitment of a random
    polynomial with n coefficients equals p(tau) G (every point takes part), and the sampled points equal tau^i G."""
    buf = torch.empty((n, 104), dtype=torch.uint8, device=device)
    ctx.srs_powers_of_tau_into(tau, n, buf.data_ptr())
    idx = sample_indices(n, seed)
    rows = buf[torch.as_tensor(idx, device=device)].cpu().numpy()
    ctx.init_ptr(buf.data_ptr(), n, 1 << 4, 1 << 7)
    del buf
    if device != "cpu":
        torch.cuda.empty_cache()
    gen = orc.g1_generator()
    p = orc.gen_fr(seed, n)
    p_tau = orc.into_repr(orc.poly_eval(p, orc.from_repr(u256(tau)[None])[0])[None])[0]
    kzg = np.array_equal(orc.normalize(ctx.commit(p)), orc.g1_mul(gen, p_tau))
    pts = all(np.array_equal(rows[j], orc.g1_mul(gen, u256(pow(tau, i, R_MOD)))) for j, i in enumerate(idx))
    return {"kzg_identity": bool(kzg), "sampled_points": bool(pts), "n_sampled": len(idx)}


@pytest.mark.parametrize("log_n", [12, 16])
def test_matches_the_oracle(orc, gpu_lib, log_n):
    n = (1 << (log_n - 6 if DRY else log_n)) + 3
    c = Context(gpu_lib, 0, 0, 1)
    ref = orc.gen_srs(u256(TAU), n)
    assert np.array_equal(c.srs_powers_of_tau(TAU, n), ref), f"n = {n}"
    c.close()


def test_kzg_identity_and_sampled_points_at_2p22(orc, gpu_lib):
    n = (1 << (8 if DRY else 22)) + 3
    c = Context(gpu_lib, 0, 0, 1)
    got = check_device_srs(orc, c, TAU, n, DEV, 14000)
    assert got["kzg_identity"] and got["sampled_points"], got
    c.close()


@pytest.mark.parametrize("quotient", ["whole", "sliced"])
def test_universal_setup_proofs_verify_at_2p16(orc, gpu_lib, quotient):
    log_n = 6 if DRY else 16
    n, seed = 1 << log_n, 14100
    c = Context(gpu_lib, 0, 0, 1)
    assert universal_setup(c, torch, n + 2, n, 8 * n, tau=TAU, device=DEV) == TAU
    pr, vk, (_, _, witness, _) = tp.tc.prover_from_circuit(orc, c, log_n, seed, DEV, quotient)
    proof, pub = pr.prove_circuit(tp.tc.witness_host(witness, DEV))             # blinded by the library
    assert tp.pv.verify(orc, pr.verifying_key(), pub, proof, TAU), f"2^{log_n}, {quotient}"
    if quotient == "whole":
        tp.check_rejections(orc, pr, witness, TAU, DEV, seed, every=False)
    c.close()
