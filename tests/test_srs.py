"""dp_srs_powers_of_tau and srs.universal_setup on the kernel-logic emulator: the points equal the oracle's [tau^i] G
byte for byte, also across the 128-point normalisation blocks and for the degenerate tau = 1 and r - 1; the argument
errors; output to host and device memory; a context's SRS is left alone; and a proof over the generated SRS equals the
proof over the oracle's and verifies."""
import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context, DpError
from distributed_plonk_b200.proof import fr_to_int
from distributed_plonk_b200.resident import N_BLIND
from distributed_plonk_b200.srs import universal_setup
from distributed_plonk_b200.transcript import R_MOD
from tests import plonk_verifier as pv
from tests import test_circuit as tc

TAU = 0x2F1D4C3B5A69788796A5B4C3D2E1F00112233445566778899AABBCCDDEEFF0


def oracle_srs(orc, tau: int, n: int) -> np.ndarray:
    return orc.gen_srs(np.frombuffer(tau.to_bytes(32, "little"), dtype=np.uint64), n)


@pytest.fixture(scope="module")
def ctx(emul_lib):
    c = Context(emul_lib, 0, 0, 1)
    yield c
    c.close()


@pytest.mark.parametrize("n", [1, 2, 3, 100, 300])      # 300: three normalisation blocks of 128, the last one partial
def test_matches_the_oracle(orc, ctx, n):
    assert np.array_equal(ctx.srs_powers_of_tau(TAU, n), oracle_srs(orc, TAU, n))


def test_tau_one_two_and_minus_one(orc, ctx):
    gen = orc.g1_generator()
    ones = ctx.srs_powers_of_tau(1, 150)                  # every denominator of a block is the same
    assert all(np.array_equal(p, gen) for p in ones)
    neg_gen = orc.g1_mul(gen, np.frombuffer((R_MOD - 1).to_bytes(32, "little"), dtype=np.uint64))
    alt = ctx.srs_powers_of_tau(R_MOD - 1, 10)
    for i, p in enumerate(alt):
        assert np.array_equal(p, gen if i % 2 == 0 else neg_gen), i
    assert np.array_equal(ctx.srs_powers_of_tau(2, 140), oracle_srs(orc, 2, 140))


def test_argument_errors(emul_lib, ctx):
    out = np.zeros((4, 104), dtype=np.uint8)
    tau = TAU.to_bytes(32, "little")
    for bad, word in ((0, "zero"), (R_MOD, "canonical"), (R_MOD + 5, "canonical"), ((1 << 256) - 1, "canonical")):
        with pytest.raises(DpError) as e:
            ctx.srs_powers_of_tau(bad, 4)
        assert e.value.code == -1 and word in str(e.value)
    for args in ((None, 4, out.ctypes.data), (tau, 4, None), (None, 4, None)):
        assert emul_lib.dp_srs_powers_of_tau(ctx.h, *args) == -1
    assert emul_lib.dp_srs_powers_of_tau(None, tau, 4, out.ctypes.data) == -1
    assert emul_lib.dp_srs_powers_of_tau(ctx.h, None, 0, None) == 0        # n = 0: nothing read, nothing written
    assert ctx.srs_powers_of_tau(TAU, 0).shape == (0, 104)
    with pytest.raises(ValueError):
        ctx.srs_powers_of_tau(-1, 4)
    assert not out.any()


def test_host_and_device_output(orc, ctx):
    """on the emulator device memory is host memory: a torch buffer stands for both, at an offset, the bytes around it
    untouched"""
    n = 70
    buf = torch.full((n + 2, 104), 0xAB, dtype=torch.uint8)
    ctx.srs_powers_of_tau_into(TAU, n, buf[1:].data_ptr())
    got = buf.numpy()
    assert np.array_equal(got[1:n + 1], oracle_srs(orc, TAU, n))
    assert (got[0] == 0xAB).all() and (got[n + 1] == 0xAB).all()


def test_leaves_an_initialised_context_alone(orc, emul_lib):
    """a call after dp_init leaves the SRS and the commitments over it as they were; the fixed-base table the first call
    builds is dropped by dp_init and rebuilt by the next call, with the same points"""
    n = 64
    bases = orc.gen_bases(5, n, 64, True)
    c = Context(emul_lib, 0, 0, 1)
    first = c.srs_powers_of_tau(TAU, 130)
    c.init(bases, 16, 128)
    sc = orc.gen_fr(6, n)
    before = c.commit(sc)
    assert np.array_equal(c.srs_powers_of_tau(TAU, 130), first)
    assert np.array_equal(first, oracle_srs(orc, TAU, 130))
    assert np.array_equal(c.commit(sc), before)
    assert np.array_equal(c.get_bases(0, n), bases)
    c.close()


def test_universal_setup_proof_equals_the_oracle_srs_proof_and_verifies(orc, emul_lib):
    log_n, seed = 6, 13000
    n = 1 << log_n
    blind = orc.gen_fr(seed + 1, N_BLIND)
    proofs = []
    for source in ("library", "oracle"):
        c = Context(emul_lib, 0, 0, 1)
        if source == "library":
            assert universal_setup(c, torch, n + 2, n, 8 * n, tau=TAU, device="cpu") == TAU
            assert np.array_equal(c.get_bases(0, n + 3), oracle_srs(orc, TAU, n + 3))
        else:
            c.init(oracle_srs(orc, TAU, n + 3), n, 8 * n)
        pr, vk, (_, _, witness, _) = tc.prover_from_circuit(orc, c, log_n, seed, "cpu")
        proof, pub = pr.prove_circuit(tc.witness_host(witness, "cpu"), blind=blind)
        assert pub == [fr_to_int(v) for v in witness[1:4]]
        assert pv.verify(orc, pr.verifying_key(), pub, proof, TAU), f"verifier rejects the proof over the {source} SRS"
        proofs.append(proof.to_bytes())
        c.close()
    assert proofs[0] == proofs[1]


def test_universal_setup_draws_tau(orc, emul_lib):
    c = Context(emul_lib, 0, 0, 1)
    tau = universal_setup(c, torch, 3, 4, 8, device="cpu")
    assert 0 < tau < R_MOD
    assert np.array_equal(c.get_bases(0, 4), oracle_srs(orc, tau, 4))
    c.close()
