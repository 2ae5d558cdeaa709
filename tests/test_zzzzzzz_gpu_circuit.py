"""Circuit preprocessing and the witness gather on the GPU: the wire permutation at 5 x 2^20 and 5 x 2^22 slots against the
stable-argsort restatement for every variable distribution of tests/test_circuit.py; identity / sigma evaluations, the
gather and load_circuit against the oracle at 2^16; the verifying-key commitments at 2^20 against (sum c_i t_i) G over a
synthetic SRS with known discrete logs t_i; prove_witness against prove in both round-3 layouts and the quotient degree of
a satisfied circuit built from variables."""
import os

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context
from distributed_plonk_b200.resident import N_SEL, N_WIRE, NumpyField, ResidentProver, bench_circuit_inputs
from tests import test_circuit as tc

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
DEV = "cpu" if DRY else "cuda"


class DevBuf:
    def __init__(self, a: np.ndarray):
        self.t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(DEV)
        self.dtype = a.dtype
        self.ptr = self.t.data_ptr()


def to_host(b: DevBuf) -> np.ndarray:
    if not DRY:
        torch.cuda.synchronize()
    return b.t.cpu().numpy().view(b.dtype)


def host(t: torch.Tensor) -> np.ndarray:
    if not DRY:
        torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("log_n", [20, 22])
def test_wire_permutation_at_scale(gpu_lib, log_n):
    if DRY:
        log_n = 10 if log_n == 20 else 11
    n = 1 << log_n
    c = Context(gpu_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, 8 * n)
    maps = tc.variable_maps(N_WIRE, n, 9700 + log_n)
    maps["bench padding"] = (bench_circuit_inputs(log_n, 4 * n), 4 * n)
    for name, (wv, num_vars) in maps.items():
        got = tc.device_succ(c, wv, N_WIRE, n, num_vars, DevBuf, to_host)
        assert np.array_equal(got, tc.succ_argsort(wv)), f"wire permutation, {name}, 5 x 2^{log_n} slots"
    c.close()


def test_perm_evals_and_gather_at_2p16(orc, gpu_lib):
    log_n = 8 if DRY else 16
    n = 1 << log_n
    c = Context(gpu_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, 8 * n)
    k = orc.gen_fr(9800, N_WIRE)
    wv, num_vars = tc.variable_maps(N_WIRE, n, 9801)["padded"]
    succ = tc.succ_argsort(wv)
    want_id, want_sig = tc.perm_evals_oracle(succ, N_WIRE, n, k)
    s, idv, sig = DevBuf(succ), DevBuf(np.zeros((N_WIRE * n, 4), dtype=np.uint64)), DevBuf(np.zeros((N_WIRE * n, 4), dtype=np.uint64))
    c.perm_evals_dev(s.ptr, N_WIRE, n, k, idv.ptr, sig.ptr)
    assert np.array_equal(to_host(idv), want_id) and np.array_equal(to_host(sig), want_sig)
    c.perm_evals_dev(None, N_WIRE, n, k, idv.ptr, sig.ptr)
    assert np.array_equal(to_host(sig), want_id)
    witness = orc.gen_fr(9802, num_vars)
    w, v = DevBuf(witness), DevBuf(wv)
    wires, pub = DevBuf(np.zeros((N_WIRE * n, 4), dtype=np.uint64)), DevBuf(np.zeros((n, 4), dtype=np.uint64))
    c.witness_gather_dev(w.ptr, num_vars, v.ptr, N_WIRE, n, 21, wires.ptr, pub.ptr)
    want_w, want_p = tc.gather_oracle(witness, wv, N_WIRE, n, 21)
    assert np.array_equal(to_host(wires), want_w) and np.array_equal(to_host(pub), want_p)
    c.close()


def test_load_circuit_at_2p16(orc, gpu_lib):
    log_n = 8 if DRY else 16
    n = 1 << log_n
    bases = orc.gen_bases(5, n + 3, n + 3, True)
    c = Context(gpu_lib, 0, 0, 1)
    c.init(bases, n, 8 * n)
    tc.check_load_circuit(orc, c, bases, log_n, 9900, DEV)
    c.close()


def splitmix_scalars(seed: int, n: int) -> np.ndarray:
    """the discrete logs t_i of dp_debug_gen_bases(seed, n): bases[i] = t_i G"""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (np.arange(n, dtype=np.uint64) + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return z | np.uint64(1)


def test_verifying_key_at_2p20_against_known_discrete_logs(orc, gpu_lib):
    log_n = 8 if DRY else 20
    n = 1 << log_n
    seed = 0xC1C5EED
    c = Context(gpu_lib, 0, 0, 1)
    bases = c.gen_bases(seed, n)
    c.init(bases, n, 8 * n)
    rng = np.random.default_rng(5)
    sel = [orc.gen_fr(9950 + i, n) for i in range(N_SEL)]
    F = NumpyField(log_n)
    k = np.stack([F.from_u64(v) for v in (1, 7, 13, 17, 23)])
    wv = bench_circuit_inputs(log_n, 4 * n, seed=int(rng.integers(1 << 30)))
    pr = ResidentProver(c, torch, log_n, DEV, F)
    vk, _ = pr.load_circuit(sel, wv, 4 * n, k, 16)
    t = splitmix_scalars(seed, n)
    gen = orc.g1_generator()
    for j, p in enumerate(pr.sel_coef + pr.sig_coef):
        dot = orc.fr_dot_u64(orc.into_repr(host(p)), t)
        assert np.array_equal(orc.normalize(vk[j]), orc.g1_mul(gen, dot)), f"verifying-key commitment {j}"
    c.close()


@pytest.mark.parametrize("quotient", ["whole", "sliced"])
def test_prove_witness_equals_prove_at_2p16(orc, gpu_lib, quotient):
    log_n = 8 if DRY else 16
    n = 1 << log_n
    c = Context(gpu_lib, 0, 0, 1)
    c.init(orc.gen_bases(5, n + 3, n + 3, True), n, 8 * n)
    tc.check_prove_witness(orc, c, log_n, 10000, DEV, quotient)
    c.close()


def test_satisfied_circuit_degree_at_2p16(orc, gpu_lib):
    log_n = 8 if DRY else 16
    n = 1 << log_n
    c = Context(gpu_lib, 0, 0, 1)
    c.init(orc.gen_bases(5, n + 3, n + 3, True), n, 8 * n)
    tc.check_satisfied_circuit_degree(orc, c, log_n, 10100, DEV)
    c.close()
