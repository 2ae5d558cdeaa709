"""Round 3 slice by slice on the GPU: the slice transform (dp_ntt_dev_quot_slice) against the strided whole-domain coset
transform and the oracle's Horner evaluation, the quotient slices against dp_quotient_evals_dev in both 1/(x - 1) modes,
the sliced resident prover against the oracle and against the whole-domain prover, and its evaluation buffers' size."""
import os

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context
from distributed_plonk_b200.resident import N_SEL, N_WIRE, NumpyField, ResidentProver

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
DEV = "cpu" if DRY else "cuda"


def dev(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64).copy()).to(DEV)


def host(t: torch.Tensor) -> np.ndarray:
    if not DRY:
        torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint64)


# (gate, quotient domain): the 2-pass plan of 2^12 and the 3-pass plan of 2^20, both with the per-slice factor tables
@pytest.mark.parametrize("logn,logq", [(4, 7), (6, 9)] if DRY else [(12, 15), (20, 23)])
def test_slice_ntt_vs_strided_padded_transform(orc, gpu_lib, logn, logq):
    n, m = 1 << logn, 1 << logq
    c = Context(gpu_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, m)
    for n_valid, seed in ((n, 5000 + logn), (n // 8, 5100 + logn), (3, 5200 + logn)):
        x = orc.gen_fr(seed, n_valid)
        xd = dev(x)
        full = torch.zeros((m, 4), dtype=torch.int64, device=DEV)
        full[:n_valid] = xd
        c.ntt_dev_padded(full.data_ptr(), n_valid, logq, False, True)
        out = torch.empty((n, 4), dtype=torch.int64, device=DEV)
        for k in range(m // n):
            c.ntt_dev_quot_slice(xd.data_ptr(), n_valid, k, out.data_ptr())
            assert torch.equal(out, full[k::m // n]), f"slice {k}, 2^{logn} -> 2^{logq}, {n_valid} coefficients"
        assert np.array_equal(host(xd), x), "the slice transform wrote to its input"
        # the last slice at a few positions against the oracle's O(n) Horner evaluation at g * omega_m^(k + 8 i)
        k, idx = m // n - 1, [0, 1, n // 2 + 3, n - 1]
        want = orc.ntt_outputs_at(x, m, np.array([k + (m // n) * i for i in idx], dtype=np.uint64), False, True)
        assert np.array_equal(host(out)[idx], want)
    c.close()


@pytest.mark.parametrize("table", ["0", "1"])
def test_quotient_slices_vs_whole(orc, gpu_lib, monkeypatch, table):
    monkeypatch.setenv("DP_QUOT_TABLE", table)
    logn, logq = (6, 9) if DRY else (12, 15)
    n, m, ratio = 1 << logn, 1 << logq, 1 << (logq - logn)
    c = Context(gpu_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, m)
    arrs = [dev(orc.gen_fr(5300 + i, m)) for i in range(25)]
    k = orc.gen_fr(5330, 5)
    al, be, ga = (orc.gen_fr(5331 + i, 1)[0] for i in range(3))
    want = torch.empty((m, 4), dtype=torch.int64, device=DEV)
    p = [t.data_ptr() for t in arrs]
    c.quotient_evals_dev(p[:13], p[13:18], p[18:23], p[23], p[24], k, al, be, ga, want.data_ptr())
    got = torch.zeros((m, 4), dtype=torch.int64, device=DEV)
    for s in range(ratio):
        sl = [t[s::ratio].contiguous() for t in arrs]
        q = [t.data_ptr() for t in sl]
        c.quotient_evals_slice_dev(q[:13], q[13:18], q[18:23], q[23], q[24], k, al, be, ga, s, got.data_ptr())
    assert torch.equal(got, want), f"quotient slices, DP_QUOT_TABLE={table}"
    c.close()


@pytest.mark.parametrize("log_n", [6, 10])
def test_sliced_resident_prover(orc, gpu_lib, monkeypatch, log_n):
    from tests.test_quot_slices import check_sliced_prover
    n = 1 << log_n
    bases = orc.gen_bases(5, n + 32, 64, True)
    c = Context(gpu_lib, 0, 0, 1)
    c.init(bases, n, 8 * n)
    check_sliced_prover(orc, c, bases, log_n, 5400 + log_n, DEV, monkeypatch)
    c.close()


def _prover_inputs(orc, log_n, seed):
    n = 1 << log_n
    F = NumpyField(log_n)
    sel = [orc.gen_fr(seed + i, n) for i in range(N_SEL)]
    sig = [orc.gen_fr(seed + 20 + i, n) for i in range(N_WIRE)]
    key = (sel, sig, [orc.fft(s, False, False) for s in sig], [orc.gen_fr(seed + 30 + i, n) for i in range(N_WIRE)],
           np.stack([F.from_u64(v) for v in (1, 7, 13, 17, 23)]))
    w = torch.as_tensor(np.concatenate([orc.gen_fr(seed + 40 + i, n) for i in range(N_WIRE)]).view(np.int64))
    p = torch.as_tensor(orc.gen_fr(seed + 50, n).view(np.int64))
    if not DRY:
        w, p = w.pin_memory(), p.pin_memory()
    ch = {name: orc.gen_fr(seed + 60 + j, 1)[0] for j, name in enumerate(("beta", "gamma", "alpha", "zeta", "v"))}
    return F, key, (w, p, ch)


def test_sliced_and_whole_provers_agree(orc, gpu_lib):
    log_n = 8 if DRY else 16
    n = 1 << log_n
    c = Context(gpu_lib, 0, 0, 1)
    c.init(orc.gen_bases(5, n + 32, 64, True), n, 8 * n)
    F, key, inputs = _prover_inputs(orc, log_n, 5500)
    outs = {}
    for mode in ("whole", "sliced"):
        pr = ResidentProver(c, torch, log_n, DEV, F, quotient=mode)
        pr.load_key(*key)
        com, ev = pr.prove(*inputs)
        outs[mode] = [np.asarray(x) for x in com + ev]
        del pr
    assert len(outs["whole"]) == 23
    for j, (a, b) in enumerate(zip(outs["whole"], outs["sliced"])):
        assert np.array_equal(a, b), f"output {j} of the proof differs between the whole-domain and the sliced round 3"
    c.close()


@pytest.mark.skipif(DRY, reason="torch's CUDA allocator statistics")
def test_sliced_prover_allocates_n_sized_evaluation_buffers(orc, gpu_lib):
    log_n = 16
    n, m = 1 << log_n, 8 << log_n
    c = Context(gpu_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, m)
    F = NumpyField(log_n)
    own = {}
    for mode in ("whole", "sliced"):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        pr = ResidentProver(c, torch, log_n, "cuda", F, quotient=mode)
        own[mode] = torch.cuda.max_memory_allocated() - base
        del pr
    # everything else is the same n-sized buffers and the m-point quotient: the difference is 25 x (m - n) points
    assert own["whole"] - own["sliced"] == 25 * (m - n) * 32, own
    assert own["sliced"] < 25 * m * 32, own
    c.close()
