"""Blinded proofs on the GPU: dp_poly_blind_dev, the quotient with tails in both 1/(x - 1) modes over the whole coset and
every slice (against the oracle at 2^12, and at a 2^20-point gate domain, whose slice transforms take the multi-pass plans,
against the quotient of the full polynomials' coset evaluations), the blinded resident prover in both round-3 layouts,
and the degree of its quotient on a satisfied circuit."""
import os

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context
from distributed_plonk_b200.resident import N_BLIND, N_WIRE, ResidentProver
from tests import test_blinding as tb

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
DEV = "cpu" if DRY else "cuda"


def dev(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64).copy()).to(DEV)


def host(t: torch.Tensor) -> np.ndarray:
    if not DRY:
        torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint64)


def test_blind(orc, gpu_lib):
    n = 1 << (6 if DRY else 12)
    c = Context(gpu_lib, 0, 0, 1)
    p = orc.gen_fr(8000, n)
    for k in (2, 3):
        b = orc.gen_fr(8001 + k, k)
        t = dev(np.concatenate([p, np.zeros((k, 4), dtype=np.uint64)]))
        c.poly_blind_dev(t.data_ptr(), n, k, b)
        assert np.array_equal(host(t), tb.blinded(orc, p, b, n))
    outs = []
    for _ in range(2):
        t = dev(np.concatenate([p, np.zeros((3, 4), dtype=np.uint64)]))
        c.poly_blind_dev(t.data_ptr(), n, 3)
        outs.append(host(t))
    assert not np.array_equal(outs[0], outs[1])
    for o in outs:     # b(X) (X^n - 1) vanishes on H: p(omega^i) = the blinded polynomial's, i = 0 and 1 (X = 1, omega)
        assert np.array_equal(orc.poly_eval(o, tb.common._fr_one(orc)), orc.poly_eval(p, tb.common._fr_one(orc)))
        w = tb.NumpyField(n.bit_length() - 1).omega
        assert np.array_equal(orc.poly_eval(o, w), orc.poly_eval(p, w))
    c.close()


def tail_quotient_device(c, arrs, tails, scal, n, m):
    """whole-coset and all-slices quotients with tails of device arrays; returns both as device tensors"""
    k, al, be, ga = scal
    tl = [(t.data_ptr() if t.shape[0] else None, t.shape[0]) for t in tails]
    p = [a.data_ptr() for a in arrs]
    whole = torch.zeros((m, 4), dtype=torch.int64, device=DEV)
    c.quotient_evals_tail_dev(p[:13], p[13:18], p[18:23], p[23], p[24], k, al, be, ga, tl, whole.data_ptr())
    ratio = m // n
    sliced = torch.zeros((m, 4), dtype=torch.int64, device=DEV)
    for s in range(ratio):
        q = [a[s::ratio].contiguous() for a in arrs]
        qp = [a.data_ptr() for a in q]
        c.quotient_evals_slice_tail_dev(qp[:13], qp[13:18], qp[18:23], qp[23], qp[24], k, al, be, ga, tl, s, sliced.data_ptr())
    return whole, sliced


@pytest.mark.parametrize("table", ["0", "1"])
def test_tail_quotient_vs_oracle(orc, gpu_lib, monkeypatch, table):
    monkeypatch.setenv("DP_QUOT_TABLE", table)
    logn, logq = (6, 9) if DRY else (12, 15)
    n, m = 1 << logn, 1 << logq
    c = Context(gpu_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, m)
    for j, lens in enumerate(tb.LENS):
        arrs, tails, scal, want = tb.tail_instance(orc, n, m, 8100 + 100 * j, lens)
        whole, sliced = tail_quotient_device(c, [dev(a) for a in arrs], [dev(t) for t in tails], scal, n, m)
        assert np.array_equal(host(whole), want), f"whole coset, tails {lens}, DP_QUOT_TABLE={table}"
        assert torch.equal(sliced, whole), f"slices, tails {lens}, DP_QUOT_TABLE={table}"
    c.close()


def test_tail_quotient_on_a_2p20_gate_domain(orc, gpu_lib):
    """the slice layout at a 2^20-point gate domain: the heads through dp_ntt_dev_quot_slice (multi-pass plans), the
    tails in the kernel, against the plain quotient of the full polynomials' coset evaluations (dp_ntt_dev_padded)"""
    logn, logq = (6, 9) if DRY else (20, 23)
    n, m, ratio = 1 << logn, 1 << logq, 1 << (logq - logn)
    lens = (2, 2, 2, 2, 2, 3)
    c = Context(gpu_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, m)
    g = torch.Generator(device=DEV)
    g.manual_seed(0xB11D)

    def rand_fr(count):
        t = torch.randint(-(1 << 63), (1 << 63) - 1, (count, 4), dtype=torch.int64, device=DEV, generator=g)
        t[:, 3] &= (1 << 62) - 1
        return t

    k = orc.gen_fr(8200, 5)
    al, be, ga = (orc.gen_fr(8201 + i, 1)[0] for i in range(3))
    fixed = [rand_fr(n) for _ in range(13 + 5)] + [rand_fr(n)]         # selectors, sigmas, public input: coefficients
    polys = [rand_fr(n + t) for t in lens]                                # the five wires and z, with their tails
    tails = [p[n:] for p in polys]
    tl = [(t.data_ptr(), t.shape[0]) for t in tails]
    # reference: every polynomial in full on the m-point coset, the quotient without tails
    full = []
    for p in fixed[:18] + polys + fixed[18:]:
        buf = torch.zeros((m, 4), dtype=torch.int64, device=DEV)
        buf[:p.shape[0]] = p
        c.ntt_dev_padded(buf.data_ptr(), p.shape[0], logq, False, True)
        full.append(buf)
    want = torch.empty((m, 4), dtype=torch.int64, device=DEV)
    f = [t.data_ptr() for t in full]
    c.quotient_evals_dev(f[:13], f[13:18], f[18:23], f[23], f[24], k, al, be, ga, want.data_ptr())
    del full, f
    heads = fixed[:18] + [p[:n] for p in polys] + fixed[18:]
    bufs = [torch.empty((n, 4), dtype=torch.int64, device=DEV) for _ in range(25)]
    b = [t.data_ptr() for t in bufs]
    got = torch.zeros((m, 4), dtype=torch.int64, device=DEV)
    for s in range(ratio):
        for dst, src in zip(b, heads):
            c.ntt_dev_quot_slice(src.data_ptr(), n, s, dst)
        c.quotient_evals_slice_tail_dev(b[:13], b[13:18], b[18:23], b[23], b[24], k, al, be, ga, tl, s, got.data_ptr())
    assert torch.equal(got, want), "sliced quotient with tails at a 2^20-point gate domain"
    c.close()


@pytest.mark.parametrize("quotient", ["whole", "sliced"])
def test_blinded_prover_vs_oracle(orc, gpu_lib, quotient):
    log_n = 6 if DRY else 12
    n = 1 << log_n
    bases = orc.gen_bases(5, n + 32, n + 32, True)
    c = Context(gpu_lib, 0, 0, 1)
    c.init(bases, n, 8 * n)
    tb.check_blinded_prover(orc, c, bases, log_n, 8300 + log_n, DEV, quotient)
    c.close()


def test_blinded_provers_at_2p16(orc, gpu_lib):
    """whole and sliced give the same blinded proof; zero blinders give the unblinded proof; the library's blinders
    change the six blinded commitments"""
    log_n = 8 if DRY else 16
    n = 1 << log_n
    c = Context(gpu_lib, 0, 0, 1)
    c.init(orc.gen_bases(5, n + 32, n + 32, True), n, 8 * n)   # all distinct: G_(n+j) = G_j would hide a blinding
    F, key, wires, pub, ch = tb.prover_key(orc, log_n, 8400)
    w, p = tb.host_inputs(wires, pub, DEV)
    blind = orc.gen_fr(8450, N_BLIND)
    outs = {}
    for mode in ("whole", "sliced"):
        pr = ResidentProver(c, torch, log_n, DEV, F, quotient=mode)
        pr.load_key(*key)
        com, ev = pr.prove(w, p, ch, blind=blind)
        outs[mode] = [np.asarray(x) for x in com + ev]
        plain = pr.prove(w, p, ch)
        zero = pr.prove(w, p, ch, blind=np.zeros((N_BLIND, 4), dtype=np.uint64))
        assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(plain[0] + plain[1], zero[0] + zero[1])), mode
        r1, r2 = pr.prove(w, p, ch, blind=True), pr.prove(w, p, ch, blind=True)
        for j in range(N_WIRE + 1):
            assert not np.array_equal(orc.normalize(r1[0][j]), orc.normalize(r2[0][j])), f"{mode}: commitment {j}"
        del pr
    assert len(outs["whole"]) == 23
    for j, (a, b) in enumerate(zip(outs["whole"], outs["sliced"])):
        assert np.array_equal(a, b), f"output {j} of the blinded proof differs between the layouts"
    c.close()


@pytest.mark.parametrize("log_n", [6, 12])
def test_blinded_quotient_degree_on_a_satisfied_circuit(orc, gpu_lib, log_n):
    if DRY:
        log_n = min(log_n, 6)
    n = 1 << log_n
    c = Context(gpu_lib, 0, 0, 1)
    c.init(orc.gen_bases(5, n + 3, n + 3, True), n, 8 * n)
    tb.check_satisfied_degree(orc, c, log_n, 8500 + log_n, DEV)
    c.close()
