"""Round 3 slice by slice (dp_ntt_dev_quot_slice, dp_quotient_evals_slice_dev, ResidentProver(quotient="sliced")) on the
kernel-logic emulator: every slice transform equals the strided whole-domain coset transform byte for byte on the 1-, 2-
and 3-pass plans, all slices of the quotient equal dp_quotient_evals_dev and the oracle, and the sliced prover passes the
oracle's check of all 13 commitments and 10 evaluations - also on the asynchronous-stream build under adversarial
schedules, since its 25 evaluation buffers are reused from one slice to the next."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

from distributed_plonk_b200._binding import Context, DpError
from distributed_plonk_b200.resident import ResidentProver

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def pad(c, m):
    out = np.zeros((m, 4), dtype=np.uint64)
    out[:c.shape[0]] = c
    return out


def check_slice_ntt(orc, c, log_n, log_m, seed, n_valids):
    n, m = 1 << log_n, 1 << log_m
    for j, n_valid in enumerate(n_valids):
        x = np.ascontiguousarray(orc.gen_fr(seed + j, n_valid))
        before = x.copy()
        ref = orc.fft(pad(x, m), False, True)
        for k in range(m // n):
            out = np.zeros((n, 4), dtype=np.uint64)
            c.ntt_dev_quot_slice(x.ctypes.data, n_valid, k, out.ctypes.data)
            assert np.array_equal(out, ref[k::m // n]), f"slice {k} of 2^{log_n} -> 2^{log_m}, {n_valid} coefficients"
        assert np.array_equal(x, before), "the slice transform wrote to its input"


# (pass-planning limits set before dp_init so that the gate domain takes the 1-, 2- or 3-pass plan with its per-slice
# factor tables; None = defaults), gate domain, quotient domain
PLANS = [(None, 3, 6), ((3, 2), 3, 6), ((3, 2), 4, 7), ((3, 3), 6, 9), ((3, 2), 6, 9), ((2, 2), 6, 10), ((2, 2), 5, 5),
         ((2, 2), 5, 6), ((3, 2), 5, 9)]


@pytest.mark.parametrize("limits,log_n,log_m", PLANS)
def test_slice_ntt_equals_the_strided_coset_transform(orc, emul_lib, limits, log_n, log_m):
    c = Context(emul_lib, 0, 0, 1)
    if limits:
        c.debug_set_limits(limits[0], limits[1], 0)
    c.init(np.zeros(0, dtype=np.uint8), 1 << log_n, 1 << log_m)
    n = 1 << log_n
    check_slice_ntt(orc, c, log_n, log_m, 3000 + log_n + log_m, sorted({n, max(1, n // 8), min(3, n), 1}, reverse=True))
    c.close()


def test_slice_ntt_after_the_split_changes(orc, emul_lib):
    """limits lowered after dp_init: the per-slice tables no longer fit the split, the scale-and-copy path takes over"""
    c = Context(emul_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), 1 << 6, 1 << 9)
    c.debug_set_limits(3, 2, 0)
    check_slice_ntt(orc, c, 6, 9, 3100, (64, 8))
    c.close()


def test_slice_errors(orc, emul_lib):
    c = Context(emul_lib, 0, 0, 1)
    x = np.ascontiguousarray(orc.gen_fr(3200, 16))
    out = np.zeros((16, 4), dtype=np.uint64)
    arrs = [np.zeros((16, 4), dtype=np.uint64) for _ in range(25)]
    one = orc.gen_fr(3201, 1)[0]
    k5 = orc.gen_fr(3202, 5)
    q_out = np.zeros((128, 4), dtype=np.uint64)

    def quot(k, out_ptr=q_out.ctypes.data, a=arrs):
        c.quotient_evals_slice_dev([t.ctypes.data for t in a[:13]], [t.ctypes.data for t in a[13:18]], [t.ctypes.data for t in a[18:23]],
                                   a[23].ctypes.data, a[24].ctypes.data, k5, one, one, one, k, out_ptr)

    def code(f):
        with pytest.raises(DpError) as e:
            f()
        return e.value.code

    assert code(lambda: c.ntt_dev_quot_slice(x.ctypes.data, 16, 0, out.ctypes.data)) == -2       # before dp_init
    assert code(lambda: quot(0)) == -2
    c.init(np.zeros(0, dtype=np.uint8), 16, 128)
    assert code(lambda: c.ntt_dev_quot_slice(x.ctypes.data, 16, 8, out.ctypes.data)) == -1        # slice >= m/n
    assert code(lambda: c.ntt_dev_quot_slice(x.ctypes.data, 17, 0, out.ctypes.data)) == -1        # n_valid > n
    assert code(lambda: c.ntt_dev_quot_slice(None, 16, 0, out.ctypes.data)) == -1
    assert code(lambda: c.ntt_dev_quot_slice(x.ctypes.data, 16, 0, None)) == -1
    assert code(lambda: c.ntt_dev_quot_slice(x.ctypes.data, 16, 0, x.ctypes.data + 32 * 15)) == -1  # output overlaps input
    assert code(lambda: quot(8)) == -1
    assert code(lambda: quot(0, None)) == -1
    assert code(lambda: quot(0, arrs[7].ctypes.data)) == -1                                          # output overlaps input 7
    c.ntt_dev_quot_slice(x.ctypes.data, 16, 7, out.ctypes.data)                                      # the last slice is fine
    c.ntt_dev_quot_slice(x.ctypes.data, 0, 1, out.ctypes.data)                                       # the zero polynomial
    assert not out.any()
    c.close()


def check_quotient_slices(orc, c, n, m, seed):
    """all slices into one buffer == dp_quotient_evals_dev on the whole arrays == the oracle, byte for byte"""
    ratio = m // n
    sel = [orc.gen_fr(seed + i, m) for i in range(13)]
    sig = [orc.gen_fr(seed + 20 + i, m) for i in range(5)]
    w = [orc.gen_fr(seed + 30 + i, m) for i in range(5)]
    z, pi = orc.gen_fr(seed + 40, m), orc.gen_fr(seed + 41, m)
    k = orc.gen_fr(seed + 42, 5)
    al, be, ga = (orc.gen_fr(seed + 43 + i, 1)[0] for i in range(3))
    whole = sel + sig + w + [z, pi]
    ptr = [a.ctypes.data for a in whole]
    want = np.zeros((m, 4), dtype=np.uint64)
    c.quotient_evals_dev(ptr[:13], ptr[13:18], ptr[18:23], ptr[23], ptr[24], k, al, be, ga, want.ctypes.data)
    assert np.array_equal(want, orc.quotient_evals(np.stack(sel), np.stack(sig), np.stack(w), z, pi, k, al, be, ga, n))
    got = np.zeros((m, 4), dtype=np.uint64)
    for s in range(ratio):
        sl = [np.ascontiguousarray(a[s::ratio]) for a in whole]
        p = [a.ctypes.data for a in sl]
        before = got.copy()
        c.quotient_evals_slice_dev(p[:13], p[13:18], p[18:23], p[23], p[24], k, al, be, ga, s, got.ctypes.data)
        touched = np.zeros(m, dtype=bool)
        touched[s::ratio] = True
        assert np.array_equal(got[~touched], before[~touched]), f"slice {s} wrote outside its points"
    assert np.array_equal(got, want), f"quotient slices n={n} m={m}"


@pytest.mark.parametrize("table", ["0", "1"])
@pytest.mark.parametrize("n,m", [(64, 512), (4, 32), (16, 16), (2, 32), (64, 128), (8, 16)])
def test_quotient_slices_equal_the_whole_quotient(orc, emul_lib, monkeypatch, table, n, m):
    monkeypatch.setenv("DP_QUOT_TABLE", table)          # read by dp_create: 0 = product-tree variant, 1 = cached table
    c = Context(emul_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, m)
    check_quotient_slices(orc, c, n, m, 3300 + n + m)
    c.close()


def check_sliced_prover(orc, ctx, bases, log_n, seed, device, monkeypatch):
    """tests/test_resident.py's oracle check of all 13 commitments and 10 evaluations, with the prover in sliced mode"""
    from tests import test_resident
    monkeypatch.setattr(test_resident, "ResidentProver", functools.partial(ResidentProver, quotient="sliced"))
    test_resident.check_resident_prover(orc, ctx, bases, log_n, seed, device)


def test_sliced_resident_prover(orc, emul_lib, monkeypatch):
    bases = orc.gen_bases(5, 80, 64, True)
    c = Context(emul_lib, 0, 0, 1)
    c.init(bases, 1 << 6, 1 << 9)
    check_sliced_prover(orc, c, bases, 6, 2100, "cpu", monkeypatch)
    c.close()


def test_prover_modes(emul_lib):
    import torch
    from distributed_plonk_b200.resident import NumpyField
    c = Context(emul_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), 1 << 4, 1 << 7)
    F = NumpyField(4)
    assert ResidentProver(c, torch, 4, "cpu", F).quotient == "whole"          # what fits keeps today's layout
    pr = ResidentProver(c, torch, 4, "cpu", F, quotient="sliced")
    assert pr.big is None and len(pr.slices) == 25 and all(t.shape[0] == 16 for t in pr.slices)
    with pytest.raises(ValueError):
        ResidentProver(c, torch, 4, "cpu", F, quotient="tiled")
    c.close()


@pytest.mark.timeout(1500)
@pytest.mark.skipif(os.environ.get("DP_TEST_EMUL_ASYNC", "0") == "1", reason="this test starts the asynchronous runs itself")
def test_slices_under_adversarial_stream_schedules():
    """the slice transforms, the quotient slices and the sliced prover on the asynchronous-stream emulator build, with
    the compute, copy-in and MSM tail streams in turn made pathologically slow (tests/test_emul_async.py)"""
    from tests.emul import build as emul_build
    emul_build.build(async_streams=True)
    select = "sliced_resident_prover or (strided_coset_transform and 6-9) or (whole_quotient and 64-512)"
    procs = []
    for slow in (0, 1, 3):
        env = dict(os.environ, DP_TEST_EMUL_ASYNC="1", DP_EMUL_SLOW=f"{slow}:1500")
        procs.append(subprocess.Popen(
            [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider", "-k", select],
            cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    for slow, p in zip((0, 1, 3), procs):
        out, _ = p.communicate()
        assert p.returncode == 0, f"adversarial schedule {slow}:\n{out[-3000:]}"
        assert " passed" in out and "failed" not in out
