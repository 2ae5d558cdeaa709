"""The batched-affine MSM levels (DP_MSM_AFFINE / DP_MSM_TUNE) on the GPU.  Last file of the suite on purpose: these
kernels are the newest of the library, so nothing else in the suite runs after the forced-level cases and the wider
search exercised here."""
import os

import numpy as np
import pytest

from distributed_plonk_b200._binding import Context
from tests import common

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
N_BIG, N_DISTINCT = ((1 << 8) + 8, 64) if DRY else ((1 << 16) + 32, 2048)


@pytest.fixture(scope="module")
def bases(orc):
    return orc.gen_bases(5, N_BIG, N_DISTINCT, True)


@pytest.mark.parametrize("levels", [2, 1, 3])
def test_forced_levels_vs_oracle(orc, gpu_lib, bases, monkeypatch, levels):
    monkeypatch.setenv("DP_MSM_AFFINE", str(levels))
    monkeypatch.setenv("DP_MSM_AFFINE_MIN", "0")
    c = Context(gpu_lib, 0, 0, 1)
    c.init(bases, 1 << 12, 1 << 15)
    assert c.msm_tuning()["levels"] == levels
    sizes = (1, 33, 1000, (1 << 12) + 32, N_BIG) if levels == 2 else (1000, N_BIG)
    for n in [min(n, N_BIG) for n in sizes][: 2 if DRY else None]:
        common.check_msm(orc, c, bases, n, 4000 + n)          # uniform, witness-like, all r-1, all zero, all one
    for cbits in (5, 12, 17)[: 1 if DRY else None]:            # per-window bucket sets
        c.debug_set_limits(11, 9, cbits)
        common.check_msm(orc, c, bases, min(3000, N_BIG), 4100 + cbits, which=("uniform", "witness-like"))
    c.debug_set_limits(11, 9, 0)
    s2 = np.zeros((N_DISTINCT + 1, 4), dtype=np.uint64)        # bases 0 and N_DISTINCT are the same point (tiled)
    s2[0] = common.u256(5)
    s2[N_DISTINCT] = common.u256(common.R_MOD - 5)
    assert orc.normalize(c.msm(0, N_DISTINCT + 1, s2))[96] == 1          # P + (-P)
    s2[N_DISTINCT] = common.u256(5)
    common.assert_point_eq(orc, c.msm(0, N_DISTINCT + 1, s2), orc.msm(bases[:N_DISTINCT + 1], s2), "same point twice")
    nb = N_BIG - 32 if not DRY else N_BIG - 8
    sc = orc.gen_fr(4200, nb, False)
    ranges = [(0, nb), (100, nb // 2 + 100), (0, 0)]
    outs = c.msm_batch([(lo, hi, sc, hi - lo) for lo, hi in ranges])
    for k, (lo, hi) in enumerate(ranges):
        common.assert_point_eq(orc, outs[k], orc.msm(bases[lo:hi], sc[: hi - lo]), f"batch job {k}")
    c.close()


def test_tuning_at_init_agrees(orc, gpu_lib, monkeypatch):
    """dp_init times the plain pipeline and 1, 2, 3 tree levels over the context's own table (DP_MSM_TUNE=2: the wider
    search; the default compares plain and two levels); all must give the same 144 bytes"""
    monkeypatch.delenv("DP_MSM_AFFINE", raising=False)
    monkeypatch.setenv("DP_MSM_TUNE", "2")
    if DRY:
        monkeypatch.setenv("DP_MSM_AFFINE_MIN", "0")
    n = (1 << (11 if DRY else 20)) + 32
    c = Context(gpu_lib, 0, 0, 1)
    b = c.gen_bases(77, n)
    c.init(b, 1 << 4 if DRY else 1 << 20, 1 << 7 if DRY else 1 << 23)
    t = c.msm_tuning()
    print("msm tuning at 2^20:", t)
    assert t["equal"] == 1, f"the two MSM pipelines disagree: {t}"
    assert t["plain_ms"] > 0 and t["affine_ms"] > 0 and t["levels"] in (0, 1, 2, 3)
    sc = orc.gen_fr(4300, n, False)
    sc[::5] = 0
    common.assert_point_eq(orc, c.msm(0, n, sc), orc.msm(b, sc), "2^20 MSM through the tuned pipeline")
    c.close()


@pytest.mark.skipif(DRY, reason="the probe's child loads the CUDA library")
def test_probe_in_a_child_process(gpu_lib):
    from distributed_plonk_b200 import tune
    res = tune.probe(0, 0, 1, 18)
    print("probe at 2^18:", res)
    assert "error" not in res and res["equal"] in (1, -1)
    assert tune.choose(res) in (0, 1, 2, 3)
