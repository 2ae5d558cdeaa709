"""The window-multiple table at widths pinned with DP_MSM_PRE_C, on the kernel-logic emulator: widths 8 to 12 over
2^11+ bases (what dp_init's cost model picks for such an SRS, and the narrower ones it never picks), with and without
batched-affine tree levels, against the oracle on the usual scalar distributions and on the edges of the signed-digit
recoding; no table at all (DP_MSM_PRE_C=0); widths dp_init must refuse.  The wider tables and the production sizes run
on the GPU (tests/test_zzzzzzzzzz_gpu_msm_geometry.py)."""
import numpy as np
import pytest

from distributed_plonk_b200._binding import Context, DpError
from tests import common, msm_recoding

N = 2048 + 37                    # >= 2^11 bases: dp_init builds a table; the full range uses it at every width 8..12
SEED = 20500


@pytest.fixture(scope="module")
def bases(orc):
    return orc.gen_bases(SEED, N, 64, True)                   # tiled distinct points with infinity among them


@pytest.fixture(scope="module")
def expected(orc, bases):
    """oracle points, one per scalar set; they do not depend on the width"""
    sets = common.scalar_sets(orc, N, SEED + 1)
    return {name: (sc, orc.msm(bases, sc)) for name, sc in sets.items()}


def pinned_ctx(lib, monkeypatch, bases, pre_c, levels, W=1, me=0):
    monkeypatch.setenv("DP_MSM_PRE_C", str(pre_c))
    monkeypatch.setenv("DP_MSM_AFFINE", str(levels))
    monkeypatch.setenv("DP_MSM_AFFINE_MIN", "0")
    c = Context(lib, 0, me, W)
    c.init(bases, 1 << 4, 1 << 7)
    return c


@pytest.mark.parametrize("levels", [0, 2])
@pytest.mark.parametrize("pre_c", [8, 9, 10, 11, 12])
def test_pinned_width_vs_oracle(orc, emul_lib, monkeypatch, bases, expected, pre_c, levels):
    c = pinned_ctx(emul_lib, monkeypatch, bases, pre_c, levels)
    assert c.msm_tuning()["levels"] == levels
    for name, (sc, ref) in expected.items():
        common.assert_point_eq(orc, c.msm(0, N, sc), ref, f"c={pre_c} L={levels} {name}")
    sc, _ = msm_recoding.place_recoding_edges(pre_c, N, SEED + 2, 12, expected["uniform"][0])
    common.assert_point_eq(orc, c.msm(0, N, sc), orc.msm(bases, sc), f"c={pre_c} L={levels} recoding edges over uniform")
    sc, _ = msm_recoding.place_recoding_edges(pre_c, N, SEED + 3, 40)
    common.assert_point_eq(orc, c.msm(0, N, sc), orc.msm(bases, sc), f"c={pre_c} L={levels} recoding edges over zeros")
    for name, v in msm_recoding.recoding_edge_scalars(pre_c).items():          # one edge in every slot: one bucket per window
        sc = np.tile(common.u256(v), (N, 1))
        common.assert_point_eq(orc, c.msm(0, N, sc), orc.msm(bases, sc), f"c={pre_c} L={levels} all '{name}'")
    c.close()


def test_no_table_gives_the_same_points(orc, emul_lib, monkeypatch, bases, expected):
    """DP_MSM_PRE_C=0: dp_init builds no table, so every MSM takes the per-window pipeline (a GPU short of memory)"""
    for levels in (0, 2):
        c = pinned_ctx(emul_lib, monkeypatch, bases, 0, levels)
        for name, (sc, ref) in expected.items():
            common.assert_point_eq(orc, c.msm(0, N, sc), ref, f"no table, L={levels}, {name}")
        c.close()
    monkeypatch.delenv("DP_MSM_AFFINE")
    monkeypatch.delenv("DP_MSM_AFFINE_MIN")
    c = Context(emul_lib, 0, 0, 1)
    c.init(bases, 1 << 4, 1 << 7)
    assert c.msm_tuning()["equal"] == -1                       # no table: nothing for dp_init to tune
    c.close()


def test_pinned_width_own_shard(orc, emul_lib, monkeypatch):
    """worker 1 of 2 with a pinned width: the table covers its shard [n, 2n) only"""
    n = 2048
    bases = orc.gen_bases(SEED + 4, 2 * n + 5, 61, True)        # a period that does not divide the shard start
    hi = 2 * n + 5
    sc = orc.gen_fr(SEED + 5, hi, False)
    for pre_c in (8, 11):
        c = pinned_ctx(emul_lib, monkeypatch, bases, pre_c, 0, W=2, me=1)
        for lo, h, what in ((n + 2, hi, "own shard (table)"), (n + 600, n + 1900, "inside the shard"),
                            (n - 7, hi, "straddling the shard start"), (0, n, "other shard")):
            common.assert_point_eq(orc, c.msm(lo, h, sc[:h - lo]), orc.msm(bases[lo:h], sc[:h - lo]), f"c={pre_c} {what}")
        c.close()


@pytest.mark.parametrize("value", ["7", "23", "1", "-1", "abc", "12x"])
def test_width_out_of_range_is_refused(orc, emul_lib, monkeypatch, bases, value):
    monkeypatch.setenv("DP_MSM_PRE_C", value)
    c = Context(emul_lib, 0, 0, 1)
    with pytest.raises(DpError) as e:
        c.init(bases, 1 << 4, 1 << 7)
    assert e.value.code == -1 and "DP_MSM_PRE_C" in str(e.value), str(e.value)
    with pytest.raises(DpError) as e:
        c.msm(0, 1, np.zeros((1, 4), dtype=np.uint64))
    assert e.value.code == -2                                  # the context stays uninitialised
    c.close()


def test_pinned_width_needs_2p11_bases(orc, emul_lib, monkeypatch):
    """a shard below 2^11 bases cannot take a pinned table: refused, never a quiet fall-back to the per-window pipeline"""
    monkeypatch.setenv("DP_MSM_PRE_C", "10")
    c = Context(emul_lib, 0, 0, 1)
    with pytest.raises(DpError) as e:
        c.init(orc.gen_bases(SEED, 2047, 64, True), 1 << 4, 1 << 7)
    assert e.value.code == -1 and "DP_MSM_PRE_C" in str(e.value)
    c.init(orc.gen_bases(SEED, 2048, 64, True), 1 << 4, 1 << 7)       # exactly 2^11: accepted
    c.close()
    c = Context(emul_lib, 0, 1, 2)                                     # 2^12 - 2 bases over two workers: 2047 in shard 1
    with pytest.raises(DpError) as e:
        c.init(orc.gen_bases(SEED, 4094, 64, True), 1 << 4, 1 << 7)
    assert e.value.code == -1
    c.close()
    monkeypatch.setenv("DP_MSM_PRE_C", "0")                            # no table asked for: any size is fine
    c = Context(emul_lib, 0, 0, 1)
    c.init(orc.gen_bases(SEED, 100, 64, True), 1 << 4, 1 << 7)
    c.close()
