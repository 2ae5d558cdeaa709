"""The MSM at every window-table width dp_init can choose (DP_MSM_PRE_C pins it), on the GPU.  Which pipeline a
commitment takes otherwise depends on the SRS size, the free device memory at dp_init and a timing race, so the suite
pins each one it means to test:
  a. widths 8..22 x tree levels 0 and 2 (1 and 3 at 8, 16, 22) over 2^20 + 32 bases with infinity among them;
  b. the edges of the signed-digit recoding at every width, written into a few hundred slots of a 2^20 range;
  c. every digit in one bucket (one repeated scalar) at widths 20..22, which sends 2^20 digits through msm_collapse;
  d. the table-use threshold, a worker's shard table (W = 2, me = 1), dp_msm_dev_batch and dp_msm_submit / collect;
  e. 2^24 + 3 and 2^22 + 32 bases, the sizes of the largest provers: without a table (the per-window pipeline a GPU
     short of memory runs) and with the widest tables, checked against the known discrete logs of the bases.
Last file of the suite: it needs up to ~28 GB of device memory and the newest-runs-last order of the other files."""
import os

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context, DpError
from tests import common, msm_recoding
from tests.test_zzzzzzz_gpu_circuit import splitmix_scalars

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
DEV = "cpu" if DRY else "cuda"
N = (1 << 12) + 32 if DRY else (1 << 20) + 32          # bases of the sweep (each half >= 2^11: a worker's shard gets a table)
R = 1 << 11 if DRY else 1 << 20                        # range of the recoding-edge and bucket-skew MSMs
WIDTHS = [8, 12] if DRY else list(range(8, 23))
SWEEP = [(c, lv) for c in WIDTHS for lv in (0, 2)] + [(c, lv) for c in ((8,) if DRY else (8, 16, 22)) for lv in (1, 3)]
SEED = 21000
E_OOM = -3


def table_threshold(c: int) -> int:
    """fewest points an MSM inside the table's range needs to use it: n * windows >= 4 * 2^(c-1) (msm_enqueue)"""
    nw = (256 + c - 1) // c
    return -(-(4 << (c - 1)) // nw)


def pinned(lib, monkeypatch, bases, pre_c, levels=0, W=1, me=0):
    """a context over `bases` (host array or (device pointer, count)) with the table width pinned (None: dp_init's choice)"""
    if pre_c is None:
        monkeypatch.delenv("DP_MSM_PRE_C", raising=False)
    else:
        monkeypatch.setenv("DP_MSM_PRE_C", str(pre_c))
    monkeypatch.setenv("DP_MSM_AFFINE", str(levels))
    monkeypatch.setenv("DP_MSM_AFFINE_MIN", "0")
    c = Context(lib, 0, me, W)
    if isinstance(bases, tuple):
        c.init_ptr(bases[0], bases[1], 1 << 4, 1 << 7)
    else:
        c.init(bases, 1 << 4, 1 << 7)
    return c


@pytest.fixture(scope="module")
def bases(orc, gpu_lib):
    """N distinct points (the library's k_i G), every 997th the point at infinity"""
    c = Context(gpu_lib, 0, 0, 1)
    b = c.gen_bases(SEED, N)
    c.close()
    inf = orc.gen_bases(5, 4, 4, True)[3]
    assert inf[96] == 1
    b[5::997] = inf
    return b


@pytest.fixture(scope="module")
def expected(orc, bases):
    """oracle point per scalar set, computed once: it does not depend on the width"""
    return {name: (sc, orc.msm(bases, sc)) for name, sc in common.scalar_sets(orc, N, SEED + 1).items()}


@pytest.fixture(scope="module")
def uniform_background(orc, bases):
    """uniform scalars over the range R with the recoding-edge slots zeroed, and its oracle point"""
    _, slots = msm_recoding.place_recoding_edges(8, R, SEED + 3, 50)
    bg = orc.gen_fr(SEED + 2, R, False)
    bg[slots] = 0
    return bg, orc.msm(bases[:R], bg)


@pytest.mark.parametrize("pre_c,levels", SWEEP)
def test_width_and_levels_vs_oracle(orc, gpu_lib, monkeypatch, bases, expected, pre_c, levels):
    c = pinned(gpu_lib, monkeypatch, bases, pre_c, levels)
    assert c.msm_tuning()["levels"] == levels
    for name, (sc, ref) in expected.items():
        common.assert_point_eq(orc, c.msm(0, N, sc), ref, f"c={pre_c} L={levels} {name}")
    c.close()


@pytest.mark.parametrize("pre_c", WIDTHS)
def test_recoding_edges_and_bucket_skew(orc, gpu_lib, monkeypatch, bases, expected, uniform_background, pre_c):
    """every recoding edge of width pre_c in 50 slots each, over zeros and over uniform scalars (oracle: the background's
    point plus the slots' MSM); at widths 20..22 also one repeated random scalar (oracle: v * sum of the bases)"""
    assert R * ((256 + pre_c - 1) // pre_c) >= 4 << (pre_c - 1) or DRY       # the range uses the table
    c = pinned(gpu_lib, monkeypatch, bases, pre_c)
    sc, slots = msm_recoding.place_recoding_edges(pre_c, R, SEED + 3, 50)
    edges_ref = orc.msm(np.ascontiguousarray(bases[slots]), np.ascontiguousarray(sc[slots]))
    common.assert_point_eq(orc, c.msm(0, R, sc), edges_ref, f"c={pre_c} recoding edges over zeros")
    bg, bg_ref = uniform_background
    sc, _ = msm_recoding.place_recoding_edges(pre_c, R, SEED + 3, 50, bg)
    common.assert_point_eq(orc, c.msm(0, R, sc), orc.g1_add(bg_ref, edges_ref), f"c={pre_c} recoding edges over uniform")
    if pre_c >= 20 or (DRY and pre_c == WIDTHS[-1]):
        total = orc.normalize(expected["all one"][1])                  # sum of all N bases
        v = orc.gen_fr(SEED + 4 + pre_c, 1, False)[0]
        got = c.msm(0, N, np.tile(v, (N, 1)))
        assert np.array_equal(orc.normalize(got), orc.g1_mul(total, v)), f"c={pre_c}: one repeated random scalar"
    c.close()


@pytest.mark.parametrize("pre_c", [12, 16, 22] if not DRY else [8])
def test_table_threshold(orc, gpu_lib, monkeypatch, bases, pre_c):
    """sub-ranges with just enough points to use the table and one point fewer (the per-window pipeline)"""
    c = pinned(gpu_lib, monkeypatch, bases, pre_c)
    t = table_threshold(pre_c)
    sc = orc.gen_fr(SEED + 5, t, False)
    sc[1::3] = 0
    for lo, n in ((1000, t), (1000, t - 1), (N - t, t), (N - t + 1, t - 1)):
        common.assert_point_eq(orc, c.msm(lo, lo + n, sc[:n]), orc.msm(bases[lo:lo + n], sc[:n]), f"c={pre_c} [{lo}, +{n})")
    c.close()


@pytest.mark.parametrize("pre_c", [16, 21] if not DRY else [8])
def test_shard_table(orc, gpu_lib, monkeypatch, bases, pre_c):
    """worker 1 of 2: the table covers its shard [N/2, N) only; ranges inside it, all of it, straddling its start"""
    c = pinned(gpu_lib, monkeypatch, bases, pre_c, W=2, me=1)
    h = N // 2
    sc = orc.gen_fr(SEED + 6, h + 300, False)
    sc[::4] = 0
    for lo, hi, what in ((h, N, "whole shard"), (h + 3, N - 5, "inside the shard"), (h - 300, N, "straddling the shard start"),
                         (h - 7, h + 9, "a few points across the start")):
        common.assert_point_eq(orc, c.msm(lo, hi, sc[:hi - lo]), orc.msm(bases[lo:hi], sc[:hi - lo]), f"c={pre_c} {what}")
    c.close()


def test_batch_and_async_under_pinned_widths(orc, gpu_lib, monkeypatch, bases):
    """dp_msm_dev_batch at width 21 (the first two jobs use the table), dp_msm_submit / collect at width 18"""
    c = pinned(gpu_lib, monkeypatch, bases, 12 if DRY else 21)
    ranges = [(0, R), (5000 % N, 5000 % N + R // 2 + 7), (0, 0)] if not DRY else [(0, R), (50, 50 + R // 2 + 7), (0, 0)]
    scs = [np.ascontiguousarray(orc.gen_fr(SEED + 7 + k, max(hi - lo, 1), False)) for k, (lo, hi) in enumerate(ranges)]
    dev = [torch.from_numpy(s.view(np.uint8).copy()).to(DEV) for s in scs]
    outs = torch.zeros((len(ranges), 144), dtype=torch.uint8, device=DEV)
    c.msm_dev_batch([(lo, hi, dev[k].data_ptr(), hi - lo, outs[k].data_ptr()) for k, (lo, hi) in enumerate(ranges)])
    outs = outs.cpu().numpy()
    for k, (lo, hi) in enumerate(ranges):
        common.assert_point_eq(orc, outs[k], orc.msm(bases[lo:hi], scs[k][:hi - lo]), f"dev batch job {k}")
    c.close()
    c = pinned(gpu_lib, monkeypatch, bases, 8 if DRY else 18)
    common.check_async_msm(orc, c, bases, (1 << 10) if DRY else (1 << 17), SEED + 10)
    c.close()


def random_canonical(n: int, seed: int) -> np.ndarray:
    """n scalars below 2^254 (< r), with zeros and r - 1 among them"""
    sc = np.random.default_rng(seed).integers(0, 1 << 64, size=(n, 4), dtype=np.uint64, endpoint=False)
    sc[:, 3] &= np.uint64((1 << 62) - 1)
    sc[::1001] = 0
    sc[7::1003] = common.u256(common.R_MOD - 1)
    return sc


def check_known_logs(orc, lib, monkeypatch, log_n: int, extra: int, pre_c, table_bytes: int, seed: int):
    """n = 2^log_n + extra bases k_i G generated on the device; commitments of random scalars at lengths n, n - 1, 2^log_n
    and a sub-range equal (sum s_i k_i) G: an O(n) check on the host"""
    n = (1 << log_n) + extra
    if not DRY:
        free = torch.cuda.mem_get_info()[0]
        need = table_bytes + n * (96 + 104) + (6 << 30)                # table, bases, generation buffer, MSM scratch
        if free < need:
            pytest.skip(f"DP_MSM_PRE_C={pre_c} at {n} bases needs ~{need / 2**30:.1f} GiB, the GPU has {free / 2**30:.1f} GiB free")
    gen = Context(lib, 0, 0, 1)
    buf = torch.empty((n, 104), dtype=torch.uint8, device=DEV)
    gen.gen_bases_into(seed, n, buf.data_ptr())
    gen.close()
    try:
        c = pinned(lib, monkeypatch, (buf.data_ptr(), n), pre_c)
    except DpError as e:
        if e.code != E_OOM or DRY:
            raise
        free = torch.cuda.mem_get_info()[0]
        pytest.skip(f"DP_MSM_PRE_C={pre_c} at {n} bases: the table did not fit, {free / 2**30:.1f} GiB free after the failed dp_init ({e})")
    finally:
        del buf
        if not DRY:
            torch.cuda.empty_cache()
    t = splitmix_scalars(seed, n)
    g = orc.g1_generator()
    sc = random_canonical(n, seed)
    sub_lo = 37 if DRY else 12345
    for lo, hi in ((0, n), (0, n - 1), (0, 1 << log_n), (sub_lo, sub_lo + (1 << (log_n - 1)) + 1)):
        got = c.msm(lo, hi, sc[:hi - lo])
        ref = orc.g1_mul(g, orc.fr_dot_u64(sc[:hi - lo], t[lo:hi]))
        assert np.array_equal(orc.normalize(got), ref), f"DP_MSM_PRE_C={pre_c}: [{lo}, {hi}) of {n} bases"
    c.close()


@pytest.mark.parametrize("pre_c", [0, 22])
def test_known_discrete_logs_at_2p24(orc, gpu_lib, monkeypatch, pre_c):
    """the 2^24-gate prover's SRS: no table (the per-window pipeline, c = 18, 15 windows x 2^17 buckets) and the width-22
    table (19.3 GB, 2^21 buckets); skipped with the free memory named when the card cannot hold the table"""
    log_n, extra = (11, 3) if DRY else (24, 3)
    width = (12 if DRY else 22) if pre_c else 0
    nw = (256 + width - 1) // width if width else 0
    check_known_logs(orc, gpu_lib, monkeypatch, log_n, extra, width, nw * ((1 << log_n) + extra) * 96, SEED + 20)


@pytest.mark.parametrize("pre_c", [None, 21])
def test_known_discrete_logs_at_2p22(orc, gpu_lib, monkeypatch, pre_c):
    """the 2^22-gate prover's SRS: dp_init's own choice (width 20 when a quarter of the free memory holds 5.2 GB) and 21"""
    log_n, extra = (11, 32) if DRY else (22, 32)
    width = pre_c if not DRY or pre_c is None else 11
    nw = (256 + width - 1) // width if width else 0
    check_known_logs(orc, gpu_lib, monkeypatch, log_n, extra, width, nw * ((1 << log_n) + extra) * 96, SEED + 30)


def test_width_too_wide_for_the_shard_is_refused(orc, gpu_lib, monkeypatch):
    """a width whose table would hold 2^31 points or more is refused by dp_init, not replaced by another width"""
    n = 2048 if DRY else 1 << 26                              # 32 windows x 2^26 = 2^31
    if DRY:
        monkeypatch.setenv("DP_MSM_PRE_C", "7")
    else:
        monkeypatch.setenv("DP_MSM_PRE_C", "8")
        if torch.cuda.mem_get_info()[0] < n * 104 * 2 + (n * 96) + (2 << 30):
            pytest.skip(f"{n} bases need ~{(n * 304) / 2**30:.0f} GiB, the GPU has {torch.cuda.mem_get_info()[0] / 2**30:.1f} GiB free")
    c = Context(gpu_lib, 0, 0, 1)
    buf = torch.empty((n, 104), dtype=torch.uint8, device=DEV)
    c.gen_bases_into(SEED, n, buf.data_ptr())
    with pytest.raises(DpError) as e:
        c.init_ptr(buf.data_ptr(), n, 1 << 4, 1 << 7)
    assert e.value.code == -1 and "DP_MSM_PRE_C" in str(e.value), str(e.value)
    del buf
    c.close()
    if not DRY:
        torch.cuda.empty_cache()
