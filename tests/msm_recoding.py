"""Scalars at the edges of the MSM's signed-digit recoding, shared by the emulator and GPU files that pin the width of the
window-multiple table (tests/test_msm_geometry.py, tests/test_zzzzzzzzzz_gpu_msm_geometry.py)."""
import numpy as np

from tests.common import R_MOD, u256


def recoding_edge_scalars(c: int) -> dict:
    """Canonical scalars at the edges of the signed-digit recoding with c-bit windows (msm.cuh for_each_digit: a window's
    raw value plus the carry in becomes a digit in [-2^(c-1), 2^(c-1)]; above 2^(c-1) it is negative and carries).
    The top window of a canonical scalar never reaches 2^(c-1), even after a carry (r's top window is below 2^(c-1) - 1
    for every c in 8..22), so none of these may set the carry-out error."""
    nw = (256 + c - 1) // c
    assert (R_MOD >> (c * (nw - 1))) + 1 < 1 << (c - 1)
    low = [w for w in range(nw) if c * w + c - 1 < 254]        # windows whose bit c-1 lies below 2^254 < r
    half = sum(1 << (c * w + c - 1) for w in low)
    T = c * ((R_MOD.bit_length() - 1) // c)                     # the window that holds r's top bit
    edges = {
        "every window 2^(c-1)": half,                           # the largest positive digit, no carry anywhere
        "every window 2^(c-1)+1": sum(((1 << (c - 1)) + 1) << (c * w) for w in low),   # negative digits, carries
        "carry makes every window 2^(c-1)+1": half + 1,         # window 0 carries into 2^(c-1) above it, and so on up
        "2^(ck)-1": (1 << (c * (254 // c))) - 1,                # raw 2^c - 1 + carry = 2^c: digit 0, carry through every window
        "r-1": R_MOD - 1,
        "r-2": R_MOD - 2,
        "carry into the top window": ((R_MOD >> T) << T) - 1,   # largest canonical scalar whose low windows all carry
    }
    for name, v in edges.items():
        assert 0 < v < R_MOD, (c, name)
    return edges


def place_recoding_edges(c: int, n: int, seed: int, per_edge: int, background=None):
    """n scalars: `background` (zeros when None) with every recoding edge of width c written into per_edge slots.  The slots
    depend on (n, seed, per_edge) only, not on c.  Returns (scalars, slots)."""
    edges = list(recoding_edge_scalars(c).values())
    slots = np.random.default_rng(seed).choice(n, size=len(edges) * per_edge, replace=False)
    sc = np.zeros((n, 4), dtype=np.uint64) if background is None else np.array(background[:n], dtype=np.uint64)
    for k, v in enumerate(edges):
        sc[slots[k * per_edge:(k + 1) * per_edge]] = u256(v)
    return sc, slots
