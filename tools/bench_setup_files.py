#!/usr/bin/env python
"""Setup files (DESIGN.md section 3.9): encoding, decoding and checking an SRS of 2^L + 3 points.  Prints one JSON line.

    python tools/bench_setup_files.py --log-n 22
    python tools/bench_setup_files.py --log-n 24

Before anything is timed: universal_setup, dp_get_bases_compressed of every point, dp_init_compressed of those bytes in a
second context, whose dp_get_bases must equal the first context's (sampled blocks), dp_srs_check must accept it and
refuse the open key of another tau, and the G2 pair must survive dp_g2_compress -> dp_g2_decompress; else exit code 3.
Then, each a host clock around a call that ends in a device synchronise, median of --steps calls after one warm-up:
  * get_bases_compressed   all points to host memory, and to a device buffer: the second is the kernel with its staging
                           copy and is reported as bytes/s against the 96 B read + 48 B written per point
  * init_compressed        dp_init_compressed from host memory with and without the subgroup check (one call each: the
                           check is a 255-bit scalar multiplication per point)
  * srs_check              total and dp_last_srs_check's split into scalar generation, the two MSMs and the pairing
  * g2                     dp_g2_compress and dp_g2_decompress (with the subgroup check) of the two points of a file
It fails without a GPU."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import gpu_identity  # noqa: E402

TAU = 0x5BE0CD19137E2179A54FF53A5F1D36F1510E527FADE682D19B05688C2B3E6C1F


def median_ms(fn, steps: int) -> float:
    fn()
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return round(1e3 * float(np.median(times)), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22, dest="log_n")
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_setup_files.py measures on a GPU: none is available")

    import distributed_plonk_b200 as dp
    from distributed_plonk_b200.srs import universal_setup

    lib = dp.load()
    n_gates = 1 << args.log_n
    n = n_gates + 3
    line = {"metric": "setup_files", "points": n, "steps": args.steps, "gpu": gpu_identity(0)}
    a = dp.Context(lib, 0, 0, 1)
    universal_setup(a, torch, n - 1, n_gates, 8 * n_gates, tau=TAU)
    g2 = a.srs_open_key(TAU)
    comp = a.get_bases_compressed(0, n)
    b = dp.Context(lib, 0, 0, 1)
    t0 = time.perf_counter()
    b.init_compressed(comp, n_gates, 8 * n_gates, check_subgroup=False)
    init_unchecked_ms = 1e3 * (time.perf_counter() - t0)
    blocks = [0, n // 3, n - 4096] if n > 8192 else [0]
    m = min(n, 4096)
    g2_back = b.g2_decompress(b.g2_compress(g2))
    checks = {
        "bases_round_trip": all(np.array_equal(a.get_bases(s, m), b.get_bases(s, m)) for s in blocks),
        "srs_check_accepts": b.srs_check(g2),
        "srs_check_refuses_another_tau": not b.srs_check(a.srs_open_key(TAU + 1)),
        "g2_round_trip": bool(np.array_equal(g2_back, g2)),
    }
    line["checks"] = checks
    ok = all(checks.values())
    if ok:
        dev = torch.empty((n, 48), dtype=torch.uint8, device="cuda")
        to_dev = median_ms(lambda: b.lib.dp_get_bases_compressed(b.h, 0, n, dev.data_ptr()), args.steps)
        to_host = median_ms(lambda: b.get_bases_compressed(0, n, comp), args.steps)
        line["get_bases_compressed"] = {
            "to_device_ms": to_dev, "to_host_ms": to_host, "needed_bytes": n * (96 + 48),
            "to_device_gb_per_s": round(n * (96 + 48) / (to_dev * 1e-3) / 1e9, 1),
            "what": "needed_bytes = 96 B read + 48 B written per point; the call also copies its 48 B staging chunks to the destination"}
        del dev
        parts = {"scalars_ms": [], "msm_ms": [], "pairing_ms": [], "total_ms": []}
        for i in range(args.steps + 1):
            t0 = time.perf_counter()
            ok &= b.srs_check(g2)
            total = 1e3 * (time.perf_counter() - t0)
            if i:
                last = b.last_srs_check()
                for k in ("scalars_ms", "msm_ms", "pairing_ms"):
                    parts[k].append(last[k])
                parts["total_ms"].append(total)
        line["srs_check"] = {k: round(float(np.median(v)), 3) for k, v in parts.items()}
        enc = b.g2_compress(g2)
        line["g2"] = {"compress_2_ms": median_ms(lambda: b.g2_compress(g2), args.steps),
                      "decompress_2_checked_ms": median_ms(lambda: b.g2_decompress(enc), args.steps)}
        t0 = time.perf_counter()
        b.init_compressed(comp, n_gates, 8 * n_gates, check_subgroup=True)
        line["init_compressed"] = {"unchecked_ms": round(init_unchecked_ms, 1), "subgroup_checked_ms": round(1e3 * (time.perf_counter() - t0), 1),
                                   "what": "one call each from pageable host memory, dp_init's table build and MSM tuning included"}
    a.close()
    b.close()
    line["what"] = "host clock around each call (every entry ends in a device synchronise), median after a warm-up"
    if not ok:
        line["error"] = "a round trip or a check failed"
    print(json.dumps(line), flush=True)
    if not ok:
        raise SystemExit(3)


if __name__ == "__main__":
    main()
