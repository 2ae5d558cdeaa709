#!/usr/bin/env python
"""The setup ceremony (DESIGN.md section 3.10): one contribution to an SRS of 2^L + 3 points.  Prints one JSON line.

    python tools/bench_srs_update.py --log-n 22
    python tools/bench_srs_update.py --log-n 24

Before anything is timed: dp_srs_update of universal_setup(tau) with a fixed s, to device memory and to host memory, must
equal dp_g1_compress(dp_srs_powers_of_tau(tau s)) byte for byte, its G2 outputs dp_srs_open_key(s) and (tau s), and the
plain 255-bit double-and-add (dp_debug_srs_update_plain) must give the same bytes; else exit code 3.
Then, each a host clock around a call that ends in a device synchronise, median of --steps calls after one warm-up:
  * update                 dp_srs_update to a device buffer and to host memory, and dp_debug_srs_update_plain to the
                           device buffer: the method comparison that fixed the kernel
  * contribute             srs.contribute end to end (load_srs with all checks, the update into a memory map, the receipt)
                           from a file on local disk to another, in a fresh context each time: the 2nd and 3rd of the chain
  * load_ceremony_srs      for the final file of a chain of 3 contributions, in a fresh context each time
It fails without a GPU."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import gpu_identity  # noqa: E402

TAU = 0x6A09E667F3BCC908B2FB1366EA957D3E3ADEC17512775099DA2F590B0667322A
S = 0x3C6EF372FE94F82BA54FF53A5F1D36F1510E527FADE682D19B05688C2B3E6C1F


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
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_srs_update.py measures on a GPU: none is available")

    import distributed_plonk_b200 as dp
    from distributed_plonk_b200.srs import ceremony_start, contribute, load_ceremony_srs, universal_setup
    from distributed_plonk_b200.transcript import R_MOD

    lib = dp.load()
    n_gates = 1 << args.log_n
    n = n_gates + 3
    line = {"metric": "srs_update", "points": n, "steps": args.steps, "gpu": gpu_identity(0)}
    a = dp.Context(lib, 0, 0, 1)
    universal_setup(a, torch, n - 1, n_gates, 8 * n_gates, tau=TAU)
    g2 = a.srs_open_key(TAU)
    t = TAU * S % R_MOD
    ref = torch.empty((n, 104), dtype=torch.uint8, device="cuda")
    a.srs_powers_of_tau_into(t, n, ref.data_ptr())
    want = torch.empty((n, 48), dtype=torch.uint8, device="cuda")
    a._ck(lib.dp_g1_compress(a.h, ref.data_ptr(), n, want.data_ptr()))
    del ref
    torch.cuda.empty_cache()
    dev = torch.empty((n, 48), dtype=torch.uint8, device="cuda")
    host = np.empty((n, 48), dtype=np.uint8)
    _, g2_dev = a.srs_update(g2, n, S, out48=dev.data_ptr())
    checks = {"device_equals_powers_of_tau_s": bool(torch.equal(dev, want))}
    _, g2_host = a.srs_update(g2, n, S, out48=host)
    want_host = want.cpu().numpy()
    checks["host_equals_powers_of_tau_s"] = bool(np.array_equal(host, want_host))
    checks["g2_equals_open_keys"] = bool(np.array_equal(g2_dev, g2_host) and np.array_equal(g2_host[0], a.srs_open_key(S)[1])
                                         and np.array_equal(g2_host[1], a.srs_open_key(t)[1]))
    a.srs_update(g2, n, S, out48=dev.data_ptr(), plain=True)
    checks["plain_double_and_add_equal"] = bool(torch.equal(dev, want))
    del want, want_host
    line["checks"] = checks
    ok = all(checks.values())
    if ok:
        line["update"] = {
            "glv_to_device_ms": median_ms(lambda: a.srs_update(g2, n, None, out48=dev.data_ptr()), args.steps),
            "glv_to_host_ms": median_ms(lambda: a.srs_update(g2, n, None, out48=host), args.steps),
            "plain_to_device_ms": median_ms(lambda: a.srs_update(g2, n, None, out48=dev.data_ptr(), plain=True), args.steps),
            "what": "whole calls: host power tables, the G2 kernel, the G1 kernel in SRS_CHUNK launches, the copies"}
        line["update"]["plain_over_glv"] = round(line["update"]["plain_to_device_ms"] / line["update"]["glv_to_device_ms"], 2)
    del dev
    a.close()
    torch.cuda.empty_cache()
    if ok:
        with tempfile.TemporaryDirectory() as d:
            paths = [os.path.join(d, f"srs{j}.bin") for j in range(4)]
            ceremony_start(paths[0], n)
            times, receipts = [], []
            for j in range(3):                                       # the first is the warm-up; the chain goes on from it
                c = dp.Context(lib, 0, 0, 1)
                t0 = time.perf_counter()
                receipts.append(contribute(c, paths[j], paths[j + 1], n_gates, 8 * n_gates))
                times.append(time.perf_counter() - t0)
                c.close()
                os.remove(paths[j])
            line["contribute_ms"] = round(1e3 * statistics.median(times[1:]), 1)
            times = []
            for _ in range(args.steps + 1):
                c = dp.Context(lib, 0, 0, 1)
                t0 = time.perf_counter()
                load_ceremony_srs(c, paths[-1], receipts, n_gates, 8 * n_gates)
                times.append(time.perf_counter() - t0)
                c.close()
            line["load_ceremony_srs_ms"] = round(1e3 * statistics.median(times[1:]), 1)
            line["chain_length"] = len(receipts)
    line["what"] = "host clock around each call (every entry ends in a device synchronise), median after a warm-up"
    if not ok:
        line["error"] = "an update differs from the SRS of tau s"
    print(json.dumps(line), flush=True)
    if not ok:
        raise SystemExit(3)


if __name__ == "__main__":
    main()
