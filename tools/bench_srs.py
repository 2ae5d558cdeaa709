#!/usr/bin/env python
"""The KZG setup on the GPU (dp_srs_powers_of_tau: [tau^i] G1, i < 2^L + 3, the bases a blinded 2^L-gate prover needs).
Prints one JSON line.

    python tools/bench_srs.py --log-n 24
    python tools/bench_srs.py --log-n 22 --prove
    python tools/bench_srs.py --log-n 20 --cpu

Before anything is timed, the points are checked (tests/test_zzzzzzzzz_gpu_srs.py: check_device_srs): the library's
commitment of a random polynomial with 2^L + 3 coefficients over the generated SRS equals p(tau) G, which involves every
point, and 64 sampled points (0, 1, n - 1, both sides of every launch chunk, random ones) equal tau^i G.  A mismatch
exits with code 3.  Then dp_srs_powers_of_tau into device memory is timed: one warm-up call (which builds the context's
fixed-base table), then --steps calls, host clock around a device synchronise.

--cpu: also times the oracle's gen_srs (oracle/c/ark_oracle.c) at the same size on every host thread.  That is a
restatement by 256-bit double-and-add per point, not arkworks' FixedBase windowed multiplication that jf-plonk's
universal_setup uses, so it is a bound on what a plain CPU loop costs, not the reference's time.

--prove: universal_setup (fresh tau, SRS freed before the prover is built), then tests/test_circuit.py's satisfied
circuit at 2^L gates, load_circuit and two prove_circuit calls blinded by the library; the verifier
(tests/plonk_verifier.py, with the trapdoor) must accept both (exit code 3 otherwise)."""
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

WINDOW_BITS = 16                 # SRS_C in csrc/srs.cuh
TAU = 0x1B4D5E6F708192A3B4C5D6E7F8091A2B3C4D5E6F708192A3B4C5D6E7F80912


def prove_leg(orc, torch, ctx, log_n: int, line: dict) -> bool:
    from distributed_plonk_b200.srs import universal_setup
    from distributed_plonk_b200.resident import NumpyField, ResidentProver
    from tests import plonk_verifier as pv
    from tests import test_circuit as tc
    n = 1 << log_n
    t0 = time.perf_counter()
    tau = universal_setup(ctx, torch, n + 2, n, 8 * n)
    setup_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    sel, wv, witness, k = tc.satisfied_circuit(orc, log_n, 0x5E7)
    build_s = time.perf_counter() - t0
    pr = ResidentProver(ctx, torch, log_n, "cuda", NumpyField(log_n))
    t0 = time.perf_counter()
    pr.load_circuit(sel, wv, witness.shape[0], k, 3)
    torch.cuda.synchronize()
    load_s = time.perf_counter() - t0
    del sel, wv
    wit = tc.witness_host(witness, "cuda")
    vk, ok, proof_s = pr.verifying_key(), True, []
    for _ in range(2):
        t0 = time.perf_counter()
        proof, pub = pr.prove_circuit(wit)
        torch.cuda.synchronize()
        proof_s.append(time.perf_counter() - t0)
        ok &= bool(pv.verify(orc, vk, pub, proof, tau))
    line["verify"]["full_size_proof_verifies"] = ok
    line["prove"] = {"log_gates": log_n, "quotient": pr.quotient, "universal_setup_ms": round(setup_s * 1e3, 1),
                     "circuit_build_on_host_s": round(build_s, 2), "load_circuit_ms": round(load_s * 1e3, 1),
                     "prove_circuit_ms": [round(s * 1e3, 1) for s in proof_s],
                     "what": "universal_setup = generate 2^L + 3 points on the device + dp_init from them; load_circuit and each "
                             "prove_circuit (blinded by the library) end in a device synchronise; host clock"}
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22, dest="log_n")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--cpu", action="store_true", help="also time the oracle's double-and-add gen_srs on every host thread")
    ap.add_argument("--prove", action="store_true", help="universal_setup, then a full-size proof the verifier must accept")
    args = ap.parse_args()

    import torch

    import distributed_plonk_b200 as dp
    from oracle import loader as orc
    from tests.test_zzzzzzzzz_gpu_srs import check_device_srs
    orc.build()

    n = (1 << args.log_n) + 3
    ctx = dp.Context(dp.load(), 0, 0, 1)
    line = {"metric": "srs_powers_of_tau", "log_n": args.log_n, "points": n, "window_bits": WINDOW_BITS, "steps": args.steps,
            "gpu": gpu_identity(0)}
    line["verify"] = check_device_srs(orc, ctx, TAU, n, "cuda", 0x5125)
    ok = line["verify"]["kzg_identity"] and line["verify"]["sampled_points"]
    if ok:
        out = torch.empty((n, 104), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ctx.srs_powers_of_tau_into(TAU, n, out.data_ptr())           # warm-up, builds the table
        first_ms = 1e3 * (time.perf_counter() - t0)
        times = []
        for _ in range(args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ctx.srs_powers_of_tau_into(TAU, n, out.data_ptr())
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        del out
        torch.cuda.empty_cache()
        windows = (256 + WINDOW_BITS - 1) // WINDOW_BITS
        ms = 1e3 * float(np.median(times))
        line["gpu_ms"] = {"median": round(ms, 3), "min": round(1e3 * min(times), 3), "values": [round(1e3 * t, 3) for t in times],
                          "first_call": round(first_ms, 3)}
        line["points_per_s"] = round(n / (ms / 1e3), 1)
        line["mixed_adds_per_s"] = round(n * windows / (ms / 1e3), 1)
        line["what"] = (f"one dp_srs_powers_of_tau call into device memory, host clock around a device synchronise; mixed additions "
                        f"counted as n * {windows} (one per {WINDOW_BITS}-bit signed digit; a zero digit, probability 2^-{WINDOW_BITS}, "
                        "skips one); the fixed-base table is built by the warm-up call and kept by the context, so it is not in the time")
        if args.cpu:
            orc.set_num_threads(os.cpu_count() or 1)
            t0 = time.perf_counter()
            orc.gen_srs(np.frombuffer(TAU.to_bytes(32, "little"), dtype=np.uint64), n)
            cpu_s = time.perf_counter() - t0
            line["cpu_oracle"] = {"s": round(cpu_s, 3), "threads": os.cpu_count(), "speedup_of_gpu": round(cpu_s * 1e3 / ms, 1),
                                  "what": "oracle/c gen_srs at the same size: one 256-bit double-and-add per point on every host "
                                          "thread; a restatement, not arkworks' FixedBase"}
        if args.prove:
            ok = prove_leg(orc, torch, ctx, args.log_n, line)
    if not ok:
        line["error"] = "the generated SRS or the proof over it failed its check"
    print(json.dumps(line), flush=True)
    ctx.close()
    if not ok:
        raise SystemExit(3)


if __name__ == "__main__":
    main()
