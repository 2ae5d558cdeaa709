#!/usr/bin/env python
"""Batch proofs (ResidentProver.prove_batch, DESIGN.md 3.11) against the same number of prove_circuit calls, on one prover.
Prints one JSON line per batch size.

    python tools/bench_batch.py --log-n 22 --batch 4            # K = 4 at 2^22 gates
    python tools/bench_batch.py --log-n 22 --batch 1,2,4,8      # several K on one prover (one setup)
    python tools/bench_batch.py --log-n 23 --batch max          # K = max_batch()

Before anything is timed, over universal_setup at 2^L gates and tests/test_circuit.py's satisfied circuit: a batch of one
with fixed blinders must equal prove_circuit with the same blinders in all 13 commitments and 10 evaluations; a batch of K
must be accepted by verify_batch_proof; the same batch with one evaluation changed must be rejected.  Exit code 3 otherwise.
Then, per K, --steps rounds that alternate one prove_batch(K) with K prove_circuit calls (host clock around each; every
library entry ends in a device synchronise), after one warm-up of each.  Reported: the medians, proofs per second of both,
their ratio, verify_batch_proof's median, device memory in use after the batch (torch's cache and the library's pool keep
their blocks, so this bounds the peak), and the card's name and power limit."""
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


def changed_eval(bp):
    """the batch with instance 0's first wire evaluation + 1"""
    from distributed_plonk_b200.proof import BatchProof, ProofEvaluations
    from distributed_plonk_b200.transcript import R_MOD
    e0 = bp.poly_evals_vec[0]
    bad = ProofEvaluations([(e0.wires_evals[0] + 1) % R_MOD] + list(e0.wires_evals[1:]), e0.wire_sigma_evals, e0.perm_next_eval)
    return BatchProof(bp.wires_poly_comms_vec, bp.prod_perm_poly_comms_vec, [bad] + bp.poly_evals_vec[1:], bp.split_quot_poly_comms,
                      bp.opening_proof, bp.shifted_opening_proof)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22, dest="log_n")
    ap.add_argument("--batch", default="4", help="K, a comma-separated list of K, or 'max' (max_batch())")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--quotient", default="auto", choices=("auto", "whole", "sliced"))
    args = ap.parse_args()

    import torch

    import distributed_plonk_b200 as dp
    from distributed_plonk_b200.resident import N_BLIND, NumpyField, ResidentProver
    from distributed_plonk_b200.srs import open_key, universal_setup
    from distributed_plonk_b200.verifier import verify_batch_proof
    from oracle import loader as orc
    from tests import test_circuit as tc
    orc.build()

    lib = dp.load()
    gpu = gpu_identity(0)
    ctx = dp.Context(lib, 0, 0, 1)
    n = 1 << args.log_n
    tau = universal_setup(ctx, torch, n + 2, n, 8 * n)
    key = open_key(ctx, tau)
    sel, wv, witness, k5 = tc.satisfied_circuit(orc, args.log_n, 0xBA7)
    pr = ResidentProver(ctx, torch, args.log_n, "cuda", NumpyField(args.log_n), quotient=args.quotient)
    pr.load_circuit(sel, wv, witness.shape[0], k5, 3)
    vk = pr.verifying_key()
    wit = tc.witness_host(witness, "cuda")
    blind = orc.gen_fr(0xB1, N_BLIND)
    single, _ = pr.prove_circuit(wit, blind=blind)
    one, _ = pr.prove_batch([wit], blind=[blind])
    cap = pr.max_batch()                                      # after a proof: the library's pool has its scratch by now
    sizes = [cap] if args.batch == "max" else [min(int(x), cap) for x in args.batch.split(",")]
    base = {"metric": "plonk_batch_proof", "log_n": args.log_n, "quotient": pr.quotient, "steps": args.steps, "max_batch": cap,
            "instance_gib": round(pr.instance_bytes() / 2**30, 3), "gpu": gpu}
    ok = True
    for K in sizes:
        line = dict(base, batch=K)
        bp, pubs = pr.prove_batch([wit] * K)
        checks = {"batch_of_one_equals_prove_circuit": one.instance(0) == single,
                  "accepted": verify_batch_proof(ctx, vk, key, pubs, bp),
                  "changed_evaluation_rejected": not verify_batch_proof(ctx, vk, key, pubs, changed_eval(bp))}
        line["checks"] = checks
        if not all(checks.values()):
            ok = False
            line["error"] = "a check failed"
            print(json.dumps(line), flush=True)
            continue
        torch.cuda.synchronize()
        tb, ts = [], []
        for step in range(args.steps + 1):                    # step 0 warms both up
            t0 = time.perf_counter()
            pr.prove_batch([wit] * K)
            t1 = time.perf_counter()
            for _ in range(K):
                pr.prove_circuit(wit)
            t2 = time.perf_counter()
            if step:
                tb.append(t1 - t0)
                ts.append(t2 - t1)
        free, total = torch.cuda.mem_get_info()
        vt = []
        for _ in range(args.steps + 1):
            t0 = time.perf_counter()
            verify_batch_proof(ctx, vk, key, pubs, bp)
            vt.append(time.perf_counter() - t0)
        mb, ms = float(np.median(tb)), float(np.median(ts))
        line.update({
            "batch_ms": round(1e3 * mb, 1), "batch_ms_values": [round(1e3 * t, 1) for t in tb],
            "separate_ms": round(1e3 * ms, 1), "separate_ms_values": [round(1e3 * t, 1) for t in ts],
            "batch_proofs_per_s": round(K / mb, 3), "separate_proofs_per_s": round(K / ms, 3), "speedup": round(ms / mb, 3),
            "verify_batch_proof_ms": round(1e3 * float(np.median(vt[1:])), 2),
            "proof_bytes": {"batch": len(bp.to_bytes()), "separate": 976 * K},
            "device_in_use_gib": round((total - free) / 2**30, 2), "torch_peak_reserved_gib": round(torch.cuda.max_memory_reserved() / 2**30, 2),
            "what": "medians over --steps rounds that alternate prove_batch(K) with K prove_circuit calls on one prover, blinded "
                    "with library-drawn scalars; host clock; device_in_use after the batch bounds the peak"})
        print(json.dumps(line), flush=True)
    ctx.close()
    if not ok:
        raise SystemExit(3)


if __name__ == "__main__":
    main()
