#!/usr/bin/env python
"""The verifier without the trapdoor (distributed_plonk_b200/verifier.py): one dp_multi_pairing, verify per proof and
batch_verify per proof.  Prints one JSON line.

    python tools/bench_verify.py                    # proofs at 2^16 gates
    python tools/bench_verify.py --big-log-n 22     # also one 2^22-gate proof over a generated SRS

Before anything is timed: universal_setup at 2^L gates, open_key of the same tau, tests/test_circuit.py's satisfied
circuit, 8 proofs blinded by the library; verify must accept every one (also after proof_from_bytes) and reject the
first with one evaluation changed, batch_verify must accept the 8 and reject them with that proof in the middle, else
exit code 3.  Then, each a host clock around the call (every entry ends in a device synchronise), median of --steps
calls after one warm-up:
  * pairing_k2_ms        one dp_multi_pairing of 2 pairs (what verify calls)
  * verify_ms            verify per proof, split into decode (proof_from_bytes: 13 points decompressed and
                         subgroup-checked on the GPU), transcript_scalars (merlin transcript and the Fr scalars, host),
                         msm (the two dp_msm_points calls) and pairing
  * batch_verify_ms      batch_verify of k proofs, k = 1, 8, 64, 256, total and per proof; the batches repeat the 8
                         distinct proofs (every item is still hashed and folded on its own)
--big-log-n L': universal_setup, load_circuit and one prove_circuit at 2^L' gates; verify must accept the proof and
reject it with one evaluation changed (exit code 3 otherwise)."""
from __future__ import annotations

import argparse
import json
import os
import secrets
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import gpu_identity  # noqa: E402


def tampered(proof):
    from distributed_plonk_b200.proof import Proof
    from distributed_plonk_b200.transcript import R_MOD
    ev = proof.evaluations()
    ev[0] = (ev[0] + 1) % R_MOD
    c = proof.commitments()
    return Proof(c[0:5], c[5], c[6:11], c[11], c[12], ev[0:5], ev[5:9], ev[9])


def median_ms(fn, steps: int) -> tuple:
    fn()
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return round(1e3 * float(np.median(times)), 3), [round(1e3 * t, 3) for t in times]


def circuit_prover(orc, torch, ctx, log_n: int):
    from distributed_plonk_b200.resident import NumpyField, ResidentProver
    from tests import test_circuit as tc
    sel, wv, witness, k = tc.satisfied_circuit(orc, log_n, 0x7E1)
    pr = ResidentProver(ctx, torch, log_n, "cuda", NumpyField(log_n))
    pr.load_circuit(sel, wv, witness.shape[0], k, 3)
    return pr, tc.witness_host(witness, "cuda")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=16, dest="log_n")
    ap.add_argument("--big-log-n", type=int, default=0, dest="big_log_n")
    ap.add_argument("--steps", type=int, default=7)
    args = ap.parse_args()

    import torch

    import distributed_plonk_b200 as dp
    from distributed_plonk_b200.srs import open_key, universal_setup
    from distributed_plonk_b200.proof import g2_to_raw, point_to_raw
    from distributed_plonk_b200.verifier import batch_verify, proof_from_bytes, verify
    from oracle import loader as orc
    orc.build()

    lib = dp.load()
    line = {"metric": "plonk_verify", "log_n": args.log_n, "steps": args.steps, "gpu": gpu_identity(0)}
    ctx = dp.Context(lib, 0, 0, 1)
    n = 1 << args.log_n
    tau = universal_setup(ctx, torch, n + 2, n, 8 * n)
    ok_key = open_key(ctx, tau)
    pr, wit = circuit_prover(orc, torch, ctx, args.log_n)
    vk = pr.verifying_key()
    proofs = [pr.prove_circuit(wit) for _ in range(8)]
    encoded = [p.to_bytes() for p, _ in proofs]
    checks = {
        "all_accepted": all(verify(ctx, vk, ok_key, pub, p) for p, pub in proofs),
        "all_accepted_after_decoding": all(verify(ctx, vk, ok_key, pub, proof_from_bytes(ctx, b)) for (_, pub), b in zip(proofs, encoded)),
        "tampered_rejected": not verify(ctx, vk, ok_key, proofs[0][1], tampered(proofs[0][0])),
        "batch_accepted": batch_verify(ctx, ok_key, [(vk, pub, p) for p, pub in proofs]),
        "batch_with_tampered_rejected": not batch_verify(ctx, ok_key, [(vk, pub, tampered(p) if i == 4 else p) for i, (p, pub) in enumerate(proofs)]),
    }
    line["checks"] = checks
    ok = all(checks.values())
    if ok:
        g1 = np.frombuffer(point_to_raw(ok_key.g) * 2, dtype=np.uint8).reshape(2, 104)
        g2 = np.frombuffer(g2_to_raw(ok_key.beta_h) + g2_to_raw(ok_key.h), dtype=np.uint8).reshape(2, 200)
        med, vals = median_ms(lambda: ctx.multi_pairing(g1, g2), args.steps)
        line["pairing_k2_ms"] = {"median": med, "values": vals}
        parts = {"decode_ms": [], "transcript_scalars_ms": [], "msm_ms": [], "pairing_ms": [], "total_ms": []}
        for i in range(args.steps + 1):
            b, pub = encoded[i % 8], proofs[i % 8][1]
            t = {}
            t0 = time.perf_counter()
            p = proof_from_bytes(ctx, b)
            t["decode_ms"] = 1e3 * (time.perf_counter() - t0)
            ok &= verify(ctx, vk, ok_key, pub, p, t)
            t["total_ms"] = 1e3 * (time.perf_counter() - t0)
            if i:                                                        # the first is the warm-up
                for k, v in t.items():
                    parts[k].append(v)
        line["verify_ms"] = {k: round(float(np.median(v)), 3) for k, v in parts.items()}
        line["batch_verify_ms"] = {}
        for k in (1, 8, 64, 256):
            items = [(vk, proofs[i % 8][1], proofs[i % 8][0]) for i in range(k)]
            res = []
            med, vals = median_ms(lambda: res.append(batch_verify(ctx, ok_key, items)), max(3, args.steps // 2) if k >= 64 else args.steps)
            ok &= all(res)
            line["batch_verify_ms"][str(k)] = {"total": med, "per_proof": round(med / k, 3)}
    del pr, wit
    ctx.close()
    torch.cuda.empty_cache()
    if ok and args.big_log_n:
        ctx = dp.Context(lib, 0, 0, 1)
        big = 1 << args.big_log_n
        t0 = time.perf_counter()
        tau = universal_setup(ctx, torch, big + 2, big, 8 * big)
        setup_s = time.perf_counter() - t0
        key = open_key(ctx, tau)
        pr, wit = circuit_prover(orc, torch, ctx, args.big_log_n)
        t0 = time.perf_counter()
        proof, pub = pr.prove_circuit(wit)
        prove_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        accepted = verify(ctx, pr.verifying_key(), key, pub, proof_from_bytes(ctx, proof.to_bytes()))
        verify_s = time.perf_counter() - t0
        rejected = not verify(ctx, pr.verifying_key(), key, pub, tampered(proof))
        line["big"] = {"log_gates": args.big_log_n, "accepted": accepted, "tampered_rejected": rejected,
                       "universal_setup_ms": round(setup_s * 1e3, 1), "prove_circuit_ms": round(prove_s * 1e3, 1),
                       "decode_and_verify_ms": round(verify_s * 1e3, 3)}
        ok &= accepted and rejected
        del pr, wit
        ctx.close()
    line["what"] = ("host clock around each call (every library entry ends in a device synchronise), median after a warm-up; "
                    "verify_ms splits one decode + verify; the batches repeat 8 distinct proofs")
    if not ok:
        line["error"] = "a proof was not accepted or a tampered one was"
    print(json.dumps(line), flush=True)
    if not ok:
        raise SystemExit(3)


if __name__ == "__main__":
    main()
