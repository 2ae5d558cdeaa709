#!/usr/bin/env python
"""Resident prover (distributed_plonk_b200/resident.py) on its own, at any size that fits one GPU: the round-3 layout it
picks, its proofs/s and its peak device memory, and at log_n <= 22 the whole-domain and the sliced round 3 on one prover,
timed alternately (DESIGN.md 3.4).  Prints one JSON line.

    python tools/bench_resident.py --log-n 24 --steps 2
    python tools/bench_resident.py --log-n 22 --steps 3            # + e2e_resident_sliced, alternated with whole
    python tools/bench_resident.py --log-n 24 --zk                 # blinded (e2e_resident_zk) and unblinded, alternated

Before anything is timed: one seeded slice transform (dp_ntt_dev_quot_slice) at a few positions against the oracle's
O(n) Horner evaluation, and at log_n <= 22 the 13 commitments and 10 evaluations of both layouts compared byte for byte.
With --zk, instead of the two layouts: a proof with all-zero blinders must equal the unblinded proof in all 13 commitments
and 10 evaluations, then blinded proofs (the library draws the 13 scalars) and unblinded ones are timed alternately on one
prover in its chosen layout.  A mismatch exits with code 3.  Set-up as bench.py's (synthetic SRS generated on the GPU, dp_init's own MSM tuning), with
nothing else allocated: no schedule buffers, no host-buffer leg, no CPU baseline."""
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

from bench import GEN_SEED, gpu_identity  # noqa: E402


def check_slice_ntt(torch, ctx, log_n, rand_fr):
    """slice 5 of 8 of a seeded polynomial at a few positions i against the oracle at g * omega_m^(5 + 8 i)"""
    from oracle import loader as orc
    orc.build()
    n, m, k = 1 << log_n, 8 << log_n, 5
    g = torch.Generator(device="cuda")
    g.manual_seed(0x511CE)
    p = rand_fr(n, g)
    out = torch.empty_like(p)
    torch.cuda.synchronize()
    ctx.ntt_dev_quot_slice(p.data_ptr(), n, k, out.data_ptr())
    idx = sorted({0, 1, (7919 * 13) % n, n // 2 + 1, n - 1})
    got = out[idx].cpu().numpy().view(np.uint64)
    want = orc.ntt_outputs_at(p.cpu().numpy().view(np.uint64), m, np.array([k + 8 * i for i in idx], dtype=np.uint64), False, True)
    return bool(np.array_equal(got, want))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22, dest="log_n")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the two layouts (log_n <= 22) or of blinded and unblinded (--zk)")
    ap.add_argument("--zk", action="store_true", help="time blinded (zero-knowledge) against unblinded proofs instead of the layouts")
    args = ap.parse_args()

    import torch

    import distributed_plonk_b200 as dp
    from distributed_plonk_b200 import resident

    log_n = args.log_n
    n, nb = 1 << log_n, (1 << log_n) + 32
    lib = dp.load()
    ctx = dp.Context(lib, 0, 0, 1)
    bases_t = torch.empty((nb, 104), dtype=torch.uint8, device="cuda")
    ctx.gen_bases_into(GEN_SEED, nb, bases_t.data_ptr())
    inf = torch.zeros(104, dtype=torch.uint8, device="cuda")
    inf[96] = 1
    bases_t[3] = inf
    bases_t[n:] = inf
    torch.cuda.synchronize()
    ctx.init_ptr(bases_t.data_ptr(), nb, n, 8 * n)
    del bases_t, inf
    gen = torch.Generator(device="cuda")
    gen.manual_seed(0xB200)

    def rand_fr(count, g=gen):
        t = torch.randint(-(1 << 63), (1 << 63) - 1, (count, 4), dtype=torch.int64, device="cuda", generator=g)
        t[:, 3] &= (1 << 62) - 1
        return t

    def timed(fn, steps, warmup, device_events=False):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        ctx.sync()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
        ctx.sync()
        return time.perf_counter() - t0, 0

    line = {"metric": "resident_proofs_per_sec", "value": None, "unit": "proofs/s", "log_gates": log_n, "steps": args.steps,
            "gpu": gpu_identity(0), "verify": {"slice_ntt_horner": check_slice_ntt(torch, ctx, log_n, rand_fr)}}
    ok = line["verify"]["slice_ntt_horner"]
    if ok:
        torch.cuda.empty_cache()
        prover = resident.make_bench_prover(ctx, torch, log_n, rand_fr)
        pr, (wires, pub, ch) = prover
        line["chosen"] = pr.quotient
        modes = ["whole", "sliced"] if log_n <= 22 and pr.quotient == "whole" and not args.zk else [pr.quotient]
        if args.zk:
            plain = pr.prove(wires, pub, ch)
            zero = pr.prove(wires, pub, ch, blind=np.zeros((resident.N_BLIND, 4), dtype=np.uint64))
            ok = len(plain[0] + plain[1]) == 23 and all(np.array_equal(np.asarray(a), np.asarray(b))
                                                         for a, b in zip(plain[0] + plain[1], zero[0] + zero[1]))
            line["verify"]["zero_blinders_equal_unblinded"] = ok
            if ok:
                legs = {False: [], True: []}
                for _ in range(args.rounds):                              # unblinded, blinded, unblinded, blinded, ...
                    for b in (False, True):
                        legs[b].append(resident.bench_leg(ctx, torch, log_n, rand_fr, timed, args.steps, prover=prover, blind=b))
                for b, rs in legs.items():
                    dt, st = sum(r["steps"] / r["value"] for r in rs), sum(r["steps"] for r in rs)
                    line["e2e_resident_zk" if b else "e2e_resident"] = dict(rs[-1], value=st / dt, ms_per_step=dt / st * 1e3, steps=st,
                                                                            values=[r["value"] for r in rs])
                line["value"] = line["e2e_resident"]["value"]
                line["zk_cost"] = {"slowdown": round(line["e2e_resident"]["value"] / line["e2e_resident_zk"]["value"] - 1, 4),
                                   "what": "unblinded proofs/s over blinded proofs/s, minus 1, alternated on one prover"}
        elif len(modes) == 2:
            outs = {}
            for mode in modes:
                pr.quotient = mode
                com, ev = pr.prove(wires, pub, ch)
                outs[mode] = [np.asarray(x) for x in com + ev]
            ok = len(outs["whole"]) == 23 and all(np.array_equal(a, b) for a, b in zip(outs["whole"], outs["sliced"]))
            line["verify"]["resident_sliced_equals_whole"] = ok
        if ok and not args.zk:
            legs = {mode: [] for mode in modes}
            for _ in range(args.rounds if len(modes) == 2 else 1):     # whole, sliced, whole, sliced, ...
                for mode in modes:
                    pr.quotient = mode
                    legs[mode].append(resident.bench_leg(ctx, torch, log_n, rand_fr, timed, args.steps, prover=prover))
            for mode, rs in legs.items():
                dt, st = sum(r["steps"] / r["value"] for r in rs), sum(r["steps"] for r in rs)
                key = "e2e_resident" if mode == line["chosen"] else "e2e_resident_" + mode
                line[key] = dict(rs[-1], value=st / dt, ms_per_step=dt / st * 1e3, steps=st, values=[r["value"] for r in rs])
            line["value"] = line["e2e_resident"]["value"]
    if not ok:
        line["error"] = ("a proof with zero blinders differs from the unblinded proof" if args.zk and "zero_blinders_equal_unblinded" in line["verify"]
                         else "the sliced resident prover disagrees with the oracle or with the whole-domain prover")
    print(json.dumps(line), flush=True)
    ctx.close()
    if not ok:
        raise SystemExit(3)


if __name__ == "__main__":
    main()
