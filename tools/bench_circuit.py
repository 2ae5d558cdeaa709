#!/usr/bin/env python
"""The resident prover from a circuit (ResidentProver.load_circuit / prove_witness): the time of the preprocessing, split
into its steps, then prove_witness (witness in, wires gathered on the device) timed alternately against prove (5n wire +
n public-input evaluations in) on one prover.  Prints one JSON line.

    python tools/bench_circuit.py --log-n 22
    python tools/bench_circuit.py --log-n 24 --steps 2 --rounds 1
    python tools/bench_circuit.py --log-n 22 --proof

--proof: proofs a verifier accepts (prove_circuit, challenges from the transcript) instead of the prove_witness / prove
alternation.  First prove_circuit with fixed blinders must equal prove_witness on the challenges it derived with the same
blinders (13 commitments, 10 evaluations; exit code 3 otherwise), then prove_circuit and prove_witness (both blinded by
the library) are timed alternately on one prover, with transcript_ms: the host time inside the transcript per proof.

The circuit is bench_circuit_inputs' synthetic one: num_vars = 4n variables, slots on uniform random variables except the
last n/8 gates, which all hold one padding variable.  Before anything is timed: the identity / sigma evaluations at 4096
sampled slots against a stable-argsort restatement of the wire permutation; three verifying-key commitments (selector 0,
sigmas 0 and 4) against (sum_i c_i t_i) G over the synthetic SRS, whose discrete logs t_i are known; the coefficient forms
at a few points of the gate domain against the evaluations they came from; one prove_witness against prove of the
gathered evaluations, all 13 commitments and 10 evaluations.  A mismatch exits with code 3."""
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

SRS_SEED = 0xC1C5EED


def splitmix_scalars(seed: int, n: int) -> np.ndarray:
    """the discrete logs t_i of dp_debug_gen_bases(seed, n): bases[i] = t_i G"""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (np.arange(n, dtype=np.uint64) + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return z | np.uint64(1)


def succ_argsort(v: np.ndarray) -> np.ndarray:
    order = np.argsort(v, kind="stable")
    keys = v[order]
    head = np.ones(v.shape[0], dtype=bool)
    head[1:] = keys[1:] != keys[:-1]
    first = np.maximum.accumulate(np.where(head, np.arange(v.shape[0]), 0))
    same_next = np.zeros(v.shape[0], dtype=bool)
    same_next[:-1] = ~head[1:]
    succ = np.empty(v.shape[0], dtype=np.int64)
    succ[order] = np.where(same_next, np.roll(order, -1), order[first])
    return succ


def verify(ctx, torch, pr, vk, log_n, wire_vars, witness, ch):
    from oracle import loader as orc
    from distributed_plonk_b200.resident import N_SEL, N_WIRE
    orc.build()
    n, F = 1 << log_n, pr.F
    host = lambda t: t.cpu().numpy().view(np.uint64)
    out = {}
    # identity / sigma at sampled slots
    rng = np.random.default_rng(1)
    slots = np.unique(np.concatenate([rng.integers(0, N_WIRE * n, 4096), [0, n - 1, 4 * n, N_WIRE * n - 1]]))
    succ = succ_argsort(wire_vars)
    idx = torch.as_tensor(slots, device=pr.id_eval.device)
    idv, sig = host(pr.id_eval[idx]), host(pr.sig_eval[idx])
    val = lambda s: F.mul(pr.k[s >> log_n], F.pow_u64(F.omega, int(s) & (n - 1)))
    out["perm_evals"] = all(np.array_equal(idv[j], val(int(s))) and np.array_equal(sig[j], val(int(succ[s]))) for j, s in enumerate(slots))
    # verifying key over known discrete logs
    t, gen = splitmix_scalars(SRS_SEED, n), orc.g1_generator()
    polys = pr.sel_coef + pr.sig_coef
    out["vk_known_logs"] = all(np.array_equal(orc.normalize(vk[j]), orc.g1_mul(gen, orc.fr_dot_u64(orc.into_repr(host(polys[j])), t)))
                               for j in (0, N_SEL, N_SEL + N_WIRE - 1))
    # coefficient forms evaluate back to their evaluations
    ok = True
    for j, p in enumerate(polys):
        ev = pr.sel_eval_check[j] if j < N_SEL else pr.sig_eval[(j - N_SEL) * n:(j - N_SEL + 1) * n]
        for i in (0, 1, n // 3, n - 1):
            ok &= np.array_equal(ctx.poly_eval(p.data_ptr(), F.pow_u64(F.omega, i), n), host(ev[i:i + 1])[0])
    out["coefficient_forms"] = bool(ok)
    # one proof both ways
    com, ev, _ = pr.prove_witness(witness, ch)
    # the wire evaluations stay as gathered; the public input is rebuilt on the host (round 2 transforms pr.pub in place)
    wires = pr.wire_eval.cpu().pin_memory()
    pub_np = np.zeros((n, 4), dtype=np.uint64)
    pub_np[:pr.num_inputs] = witness.numpy().view(np.uint64)[wire_vars[(N_WIRE - 1) * n:(N_WIRE - 1) * n + pr.num_inputs].astype(np.int64)]
    pub = torch.as_tensor(pub_np.view(np.int64)).pin_memory()
    com2, ev2 = pr.prove(wires, pub, ch)
    out["prove_witness_equals_prove"] = len(com + ev) == 23 and all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(com + ev, com2 + ev2))
    return out, (wires, pub)


def proof_leg(torch, pr, witness, args, line) -> bool:
    """--proof: the equality check, then prove_circuit and prove_witness alternately (both blinded by the library)"""
    from distributed_plonk_b200.proof import Proof, fr_from_int
    from distributed_plonk_b200.resident import N_BLIND
    rng = np.random.default_rng(0xB11D)
    fixed = np.stack([fr_from_int(int(rng.integers(1 << 62)) << 180 | int(rng.integers(1 << 62))) for _ in range(N_BLIND)])
    proof, _ = pr.prove_circuit(witness, blind=fixed)
    com, ev, _ = pr.prove_witness(witness, pr.last_challenges, blind=fixed)
    ok = Proof.from_raw(com, ev) == proof
    line["verify"]["prove_circuit_equals_prove_witness"] = bool(ok)
    if not ok:
        line["error"] = "prove_circuit and prove_witness on its challenges disagree"
        return False
    legs, tms = {"prove_circuit": [], "prove_witness": []}, []
    ch = pr.last_challenges
    for _ in range(args.rounds):
        for name in legs:
            fn = (lambda: pr.prove_circuit(witness)) if name == "prove_circuit" else (lambda: pr.prove_witness(witness, ch, blind=True))
            fn()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                fn()
                if name == "prove_circuit":
                    tms.append(pr.last_transcript_ms)
            torch.cuda.synchronize()
            legs[name].append(args.steps / (time.perf_counter() - t0))
    for name, vals in legs.items():
        line[name] = {"proofs_per_s": round(float(np.mean(vals)), 4), "values": [round(v, 4) for v in vals], "blind": True}
    ms_per_proof = 1e3 / line["prove_circuit"]["proofs_per_s"]
    line["transcript_ms"] = {"mean": round(float(np.mean(tms)), 3), "max": round(float(np.max(tms)), 3),
                             "share_of_proof": round(float(np.mean(tms)) / ms_per_proof, 5),
                             "what": "host time inside the transcript per prove_circuit: public inputs, 11 commitments converted "
                                     "to affine and hashed, 10 evaluations, 5 challenges (the verifying-key prefix is hashed once, "
                                     "by load_circuit), plus the proof object; host clock"}
    line["proof_bytes"] = len(proof.to_bytes())
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=22, dest="log_n")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of prove_witness and prove")
    ap.add_argument("--proof", action="store_true", help="time prove_circuit against prove_witness instead (module docstring)")
    args = ap.parse_args()

    import torch

    import distributed_plonk_b200 as dp
    from distributed_plonk_b200 import resident

    log_n = args.log_n
    n, nb = 1 << log_n, (1 << log_n) + 32
    lib = dp.load()
    ctx = dp.Context(lib, 0, 0, 1)
    bases_t = torch.empty((nb, 104), dtype=torch.uint8, device="cuda")
    ctx.gen_bases_into(SRS_SEED, nb, bases_t.data_ptr())        # distinct k_i G everywhere: the discrete logs stay known
    torch.cuda.synchronize()
    ctx.init_ptr(bases_t.data_ptr(), nb, n, 8 * n)
    del bases_t
    torch.cuda.empty_cache()
    gen = torch.Generator(device="cuda")
    gen.manual_seed(0xC1C)

    def rand_fr(count):
        t = torch.randint(-(1 << 63), (1 << 63) - 1, (count, 4), dtype=torch.int64, device="cuda", generator=gen)
        t[:, 3] &= (1 << 62) - 1
        return t

    free0, total = torch.cuda.mem_get_info()
    torch.cuda.reset_peak_memory_stats()
    pr, vk, (witness, ch) = resident.make_bench_circuit(ctx, torch, log_n, rand_fr)
    first_load_ms = dict(pr.load_ms)
    # a second, warm load from selector evaluations kept on the host for the coefficient check
    rng_sel = [rand_fr(n).cpu().numpy().view(np.uint64) for _ in range(resident.N_SEL)]
    wire_vars = resident.bench_circuit_inputs(log_n, pr.num_vars)
    t0 = time.perf_counter()
    vk, _ = pr.load_circuit(rng_sel, wire_vars, pr.num_vars, pr.k, pr.num_inputs)   # timed load, warm
    load_s = time.perf_counter() - t0
    pr.sel_eval_check = [torch.as_tensor(s.view(np.int64)) for s in rng_sel]
    line = {"metric": "circuit_load_and_prove", "log_gates": log_n, "num_vars": pr.num_vars, "steps": args.steps, "gpu": gpu_identity(0),
            "quotient": pr.quotient}
    line["verify"], (wires, pub) = verify(ctx, torch, pr, vk, log_n, wire_vars, witness, ch)
    ok = all(line["verify"].values())
    if ok:
        line["load_circuit"] = {"ms": round(load_s * 1e3, 2), "steps_ms": {k: round(v, 2) for k, v in pr.load_ms.items()},
                                "first_call_ms": {k: round(v, 2) for k, v in first_load_ms.items()},
                                "what": "wire_permutation = sort + successor; perm_evals = identity and sigma evaluations; intt = 18 in-place "
                                        "iNTT(n); commit = the 18 verifying-key commitments (one MSM batch, or one per polynomial when round 3 is sliced); host clock, every step ends in a "
                                        "device synchronise; steps_ms is a second, warm call"}
        legs = {} if args.proof else {"prove_witness": [], "prove": []}
        if args.proof:
            ok = proof_leg(torch, pr, witness, args, line)
        for _ in range(args.rounds):
            for name in legs:
                fn = (lambda: pr.prove_witness(witness, ch)) if name == "prove_witness" else (lambda: pr.prove(wires, pub, ch))
                fn()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    fn()
                torch.cuda.synchronize()
                ctx.sync()
                legs[name].append(args.steps / (time.perf_counter() - t0))
        for name, vals in legs.items():
            line[name] = {"proofs_per_s": round(float(np.mean(vals)), 4), "values": [round(v, 4) for v in vals]}
        if not args.proof:
            line["prove_witness"]["h2d_bytes_per_proof"] = int(pr.num_vars * 32)
            line["prove"]["h2d_bytes_per_proof"] = int((resident.N_WIRE + 1) * n * 32)
        free1, _ = torch.cuda.mem_get_info()
        torch_peak, torch_now = torch.cuda.max_memory_reserved(), torch.cuda.memory_reserved()
        line["device_memory"] = {"peak_gib_bound": round(((total - free1) - torch_now + torch_peak) / 2**30, 3),
                                 "in_use_before_gib": round((total - free0) / 2**30, 3), "device_total_gib": round(total / 2**30, 3),
                                 "how": "device memory in use at the end (the library's pool keeps its peak), minus torch's reserve now, "
                                        "plus torch's peak reserve since the prover was built (an upper bound of the peak)"}
        if ok:
            line["value"] = line["prove_circuit" if args.proof else "prove_witness"]["proofs_per_s"]
    if not ok:
        line.setdefault("error", "the preprocessing or the proof from the witness disagrees with its check")
    print(json.dumps(line), flush=True)
    ctx.close()
    if not ok:
        raise SystemExit(3)


if __name__ == "__main__":
    main()
