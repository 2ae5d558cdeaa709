"""One TurboPlonk proof's polynomial arithmetic with every polynomial RESIDENT on the worker.

What the reference's dispatcher does between its worker calls (src/dispatcher2.rs:192-713) - and ships
every polynomial over the wire for, twice per transform - restated over the worker-resident entries of
the C ABI (SURVEY.md 8f-1; the schema already declares round3*/round4*/round5* RPCs for exactly this,
src/hello_world.capnp:26-44, the worker implements none of them).  The witness (wire and public-input
evaluations) goes in once; 13 commitments and 10 evaluations come back:

  round 1  5 x (iNTT(n) -> commit)                                        dispatcher2.rs:294-321
  round 2  grand product -> iNTT(n) -> commit                             329-361
  round 3  25 x coset-NTT(8n) of n coefficients, quotient evaluations,    363-532
           coset-iNTT(8n), 5 commitments of the (n+2)-coefficient chunks
  round 4  10 evaluations at zeta / zeta*omega                            535-555
  round 5  linearisation and batch polynomials, two divisions by          557-690
           (X - point), 2 commitments

prove(..., blind=True) blinds as the reference prover does (dispatcher2.rs:294-361), which makes the proof
zero-knowledge: every wire gets + (b_0 + b_1 X) * Z_H and z gets + (b_0 + b_1 X + b_2 X^2) * Z_H (dp_poly_blind_dev,
13 secret scalars drawn inside the library), so they have n + 2 and n + 3 coefficients, and the quotient has degree
5(n+1)+2 on a satisfied circuit, the degree the reference's split_quot_polys requires.  Round 3 still transforms the
first n coefficients of each polynomial; the quotient kernel adds x^n * tail(x) for the last 2 or 3 (DESIGN.md 3.4).
blind=False (the default) leaves the proof unblinded, the computation as before.

prove_circuit derives the challenges itself: a Fiat-Shamir transcript (transcript.py: merlin over Strobe-128 / Keccak, fed
what the reference's FakeStandardTranscript feeds it, dispatcher2.rs:44-154) of the verifying key, the public inputs and
each round's commitments and evaluations, so it returns a Proof (proof.py) that a PLONK verifier accepts; blinded by
default.  The hashing is host work on a few kilobytes; the verifying-key prefix is hashed once per load_circuit.
prove and prove_witness still take the challenges as inputs (tests, benchmarks), and make the same library calls.
prove_batch proves k witnesses of the loaded circuit with one transcript, one quotient sum_i alpha^(3i) Q_i and one pair of
openings (DESIGN.md 3.11); every path runs the same per-round helpers over a list of instances.
The proving key (13 selector + 5 sigma polynomials in coefficient form, sigma / identity permutation
evaluations) stays resident across proofs, as `State` keeps the bases (worker.rs:42-59).

Buffers are torch tensors (int64 [count, 4] = raw Fr) on the worker's device - or CPU tensors when the
library under test is the kernel-logic emulator, whose "device" memory is host memory.
"""
from __future__ import annotations

import numpy as np

from .proof import Proof, VerifyingKey, fr_from_int, fr_to_int, point_from_jacobian
from .transcript import PlonkTranscript

N_SEL, N_WIRE = 13, 5
N_COEF = N_SEL + 2 * N_WIRE + 2       # polynomials evaluated on the quotient coset in round 3
BLIND_WIRE, BLIND_Z = 2, 3            # blinding scalars of each wire (rand(1) * Z_H) and of z (rand(2) * Z_H)
N_BLIND = N_WIRE * BLIND_WIRE + BLIND_Z


class ResidentProver:
    # Round 3 evaluates 25 polynomials of n coefficients on the m = 8n-point quotient coset.  "whole": 25 buffers of m points
    # (25 x 8n x 32 B: 25 GiB at 2^22), one coset-NTT(8n) each, one quotient launch.  "sliced": the coset is the disjoint union
    # of the 8 gate-domain cosets s_k * H_n (s_k = g * omega_m^k), so round 3 runs slice by slice through 25 n-point buffers:
    # 25 slice transforms (dp_ntt_dev_quot_slice), then the quotient of that slice (dp_quotient_evals_slice_dev), which
    # writes quot[k + 8i].  Same quotient bytes either way.  "auto" takes "whole" when its buffers fit the device's free memory
    # with WHOLE_MARGIN_M quotient-domain buffers (the final iNTT(8n)'s scratch) and WHOLE_MARGIN_BYTES to spare, "sliced"
    # otherwise.  (The cached 1/(x - 1) table of m points is optional: the quotient falls back to its tree variant without it.)
    WHOLE_MARGIN_M, WHOLE_MARGIN_BYTES = 1, 1 << 30
    # prove_batch: device memory left free beside the batch's instances (MSM and quotient scratch), and the emulator's cap
    BATCH_MARGIN_BYTES, CPU_MAX_BATCH = 1 << 30, 64

    def __init__(self, ctx, torch, log_n: int, device: str, field, quotient: str = "auto"):
        """field: helpers over raw Montgomery Fr as np.uint64[4] - mul(a,b), add(a,b), sub(a,b), inv(a), from_u64(v),
        pow_u64(a, e), omega (the generator of the n-point domain); tests and the bench pass the oracle's / numpy ones:
        the handful of scalar challenge products of rounds 4-5 are host-side glue, not hot-path work.
        quotient: "auto" (default), "whole" or "sliced" - how round 3 lays out its evaluations (above)"""
        if quotient not in ("auto", "whole", "sliced"):
            raise ValueError(f"quotient must be 'auto', 'whole' or 'sliced', not {quotient!r}")
        self.ctx, self.torch, self.F = ctx, torch, field
        self.log_n, self.n, self.m = log_n, 1 << log_n, 8 << log_n
        self.dev = device
        n, m = self.n, self.m

        def buf(count):
            return torch.zeros((count, 4), dtype=torch.int64, device=device)

        self.sel_coef = [buf(n) for _ in range(N_SEL)]
        self.sig_coef = [buf(n) for _ in range(N_WIRE)]
        self.sig_eval = buf(N_WIRE * n)
        self.id_eval = buf(N_WIRE * n)
        self.wire_eval = buf(N_WIRE * n)
        self.pub = buf(n)
        # coefficient buffers with room for the blinding tails (prove(blind=...)); unblinded, only the first n are used
        self.wire_coef = [buf(n + BLIND_WIRE) for _ in range(N_WIRE)]
        self.z = buf(n + BLIND_Z)
        self.quot = buf(m)
        self.lin = buf(n + BLIND_Z)
        self.batch = buf(n + BLIND_Z)
        self.wit = [buf(n + 2), buf(n + 2)]
        if quotient == "auto":
            quotient = "whole" if self.whole_fits(torch, device, m) else "sliced"
        self.quotient = quotient
        # coset evaluations: 13 sel, 5 sigma, 5 wires, z, pub.  A whole-domain prover can also run the sliced round 3 (its
        # slice buffers are the heads of the whole-domain ones): tools/bench_resident.py times both modes on one prover that way.
        self.big = [buf(m) for _ in range(N_COEF)] if quotient == "whole" else None
        self.slices = [t[:n] for t in self.big] if self.big is not None else [buf(n) for _ in range(N_COEF)]
        self._own = _Instance(self.wire_eval, self.pub, self.wire_coef, self.z)   # a single proof's instance, instance 0 of a batch
        self._extra = []                                       # prove_batch: instances 1, 2, ... (kept for the next batch)
        self._srs_checked = False
        self.vars = self.witness = None                       # load_circuit: the variable map and the witness buffer
        self.vk = self._vk_transcript = None                  # load_circuit: the verifying key, the transcript after it
        self.last_challenges, self.last_transcript_ms = None, None

    @classmethod
    def whole_fits(cls, torch, device: str, m: int) -> bool:
        """the whole-domain layout fits the device's free memory with the stated margin (always on the CPU emulator)"""
        if device == "cpu":
            return True
        free, _ = torch.cuda.mem_get_info(torch.device(device))
        return (N_COEF + cls.WHOLE_MARGIN_M) * m * 32 + cls.WHOLE_MARGIN_BYTES <= free

    # ---- setup: the proving key, once
    def load_key(self, sel_coef, sig_coef, sig_eval, id_eval, k):
        """selector / sigma polynomials in coefficient form ([n,4] each), sigma and identity permutation evaluations
        ([5][n,4]), the coset representatives k[5]"""
        t = self.torch
        for dst, src in zip(self.sel_coef + self.sig_coef, list(sel_coef) + list(sig_coef)):
            dst.copy_(t.as_tensor(np.ascontiguousarray(src).view(np.int64)))
        self.sig_eval.copy_(t.as_tensor(np.concatenate(sig_eval).view(np.int64)))
        self.id_eval.copy_(t.as_tensor(np.concatenate(id_eval).view(np.int64)))
        self.k = np.ascontiguousarray(k, dtype=np.uint64)

    def load_circuit(self, selector_evals, wire_vars, num_vars: int, k, num_inputs: int):
        """the proving key from a circuit, on the device: selector_evals [13][n,4] raw Fr (evaluations over the gate domain),
        wire_vars [5n] u32 variable ids in slot order (wire type * n + gate), num_vars, the coset representatives k[5] and
        the number of public inputs (the output wires of the first num_inputs gates).  Builds the wire permutation, the
        identity and sigma evaluations, the 13 + 5 coefficient forms (in-place iNTTs) and commits all 18 in one MSM batch
        (one per polynomial in the sliced layout, where memory is short).
        The variable map and a num_vars-entry witness buffer stay resident for prove_witness.  Returns (verifying-key
        commitments: 13 selector + 5 sigma, 144 B each; k).  self.load_ms: milliseconds of each step (host clock; each
        library call returns when its kernels are done)."""
        import time
        t, ctx, n, P = self.torch, self.ctx, self.n, lambda x: x.data_ptr()
        wire_vars = np.ascontiguousarray(wire_vars, dtype=np.uint32)
        if wire_vars.shape != (N_WIRE * n,):
            raise ValueError(f"wire_vars: {N_WIRE * n} u32 variable ids, not shape {wire_vars.shape}")
        if not 0 <= num_inputs <= n:
            raise ValueError(f"num_inputs = {num_inputs} outside 0..n")
        self.k = np.ascontiguousarray(k, dtype=np.uint64)
        for dst, src in zip(self.sel_coef, list(selector_evals)):
            dst.copy_(t.as_tensor(np.ascontiguousarray(src).view(np.int64)))
        self.vars = t.as_tensor(wire_vars.view(np.int32)).to(self.dev)
        self.num_vars, self.num_inputs = int(num_vars), int(num_inputs)
        self.witness = None
        self._sync()
        ms = {}
        t0 = time.perf_counter()
        scratch_bytes = ctx.wire_permutation_scratch_bytes(N_WIRE, n, self.num_vars)
        scratch = t.empty(scratch_bytes, dtype=t.uint8, device=self.dev)
        succ = t.empty(N_WIRE * n, dtype=t.int32, device=self.dev)
        ctx.wire_permutation_dev(P(self.vars), N_WIRE, n, self.num_vars, P(scratch), scratch_bytes, P(succ))
        t1 = time.perf_counter()
        ms["wire_permutation"] = (t1 - t0) * 1e3
        del scratch
        ctx.perm_evals_dev(P(succ), N_WIRE, n, self.k, P(self.id_eval), P(self.sig_eval))
        t2 = time.perf_counter()
        ms["perm_evals"] = (t2 - t1) * 1e3
        del succ
        if self.dev != "cpu":
            t.cuda.empty_cache()                              # the sort scratch goes back to the device, not to torch's cache
        for i in range(N_WIRE):
            self.sig_coef[i].copy_(self.sig_eval[i * n:(i + 1) * n])
        self._sync()
        t3 = time.perf_counter()
        polys = self.sel_coef + self.sig_coef
        for p in polys:
            ctx.ntt_dev(P(p), self.log_n, True, False)
        t4 = time.perf_counter()
        ms["intt"] = (t4 - t3) * 1e3
        # one MSM batch of all 18 holds every job's sort scratch at once: that fits beside the whole-domain layout, which is
        # only chosen with memory to spare; a sliced prover (2^23, 2^24 gates) commits one polynomial per batch
        group = len(polys) if self.quotient == "whole" else 1
        vk = []
        for g0 in range(0, len(polys), group):
            vk += ctx.commit_dev_batch([P(p) for p in polys[g0:g0 + group]], [n] * len(polys[g0:g0 + group]))
        t5 = time.perf_counter()
        ms["commit"] = (t5 - t4) * 1e3
        self.witness = t.zeros((self.num_vars, 4), dtype=t.int64, device=self.dev)
        # the verifying key as a verifier sees it, and the transcript after it: the same prefix for every proof
        pts = [point_from_jacobian(c) for c in vk]
        self.vk = VerifyingKey(n, self.num_inputs, [fr_to_int(x) for x in self.k], pts[:N_SEL], pts[N_SEL:])
        self._vk_transcript = PlonkTranscript()
        self._vk_transcript.append_vk(self.vk)
        ms["vk_transcript"] = (time.perf_counter() - t5) * 1e3
        self.load_ms = ms
        return vk, self.k

    def verifying_key(self) -> VerifyingKey:
        """the verifying key of the circuit given to load_circuit"""
        if self.vk is None:
            raise ValueError("no verifying key: call load_circuit first")
        return self.vk

    def _sync(self):
        if self.dev != "cpu":
            self.torch.cuda.current_stream().synchronize()

    def _check_srs(self):
        """a blinded proof commits z with n + 3 coefficients: the SRS must have that many bases"""
        if self._srs_checked:
            return
        from ._binding import DpError
        try:
            self.ctx.get_bases(self.n + BLIND_Z - 1, 1)
        except DpError as e:
            raise ValueError(f"a blinded proof of 2^{self.log_n} gates commits polynomials of n + {BLIND_Z} coefficients: the SRS "
                             f"given to dp_init needs at least {self.n + BLIND_Z} bases") from e
        self._srs_checked = True

    # ---- one proof
    def prove(self, wire_evals_host, pub_host, ch, blind=False):
        """wire_evals_host: torch tensor [5n,4] (pinned host memory on a GPU), pub_host [n,4]; ch: dict of the
        challenges beta, gamma, alpha, zeta, v as raw Fr.  Returns (commitments: list of 13 x 144 B, evals: list).
        blind: False (unblinded), True (the library draws the N_BLIND = 13 blinding scalars from the OS entropy pool) or
        an [13,4] array of raw Fr below r (wire i takes rows 2i, 2i+1, z rows 10-12; reproducible proofs for tests)"""
        blinded, scalars = self._blinding(blind)
        # witness in: the only bulk host->device traffic of the proof
        self.wire_eval.copy_(wire_evals_host, non_blocking=True)
        self.pub.copy_(pub_host, non_blocking=True)
        return self._rounds(lambda stage, outputs: ch, blinded, scalars)

    def prove_witness(self, witness_host, ch, blind=False):
        """prove() from the circuit given to load_circuit: witness_host = torch tensor [num_vars,4] raw Fr (pinned host
        memory on a GPU), the proof's only bulk host->device copy; the wire and public-input evaluations are gathered on the
        device (dp_witness_gather_dev), then the rounds run exactly as in prove().  Returns (commitments, evals, public
        inputs [num_inputs,4] - what the verifier needs besides the proof)"""
        if self.vars is None:
            raise ValueError("prove_witness needs a circuit: call load_circuit first")
        if tuple(witness_host.shape) != (self.num_vars, 4):
            raise ValueError(f"witness: shape ({self.num_vars}, 4), not {tuple(witness_host.shape)}")
        blinded, scalars = self._blinding(blind)
        pub = self._gather(witness_host)
        com, evals = self._rounds(lambda stage, outputs: ch, blinded, scalars)
        return com, evals, pub

    def prove_circuit(self, witness_host, blind=True):
        """a proof of the circuit given to load_circuit that a PLONK verifier accepts: the challenges come from the
        transcript (PlonkTranscript over merlin) of the verifying key, the public inputs and each round's commitments and
        evaluations, as in the reference prover (dispatcher2.rs:239-243, 322-328, 357-362, 533-544, 556-560, 634).
        witness_host as in prove_witness; blind as in prove, True by default, because a proof for a verifier should be
        zero-knowledge.  Returns (Proof, public inputs as canonical ints).  Leaves the challenges in self.last_challenges
        (raw Fr, the dict prove_witness takes) and the host time spent in the transcript - point conversions, hashing -
        in self.last_transcript_ms"""
        if self._vk_transcript is None:
            raise ValueError("prove_circuit needs a circuit: call load_circuit first")
        if tuple(witness_host.shape) != (self.num_vars, 4):
            raise ValueError(f"witness: shape ({self.num_vars}, 4), not {tuple(witness_host.shape)}")
        import time
        blinded, scalars = self._blinding(blind)
        pub = self._gather(witness_host)
        t0 = time.perf_counter()
        pub_int = [fr_to_int(v) for v in pub]
        tr = self._vk_transcript.clone()
        tr.append_pub_input(pub_int)
        clock = [time.perf_counter() - t0]

        def challenges(stage, outputs):
            t1 = time.perf_counter()
            if stage == "evals":
                ev = [fr_to_int(v) for v in outputs]
                tr.append_proof_evaluations(ev[:N_WIRE], ev[N_WIRE:2 * N_WIRE - 1], ev[-1])
            else:
                tr.append_commitments({"wires": b"witness_poly_comms", "perm": b"perm_poly_comms", "quot": b"quot_poly_comms"}[stage],
                                      [point_from_jacobian(c) for c in outputs])
            names = {"wires": ("beta", "gamma"), "perm": ("alpha",), "quot": ("zeta",), "evals": ("v",)}[stage]
            out = {name: fr_from_int(tr.get_and_append_challenge(name.encode())) for name in names}
            derived.update(out)
            clock[0] += time.perf_counter() - t1
            return out

        derived = {}
        com, evals = self._rounds(challenges, blinded, scalars)
        t2 = time.perf_counter()
        proof = Proof.from_raw(com, evals)
        self.last_transcript_ms = (clock[0] + time.perf_counter() - t2) * 1e3
        self.last_challenges = derived
        return proof, pub_int

    def _gather(self, witness_host, inst=None):
        """the witness in, the wire and public-input evaluations gathered on the device (into inst's buffers, or the single
        proof's); returns the public inputs"""
        inst = self._own if inst is None else inst
        self.witness.copy_(witness_host, non_blocking=True)
        self._sync()                                           # torch's stream -> the library's stream
        P = lambda t: t.data_ptr()
        self.ctx.witness_gather_dev(P(self.witness), self.num_vars, P(self.vars), N_WIRE, self.n, self.num_inputs, P(inst.wire_eval), P(inst.pub))
        return inst.pub[:self.num_inputs].cpu().numpy().view(np.uint64).copy()

    # ---- a batch of proofs of one circuit (DESIGN.md 3.11)
    def instance_bytes(self) -> int:
        """device memory of one more batch instance: 5 wire evaluations, the public input (n each), 5 wires (n + 2) and z (n + 3)"""
        n = self.n
        return 32 * (N_WIRE * n + n + N_WIRE * (n + BLIND_WIRE) + n + BLIND_Z)

    def max_batch(self) -> int:
        """the largest k prove_batch takes: instance 0 lives in the single proof's buffers, each further one needs
        instance_bytes(), from the device's free memory (plus what torch caches and the instances already allocated) less
        one quotient-domain buffer (the final iNTT's scratch) and BATCH_MARGIN_BYTES; never below a batch that has already
        run (its instances are kept, and the library's pool has grown to serve it).  CPU_MAX_BATCH on the CPU emulator"""
        if self.dev == "cpu":
            return self.CPU_MAX_BATCH
        t = self.torch
        free, _ = t.cuda.mem_get_info(t.device(self.dev))
        free += t.cuda.memory_reserved(self.dev) - t.cuda.memory_allocated(self.dev) + len(self._extra) * self.instance_bytes()
        return 1 + max(len(self._extra), (free - self.m * 32 - self.BATCH_MARGIN_BYTES) // self.instance_bytes())

    def _instances(self, k):
        """instance 0 and k - 1 resident instances, allocated on first use and kept"""
        def buf(count):
            return self.torch.zeros((count, 4), dtype=self.torch.int64, device=self.dev)
        n = self.n
        while len(self._extra) < k - 1:
            self._extra.append(_Instance(buf(N_WIRE * n), buf(n), [buf(n + BLIND_WIRE) for _ in range(N_WIRE)], buf(n + BLIND_Z)))
        return [self._own] + self._extra[:k - 1]

    def prove_batch(self, witnesses_host, blind=True):
        """one BatchProof of k = len(witnesses_host) instances of the circuit given to load_circuit (DESIGN.md 3.11): the
        instances share one transcript, one quotient (sum_i alpha^(3i) Q_i) and one pair of openings.  witnesses_host: k
        witnesses as in prove_circuit; blind: True (library-drawn scalars), False, or k arrays of shape [13, 4] (one per
        instance, as prove's).  A batch of one is prove_circuit's proof, call for call.  Returns (BatchProof, [public inputs
        of each instance as canonical ints]); sets last_challenges and last_transcript_ms as prove_circuit does.
        ValueError for k = 0, k > max_batch(), or wrong shapes"""
        from .proof import BatchProof
        if self._vk_transcript is None:
            raise ValueError("prove_batch needs a circuit: call load_circuit first")
        k = len(witnesses_host)
        if k == 0:
            raise ValueError("prove_batch needs at least one witness")
        if k > self.max_batch():
            raise ValueError(f"a batch of {k} needs {k - 1} x {_gib(self.instance_bytes())} GiB beside the prover: max_batch() = {self.max_batch()}")
        for i, w in enumerate(witnesses_host):
            if tuple(w.shape) != (self.num_vars, 4):
                raise ValueError(f"witness {i}: shape ({self.num_vars}, 4), not {tuple(w.shape)}")
        if blind is True or blind is False:
            blinded, scalars = self._blinding(blind)
            scalars = [scalars] * k
        else:
            if len(blind) != k:
                raise ValueError(f"blind: {len(blind)} blinding arrays for {k} witnesses")
            if any(b is True or b is False for b in blind):
                raise ValueError("blind: True, False, or one [13, 4] array per witness")
            blinded, scalars = True, [self._blinding(b)[1] for b in blind]
        import time
        insts = self._instances(k)
        pubs = [self._gather(w, inst) for w, inst in zip(witnesses_host, insts)]
        t0 = time.perf_counter()
        pub_int = [[fr_to_int(v) for v in pub] for pub in pubs]
        tr = self._vk_transcript.clone()
        tr.append_pub_input(pub_int[0])
        for pi in pub_int[1:]:
            tr.append_vk(self.vk)
            tr.append_pub_input(pi)
        clock = [time.perf_counter() - t0]

        def challenges(stage, outputs):
            t1 = time.perf_counter()
            if stage == "evals":
                ev = [fr_to_int(v) for v in outputs]
                for i in range(0, len(ev), 2 * N_WIRE):
                    tr.append_proof_evaluations(ev[i:i + N_WIRE], ev[i + N_WIRE:i + 2 * N_WIRE - 1], ev[i + 2 * N_WIRE - 1])
            else:
                tr.append_commitments({"wires": b"witness_poly_comms", "perm": b"perm_poly_comms", "quot": b"quot_poly_comms"}[stage],
                                      [point_from_jacobian(c) for c in outputs])
            names = {"wires": ("beta", "gamma"), "perm": ("alpha",), "quot": ("zeta",), "evals": ("v",)}[stage]
            out = {name: fr_from_int(tr.get_and_append_challenge(name.encode())) for name in names}
            derived.update(out)
            clock[0] += time.perf_counter() - t1
            return out

        derived = {}
        com, evals = self._rounds(challenges, blinded, scalars, insts)
        t2 = time.perf_counter()
        proof = BatchProof.from_raw(k, com, evals)
        self.last_transcript_ms = (clock[0] + time.perf_counter() - t2) * 1e3
        self.last_challenges = derived
        return proof, pub_int

    def _blinding(self, blind):
        """(blinded, scalars or None) from prove's `blind` argument"""
        blinded = blind is not False
        scalars = None
        if blinded:
            self._check_srs()
            if blind is not True:
                scalars = np.ascontiguousarray(blind, dtype=np.uint64)
                if scalars.shape != (N_BLIND, 4):
                    raise ValueError(f"blind: an array of shape ({N_BLIND}, 4) of raw Fr, True or False, not shape {scalars.shape}")
        return blinded, scalars

    def _rounds(self, challenges, blinded, scalars, insts=None):
        """rounds 1-5 from the wire and public-input evaluations in self.wire_eval / self.pub (insts None), or of the
        instances of a batch (insts: _Instance list, scalars: one blinding array or None per instance).  challenges(stage,
        outputs) -> dict of raw Fr challenges, asked where the reference asks its transcript: "wires" (the 5 wire
        commitments of each instance) -> beta, gamma; "perm" (each instance's commitment of z) -> alpha; "quot" (the 5
        quotient-chunk commitments) -> zeta; "evals" (the 10 evaluations of each instance) -> v.  Returns (commitments:
        5k wires, k z, 5 quotient chunks, 2 openings; evaluations: 10 per instance).  A batch of one makes exactly the
        library calls of a single proof."""
        if insts is None:
            insts, scalars = [self._own], [scalars]
        com = []
        for inst, sc in zip(insts, scalars):
            com += self._round1(inst, blinded, sc)
        ch = dict(challenges("wires", com))
        for inst, sc in zip(insts, scalars):
            com.append(self._round2(inst, ch, blinded, sc))
        ch.update(challenges("perm", com[len(insts) * N_WIRE:]))
        for inst in insts:
            self.ctx.ntt_dev(inst.pub.data_ptr(), self.log_n, True, False)
        com += self._round3(insts, ch, blinded)
        ch.update(challenges("quot", com[-N_WIRE:]))
        evals = self._round4(insts, ch, blinded)
        ch.update(challenges("evals", [v for ev in evals for v in ev]))
        com += self._round5(insts, ch, blinded, evals)
        return com, [v for ev in evals for v in ev]

    def _lens(self, blinded):
        n = self.n
        return (n + BLIND_WIRE, n + BLIND_Z) if blinded else (n, n)   # coefficients of each wire / of z

    def _round1(self, inst, blinded, scalars):
        """the wires' coefficient forms (blinded: + (b_0 + b_1 X) Z_H) and their 5 commitments"""
        ctx, n, log_n, P = self.ctx, self.n, self.log_n, lambda t: t.data_ptr()
        nw, _ = self._lens(blinded)
        for i in range(N_WIRE):
            inst.wire_coef[i][:n].copy_(inst.wire_eval[i * n:(i + 1) * n])
        if blinded:                                            # the blinding adds to coefficients n, n+1, ...
            for t in inst.wire_coef + [inst.z]:
                t[n:].zero_()
        self._sync()                                           # torch's stream -> the library's streams
        com = []
        for i in range(N_WIRE):
            ctx.ntt_dev(P(inst.wire_coef[i]), log_n, True, False)
            if blinded:
                ctx.poly_blind_dev(P(inst.wire_coef[i]), n, BLIND_WIRE, None if scalars is None else scalars[BLIND_WIRE * i:BLIND_WIRE * (i + 1)])
            com.append(ctx.commit_dev(P(inst.wire_coef[i]), nw))
        return com

    def _round2(self, inst, ch, blinded, scalars):
        """the permutation product z (blinded: + (b_0 + b_1 X + b_2 X^2) Z_H) and its commitment"""
        ctx, n, P = self.ctx, self.n, lambda t: t.data_ptr()
        _, nz = self._lens(blinded)
        ctx.perm_product_dev(P(inst.wire_eval), P(self.id_eval), P(self.sig_eval), N_WIRE, n, ch["beta"], ch["gamma"], P(inst.z))
        ctx.ntt_dev(P(inst.z), self.log_n, True, False)
        if blinded:
            ctx.poly_blind_dev(P(inst.z), n, BLIND_Z, None if scalars is None else scalars[N_WIRE * BLIND_WIRE:])
        return ctx.commit_dev(P(inst.z), nz)

    def _alpha_powers(self, alpha, count, step=3):
        """alpha^(step i), i < count (raw Fr): the weights of the instances of a batch"""
        F = self.F
        a3, cur, out = F.pow_u64(alpha, step), F.from_u64(1), []
        for _ in range(count):
            out.append(cur)
            cur = F.mul(cur, a3)
        return out

    def _round3(self, insts, ch, blinded):
        """25 coset evaluations on the 8n domain, the quotient evaluations, one coset-iNTT(8n), 5 commitments of the
        (n+2)-coefficient chunks.  Blinded, the wires and z are transformed on their first n coefficients and the quotient
        kernel adds the rest (their tails).  A batch: the 18 key polynomials are transformed once (per slice, sliced); each
        instance i then transforms its 7 and adds alpha^(3i) times its quotient (instance 0 writes it)"""
        ctx, n, m, P = self.ctx, self.n, self.m, lambda t: t.data_ptr()
        log_m = self.log_n + 3
        keys = self.sel_coef + self.sig_coef
        own = lambda inst: inst.wire_coef + [inst.z, inst.pub]
        qargs = (self.k, ch["alpha"], ch["beta"], ch["gamma"])
        scale = self._alpha_powers(ch["alpha"], len(insts))

        def tails(inst):
            return [(P(t) + 32 * n, BLIND_WIRE) for t in inst.wire_coef] + [(P(inst.z) + 32 * n, BLIND_Z)] if blinded else None

        def quotient(b, i, inst, slice_=None):
            if i:
                ctx.quotient_evals_acc_dev(b[:13], b[13:18], b[18:23], b[23], b[24], *qargs, tails(inst), scale[i], P(self.quot), slice_)
            elif slice_ is None:
                if blinded:
                    ctx.quotient_evals_tail_dev(b[:13], b[13:18], b[18:23], b[23], b[24], *qargs, tails(inst), P(self.quot))
                else:
                    ctx.quotient_evals_dev(b[:13], b[13:18], b[18:23], b[23], b[24], *qargs, P(self.quot))
            elif blinded:
                ctx.quotient_evals_slice_tail_dev(b[:13], b[13:18], b[18:23], b[23], b[24], *qargs, tails(inst), slice_, P(self.quot))
            else:
                ctx.quotient_evals_slice_dev(b[:13], b[13:18], b[18:23], b[23], b[24], *qargs, slice_, P(self.quot))

        if self.quotient == "whole":   # only the n coefficients at the head of each buffer are read
            b = [P(t) for t in self.big]
            for i, inst in enumerate(insts):
                dsts = self.big if i == 0 else self.big[len(keys):]
                for dst, src in zip(dsts, (keys if i == 0 else []) + own(inst)):
                    dst[:n].copy_(src[:n])
                self._sync()                                   # (the previous quotient call has returned: its reads are done)
                for dst in dsts:
                    ctx.ntt_dev_padded(P(dst), n, log_m, False, True, wait=False)
                quotient(b, i, inst)
        else:                          # slice k into the same 25 n-point buffers, every k; all of it on the library's stream
            b = [P(t) for t in self.slices]
            for k in range(m // n):
                for i, inst in enumerate(insts):
                    srcs = (keys if i == 0 else []) + own(inst)
                    for dst, src in zip(b[len(b) - len(srcs):], srcs):
                        ctx.ntt_dev_quot_slice(P(src), n, k, dst, wait=False)
                    quotient(b, i, inst, k)
        ctx.ntt_dev(P(self.quot), log_m, True, True)
        chunk = n + 2
        return [ctx.commit_dev(P(self.quot) + 32 * j * chunk, chunk) for j in range(N_WIRE)]

    def _round4(self, insts, ch, blinded):
        """per instance the 5 wires and 4 sigmas at zeta and z at zeta * omega; the sigma values are the same for every
        instance and are computed once"""
        ctx, n, P = self.ctx, self.n, lambda t: t.data_ptr()
        nw, nz = self._lens(blinded)
        zeta = ch["zeta"]
        zeta_w = self.F.mul(zeta, self.F.omega)
        out, s_ev = [], None
        for inst in insts:
            w_ev = [ctx.poly_eval(P(inst.wire_coef[i]), zeta, nw) for i in range(N_WIRE)]
            if s_ev is None:
                s_ev = [ctx.poly_eval(P(self.sig_coef[i]), zeta, n) for i in range(N_WIRE - 1)]
            out.append(w_ev + s_ev + [ctx.poly_eval(P(inst.z), zeta_w, nz)])
        return out

    def _lin_scalars(self, ev, ch, vanish, lag1):
        """one instance's linearisation scalars from its 10 evaluations: the 13 selectors', z's and sigma_4's (host glue, a
        few dozen field operations)"""
        F = self.F
        w_ev, s_ev, z_next = ev[:N_WIRE], ev[N_WIRE:2 * N_WIRE - 1], ev[-1]
        a, bb, c, d, e = w_ev
        ab, cd = F.mul(a, bb), F.mul(c, d)
        p5 = lambda x: F.mul(F.mul(F.mul(x, x), F.mul(x, x)), x)
        neg = lambda x: F.sub(F.from_u64(0), x)
        zeta = ch["zeta"]
        cz = ch["alpha"]
        for wv, kk in zip(w_ev, self.k):
            cz = F.mul(cz, F.add(F.add(wv, F.mul(F.mul(ch["beta"], kk), zeta)), ch["gamma"]))
        cz = F.add(cz, F.mul(F.mul(ch["alpha"], ch["alpha"]), lag1))
        cs = F.mul(F.mul(ch["alpha"], ch["beta"]), z_next)
        for wv, sv in zip(w_ev[:-1], s_ev):
            cs = F.mul(cs, F.add(F.add(wv, F.mul(ch["beta"], sv)), ch["gamma"]))
        cs = neg(cs)
        return [a, bb, c, d, ab, cd, p5(a), p5(bb), p5(c), p5(d), neg(e), F.from_u64(1), F.mul(F.mul(ab, cd), e)], cz, cs

    def _round5(self, insts, ch, blinded, evals):
        """the linearisation polynomial, the batch polynomial at zeta and its opening W, the (batched) z at zeta * omega and
        its opening W'.  A batch weights instance i's linearisation scalars with alpha^(3i) and its openings with v powers
        (DESIGN.md 3.11); the polynomials stay put"""
        ctx, n, F, P = self.ctx, self.n, self.F, lambda t: t.data_ptr()
        nw, nz = self._lens(blinded)
        k = len(insts)
        zeta = ch["zeta"]
        zeta_w = F.mul(zeta, F.omega)
        one = F.from_u64(1)
        vanish = F.sub(F.pow_u64(zeta, n), one)
        lag1 = F.mul(vanish, F.inv(F.mul(F.from_u64(n), F.sub(zeta, one))))
        zn2 = F.mul(F.add(vanish, one), F.mul(zeta, zeta))
        qc, cur = [], F.sub(F.from_u64(0), vanish)
        for _ in range(N_WIRE):
            qc.append(cur)
            cur = F.mul(cur, zn2)
        scale = self._alpha_powers(ch["alpha"], k)
        sel, cz, cs = None, [], None
        for i, ev in enumerate(evals):
            q_i, cz_i, cs_i = self._lin_scalars(ev, ch, vanish, lag1)
            if i:
                q_i, cz_i, cs_i = [F.mul(scale[i], x) for x in q_i], F.mul(scale[i], cz_i), F.mul(scale[i], cs_i)
            sel = q_i if sel is None else [F.add(x, y) for x, y in zip(sel, q_i)]
            cs = cs_i if cs is None else F.add(cs, cs_i)
            cz.append(cz_i)
        chunk = n + 2
        # instance 0's z where the single proof has it, the other instances' z after the quotient chunks
        coeffs = sel + [cz[0], cs] + qc + cz[1:]
        polys = [P(t) for t in self.sel_coef] + [P(insts[0].z), P(self.sig_coef[N_WIRE - 1])] + [P(self.quot) + 32 * j * chunk for j in range(N_WIRE)] \
            + [P(inst.z) for inst in insts[1:]]
        lens = [n] * N_SEL + [nz, n] + [chunk] * N_WIRE + [nz] * (k - 1)
        lin_len = max(chunk, nz)                               # n + 2, or n + 3 with the blinded z
        ctx.poly_lincomb(polys, np.stack(coeffs), out_len=lin_len, lens=lens, out_ptr=P(self.lin))
        vp = self._alpha_powers(ch["v"], 1 + 9 * k, step=1)   # v^(1 + 9i + j): wire j of instance i; v^(6 + 9i + j): sigma j
        sig_c = [vp[6 + j] for j in range(N_WIRE - 1)]
        for i in range(1, k):
            sig_c = [F.add(x, vp[6 + 9 * i + j]) for j, x in enumerate(sig_c)]
        coeffs = [one] + vp[1:1 + N_WIRE] + sig_c + [vp[1 + 9 * i + j] for i in range(1, k) for j in range(N_WIRE)]
        polys = [P(self.lin)] + [P(t) for t in insts[0].wire_coef] + [P(t) for t in self.sig_coef[:-1]] \
            + [P(t) for inst in insts[1:] for t in inst.wire_coef]
        lens = [lin_len] + [nw] * N_WIRE + [n] * (N_WIRE - 1) + [nw] * (N_WIRE * (k - 1))
        ctx.poly_lincomb(polys, np.stack(coeffs), out_len=lin_len, lens=lens, out_ptr=P(self.batch))
        ctx.poly_div_linear(P(self.batch), zeta, lin_len, P(self.wit[0]))
        com = [ctx.commit_dev(P(self.wit[0]), lin_len - 1)]
        shifted = insts[0].z
        if k > 1:                                              # sum_i v^i z_i, in the linearisation's buffer (done with)
            ctx.poly_lincomb([P(inst.z) for inst in insts], np.stack(vp[:k]), out_len=nz, lens=[nz] * k, out_ptr=P(self.lin))
            shifted = self.lin
        ctx.poly_div_linear(P(shifted), zeta_w, nz, P(self.wit[1]))
        com.append(ctx.commit_dev(P(self.wit[1]), nz - 1))
        return com


class _Instance:
    """one instance's resident state: the wire and public-input evaluations, the wires' and z's coefficient forms"""

    def __init__(self, wire_eval, pub, wire_coef, z):
        self.wire_eval, self.pub, self.wire_coef, self.z = wire_eval, pub, wire_coef, z


class NumpyField:
    """raw Montgomery Fr scalars (np.uint64[4]) through Python integers - the few dozen challenge products of rounds 4-5"""
    R_MOD = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
    R = (1 << 256) % R_MOD

    def __init__(self, log_n: int):
        root = pow(7, (self.R_MOD - 1) >> 32, self.R_MOD)
        self.omega = self._enc(pow(root, 1 << (32 - log_n), self.R_MOD))

    @classmethod
    def _dec(cls, a) -> int:
        v = sum(int(a[i]) << (64 * i) for i in range(4))
        return v * pow(cls.R, -1, cls.R_MOD) % cls.R_MOD

    @classmethod
    def _enc(cls, v: int) -> np.ndarray:
        v = v % cls.R_MOD * cls.R % cls.R_MOD
        return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)

    def mul(self, a, b):
        return self._enc(self._dec(a) * self._dec(b))

    def add(self, a, b):
        return self._enc(self._dec(a) + self._dec(b))

    def sub(self, a, b):
        return self._enc(self._dec(a) - self._dec(b))

    def inv(self, a):
        return self._enc(pow(self._dec(a), -1, self.R_MOD))

    def from_u64(self, v):
        return self._enc(v)

    def pow_u64(self, a, e):
        return self._enc(pow(self._dec(a), e, self.R_MOD))


def _gib(b) -> float:
    return round(b / 2**30, 3)


def make_bench_prover(ctx, torch, log_n: int, rand_fr, quotient: str = "auto"):
    """a ResidentProver on synthetic data (random polynomials: the arithmetic is data-independent; the quotient is then not
    a polynomial of the expected degree, which changes nothing about the work), with the witness in pinned host memory"""
    n = 1 << log_n
    F = NumpyField(log_n)
    pr = ResidentProver(ctx, torch, log_n, "cuda", F, quotient=quotient)
    for t in pr.sel_coef + pr.sig_coef:
        t.copy_(rand_fr(n))
    pr.sig_eval.copy_(rand_fr(N_WIRE * n))
    pr.id_eval.copy_(rand_fr(N_WIRE * n))
    pr.k = np.stack([F.from_u64(v) for v in (1, 7, 13, 17, 23)])
    wires = rand_fr(N_WIRE * n).cpu().pin_memory()
    pub = rand_fr(n).cpu().pin_memory()
    ch = {name: F.from_u64(v) for name, v in (("beta", 0xB17A), ("gamma", 0x6A33A), ("alpha", 0xA1FA), ("zeta", 0x2E7A), ("v", 0x55))}
    return pr, (wires, pub, ch)


def bench_circuit_inputs(log_n: int, num_vars: int, seed: int = 0xC1C):
    """a synthetic variable map: slots on uniform random variables 1..num_vars-1, except the last n/8 gates, whose five wires
    all hold variable 0 - the one large shared variable that padding a circuit to a power of two produces"""
    n = 1 << log_n
    rng = np.random.default_rng(seed)
    wire_vars = rng.integers(1, max(num_vars, 2), size=(N_WIRE, n), dtype=np.uint32) if num_vars > 1 else np.zeros((N_WIRE, n), dtype=np.uint32)
    wire_vars[:, n - n // 8:] = 0
    return wire_vars.reshape(-1)


def make_bench_circuit(ctx, torch, log_n: int, rand_fr, num_vars: int | None = None, quotient: str = "auto", num_inputs: int = 16):
    """a ResidentProver preprocessed from a synthetic circuit (load_circuit): random selector evaluations, the variable map
    of bench_circuit_inputs with num_vars variables (default 4n), k = (1, 7, 13, 17, 23); the witness (random, so the circuit
    is not satisfied, which changes nothing about the work) in pinned host memory.  Returns (prover, vk, (witness, ch))"""
    n = 1 << log_n
    num_vars = 4 * n if num_vars is None else num_vars
    F = NumpyField(log_n)
    pr = ResidentProver(ctx, torch, log_n, "cuda", F, quotient=quotient)
    sel = [rand_fr(n).cpu().numpy().view(np.uint64) for _ in range(N_SEL)]
    k = np.stack([F.from_u64(v) for v in (1, 7, 13, 17, 23)])
    vk, _ = pr.load_circuit(sel, bench_circuit_inputs(log_n, num_vars), num_vars, k, num_inputs)
    witness = rand_fr(num_vars).cpu().pin_memory()
    ch = {name: F.from_u64(v) for name, v in (("beta", 0xB17A), ("gamma", 0x6A33A), ("alpha", 0xA1FA), ("zeta", 0x2E7A), ("v", 0x55))}
    return pr, vk, (witness, ch)


def bench_leg(ctx, torch, log_n: int, rand_fr, timed, steps: int = 3, quotient: str = "auto", prover=None, blind=False):
    """bench.py's e2e_resident: proofs/s of ResidentProver.prove on synthetic data, witness copied from pinned host memory
    inside the timed region.  The prover picks its round-3 layout (quotient="auto") unless told; `prover` = (pr, inputs) of
    make_bench_prover to time an existing one (tools/bench_resident.py); `blind` is passed to prove.  Also records the layout and the leg's peak device
    memory: torch's peak plus what the library's pool added (cudaMemGetInfo before and after; the pool keeps what it
    allocates).  Torch's cached free blocks are returned to the device first, so that the layout is chosen on what is free."""
    if prover is None:
        torch.cuda.empty_cache()
    free0, total = torch.cuda.mem_get_info()
    res0 = torch.cuda.memory_reserved()
    torch.cuda.reset_peak_memory_stats()
    pr, (wires, pub, ch) = prover if prover is not None else make_bench_prover(ctx, torch, log_n, rand_fr, quotient)
    n = 1 << log_n
    out = {}

    def step():
        out["r"] = pr.prove(wires, pub, ch, blind=blind)

    dt, _ = timed(step, steps, 1, False)
    com, ev = out["r"]
    free1, _ = torch.cuda.mem_get_info()
    res1, torch_peak = torch.cuda.memory_reserved(), torch.cuda.max_memory_reserved()
    lib_added = max(0, (free0 - free1) - (res1 - res0))
    in_use_before = total - free0
    mem = {"peak_gib": _gib(in_use_before - res0 + torch_peak + lib_added), "torch_peak_reserved_gib": _gib(torch_peak),
           "library_added_gib": _gib(lib_added), "in_use_before_gib": _gib(in_use_before), "device_total_gib": _gib(total),
           "how": "device memory in use before the leg, minus torch's reserve then, plus torch's peak reserve during the leg, plus "
                  "what the library's pool grew by (its blocks are cached, so its end size is its peak)"}
    return {"value": steps / dt, "unit": "proofs/s", "ms_per_step": dt / steps * 1e3, "steps": steps, "quotient": pr.quotient,
            "device_memory": mem, "h2d_bytes_per_step": int((N_WIRE + 1) * n * 32), "d2h_bytes_per_step": int(len(com) * 144 + len(ev) * 32),
            "what": ("rounds 1-5 of one proof on worker-resident polynomials (distributed_plonk_b200/resident.py): witness in once, "
                     "13 commitments + 10 evaluations out; includes the round-2 grand product, the quotient evaluations, the round-4 "
                     "evaluations and the round-5 folds / divisions that the 33-transform + 13-MSM schedule of `value` leaves to the dispatcher; "
                     "quotient = round 3's layout: whole (25 buffers of 8n points) or sliced (8 slices through 25 buffers of n points)"),
            "timing": "host clock between barrier+synchronize"}
