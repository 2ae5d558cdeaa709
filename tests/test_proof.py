"""ResidentProver.prove_circuit on the kernel-logic emulator: the proof equals prove_witness on the challenges it derived,
in both round-3 layouts, blinded and not; the test verifier (tests/plonk_verifier.py) re-derives the same challenges from
(verifying key, public inputs, proof) and accepts, over an SRS with a known trapdoor; it rejects every tampered proof;
the transcript is fed exactly what the reference's FakeStandardTranscript feeds merlin; Proof.to_bytes decodes back -
also under adversarial asynchronous stream schedules."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle.py import bls12_381 as B
from distributed_plonk_b200._binding import Context
from distributed_plonk_b200 import transcript as T
from distributed_plonk_b200.proof import Proof, fr_from_int, fr_to_int
from distributed_plonk_b200.resident import N_BLIND, N_SEL, NumpyField, ResidentProver
from tests import plonk_verifier as pv
from tests import test_circuit as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NUM_INPUTS = 3


def setup(orc, lib, log_n, seed, device, quotient="auto"):
    """a context over the SRS [tau^i] G (i < n + 3) and a prover loaded with tests/test_circuit.py's satisfied circuit;
    returns (ctx, prover, witness, tau)"""
    n = 1 << log_n
    tau = orc.gen_fr(seed, 1, False)[0]
    c = Context(lib, 0, 0, 1)
    c.init(orc.gen_srs(tau, n + 3), n, 8 * n)
    pr, _, (_, _, witness, _) = tc.prover_from_circuit(orc, c, log_n, seed, device, quotient)
    return c, pr, witness, int.from_bytes(tau.tobytes(), "little")


def check_equals_prove_witness(orc, pr, witness, tau, device, seed):
    """prove_circuit == prove_witness(last_challenges), unblinded and with fixed blinders; the verifier derives the same
    challenges and accepts.  Returns the blinded proof and its public inputs"""
    wit = tc.witness_host(witness, device)
    vk = pr.verifying_key()
    for blind in (False, orc.gen_fr(seed + 70, N_BLIND)):
        proof, pub = pr.prove_circuit(wit, blind=blind)
        assert pub == [fr_to_int(v) for v in witness[1:1 + NUM_INPUTS]]
        ch = pr.last_challenges
        assert sorted(ch) == ["alpha", "beta", "gamma", "v", "zeta"]
        com, ev, pi = pr.prove_witness(wit, ch, blind=blind)
        assert [fr_to_int(v) for v in pi] == pub
        assert Proof.from_raw(com, ev) == proof, f"prove_circuit != prove_witness ({pr.quotient}, blinded={blind is not False})"
        derived = pv.challenges(vk, pub, proof)
        assert {k: derived[k] for k in ch} == {k: fr_to_int(v) for k, v in ch.items()}, "the verifier derives other challenges"
        assert pv.verify(orc, vk, pub, proof, tau), f"verifier rejects ({pr.quotient}, blinded={blind is not False})"
        assert pr.last_transcript_ms > 0
    return proof, pub


@pytest.mark.parametrize("log_n", [6, 8])
@pytest.mark.parametrize("quotient", ["whole", "sliced"])
def test_prove_circuit_equals_prove_witness_and_verifies(orc, emul_lib, quotient, log_n):
    c, pr, witness, tau = setup(orc, emul_lib, log_n, 11000 + log_n, "cpu", quotient)
    check_equals_prove_witness(orc, pr, witness, tau, "cpu", 11000 + log_n)
    c.close()


def test_library_blinded_proofs_verify_and_differ(orc, emul_lib):
    c, pr, witness, tau = setup(orc, emul_lib, 6, 11100, "cpu")
    wit = tc.witness_host(witness, "cpu")
    vk = pr.verifying_key()
    (p1, pub1), (p2, pub2) = pr.prove_circuit(wit), pr.prove_circuit(wit)
    assert pub1 == pub2 and p1 != p2
    assert p1.wires_poly_comms[0] != p2.wires_poly_comms[0] and p1.wires_evals[0] != p2.wires_evals[0]
    assert pv.verify(orc, vk, pub1, p1, tau) and pv.verify(orc, vk, pub2, p2, tau)
    c.close()


def another_point(p):
    return B.g1_add(p, B.G1_GEN) if p != B.G1_GEN else B.g1_add(p, p)


def check_rejections(orc, pr, witness, tau, device, seed, every=True):
    """each commitment replaced by another valid point, each evaluation + 1, a changed public input, a proof of a witness
    with one free variable changed, a proof made with challenges that do not come from the transcript: all rejected"""
    wit = tc.witness_host(witness, device)
    vk = pr.verifying_key()
    proof, pub = pr.prove_circuit(wit, blind=orc.gen_fr(seed, N_BLIND))
    assert pv.verify(orc, vk, pub, proof, tau)
    com, ev = proof.commitments(), proof.evaluations()

    def rebuild(c, e):
        p = Proof(c[0:5], c[5], c[6:11], c[11], c[12], e[0:5], e[5:9], e[9])
        assert len(p.commitments()) == 13
        return p

    for j in (range(13) if every else (0, 5, 8, 11, 12)):
        bad = list(com)
        bad[j] = another_point(bad[j])
        assert not pv.verify(orc, vk, pub, rebuild(bad, ev), tau), f"accepted a proof with commitment {j} replaced"
    for j in (range(10) if every else (0, 4, 5, 9)):
        bad = list(ev)
        bad[j] = (bad[j] + 1) % T.R_MOD
        assert not pv.verify(orc, vk, pub, rebuild(com, bad), tau), f"accepted a proof with evaluation {j} + 1"
    assert not pv.verify(orc, vk, [pub[0] + 1] + pub[1:], proof, tau), "accepted a changed public input"
    # a free variable changed: the gates that use it no longer hold; the prover still runs
    w2 = witness.copy()
    w2[1 + NUM_INPUTS] = orc.gen_fr(seed + 1, 1)[0]
    bad_proof, bad_pub = pr.prove_circuit(tc.witness_host(w2, device), blind=orc.gen_fr(seed, N_BLIND))
    assert bad_pub == pub and not pv.verify(orc, vk, bad_pub, bad_proof, tau), "accepted a proof of an unsatisfying witness"
    # the right witness, but challenges the caller chose
    ch = {name: fr_from_int(v) for name, v in zip(("beta", "gamma", "alpha", "zeta", "v"), (11, 22, 33, 44, 55))}
    com2, ev2, _ = pr.prove_witness(wit, ch, blind=orc.gen_fr(seed, N_BLIND))
    assert not pv.verify(orc, vk, pub, Proof.from_raw(com2, ev2), tau), "accepted a proof made with chosen challenges"


def test_verifier_rejects_tampered_proofs(orc, emul_lib):
    c, pr, witness, tau = setup(orc, emul_lib, 6, 11200, "cpu")
    check_rejections(orc, pr, witness, tau, "cpu", 11200)
    c.close()


def test_proof_bytes(orc, emul_lib):
    c, pr, witness, tau = setup(orc, emul_lib, 6, 11300, "cpu")
    proof, pub = pr.prove_circuit(tc.witness_host(witness, "cpu"))
    b = proof.to_bytes()
    assert len(b) == 976
    back = pv.proof_from_bytes(b)
    for name in ("wires_poly_comms", "prod_perm_poly_comm", "split_quot_poly_comms", "opening_proof", "shifted_opening_proof",
                 "wires_evals", "wire_sigma_evals", "perm_next_eval"):
        assert getattr(back, name) == getattr(proof, name), name
    comp = [b[8 + 48 * i:8 + 48 * (i + 1)] for i in range(5)] + [b[248:296]]
    pts = proof.wires_poly_comms + [proof.prod_perm_poly_comm]
    for cb, p in zip(comp, pts):
        assert cb == B.g1_compress(p)
        assert cb == orc.g1_compress(np.frombuffer(B.g1_affine_to_bytes(p), dtype=np.uint8))[0].tobytes()
    assert pv.verify(orc, pr.verifying_key(), pub, back, tau)
    c.close()


class Recorder:
    """merlin with a record of every call; clone() shares the record, so a prover's per-proof clone appends to it"""

    def __init__(self, inner, log):
        self.inner, self.log = inner, log

    def append_message(self, label, message):
        self.log.append((bytes(label), bytes(message)))
        self.inner.append_message(label, message)

    def challenge_bytes(self, label, k):
        self.log.append((bytes(label), k))
        return self.inner.challenge_bytes(label, k)

    def clone(self):
        return Recorder(self.inner.clone(), self.log)


def test_prove_circuit_feeds_the_transcript_what_the_reference_does(orc, emul_lib):
    """the (label, message) list of FakeStandardTranscript, on a circuit with one all-zero selector (its commitment is
    the identity, encoded (0, 1, true))"""
    log_n = 6
    n = 1 << log_n
    c = Context(emul_lib, 0, 0, 1)
    c.init(orc.gen_srs(orc.gen_fr(11400, 1, False)[0], n + 3), n, 8 * n)
    sel, wv, witness, k = tc.satisfied_circuit(orc, log_n, 11400)
    sel[12] = np.zeros_like(sel[12])                            # no ECC gates
    pr = ResidentProver(c, torch, log_n, "cpu", NumpyField(log_n))
    pr.load_circuit(sel, wv, witness.shape[0], k, NUM_INPUTS)
    vk = pr.verifying_key()
    assert vk.selector_comms[12] is None and all(p is not None for p in vk.selector_comms[:12] + vk.sigma_comms)
    log = []
    pr._vk_transcript = T.PlonkTranscript(Recorder(pv.Merlin(b"PlonkProof"), log))
    pr._vk_transcript.append_vk(vk)
    proof, pub = pr.prove_circuit(tc.witness_host(witness, "cpu"), blind=orc.gen_fr(11401, N_BLIND))
    ch = {name: fr_to_int(v) for name, v in pr.last_challenges.items()}
    fr, pt = lambda v: v.to_bytes(32, "little"), lambda p: p[0].to_bytes(48, "little") + p[1].to_bytes(48, "little") + b"\x00"
    ident = bytes(48) + (1).to_bytes(48, "little") + b"\x01"
    want = [(b"field size in bits", (255).to_bytes(8, "little")), (b"domain size", n.to_bytes(8, "little")),
            (b"input size", NUM_INPUTS.to_bytes(8, "little"))]
    want += [(b"wire subsets separators", fr(fr_to_int(x))) for x in k]
    want += [(b"selector commitments", pt(p) if p is not None else ident) for p in vk.selector_comms]
    want += [(b"sigma commitments", pt(p)) for p in vk.sigma_comms]
    want += [(b"public input", fr(v)) for v in pub]
    want += [(b"witness_poly_comms", pt(p)) for p in proof.wires_poly_comms]
    challenge = lambda name: [(name.encode(), 64), (name.encode(), fr(ch[name]))]
    want += challenge("beta") + challenge("gamma") + [(b"perm_poly_comms", pt(proof.prod_perm_poly_comm))] + challenge("alpha")
    want += [(b"quot_poly_comms", pt(p)) for p in proof.split_quot_poly_comms] + challenge("zeta")
    want += [(b"wire_evals", fr(v)) for v in proof.wires_evals] + [(b"wire_sigma_evals", fr(v)) for v in proof.wire_sigma_evals]
    want += [(b"perm_next_eval", fr(proof.perm_next_eval))] + challenge("v")
    assert log == want
    assert len([m for lbl, m in log if lbl == b"selector commitments" and m == ident]) == 1
    assert all(len(m) == 97 for lbl, m in log if lbl.endswith(b"commitments") or lbl.endswith(b"comms"))
    # the recording transcript is merlin underneath: the verifier's derivation gives the same challenges
    assert {k2: v for k2, v in pv.challenges(vk, pub, proof).items() if k2 != "u"} == ch
    c.close()


def test_prove_circuit_errors(orc, emul_lib):
    n = 64
    c = Context(emul_lib, 0, 0, 1)
    c.init(orc.gen_bases(5, n + 3, 64, True), n, 8 * n)
    pr = ResidentProver(c, torch, 6, "cpu", NumpyField(6))
    with pytest.raises(ValueError):
        pr.prove_circuit(torch.zeros((10, 4), dtype=torch.int64))
    with pytest.raises(ValueError):
        pr.verifying_key()
    sel, wv, witness, k = tc.satisfied_circuit(orc, 6, 11500)
    pr.load_circuit(sel, wv, witness.shape[0], k, NUM_INPUTS)
    with pytest.raises(ValueError):
        pr.prove_circuit(torch.zeros((witness.shape[0] + 1, 4), dtype=torch.int64))
    assert len(pr.verifying_key().selector_comms) == N_SEL
    c.close()


@pytest.mark.timeout(1500)
@pytest.mark.skipif(os.environ.get("DP_TEST_EMUL_ASYNC", "0") == "1", reason="this test starts the asynchronous runs itself")
def test_prove_circuit_under_adversarial_stream_schedules():
    """prove_circuit against prove_witness and the verifier on the asynchronous-stream emulator build, with the compute,
    copy-in and MSM tail streams in turn made pathologically slow (tests/test_emul_async.py)"""
    from tests.emul import build as emul_build
    emul_build.build(async_streams=True)
    select = "prove_circuit_equals_prove_witness and sliced and 6"
    procs = []
    for slow in (0, 1, 3):
        env = dict(os.environ, DP_TEST_EMUL_ASYNC="1", DP_EMUL_SLOW=f"{slow}:1500")
        procs.append(subprocess.Popen(
            [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-p", "no:cacheprovider", "-k", select],
            cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    for slow, p in zip((0, 1, 3), procs):
        out, _ = p.communicate()
        assert p.returncode == 0, f"adversarial schedule {slow}:\n{out[-3000:]}"
        assert " passed" in out and "failed" not in out
