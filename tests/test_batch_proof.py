"""Batch proofs on the kernel-logic emulator (DESIGN.md 3.11): the accumulating quotient entries against the oracle's
quotient (out0 + s Q, whole and slice by slice, with and without tails); dp_poly_lincomb_dev chained past 32 operands with
the output as an operand; prove_batch of one equals prove_circuit in both layouts, with its transcript; batches of 2, 3
and 7 accepted by verify_batch_proof (the pairing) and by the trapdoor check of tests/plonk_batch_verifier.py; tampered
batches rejected by both; BatchProof bytes round-trip and every malformed encoding refused; argument errors - also under
adversarial asynchronous stream schedules."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context, DpError
from distributed_plonk_b200.proof import FQ_MOD, BatchProof, ProofEvaluations
from distributed_plonk_b200.resident import N_BLIND, N_SEL, N_WIRE, ResidentProver
from distributed_plonk_b200.srs import open_key, universal_setup
from distributed_plonk_b200.transcript import R_MOD
from distributed_plonk_b200.verifier import batch_proof_from_bytes, verify_batch_proof
from tests import plonk_batch_verifier as pbv
from tests import plonk_verifier as pv
from tests import test_circuit as tc
from tests import test_proof as tp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAU = 0x510E527FADE682D19B05688C2B3E6C1F1F83D9ABFB41BD6B5BE0CD19137E2179
R_ONE = (1 << 256) % R_MOD                      # 1 in raw Montgomery form


def code(f):
    with pytest.raises(DpError) as e:
        f()
    return e.value.code


# ------------------------------------------------------------------ the accumulating quotient
def check_accumulate(orc, c, n, m, seed, tails):
    ratio = m // n
    sel = [orc.gen_fr(seed + i, m) for i in range(13)]
    sig = [orc.gen_fr(seed + 20 + i, m) for i in range(5)]
    w = [orc.gen_fr(seed + 30 + i, m) for i in range(5)]
    z, pi = orc.gen_fr(seed + 40, m), orc.gen_fr(seed + 41, m)
    k = orc.gen_fr(seed + 42, 5)
    al, be, ga, s = (orc.gen_fr(seed + 43 + i, 1)[0] for i in range(4))
    tail_arrays = [np.ascontiguousarray(orc.gen_fr(seed + 50 + j, 3)) for j in range(6)]
    tl = [(t.ctypes.data, 2) for t in tail_arrays[:5]] + [(tail_arrays[5].ctypes.data, 3)] if tails else None
    whole = sel + sig + w + [z, pi]
    ptr = [a.ctypes.data for a in whole]
    args = (ptr[:13], ptr[13:18], ptr[18:23], ptr[23], ptr[24], k, al, be, ga)
    q = np.zeros((m, 4), dtype=np.uint64)
    if tails:
        c.quotient_evals_tail_dev(*args, tl, q.ctypes.data)
    else:
        q = orc.quotient_evals(np.stack(sel), np.stack(sig), np.stack(w), z, pi, k, al, be, ga, n)
    out0 = np.ascontiguousarray(orc.gen_fr(seed + 60, m))
    want = orc.vec_op("add", out0, orc.vec_op("mul", q, np.broadcast_to(s, q.shape).copy()))
    got = out0.copy()
    c.quotient_evals_acc_dev(*args, tl, s, got.ctypes.data)
    assert np.array_equal(got, want), f"whole coset n={n} m={m} tails={tails}"
    got = out0.copy()
    for sl in range(ratio):
        arrs = [np.ascontiguousarray(a[sl::ratio]) for a in whole]
        p = [a.ctypes.data for a in arrs]
        before = got.copy()
        c.quotient_evals_acc_dev(p[:13], p[13:18], p[18:23], p[23], p[24], k, al, be, ga, tl, s, got.ctypes.data, sl)
        touched = np.zeros(m, dtype=bool)
        touched[sl::ratio] = True
        assert np.array_equal(got[~touched], before[~touched]), f"slice {sl} wrote outside its points"
        assert np.array_equal(got[touched], want[touched]), f"slice {sl} n={n} m={m} tails={tails}"
    assert np.array_equal(got, want)


@pytest.mark.parametrize("table", ["0", "1"])
@pytest.mark.parametrize("tails", [False, True])
@pytest.mark.parametrize("n,m", [(64, 512), (16, 64)])
def test_accumulate_equals_out_plus_scaled_quotient(orc, emul_lib, monkeypatch, table, tails, n, m):
    monkeypatch.setenv("DP_QUOT_TABLE", table)          # read by dp_create: 0 = product-tree variant, 1 = cached table
    c = Context(emul_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, m)
    check_accumulate(orc, c, n, m, 19000 + n + m + 7 * tails, tails)
    c.close()


def test_accumulate_errors(orc, emul_lib):
    c = Context(emul_lib, 0, 0, 1)
    arrs = [np.zeros((128, 4), dtype=np.uint64) for _ in range(25)]
    k5, one = orc.gen_fr(19100, 5), orc.gen_fr(19101, 1)[0]
    out = np.zeros((128, 4), dtype=np.uint64)
    tail = np.zeros((3, 4), dtype=np.uint64)

    def acc(out_ptr=out.ctypes.data, scale=one, sl=None, a=arrs, tails=None):
        p = [t.ctypes.data for t in a]
        c.quotient_evals_acc_dev(p[:13], p[13:18], p[18:23], p[23], p[24], k5, one, one, one, tails, scale, out_ptr, sl)

    assert code(acc) == -2                                                                    # before dp_init
    c.init(np.zeros(0, dtype=np.uint8), 16, 128)
    acc()
    acc(sl=7, a=[t[:16] for t in arrs])
    assert code(lambda: acc(sl=8, a=[t[:16] for t in arrs])) == -1                            # slice >= m/n
    assert code(lambda: acc(out_ptr=arrs[3].ctypes.data)) == -1                                # the output is input 3
    assert code(lambda: acc(out_ptr=arrs[24].ctypes.data + 32 * 100)) == -1                    # overlaps input 24
    assert code(lambda: acc(sl=2, out_ptr=arrs[9].ctypes.data, a=[t[:16] for t in arrs])) == -1
    assert code(lambda: acc(scale=np.frombuffer(R_MOD.to_bytes(32, "little"), dtype=np.uint64))) == -1   # scale = r
    big = np.zeros((256, 4), dtype=np.uint64)
    assert code(lambda: acc(out_ptr=big.ctypes.data, tails=[(big.ctypes.data + 32 * 5, 2)] + [(None, 0)] * 5)) == -1  # tail overlaps
    assert code(lambda: acc(tails=[(tail.ctypes.data, 4)] + [(None, 0)] * 5)) == -1           # tail of 4
    c.close()


# ------------------------------------------------------------------ more than 32 operands
def test_lincomb_chains_past_32_operands_in_place(orc, emul_lib):
    c = Context(emul_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), 16, 128)
    ln = 40
    polys = [np.ascontiguousarray(orc.gen_fr(19200 + i, 20 + (i % 7))) for i in range(70)]
    coeffs = orc.gen_fr(19300, 70)
    for k in (31, 32, 33, 62, 63, 70):
        want = np.zeros((ln, 4), dtype=np.uint64)
        for p, cf in zip(polys[:k], coeffs[:k]):
            term = np.zeros((ln, 4), dtype=np.uint64)
            term[:p.shape[0]] = orc.vec_op("mul", p, np.broadcast_to(cf, p.shape).copy())
            want = orc.vec_op("add", want, term)
        out = np.full((ln, 4), 7, dtype=np.uint64)
        c.poly_lincomb([p.ctypes.data for p in polys[:k]], coeffs[:k], out_len=ln, lens=[p.shape[0] for p in polys[:k]], out_ptr=out.ctypes.data)
        assert np.array_equal(out, want), f"{k} operands"
    # one call with the output as operand 0: out = 1 * out + c * p
    out = np.ascontiguousarray(orc.gen_fr(19400, ln))
    want = orc.vec_op("add", out, orc.vec_op("mul", np.pad(polys[0], ((0, ln - polys[0].shape[0]), (0, 0))), np.broadcast_to(coeffs[0], (ln, 4)).copy()))
    one = np.frombuffer(R_ONE.to_bytes(32, "little"), dtype=np.uint64)
    c.poly_lincomb([out.ctypes.data, polys[0].ctypes.data], np.stack([one, coeffs[0]]), out_len=ln, lens=[ln, polys[0].shape[0]], out_ptr=out.ctypes.data)
    assert np.array_equal(out, want)
    c.close()


# ------------------------------------------------------------------ the prover
class Setup:
    """a context over universal_setup(TAU), a prover of one satisfied circuit and three witnesses of it with distinct
    public inputs"""

    def __init__(self, orc, lib, log_n, seed, quotient="auto"):
        n = 1 << log_n
        self.ctx = Context(lib, 0, 0, 1)
        universal_setup(self.ctx, torch, n + 2, n, 8 * n, tau=TAU, device="cpu")
        self.ok = open_key(self.ctx, TAU)
        self.pr, _, (self.sel, self.wv, w0, _) = tc.prover_from_circuit(orc, self.ctx, log_n, seed, "cpu", quotient)
        self.vk = self.pr.verifying_key()
        self.witnesses = [w0] + [another_witness(orc, self.sel, self.wv, w0, seed + 1 + i) for i in range(2)]
        self.seed = seed

    def wit(self, i):
        return tc.witness_host(self.witnesses[i % len(self.witnesses)], "cpu")


def another_witness(orc, sel, wv, witness, seed, num_inputs=3, pool=12):
    """a second satisfying witness of test_circuit.satisfied_circuit's circuit: new public inputs and free variables, the
    gate outputs solved again as satisfied_circuit solves them"""
    V = orc.vec_op
    n = sel[0].shape[0]
    wv = wv.reshape(N_WIRE, n)
    gen = np.arange(num_inputs, n - n // 4)
    w = witness.copy()
    w[1:1 + num_inputs + pool] = orc.gen_fr(seed, num_inputs + pool)
    a, b, cc, d = (w[wv[i, gen].astype(np.int64)] for i in range(4))
    g = [s[gen] for s in sel]
    ab, cd = V("mul", a, b), V("mul", cc, d)
    p5 = lambda v: V("mul", V("mul", V("mul", v, v), V("mul", v, v)), v)
    rest = g[11]
    for q, v in ((g[0], a), (g[1], b), (g[2], cc), (g[3], d), (g[4], ab), (g[5], cd), (g[6], p5(a)), (g[7], p5(b)), (g[8], p5(cc)), (g[9], p5(d))):
        rest = V("add", rest, V("mul", q, v))
    w[wv[4, gen].astype(np.int64)] = V("mul", rest, V("inv", V("sub", g[10], V("mul", g[12], V("mul", ab, cd)))))
    return w


@pytest.fixture(scope="module")
def s6(orc, emul_lib):
    s = Setup(orc, emul_lib, 6, 19500)
    yield s
    s.ctx.close()


def both_verify(orc, s, pubs, bp):
    """the pairing verifier and the trapdoor check agree; returns their verdict"""
    got = verify_batch_proof(s.ctx, s.vk, s.ok, pubs, bp)
    want = pbv.verify_batch(orc, s.vk, pubs, bp, TAU)
    assert got == want, f"pairing verifier {got}, trapdoor check {want}"
    return got


@pytest.mark.parametrize("log_n", [6, 7])
@pytest.mark.parametrize("quotient", ["whole", "sliced"])
def test_batch_of_one_equals_prove_circuit(orc, emul_lib, quotient, log_n):
    s = Setup(orc, emul_lib, log_n, 19600 + log_n, quotient)
    for blind in (False, orc.gen_fr(19610, N_BLIND)):
        proof, pub = s.pr.prove_circuit(s.wit(1), blind=blind)
        ch = dict(s.pr.last_challenges)
        bp, pubs = s.pr.prove_batch([s.wit(1)], blind=blind if blind is False else [blind])
        assert pubs == [pub] and len(bp) == 1
        assert bp.instance(0) == proof, f"{quotient}, blinded={blind is not False}"
        assert sorted(s.pr.last_challenges) == sorted(ch)
        assert all(np.array_equal(s.pr.last_challenges[k], ch[k]) for k in ch), "the batch of one draws other challenges"
        derived = pbv.batch_challenges(s.vk, pubs, bp)
        assert derived == pv.challenges(s.vk, pub, proof)
        assert s.pr.last_transcript_ms > 0
        assert both_verify(orc, s, pubs, bp)
    s.ctx.close()


@pytest.mark.parametrize("k", [2, 3, 7])
def test_batches_are_accepted(orc, s6, k):
    bp, pubs = s6.pr.prove_batch([s6.wit(i) for i in range(k)])
    assert len(bp) == k and len(pubs) == k
    assert pubs[0] != pubs[1]
    assert both_verify(orc, s6, pubs, bp)
    b = bp.to_bytes()
    assert len(b) == 368 + 632 * k
    assert batch_proof_from_bytes(s6.ctx, b) == bp


def tampered(bp, where, i, j):
    """bp with instance i's commitment or evaluation j changed (the quotient chunks and openings: i ignored)"""
    wires = [list(ws) for ws in bp.wires_poly_comms_vec]
    perm = list(bp.prod_perm_poly_comms_vec)
    evals = [ProofEvaluations(list(e.wires_evals), list(e.wire_sigma_evals), e.perm_next_eval) for e in bp.poly_evals_vec]
    quot, W, Wn = list(bp.split_quot_poly_comms), bp.opening_proof, bp.shifted_opening_proof
    if where == "wire":
        wires[i][j] = tp.another_point(wires[i][j])
    elif where == "perm":
        perm[i] = tp.another_point(perm[i])
    elif where == "quot":
        quot[j] = tp.another_point(quot[j])
    elif where == "open":
        W, Wn = (tp.another_point(W), Wn) if j == 0 else (W, tp.another_point(Wn))
    else:
        ev = evals[i].evaluations()
        ev[j] = (ev[j] + 1) % R_MOD
        evals[i] = ProofEvaluations(ev[:5], ev[5:9], ev[9])
    return BatchProof(wires, perm, evals, quot, W, Wn)


def test_tampered_batches_are_rejected(orc, s6):
    k = 3
    bp, pubs = s6.pr.prove_batch([s6.wit(i) for i in range(k)], blind=[orc.gen_fr(19700 + i, N_BLIND) for i in range(k)])
    assert both_verify(orc, s6, pubs, bp)
    cases = [("wire", i, j) for i in range(k) for j in (0, 4)] + [("perm", i, 0) for i in range(k)] + [("quot", 0, j) for j in (0, 4)] \
        + [("open", 0, j) for j in (0, 1)] + [("eval", i, j) for i in range(k) for j in (0, 5, 9)]
    for where, i, j in cases:
        assert not both_verify(orc, s6, pubs, tampered(bp, where, i, j)), f"accepted a batch with {where} {i}/{j} changed"
    assert not both_verify(orc, s6, [pubs[1], pubs[0], pubs[2]], bp), "accepted swapped public inputs"
    assert not both_verify(orc, s6, pubs[:2] + [[(pubs[2][0] + 1) % R_MOD] + pubs[2][1:]], bp), "accepted a changed public input"
    # instance 1's witness does not satisfy the circuit: a free variable changed
    w = s6.witnesses[1].copy()
    w[1 + 3] = orc.gen_fr(19710, 1)[0]
    bad, bad_pubs = s6.pr.prove_batch([s6.wit(0), tc.witness_host(w, "cpu"), s6.wit(2)])
    assert bad_pubs == pubs and not both_verify(orc, s6, bad_pubs, bad), "accepted a batch with an unsatisfying witness"


def test_batch_proof_bytes_and_malformed_encodings(orc, s6):
    k = 2
    bp, pubs = s6.pr.prove_batch([s6.wit(i) for i in range(k)])
    b = bp.to_bytes()
    assert len(b) == 368 + 632 * k
    back = batch_proof_from_bytes(s6.ctx, b)
    assert back == bp and verify_batch_proof(s6.ctx, s6.vk, s6.ok, pubs, back)
    u64 = lambda v: v.to_bytes(8, "little")
    patched = lambda off, new: b[:off] + new + b[off + len(new):]
    wires_end = 8 + k * (8 + 5 * 48)
    perm_end = wires_end + 8 + k * 48
    ev0 = perm_end + 8                                           # instance 0's evaluation record
    quot = perm_end + 8 + k * 336
    not_sq = next(x for x in range(1, 100) if pow((x ** 3 + 4) % FQ_MOD, (FQ_MOD - 1) // 2, FQ_MOD) != 1)
    cases = {
        "truncated": b[:-1], "empty": b"", "trailing": b + b"\x00",
        "k = 0": u64(0) + b[8:],
        "instance 1 has 4 wires": patched(8 + 8 + 5 * 48, u64(4)),
        "3 permutation commitments": patched(wires_end, u64(3)),
        "1 evaluation record": patched(perm_end, u64(1)),
        "4 wire evals": patched(ev0, u64(4)),
        "5 sigma evals": patched(ev0 + 8 + 5 * 32, u64(5)),
        "6 quotient chunks": patched(quot, u64(6)),
        "evaluation = r": patched(ev0 + 8 + 32, R_MOD.to_bytes(32, "little")),
        "perm_next_eval >= r": patched(ev0 + 336 - 32, ((1 << 256) - 1).to_bytes(32, "little")),
        "x >= p": patched(8 + 8, FQ_MOD.to_bytes(48, "little")),
        "no such point": patched(wires_end + 8, not_sq.to_bytes(48, "little")),
        "outside the subgroup": patched(len(b) - 48, orc.g1_point_outside_subgroup().tobytes()),
        "both flags": patched(quot + 8 + 47, bytes([b[quot + 8 + 47] | 0xC0])),
    }
    for name, enc in cases.items():
        with pytest.raises(ValueError):
            batch_proof_from_bytes(s6.ctx, enc)
            pytest.fail(name)


def test_argument_errors(orc, s6, monkeypatch):
    bp, pubs = s6.pr.prove_batch([s6.wit(0), s6.wit(1)])
    bad_calls = [
        lambda: verify_batch_proof(s6.ctx, s6.vk, s6.ok, pubs[:1], bp),
        lambda: verify_batch_proof(s6.ctx, s6.vk, s6.ok, pubs + [pubs[0]], bp),
        lambda: verify_batch_proof(s6.ctx, s6.vk, s6.ok, [pubs[0][:-1], pubs[1]], bp),
        lambda: verify_batch_proof(s6.ctx, s6.vk, s6.ok, [pubs[0], [R_MOD] + pubs[1][1:]], bp),
        lambda: verify_batch_proof(s6.ctx, s6.vk, s6.ok, [], BatchProof([], [], [], bp.split_quot_poly_comms, bp.opening_proof, bp.shifted_opening_proof)),
        lambda: verify_batch_proof(s6.ctx, s6.vk, s6.ok, pubs, BatchProof([bp.wires_poly_comms_vec[0][:4], bp.wires_poly_comms_vec[1]], *[getattr(bp, f) for f in (
            "prod_perm_poly_comms_vec", "poly_evals_vec", "split_quot_poly_comms", "opening_proof", "shifted_opening_proof")])),
        lambda: verify_batch_proof(s6.ctx, s6.vk, s6.ok, pubs, tampered_eval_out_of_range(bp)),
        lambda: s6.pr.prove_batch([]),
        lambda: s6.pr.prove_batch([s6.wit(0), torch.zeros((5, 4), dtype=torch.int64)]),
        lambda: s6.pr.prove_batch([s6.wit(0), s6.wit(1)], blind=[orc.gen_fr(1, N_BLIND)]),
        lambda: s6.pr.prove_batch([s6.wit(0)], blind=[orc.gen_fr(1, N_BLIND - 1)]),
        lambda: s6.pr.prove_batch([s6.wit(0)], blind=[True]),
    ]
    for j, f in enumerate(bad_calls):
        with pytest.raises(ValueError):
            f()
            pytest.fail(f"call {j}")
    monkeypatch.setattr(ResidentProver, "CPU_MAX_BATCH", 2)
    assert s6.pr.max_batch() == 2
    with pytest.raises(ValueError):
        s6.pr.prove_batch([s6.wit(i) for i in range(3)])
    pr = ResidentProver(s6.ctx, torch, 6, "cpu", s6.pr.F)
    with pytest.raises(ValueError):
        pr.prove_batch([s6.wit(0)])                                # no circuit loaded
    assert len(s6.vk.selector_comms) == N_SEL


def tampered_eval_out_of_range(bp):
    e = bp.poly_evals_vec[1]
    evals = [bp.poly_evals_vec[0], ProofEvaluations(list(e.wires_evals), list(e.wire_sigma_evals), R_MOD)]
    return BatchProof(bp.wires_poly_comms_vec, bp.prod_perm_poly_comms_vec, evals, bp.split_quot_poly_comms, bp.opening_proof, bp.shifted_opening_proof)


@pytest.mark.timeout(1500)
@pytest.mark.skipif(os.environ.get("DP_TEST_EMUL_ASYNC", "0") == "1", reason="this test starts the asynchronous runs itself")
def test_batch_under_adversarial_stream_schedules():
    """a batch of one against prove_circuit and a batch of 3 through both verifiers on the asynchronous-stream emulator
    build, with the compute, copy-in and MSM tail streams in turn made pathologically slow (tests/test_emul_async.py):
    the instances' buffers and round 3's evaluation buffers are reused in stream order"""
    from tests.emul import build as emul_build
    emul_build.build(async_streams=True)
    select = "(batch_of_one and sliced and 6) or (batches_are_accepted and 3)"
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
