"""Blinded proofs on the kernel-logic emulator: dp_poly_blind_dev against the oracle's p + b(X)(X^n - 1); the quotient
with tails (dp_quotient_evals[_slice]_tail_dev) against the oracle's quotient of the full polynomials' coset evaluations,
for mixed tail lengths, ratios 1-16, both 1/(x - 1) modes, the whole coset and every slice; the blinded resident prover
against an oracle restatement of the proof with the same blinders, in both round-3 layouts, also under adversarial
asynchronous stream schedules; and the degree of its quotient on a satisfied circuit, which the reference requires."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context, DpError
from distributed_plonk_b200.resident import BLIND_WIRE, BLIND_Z, N_BLIND, N_SEL, N_WIRE, NumpyField, ResidentProver
from tests import common

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def code(f):
    with pytest.raises(DpError) as e:
        f()
    return e.value.code


def blinded(orc, p, b, n):
    """p + b(X) * (X^n - 1) by the oracle: p (at most n coefficients) zero-extended to n + len(b)"""
    k = b.shape[0]
    full = np.zeros((n + k, 4), dtype=np.uint64)
    full[:p.shape[0]] = p
    hi = np.zeros_like(full)
    hi[n:] = b
    lo = np.zeros_like(full)
    lo[:k] = b
    return orc.poly_lincomb([full, hi, lo], np.stack([common._fr_one(orc)] * 2 + [common._fr_neg_one(orc)]))


# ------------------------------------------------------------------ dp_poly_blind_dev
@pytest.mark.parametrize("n", [1, 2, 64])
@pytest.mark.parametrize("k", [2, 3])
def test_blind_matches_the_oracle(orc, emul_lib, n, k):
    c = Context(emul_lib, 0, 0, 1)
    p = orc.gen_fr(6000 + n + k, n)
    b = orc.gen_fr(6100 + n + k, k)
    buf = np.zeros((n + k, 4), dtype=np.uint64)
    buf[:n] = p
    c.poly_blind_dev(buf.ctypes.data, n, k, b)
    assert np.array_equal(buf, blinded(orc, p, b, n))
    c.close()


def test_blind_with_library_scalars(orc, emul_lib):
    """NULL scalars: two calls blind differently, and the blinded polynomial keeps its values on H"""
    log_n = 6
    n = 1 << log_n
    F = NumpyField(log_n)
    c = Context(emul_lib, 0, 0, 1)
    p = orc.gen_fr(6200, n)
    outs = []
    for _ in range(2):
        buf = np.zeros((n + 3, 4), dtype=np.uint64)
        buf[:n] = p
        c.poly_blind_dev(buf.ctypes.data, n, 3)
        outs.append(buf)
    assert not np.array_equal(outs[0], outs[1])
    assert outs[0][n:].any() and outs[1][n:].any()
    for i in (0, 1, 17, n - 1):
        x = F.pow_u64(F.omega, i)
        want = c.poly_eval(p, x)
        for buf in outs:
            assert np.array_equal(c.poly_eval(buf, x), want), f"the blinded polynomial at omega^{i}"
    c.close()


def test_blind_errors(orc, emul_lib):
    c = Context(emul_lib, 0, 0, 1)
    buf = np.zeros((8, 4), dtype=np.uint64)
    assert code(lambda: c.poly_blind_dev(buf.ctypes.data, 4, 4)) == -1                 # k > 3
    assert code(lambda: c.poly_blind_dev(buf.ctypes.data, 4, 4, orc.gen_fr(1, 4))) == -1
    assert code(lambda: c.poly_blind_dev(0, 4, 2)) == -1                               # NULL buffer
    r = np.array([0xffffffff00000001, 0x53bda402fffe5bfe, 0x3339d80809a1d805, 0x73eda753299d7d48], dtype=np.uint64)
    assert code(lambda: c.poly_blind_dev(buf.ctypes.data, 4, 2, np.stack([r, r]))) == -1  # a scalar not below r
    assert not buf.any()
    c.poly_blind_dev(buf.ctypes.data, 4, 0)                                            # k = 0: nothing to add
    assert not buf.any()
    c.close()


# ------------------------------------------------------------------ the quotient with tails
def tail_instance(orc, n, m, seed, lens):
    """25 arrays of m points: selectors, sigmas and the public input arbitrary; wires and z the coset evaluations of the
    HEADS of polynomials with n + lens[j] coefficients.  Returns (head arrays, tails, oracle's quotient of the full ones)"""
    sel = [orc.gen_fr(seed + i, m) for i in range(13)]
    sig = [orc.gen_fr(seed + 20 + i, m) for i in range(5)]
    pi = orc.gen_fr(seed + 41, m)
    k = orc.gen_fr(seed + 42, 5)
    ch = [orc.gen_fr(seed + 43 + i, 1)[0] for i in range(3)]

    def coset(coeffs):          # evaluations on the m-point quotient coset; Horner where the m-point transform is too short
        if coeffs.shape[0] <= m:
            return orc.fft(np.concatenate([coeffs, np.zeros((m - coeffs.shape[0], 4), dtype=np.uint64)]), False, True)
        return orc.ntt_outputs_at(coeffs, m, np.arange(m, dtype=np.uint64), False, True)

    heads, tails, full = [], [], []
    for j, t in enumerate(lens):
        coeffs = orc.gen_fr(seed + 30 + j, n + t)
        heads.append(coset(coeffs[:n]))
        tails.append(np.ascontiguousarray(coeffs[n:]))
        full.append(coset(coeffs))
    want = orc.quotient_evals(np.stack(sel), np.stack(sig), np.stack(full[:5]), full[5], pi, k, *ch, n)
    return sel + sig + heads[:5] + [heads[5], pi], tails, (k, *ch), want


def check_tail_quotient(orc, c, n, m, seed, lens):
    """the whole coset and every slice against the oracle; with every length 0, against the entries without tails"""
    arrs, tails, (k, al, be, ga), want = tail_instance(orc, n, m, seed, lens)
    tl = [(t.ctypes.data if t.shape[0] else None, t.shape[0]) for t in tails]
    p = [a.ctypes.data for a in arrs]
    got = np.zeros((m, 4), dtype=np.uint64)
    c.quotient_evals_tail_dev(p[:13], p[13:18], p[18:23], p[23], p[24], k, al, be, ga, tl, got.ctypes.data)
    assert np.array_equal(got, want), f"whole-coset quotient with tails {lens}, n={n} m={m}"
    ratio = m // n
    got = np.zeros((m, 4), dtype=np.uint64)
    for s in range(ratio):
        q = [np.ascontiguousarray(a[s::ratio]) for a in arrs]
        qp = [a.ctypes.data for a in q]
        c.quotient_evals_slice_tail_dev(qp[:13], qp[13:18], qp[18:23], qp[23], qp[24], k, al, be, ga, tl, s, got.ctypes.data)
        if not any(lens):
            plain = np.zeros((m, 4), dtype=np.uint64)
            c.quotient_evals_slice_dev(qp[:13], qp[13:18], qp[18:23], qp[23], qp[24], k, al, be, ga, s, plain.ctypes.data)
            assert np.array_equal(got[s::ratio], plain[s::ratio]), f"slice {s} without tails"
    assert np.array_equal(got, want), f"quotient slices with tails {lens}, n={n} m={m}"
    if not any(lens):
        plain = np.zeros((m, 4), dtype=np.uint64)
        c.quotient_evals_dev(p[:13], p[13:18], p[18:23], p[23], p[24], k, al, be, ga, plain.ctypes.data)
        assert np.array_equal(got, plain)


LENS = [(2, 2, 2, 2, 2, 3), (0, 1, 2, 3, 0, 3), (3, 0, 1, 0, 2, 1), (1, 3, 0, 2, 3, 0), (0, 0, 0, 0, 0, 0)]


@pytest.mark.parametrize("table", ["0", "1"])
@pytest.mark.parametrize("n,m", [(16, 16), (16, 32), (16, 128), (8, 128), (64, 512)])
def test_tail_quotient_matches_the_oracle(orc, emul_lib, monkeypatch, table, n, m):
    monkeypatch.setenv("DP_QUOT_TABLE", table)          # read by dp_create: 0 = product-tree variant, 1 = cached table
    c = Context(emul_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, m)
    for j, lens in enumerate(LENS):
        check_tail_quotient(orc, c, n, m, 6300 + 100 * j + n + m, lens)
    c.close()


def test_tail_quotient_errors(orc, emul_lib):
    n, m = 16, 128
    c = Context(emul_lib, 0, 0, 1)
    arrs = [np.zeros((m, 4), dtype=np.uint64) for _ in range(25)]
    one = orc.gen_fr(6900, 1)[0]
    k5 = orc.gen_fr(6901, 5)
    tail = orc.gen_fr(6902, 4)
    out = np.zeros((m, 4), dtype=np.uint64)
    ok = [(tail.ctypes.data, 2)] * 5 + [(tail.ctypes.data, 3)]

    def whole(tl, out_ptr=out.ctypes.data):
        p = [a.ctypes.data for a in arrs]
        c.quotient_evals_tail_dev(p[:13], p[13:18], p[18:23], p[23], p[24], k5, one, one, one, tl, out_ptr)

    def sliced(tl, s=0, out_ptr=out.ctypes.data):
        p = [a[:n].ctypes.data for a in arrs]
        c.quotient_evals_slice_tail_dev(p[:13], p[13:18], p[18:23], p[23], p[24], k5, one, one, one, tl, s, out_ptr)

    for f in (whole, sliced):
        assert code(lambda: f(ok)) == -2                                              # before dp_init
    c.init(np.zeros(0, dtype=np.uint8), n, m)
    for f in (whole, sliced):
        assert code(lambda: f(ok[:5] + [(tail.ctypes.data, 4)])) == -1                # a tail longer than 3
        assert code(lambda: f([(tail.ctypes.data, 4)] + ok[1:])) == -1
        assert code(lambda: f(ok[:2] + [(None, 1)] + ok[3:])) == -1                   # NULL with a length
        assert code(lambda: f(ok[:5] + [(out.ctypes.data + 32 * 5, 3)])) == -1        # a tail inside the output
        assert code(lambda: f(ok, out_ptr=None)) == -1
        f(ok[:2] + [(None, 0)] + ok[3:])                                             # NULL of length 0 is fine
    assert code(lambda: sliced(ok, 8)) == -1                                          # slice >= m/n
    assert c.lib.dp_quotient_evals_tail_dev(c.h, None, None, out.ctypes.data) == -1               # NULL arguments
    assert c.lib.dp_quotient_evals_slice_tail_dev(c.h, None, None, 0, out.ctypes.data) == -1
    c.close()


# ------------------------------------------------------------------ the blinded prover
def prover_key(orc, log_n, seed):
    n = 1 << log_n
    F = NumpyField(log_n)
    sel = [orc.gen_fr(seed + i, n) for i in range(N_SEL)]
    sig = [orc.gen_fr(seed + 20 + i, n) for i in range(N_WIRE)]
    key = (sel, sig, [orc.fft(s, False, False) for s in sig], [orc.gen_fr(seed + 30 + i, n) for i in range(N_WIRE)],
           np.stack([F.from_u64(v) for v in (1, 7, 13, 17, 23)]))
    wires = [orc.gen_fr(seed + 40 + i, n) for i in range(N_WIRE)]
    pub = orc.gen_fr(seed + 50, n)
    ch = {name: orc.gen_fr(seed + 60 + j, 1)[0] for j, name in enumerate(("beta", "gamma", "alpha", "zeta", "v"))}
    return F, key, wires, pub, ch


def host_inputs(wires, pub, device):
    w = torch.as_tensor(np.concatenate(wires).view(np.int64))
    p = torch.as_tensor(pub.view(np.int64))
    if device != "cpu":
        w, p = w.pin_memory(), p.pin_memory()
    return w, p


def oracle_proof(orc, bases, log_n, key, wires, pub, ch, blind):
    """the reference's sequential computation (dispatcher2.rs:294-690) with the blinders `blind` ([13,4]): 13
    commitments and 10 evaluations"""
    n, m = 1 << log_n, 8 << log_n
    F = NumpyField(log_n)
    sel, sig, sig_ev, id_ev, k = key
    pad = lambda c: np.concatenate([c, np.zeros((m - c.shape[0], 4), dtype=np.uint64)])
    w_coef = [blinded(orc, orc.fft(w, True, False), blind[BLIND_WIRE * i:BLIND_WIRE * (i + 1)], n) for i, w in enumerate(wires)]
    com = [orc.commit(bases, c) for c in w_coef]
    z_ev = orc.perm_product(np.stack(wires), np.stack(id_ev), np.stack(sig_ev), ch["beta"], ch["gamma"])
    z = blinded(orc, orc.fft(z_ev, True, False), blind[N_WIRE * BLIND_WIRE:], n)
    com.append(orc.commit(bases, z))
    pub_coef = orc.fft(pub, True, False)
    cos = [orc.fft(pad(c), False, True) for c in sel + sig + w_coef + [z, pub_coef]]
    q_ev = orc.quotient_evals(np.stack(cos[:13]), np.stack(cos[13:18]), np.stack(cos[18:23]), cos[23], cos[24], k, ch["alpha"], ch["beta"], ch["gamma"], n)
    quot = orc.fft(q_ev, True, True)
    chunk = n + 2
    chunks = [quot[j * chunk:(j + 1) * chunk] for j in range(N_WIRE)]
    com += [orc.commit(bases, c) for c in chunks]
    zeta, zeta_w = ch["zeta"], F.mul(ch["zeta"], F.omega)
    w_ev = [orc.poly_eval(c, zeta) for c in w_coef]
    s_ev = [orc.poly_eval(c, zeta) for c in sig[:-1]]
    z_next = orc.poly_eval(z, zeta_w)
    D, E, R = F._dec, F._enc, F.R_MOD
    a, b, c, d, e = (D(x) for x in w_ev)
    al, be, ga, ze, v = (D(ch[x]) for x in ("alpha", "beta", "gamma", "zeta", "v"))
    vanish = (pow(ze, n, R) - 1) % R
    lag1 = vanish * pow(n * (ze - 1) % R, -1, R) % R
    cz = al
    for wv, kk in zip((a, b, c, d, e), (1, 7, 13, 17, 23)):
        cz = cz * (wv + be * kk * ze + ga) % R
    cz = (cz + al * al * lag1) % R
    cs = al * be * D(z_next) % R
    for wv, sv in zip((a, b, c, d), (D(x) for x in s_ev)):
        cs = cs * (wv + be * sv + ga) % R
    zn2 = (vanish + 1) * ze * ze % R
    coeffs = [a, b, c, d, a * b, c * d, pow(a, 5, R), pow(b, 5, R), pow(c, 5, R), pow(d, 5, R), -e, 1, a * b * c * d * e, cz, -cs]
    coeffs += [-vanish * pow(zn2, j, R) for j in range(N_WIRE)]
    lin = orc.poly_lincomb(sel + [z, sig[-1]] + chunks, np.stack([E(x) for x in coeffs]), n + BLIND_Z)
    batch = orc.poly_lincomb([lin] + w_coef + sig[:-1], np.stack([E(pow(v, j, R)) for j in range(2 * N_WIRE)]), n + BLIND_Z)
    com.append(orc.commit(bases, orc.poly_div_linear(batch, zeta)))
    com.append(orc.commit(bases, orc.poly_div_linear(z, zeta_w)))
    return com, w_ev + s_ev + [z_next]


def check_blinded_prover(orc, ctx, bases, log_n, seed, device, quotient):
    """the blinded prover against the oracle's proof with the same blinders; blind=zeros == blind=False byte for byte;
    blind=True twice gives different commitments for the six blinded polynomials"""
    F, key, wires, pub, ch = prover_key(orc, log_n, seed)
    pr = ResidentProver(ctx, torch, log_n, device, F, quotient=quotient)
    pr.load_key(*key)
    w_host, p_host = host_inputs(wires, pub, device)
    blind = orc.gen_fr(seed + 70, N_BLIND)
    for _ in range(2 if device != "cpu" else 1):               # twice on hardware: nothing of proof k may leak into proof k+1
        com, ev = pr.prove(w_host, p_host, ch, blind=blind)
    want_com, want_ev = oracle_proof(orc, bases, log_n, key, wires, pub, ch, blind)
    assert len(ev) == len(want_ev) == 10
    for j, (got, want) in enumerate(zip(ev, want_ev)):
        assert np.array_equal(got, want), f"evaluation {j} of the blinded proof ({quotient})"
    assert len(com) == len(want_com) == 13
    for j, (got, want) in enumerate(zip(com, want_com)):
        common.assert_point_eq(orc, got, want, f"commitment {j} of the blinded proof ({quotient})")
    plain = pr.prove(w_host, p_host, ch)
    zero = pr.prove(w_host, p_host, ch, blind=np.zeros((N_BLIND, 4), dtype=np.uint64))
    for j, (a, b) in enumerate(zip(plain[0] + plain[1], zero[0] + zero[1])):
        assert np.array_equal(np.asarray(a), np.asarray(b)), f"output {j}: zero blinders differ from the unblinded proof"
    r1, r2 = pr.prove(w_host, p_host, ch, blind=True), pr.prove(w_host, p_host, ch, blind=True)
    for j in range(N_WIRE + 1):
        assert not np.array_equal(orc.normalize(r1[0][j]), orc.normalize(r2[0][j])), f"commitment {j}: two blind=True proofs agree"
        assert not np.array_equal(orc.normalize(r1[0][j]), orc.normalize(plain[0][j])), f"commitment {j}: blind=True left it unblinded"
    return pr


@pytest.mark.parametrize("quotient", ["whole", "sliced"])
def test_blinded_resident_prover(orc, emul_lib, quotient):
    bases = orc.gen_bases(5, 80, 2048, True)        # all distinct: with repeated bases, G_(n+j) = G_j hides a blinding
    c = Context(emul_lib, 0, 0, 1)
    c.init(bases, 1 << 6, 1 << 9)
    check_blinded_prover(orc, c, bases, 6, 7100, "cpu", quotient)
    c.close()


def test_blinded_prover_arguments(orc, emul_lib):
    log_n = 4
    n = 1 << log_n
    F, key, wires, pub, ch = prover_key(orc, log_n, 7200)
    w_host, p_host = host_inputs(wires, pub, "cpu")
    c = Context(emul_lib, 0, 0, 1)
    c.init(orc.gen_bases(5, n + 2, 64, True), n, 8 * n)                 # enough for an unblinded proof only
    pr = ResidentProver(c, torch, log_n, "cpu", F)
    pr.load_key(*key)
    pr.prove(w_host, p_host, ch)
    with pytest.raises(ValueError, match="bases"):
        pr.prove(w_host, p_host, ch, blind=True)
    c.init(orc.gen_bases(5, n + 3, 64, True), n, 8 * n)
    with pytest.raises(ValueError, match="shape"):
        pr.prove(w_host, p_host, ch, blind=np.zeros((12, 4), dtype=np.uint64))
    pr.prove(w_host, p_host, ch, blind=True)
    c.close()


# ------------------------------------------------------------------ the reference's degree check
def satisfied_prover(orc, ctx, log_n, seed, device):
    """a ResidentProver loaded with tests/common.py's satisfied instance; returns (prover, prove(wires, blind))"""
    n = 1 << log_n
    inst = common.make_satisfied_instance(orc, ctx, log_n, seed)
    F = NumpyField(log_n)
    pr = ResidentProver(ctx, torch, log_n, device, F)
    sel_coef = [orc.fft(v, True, False) for v in inst["sel"]]
    sig_coef = [orc.fft(v, True, False) for v in inst["sigma"]]
    pr.load_key(sel_coef, sig_coef, inst["sigma"], inst["ident"], inst["k"])
    ch = {"beta": inst["beta"], "gamma": inst["gamma"], "alpha": inst["alpha"], "zeta": orc.gen_fr(seed + 80, 1)[0],
          "v": orc.gen_fr(seed + 81, 1)[0]}

    def prove(wires, blind):
        w, p = host_inputs(wires, inst["pub"], device)
        pr.prove(w, p, ch, blind=blind)
        q = pr.quot.cpu().numpy().view(np.uint64)
        nz = np.nonzero(q.any(axis=1))[0]
        return int(nz[-1]) if nz.size else -1

    return inst, prove


def check_satisfied_degree(orc, ctx, log_n, seed, device):
    """blinded, the quotient of a satisfied circuit has degree exactly 5(n+1)+2 (dispatcher2.rs, split_quot_polys);
    with one wire value corrupted it does not divide: degree > 7n"""
    n = 1 << log_n
    inst, prove = satisfied_prover(orc, ctx, log_n, seed, device)
    assert prove(inst["w"], False) <= 5 * (n + 1) + 2
    assert prove(inst["w"], orc.gen_fr(seed + 90, N_BLIND)) == 5 * (n + 1) + 2
    assert prove(inst["w"], True) == 5 * (n + 1) + 2
    bad = [v.copy() for v in inst["w"]]
    bad[1][n // 3] = orc.gen_fr(seed + 60, 1)[0]
    assert prove(bad, True) > 7 * n


def test_blinded_quotient_degree_on_a_satisfied_circuit(orc, emul_lib):
    log_n = 6
    n = 1 << log_n
    c = Context(emul_lib, 0, 0, 1)
    c.init(orc.gen_bases(5, n + 3, 64, True), n, 8 * n)
    check_satisfied_degree(orc, c, log_n, 7300, "cpu")
    c.close()


@pytest.mark.timeout(1500)
@pytest.mark.skipif(os.environ.get("DP_TEST_EMUL_ASYNC", "0") == "1", reason="this test starts the asynchronous runs itself")
def test_blinding_under_adversarial_stream_schedules():
    """the blinding, the tail quotient and the blinded prover on the asynchronous-stream emulator build, with the
    compute, copy-in and MSM tail streams in turn made pathologically slow (tests/test_emul_async.py)"""
    from tests.emul import build as emul_build
    emul_build.build(async_streams=True)
    select = "blinded_resident_prover or blind_matches or (tail_quotient_matches and 64-512)"
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


def test_quotient_tails_layout_matches_the_binding(tmp_path):
    """dp_quotient_tails compiles as plain C11 and has the size and field offsets of _binding.QuotientTails"""
    import ctypes

    import distributed_plonk_b200 as dp
    from distributed_plonk_b200 import _binding
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    src = tmp_path / "tails.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "dplonk.h"\n'
        "int main(void) {\n"
        '  printf("%zu %zu %zu %zu %zu\\n", sizeof(dp_quotient_tails), offsetof(dp_quotient_tails, wires),\n'
        "         offsetof(dp_quotient_tails, wire_len), offsetof(dp_quotient_tails, perm), offsetof(dp_quotient_tails, perm_len));\n"
        "  int (*f)(dp_ctx *, const dp_quotient_args *, const dp_quotient_tails *, uint32_t, void *) = dp_quotient_evals_slice_tail_dev;\n"
        "  int (*g)(dp_ctx *, void *, size_t, uint32_t, const void *) = dp_poly_blind_dev;\n"
        "  (void)f; (void)g;\n"
        "  return 0;\n}\n")
    exe = tmp_path / "tails"
    lib = dp.library_path()
    subprocess.check_call([cc, "-std=c11", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{os.path.join(ROOT, 'include')}", str(src), "-o", str(exe),
                           f"-L{os.path.dirname(lib)}", f"-l:{os.path.basename(lib)}", f"-Wl,-rpath,{os.path.dirname(lib)}",
                           "-Wl,--unresolved-symbols=ignore-in-shared-libs"])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    T = _binding.QuotientTails
    assert got == [ctypes.sizeof(T), T.wires.offset, T.wire_len.offset, T.perm.offset, T.perm_len.offset]
