"""The trapdoor check of a batch proof for the tests (distributed_plonk_b200 DESIGN.md 3.11): its own merlin transcript
of the batch, written over tests/plonk_verifier.py's byte-array Keccak / Strobe-128 / merlin transcription and apart from
the package's, and the batch equation with the pairing replaced by the known trapdoor tau of a test SRS, as
plonk_verifier.verify does for one proof.

TEST INFRASTRUCTURE ONLY: the product never imports it.  vk and the batch proof are read by attribute (the package's
VerifyingKey and BatchProof); points are affine (x, y) ints or None, field elements canonical ints."""
from __future__ import annotations

import numpy as np

from tests.plonk_verifier import B, R, Merlin, _aff104, _challenge, _fr, _k, _pt


def batch_challenges(vk, pubs, bp) -> dict:
    """beta, gamma, alpha, zeta, v, u of a batch: the vk and public inputs of each instance, then each round's messages of
    every instance"""
    t = Merlin(b"PlonkProof")
    for pub_input in pubs:
        t.append_message(b"field size in bits", (255).to_bytes(8, "little"))
        t.append_message(b"domain size", vk.n.to_bytes(8, "little"))
        t.append_message(b"input size", vk.num_inputs.to_bytes(8, "little"))
        for k in vk.k:
            t.append_message(b"wire subsets separators", _fr(k))
        for c in vk.selector_comms:
            t.append_message(b"selector commitments", _pt(c))
        for c in vk.sigma_comms:
            t.append_message(b"sigma commitments", _pt(c))
        for v in pub_input:
            t.append_message(b"public input", _fr(v))
    ch = {}
    for ws in bp.wires_poly_comms_vec:
        for c in ws:
            t.append_message(b"witness_poly_comms", _pt(c))
    ch["beta"], ch["gamma"] = _challenge(t, b"beta"), _challenge(t, b"gamma")
    for c in bp.prod_perm_poly_comms_vec:
        t.append_message(b"perm_poly_comms", _pt(c))
    ch["alpha"] = _challenge(t, b"alpha")
    for c in bp.split_quot_poly_comms:
        t.append_message(b"quot_poly_comms", _pt(c))
    ch["zeta"] = _challenge(t, b"zeta")
    for e in bp.poly_evals_vec:
        for v in e.wires_evals:
            t.append_message(b"wire_evals", _fr(v))
        for v in e.wire_sigma_evals:
            t.append_message(b"wire_sigma_evals", _fr(v))
        t.append_message(b"perm_next_eval", _fr(e.perm_next_eval))
    ch["v"] = _challenge(t, b"v")
    t.append_message(b"open_proof", _pt(bp.opening_proof))
    t.append_message(b"shifted_open_proof", _pt(bp.shifted_opening_proof))
    ch["u"] = _challenge(t, b"u")
    return ch


def verify_batch(orc, vk, pubs, bp, tau: int) -> bool:
    """tau * (W + u W') == zeta W + u zeta omega W' + F - E for a batch: instance i's linearisation terms weighted with
    alpha^(3i), its openings with v^(1 + 9i + j) (wires), v^(6 + 9i + j) (sigmas) and v^i (z at zeta omega)"""
    ch = batch_challenges(vk, pubs, bp)
    be, ga, al, ze, v, u = (ch[k] for k in ("beta", "gamma", "alpha", "zeta", "v", "u"))
    n, k = vk.n, len(pubs)
    om = B.Domain(n).group_gen
    inv = lambda x: pow(x % R, -1, R)
    zh = (pow(ze, n, R) - 1) % R
    if zh == 0:
        return False
    l1 = zh * inv(n * (ze - 1)) % R
    vs = [pow(v, i, R) for i in range(1 + 9 * k)]
    points, scalars = [], []
    sel_sum, cs_sum, r0_sum, e_sc = [0] * 13, 0, 0, 0
    sig_sum = [0] * 4
    for i, (pub_input, ev) in enumerate(zip(pubs, bp.poly_evals_vec)):
        ai = pow(al, 3 * i, R)
        pi = sum(p * pow(om, j, R) * zh * inv(n * (ze - pow(om, j, R))) for j, p in enumerate(pub_input)) % R
        w, s, zw = list(ev.wires_evals), list(ev.wire_sigma_evals), ev.perm_next_eval
        prod_s = 1
        for wi, si in zip(w[:4], s):
            prod_s = prod_s * (wi + be * si + ga) % R
        r0_sum += ai * (pi - al * al * l1 - al * zw * (w[4] + ga) * prod_s)
        a, b, c, d, e = w
        ab, cd = a * b % R, c * d % R
        sel = [a, b, c, d, ab, cd, pow(a, 5, R), pow(b, 5, R), pow(c, 5, R), pow(d, 5, R), -e, 1, ab * cd * e]
        sel_sum = [x + ai * y for x, y in zip(sel_sum, sel)]
        cz = al
        for wi, ki in zip(w, vk.k):
            cz = cz * (wi + be * ki * ze + ga) % R
        cz = (cz + al * al * l1) % R
        points.append(bp.prod_perm_poly_comms_vec[i])
        scalars.append(ai * cz + u * vs[i])
        cs_sum += ai * (-al * be * zw * prod_s)
        for j in range(5):
            points.append(bp.wires_poly_comms_vec[i][j])
            scalars.append(vs[1 + 9 * i + j])
            e_sc += vs[1 + 9 * i + j] * w[j]
        for j in range(4):
            sig_sum[j] += vs[6 + 9 * i + j]
            e_sc += vs[6 + 9 * i + j] * s[j]
        e_sc += u * vs[i] * zw
    zn2 = pow(ze, n + 2, R)
    points += list(vk.selector_comms) + [vk.sigma_comms[4]] + list(bp.split_quot_poly_comms) + list(vk.sigma_comms[:4])
    scalars += sel_sum + [cs_sum] + [-zh * pow(zn2, j, R) for j in range(5)] + sig_sum
    bases = np.stack([_aff104(p) for p in points])
    sc = np.stack([np.frombuffer(B.fr_to_mont_bytes(x % R), dtype=np.uint64) for x in scalars])
    F = orc.commit(bases, sc)
    e_sc = (e_sc - r0_sum) % R
    gen = orc.g1_generator()
    J = lambda aff: orc.affine_to_jacobian(aff)
    W, Ws = _aff104(bp.opening_proof), _aff104(bp.shifted_opening_proof)
    rhs = orc.g1_add(F, J(orc.g1_mul(gen, _k(-e_sc))))
    rhs = orc.g1_add(rhs, J(orc.g1_mul(W, _k(ze))))
    rhs = orc.g1_add(rhs, J(orc.g1_mul(Ws, _k(u * ze * om))))
    lhs = orc.g1_add(J(orc.g1_mul(W, _k(tau))), J(orc.g1_mul(Ws, _k(tau * u))))
    return bool(np.array_equal(orc.normalize(lhs), orc.normalize(rhs)))
