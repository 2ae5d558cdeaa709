"""PLONK verification without the trapdoor: jf-plonk's PlonkKzgSnark::verify / batch_verify over the open key
(g, h, beta h) of the setup, with the pairing on the GPU.

The transcript (transcript.PlonkTranscript) and a few dozen Fr scalars per proof stay on the host; the group work is
two MSMs over the proof's and the verifying key's points (dp_msm_points) and one 2-pair multi-pairing
(dp_multi_pairing).  For one proof, with challenges beta, gamma, alpha, zeta, v, u from the transcript:

    A = W + u W'                     B = zeta W + u zeta omega W' + F - E
    accept  <=>  e(A, beta h) * e(-B, h) == 1          (the KZG batch-opening check tau A == B, without tau)

W, W' the two opening proofs, F the linear combination of the 29 committed polynomials jf-plonk's batch check builds
and E = e_scalar * g (DESIGN.md section 3.8).  batch_verify folds k proofs into the same two points with random
r_i: A = sum r_i A_i, B = sum r_i B_i, one MSM each and one pairing call.

verify_batch_proof checks a BatchProof of k instances of one circuit (ResidentProver.prove_batch) with the same two
MSMs and one pairing: instance i's linearisation terms weighted by alpha^(3i), its openings by powers of v (DESIGN.md
section 3.11).

Inputs: proof bytes go through proof_from_bytes, which decodes and subgroup-checks every point on the GPU.  A Proof
object handed to verify is trusted to hold curve points, as jf-plonk's typed Proof is; its evaluations and the public
inputs are range-checked here."""
from __future__ import annotations

import secrets
import struct
import time

import numpy as np

from ._binding import DP_E_ARG, FQ12_BYTES, DpError
from .proof import BatchProof, Proof, ProofEvaluations, VerifyingKey, _Reader, decompress_points, g2_to_raw, point_from_raw, point_to_raw
from .transcript import PlonkTranscript, R_MOD

N_WIRES, N_QUOT, N_SIGMA_EVALS = 5, 5, 4
_TWO_ADIC_ROOT = pow(7, (R_MOD - 1) >> 32, R_MOD)          # Fr's 2^32-th root of unity (generator 7)
_FQ12_ONE = ((1 << 384) % 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB
             ).to_bytes(48, "little") + bytes(FQ12_BYTES - 48)
_DECOMPRESS_WHY = {1: "x is not below p", 2: "both flag bits set", 3: "not a point of the curve", 4: "not in the r-torsion subgroup"}


# ------------------------------------------------------------------ the proof's bytes
def proof_from_bytes(ctx, b: bytes) -> Proof:
    """The inverse of Proof.to_bytes (ark-serialize 0.3 CanonicalDeserialize of jf-plonk's Proof, 976 B).  The 13
    points are decompressed and checked to lie in the r-torsion subgroup on the GPU (dp_g1_decompress).  Raises
    ValueError on a truncated input, trailing bytes, a vector length other than 5 / 5 / 5 / 4, a bad point encoding,
    a point off the curve or outside the subgroup, or an evaluation >= r."""
    b = bytes(b)
    off = 0

    def take(k: int) -> bytes:
        nonlocal off
        if off + k > len(b):
            raise ValueError(f"truncated proof: {len(b)} bytes")
        off += k
        return b[off - k:off]

    def vec(expected: int, size: int, what: str) -> list:
        n = struct.unpack("<Q", take(8))[0]
        if n != expected:
            raise ValueError(f"{what}: {n} entries, expected {expected}")
        return [take(size) for _ in range(n)]

    comp = vec(N_WIRES, 48, "wires_poly_comms") + [take(48)] + vec(N_QUOT, 48, "split_quot_poly_comms") + [take(48), take(48)]
    evals = vec(N_WIRES, 32, "wires_evals") + vec(N_SIGMA_EVALS, 32, "wire_sigma_evals") + [take(32)]
    if off != len(b):
        raise ValueError(f"{len(b) - off} trailing bytes after the proof")
    ev = [int.from_bytes(e, "little") for e in evals]
    for i, v in enumerate(ev):
        if v >= R_MOD:
            raise ValueError(f"evaluation {i} is not below r")
    try:
        raw = ctx.g1_decompress(np.frombuffer(b"".join(comp), dtype=np.uint8).reshape(len(comp), 48), check_subgroup=True)
    except DpError as e:
        if e.code != DP_E_ARG:
            raise
        raise ValueError(f"commitment {e.index} of the proof: {_DECOMPRESS_WHY.get(e.why, e.msg)}") from e
    p = [point_from_raw(r) for r in raw]
    return Proof(p[0:5], p[5], p[6:11], p[11], p[12], ev[0:5], ev[5:9], ev[9])


# ------------------------------------------------------------------ one proof's share of the check
def _check_pub(vk, pub):
    if len(pub) != vk.num_inputs:
        raise ValueError(f"{len(pub)} public inputs, the verifying key expects {vk.num_inputs}")
    for i, v in enumerate(pub):
        if not 0 <= int(v) < R_MOD:
            raise ValueError(f"public input {i} is not a canonical scalar (0 <= v < r)")


def _check_evals(wires_evals, wire_sigma_evals, evaluations):
    if (len(wires_evals), len(wire_sigma_evals)) != (N_WIRES, N_SIGMA_EVALS):
        raise ValueError(f"evaluation vector lengths {(len(wires_evals), len(wire_sigma_evals))}, expected (5, 4)")
    for v in evaluations:
        if not 0 <= int(v) < R_MOD:
            raise ValueError("a proof evaluation is not a canonical scalar (0 <= v < r)")


def _check_shapes(vk, pub, proof):
    _check_pub(vk, pub)
    shape = (len(proof.wires_poly_comms), len(proof.split_quot_poly_comms), len(proof.wires_evals), len(proof.wire_sigma_evals))
    if shape != (N_WIRES, N_QUOT, N_WIRES, N_SIGMA_EVALS):
        raise ValueError(f"proof vector lengths {shape}, expected (5, 5, 5, 4)")
    _check_evals(proof.wires_evals, proof.wire_sigma_evals, proof.evaluations())


def _challenges(vk_transcript: PlonkTranscript, pub, proof) -> tuple:
    """beta, gamma, alpha, zeta, v, u as jf-plonk's verifier derives them, from a transcript that has the vk"""
    t = vk_transcript.clone()
    t.append_pub_input(pub)
    t.append_commitments(b"witness_poly_comms", proof.wires_poly_comms)
    beta, gamma = t.get_and_append_challenge(b"beta"), t.get_and_append_challenge(b"gamma")
    t.append_commitment(b"perm_poly_comms", proof.prod_perm_poly_comm)
    alpha = t.get_and_append_challenge(b"alpha")
    t.append_commitments(b"quot_poly_comms", proof.split_quot_poly_comms)
    zeta = t.get_and_append_challenge(b"zeta")
    t.append_proof_evaluations(proof.wires_evals, proof.wire_sigma_evals, proof.perm_next_eval)
    v = t.get_and_append_challenge(b"v")
    t.append_commitment(b"open_proof", proof.opening_proof)
    t.append_commitment(b"shifted_open_proof", proof.shifted_opening_proof)
    u = t.get_and_append_challenge(b"u")
    return beta, gamma, alpha, zeta, v, u


def _domain(vk, zeta):
    """(omega, Z_H(zeta), L_1(zeta), L_i) of the verifying key's domain, or None when zeta lies in it"""
    n = vk.n
    omega = pow(_TWO_ADIC_ROOT, (1 << 32) // n, R_MOD)
    zh = (pow(zeta, n, R_MOD) - 1) % R_MOD                  # vanishing polynomial at zeta
    if zh == 0:
        return None
    inv = lambda x: pow(x % R_MOD, -1, R_MOD)
    lagrange = lambda w_i: w_i * zh * inv(n * (zeta - w_i)) % R_MOD       # L_i(zeta), w_i = omega^i
    return omega, zh, lagrange(1), lagrange


def _instance_scalars(vk, pub, w, s, z_next, ch, dom):
    """one instance's share of the check: (r0, the 13 selector scalars, z's scalar without u, sigma_4's scalar), from its
    public inputs and evaluations (ints) and the challenges beta, gamma, alpha, zeta"""
    beta, gamma, alpha, zeta = ch[:4]
    omega, zh, l1, lagrange = dom
    pi = sum(int(p) * lagrange(pow(omega, i, R_MOD)) for i, p in enumerate(pub)) % R_MOD
    perm_s = 1                                             # prod_{i < 4} (w_i + beta s_i + gamma)
    for wi, si in zip(w[:4], s):
        perm_s = perm_s * (wi + beta * si + gamma) % R_MOD
    r0 = (pi - alpha * alpha * l1 - alpha * z_next * (w[4] + gamma) * perm_s) % R_MOD
    a, b_, c, d, e = w
    ab, cd = a * b_ % R_MOD, c * d % R_MOD
    q_sel = [a, b_, c, d, ab, cd, pow(a, 5, R_MOD), pow(b_, 5, R_MOD), pow(c, 5, R_MOD), pow(d, 5, R_MOD), -e, 1, ab * cd % R_MOD * e]
    perm_z = alpha
    for wi, ki in zip(w, vk.k):
        perm_z = perm_z * (wi + beta * int(ki) * zeta + gamma) % R_MOD
    perm_z = (perm_z + alpha * alpha * l1) % R_MOD
    sigma_last = -alpha * beta * z_next * perm_s
    return r0, q_sel, perm_z, sigma_last


def _quot_scalars(vk, zeta, zh):
    zeta_n2 = pow(zeta, vk.n + 2, R_MOD)
    return [-zh * pow(zeta_n2, j, R_MOD) for j in range(N_QUOT)]


def _terms(vk, pub, proof, ch):
    """(A points, A scalars, B points, B scalars, scalar of g in B), or None when zeta lies in the domain (the check
    is undefined there and the proof is rejected).  B = zeta W + u zeta omega W' + F - E."""
    beta, gamma, alpha, zeta, v, u = ch
    dom = _domain(vk, zeta)
    if dom is None:
        return None
    omega, zh = dom[0], dom[1]
    w, s, z_next = [int(x) for x in proof.wires_evals], [int(x) for x in proof.wire_sigma_evals], int(proof.perm_next_eval)
    r0, q_sel, perm_z, sigma_last = _instance_scalars(vk, pub, w, s, z_next, ch, dom)
    quot = _quot_scalars(vk, zeta, zh)
    vp = [pow(v, i, R_MOD) for i in range(10)]
    f_points = list(vk.selector_comms) + [proof.prod_perm_poly_comm, vk.sigma_comms[4]] + list(proof.split_quot_poly_comms) \
        + list(proof.wires_poly_comms) + list(vk.sigma_comms[:4])
    f_scalars = q_sel + [perm_z + u, sigma_last] + quot + vp[1:6] + vp[6:10]
    e_scalar = (-r0 + sum(vp[1 + i] * w[i] for i in range(5)) + sum(vp[6 + i] * s[i] for i in range(4)) + u * z_next) % R_MOD
    W, Wn = proof.opening_proof, proof.shifted_opening_proof
    return [W, Wn], [1, u], [W, Wn] + f_points, [zeta, u * zeta % R_MOD * omega] + f_scalars, -e_scalar


def _scalars(vals) -> np.ndarray:
    return np.frombuffer(b"".join((int(x) % R_MOD).to_bytes(32, "little") for x in vals), dtype=np.uint64).reshape(-1, 4)


def _raw_points(pts) -> np.ndarray:
    return np.frombuffer(b"".join(point_to_raw(p) for p in pts), dtype=np.uint8).reshape(-1, 104)


def _jacobian_to_raw(j144: np.ndarray) -> bytes:
    """the library's normalised 144-byte Jacobian (X, Y, 1) or identity (0, 1, 0) -> raw 104-byte affine"""
    b = np.ascontiguousarray(j144, dtype=np.uint8).tobytes()
    if not any(b[96:144]):
        return point_to_raw(None)
    return b[0:96] + bytes(8)


def _check(ctx, open_key, items, rs, timings) -> bool:
    t0 = time.perf_counter()
    terms_list = []
    vk_transcripts = {}
    for vk, pub, proof in items:
        _check_shapes(vk, pub, proof)
        if id(vk) not in vk_transcripts:
            t = PlonkTranscript()
            t.append_vk(vk)
            vk_transcripts[id(vk)] = t
        terms = _terms(vk, pub, proof, _challenges(vk_transcripts[id(vk)], pub, proof))
        if terms is None:
            return False
        terms_list.append(terms)
    return _pairing_check(ctx, open_key, terms_list, rs, timings, t0)


def _pairing_check(ctx, open_key, terms_list, rs, timings, t0) -> bool:
    """sum r_i A_i and -sum r_i B_i (two MSMs), then e(A, beta h) e(-B, h) == 1 (one 2-pair multi-pairing)"""
    a_pts, a_sc, b_pts, b_sc, g_sc = [], [], [], [], 0
    for (pa, sa, pb, sb, sg), r in zip(terms_list, rs):
        a_pts += pa
        a_sc += [r * x for x in sa]
        b_pts += pb
        b_sc += [-r * x for x in sb]                       # -B: the pairing takes e(-B, h)
        g_sc -= r * sg
    b_pts.append(open_key.g)
    b_sc.append(g_sc)
    t1 = time.perf_counter()
    A = ctx.msm_points(_raw_points(a_pts), _scalars(a_sc))
    neg_B = ctx.msm_points(_raw_points(b_pts), _scalars(b_sc))
    t2 = time.perf_counter()
    g1 = np.frombuffer(_jacobian_to_raw(A) + _jacobian_to_raw(neg_B), dtype=np.uint8).reshape(2, 104)
    g2 = np.frombuffer(g2_to_raw(open_key.beta_h) + g2_to_raw(open_key.h), dtype=np.uint8).reshape(2, 200)
    ok = ctx.multi_pairing(g1, g2).tobytes() == _FQ12_ONE
    t3 = time.perf_counter()
    if timings is not None:
        for key, dt in (("transcript_scalars_ms", t1 - t0), ("msm_ms", t2 - t1), ("pairing_ms", t3 - t2)):
            timings[key] = timings.get(key, 0.0) + 1e3 * dt
    return ok


def verify(ctx, vk, open_key, public_inputs, proof, timings: dict | None = None) -> bool:
    """jf-plonk's PlonkKzgSnark::verify: True when the proof is accepted.  A wrong number of public inputs, a public
    input or evaluation outside [0, r), or wrong proof vector lengths raise ValueError; a well-formed proof that fails
    the pairing check returns False.  `timings`, if given, accumulates transcript_scalars_ms / msm_ms / pairing_ms."""
    return _check(ctx, open_key, [(vk, list(public_inputs), proof)], [1], timings)


def batch_verify(ctx, open_key, items, timings: dict | None = None) -> bool:
    """Accept (True) only if every (vk, public_inputs, proof) of `items` would be accepted by verify, up to a
    soundness error of about k / r: each item's A_i and B_i are weighted with a fresh random r_i != 0 (drawn with
    `secrets`, never from the transcript) and the sums checked with one 2-pair pairing.  The items may belong to
    different circuits over the same setup.  An empty list is a ValueError."""
    items = [(vk, list(pub), proof) for vk, pub, proof in items]
    if not items:
        raise ValueError("batch_verify needs at least one proof")
    rs = [1 + secrets.randbelow(R_MOD - 1) for _ in items]
    return _check(ctx, open_key, items, rs, timings)


def verify_bytes(ctx, vk_bytes, open_key_bytes, public_inputs, proof_bytes) -> bool:
    """verify for a party that holds nothing but three byte strings - a verifying key (VerifyingKey.to_bytes), an open key
    (OpenKey.to_bytes) and a proof (Proof.to_bytes) - and the public inputs: no tau, no SRS, no circuit, and a context that
    was never initialised.  Every point is decoded and subgroup-checked on the GPU.  ValueError for a malformed encoding
    or wrong shapes, False for a well-formed proof that is not accepted."""
    from .srs import open_key_from_bytes
    vk = VerifyingKey.from_bytes(ctx, vk_bytes)
    return verify(ctx, vk, open_key_from_bytes(ctx, open_key_bytes), public_inputs, proof_from_bytes(ctx, proof_bytes))


# ------------------------------------------------------------------ batch proofs (ResidentProver.prove_batch, DESIGN.md 3.11)
def batch_proof_from_bytes(ctx, b: bytes) -> BatchProof:
    """The inverse of BatchProof.to_bytes (368 + 632 k bytes).  Every point is decompressed and checked to lie in the
    r-torsion subgroup on the GPU (dp_g1_decompress).  ValueError on a truncated input, trailing bytes, k = 0, per-instance
    vectors whose count is not k, inner lengths other than 5 / 5 / 4, a rejected point or an evaluation >= r."""
    r = _Reader(b, "batch proof")
    k = r.u64()
    if k == 0:
        raise ValueError("batch proof: no instances")
    if 368 + 632 * k > len(r.b):
        raise ValueError(f"truncated batch proof: {len(r.b)} bytes for {k} instances")
    comp = []
    for _ in range(k):
        comp += r.vec(N_WIRES, 48, "wires_poly_comms")
    comp += r.vec(k, 48, "prod_perm_poly_comms_vec")
    if r.u64() != k:
        raise ValueError("batch proof: poly_evals_vec does not have one record per instance")
    evals = []
    for _ in range(k):
        ev = [int.from_bytes(x, "little") for x in r.vec(N_WIRES, 32, "wires_evals") + r.vec(N_SIGMA_EVALS, 32, "wire_sigma_evals") + [r.take(32)]]
        for v in ev:
            if v >= R_MOD:
                raise ValueError("batch proof: an evaluation is not below r")
        evals.append(ProofEvaluations(ev[:5], ev[5:9], ev[9]))
    comp += r.vec(N_QUOT, 48, "split_quot_poly_comms") + [r.take(48), r.take(48)]
    r.end()
    p = decompress_points(ctx, comp, "the batch proof")
    q = 6 * k
    return BatchProof([p[5 * i:5 * i + 5] for i in range(k)], p[5 * k:q], evals, p[q:q + 5], p[q + 5], p[q + 6])


def _batch_challenges(vk, pubs, bp) -> tuple:
    """beta, gamma, alpha, zeta, v, u of a batch: the vk and public inputs of every instance, then each round's messages of
    all instances (DESIGN.md 3.11); a batch of one is a single proof's transcript"""
    t = PlonkTranscript()
    for pub in pubs:
        t.append_vk(vk)
        t.append_pub_input(pub)
    for ws in bp.wires_poly_comms_vec:
        t.append_commitments(b"witness_poly_comms", ws)
    beta, gamma = t.get_and_append_challenge(b"beta"), t.get_and_append_challenge(b"gamma")
    for z in bp.prod_perm_poly_comms_vec:
        t.append_commitment(b"perm_poly_comms", z)
    alpha = t.get_and_append_challenge(b"alpha")
    t.append_commitments(b"quot_poly_comms", bp.split_quot_poly_comms)
    zeta = t.get_and_append_challenge(b"zeta")
    for e in bp.poly_evals_vec:
        t.append_proof_evaluations(e.wires_evals, e.wire_sigma_evals, e.perm_next_eval)
    v = t.get_and_append_challenge(b"v")
    t.append_commitment(b"open_proof", bp.opening_proof)
    t.append_commitment(b"shifted_open_proof", bp.shifted_opening_proof)
    u = t.get_and_append_challenge(b"u")
    return beta, gamma, alpha, zeta, v, u


def _batch_terms(vk, pubs, bp, ch):
    """_terms of a batch: instance i's linearisation scalars weighted by alpha^(3i), its openings by v^(1 + 9i + j) (wires),
    v^(6 + 9i + j) (sigmas) and v^i (z at zeta omega); None when zeta lies in the domain"""
    beta, gamma, alpha, zeta, v, u = ch
    dom = _domain(vk, zeta)
    if dom is None:
        return None
    omega, zh = dom[0], dom[1]
    k = len(pubs)
    a3 = [pow(alpha, 3 * i, R_MOD) for i in range(k)]
    vp = [pow(v, i, R_MOD) for i in range(1 + 9 * k)]
    r0, sel, sigma_last, z_sc, e_scalar = 0, [0] * 13, 0, [], 0
    sig_sc = [0] * N_SIGMA_EVALS
    w_sc = []
    for i, (pub, e) in enumerate(zip(pubs, bp.poly_evals_vec)):
        w, s, z_next = [int(x) for x in e.wires_evals], [int(x) for x in e.wire_sigma_evals], int(e.perm_next_eval)
        r0_i, q_i, perm_z_i, sigma_last_i = _instance_scalars(vk, pub, w, s, z_next, ch, dom)
        r0 += a3[i] * r0_i
        sel = [x + a3[i] * y for x, y in zip(sel, q_i)]
        sigma_last += a3[i] * sigma_last_i
        z_sc.append(a3[i] * perm_z_i + u * vp[i])
        w_sc += [vp[1 + 9 * i + j] for j in range(N_WIRES)]
        sig_sc = [x + vp[6 + 9 * i + j] for j, x in enumerate(sig_sc)]
        e_scalar += sum(vp[1 + 9 * i + j] * w[j] for j in range(N_WIRES)) + sum(vp[6 + 9 * i + j] * s[j] for j in range(N_SIGMA_EVALS)) \
            + u * vp[i] * z_next
    e_scalar = (e_scalar - r0) % R_MOD
    f_points = list(vk.selector_comms) + list(bp.prod_perm_poly_comms_vec) + [vk.sigma_comms[4]] + list(bp.split_quot_poly_comms) \
        + [p for ws in bp.wires_poly_comms_vec for p in ws] + list(vk.sigma_comms[:4])
    f_scalars = [x % R_MOD for x in sel] + z_sc + [sigma_last] + _quot_scalars(vk, zeta, zh) + w_sc + sig_sc
    W, Wn = bp.opening_proof, bp.shifted_opening_proof
    return [W, Wn], [1, u], [W, Wn] + f_points, [zeta, u * zeta % R_MOD * omega] + f_scalars, -e_scalar


def verify_batch_proof(ctx, vk, open_key, public_inputs_list, batch_proof, timings: dict | None = None) -> bool:
    """True when the BatchProof of k instances of the circuit of `vk` is accepted: one transcript, one 2-pair pairing
    (DESIGN.md 3.11).  A number of public-input lists other than k, a wrong number of public inputs, a value outside
    [0, r), k = 0 or wrong vector lengths raise ValueError; a well-formed batch that fails the check returns False.
    `timings` as in verify."""
    t0 = time.perf_counter()
    bp = batch_proof
    k = len(bp.wires_poly_comms_vec)
    pubs = [list(p) for p in public_inputs_list]
    if k == 0:
        raise ValueError("a batch proof of no instances")
    if (len(bp.prod_perm_poly_comms_vec), len(bp.poly_evals_vec), len(pubs)) != (k, k, k):
        raise ValueError(f"{k} instances, {len(bp.prod_perm_poly_comms_vec)} permutation commitments, {len(bp.poly_evals_vec)} "
                         f"evaluation records, {len(pubs)} public-input lists")
    if len(bp.split_quot_poly_comms) != N_QUOT or any(len(ws) != N_WIRES for ws in bp.wires_poly_comms_vec):
        raise ValueError("batch proof vector lengths: 5 wire commitments per instance and 5 quotient chunks expected")
    for pub, e in zip(pubs, bp.poly_evals_vec):
        _check_pub(vk, pub)
        _check_evals(e.wires_evals, e.wire_sigma_evals, e.evaluations())
    terms = _batch_terms(vk, pubs, bp, _batch_challenges(vk, pubs, bp))
    if terms is None:
        return False
    return _pairing_check(ctx, open_key, [terms], [1], timings, t0)
