"""`ref_plonk_v1.bin`: the Fiat-Shamir side of the reference pin (rust/dump_fixtures.rs; format in rust/README.md), in the
container format of tests/ref_fixture.py.  TRANSCRIPT records are merlin op sequences with the challenge bytes the crate
gave; the PLONK record is one small jf-plonk proof with its verifying key, public inputs, the six challenges jf-plonk's
verifier derives and the verify result.  Checker, and a writer that produces the same records from this repository's
transcriptions, so that the checker itself is tested while no Rust toolchain exists."""
from __future__ import annotations

import struct
from types import SimpleNamespace

from distributed_plonk_b200 import transcript as T
from distributed_plonk_b200.proof import Proof
from tests import plonk_verifier as pv

TRANSCRIPT, PLONK = 9, 10
OP_NEW, OP_APPEND, OP_CHALLENGE = 0, 1, 2
CHALLENGES = ("beta", "gamma", "alpha", "zeta", "v", "u")


def encode_ops(ops) -> bytes:
    out = bytearray()
    for kind, label, arg in ops:
        out += bytes([kind]) + struct.pack("<I", len(label)) + label
        if kind == OP_APPEND:
            out += struct.pack("<I", len(arg)) + arg
        elif kind == OP_CHALLENGE:
            out += struct.pack("<I", arg)
    return bytes(out)


def decode_ops(b: bytes):
    ops, off = [], 0
    while off < len(b):
        kind = b[off]
        (ln,) = struct.unpack_from("<I", b, off + 1)
        label = b[off + 5:off + 5 + ln]
        off += 5 + ln
        arg = None
        if kind == OP_APPEND:
            (ml,) = struct.unpack_from("<I", b, off)
            arg = b[off + 4:off + 4 + ml]
            off += 4 + ml
        elif kind == OP_CHALLENGE:
            (arg,) = struct.unpack_from("<I", b, off)
            off += 4
        else:
            assert kind == OP_NEW, f"unknown op {kind}"
        ops.append((kind, label, arg))
    return ops


def replay(ops, make) -> bytes:
    t, out = None, bytearray()
    for kind, label, arg in ops:
        if kind == OP_NEW:
            t = make(label)
        elif kind == OP_APPEND:
            t.append_message(label, arg)
        else:
            out += t.challenge_bytes(label, arg)
    return bytes(out)


def _point(b: bytes):
    """ark-ec 0.3 GroupAffine ToBytes (97 B) -> (x, y) or None"""
    assert len(b) == 97 and b[96] in (0, 1)
    return None if b[96] else (int.from_bytes(b[:48], "little"), int.from_bytes(b[48:96], "little"))


def check(records) -> int:
    """every record against both transcriptions and the package's proof encoder; returns how many were compared"""
    n = 0
    for tag, (a, b, c, d), blobs in records:
        if tag == TRANSCRIPT:
            ops = decode_ops(blobs[0])
            assert len(ops) == a
            assert replay(ops, T.Transcript) == blobs[1], "the package's merlin differs from the record"
            assert replay(ops, pv.Merlin) == blobs[1], "the test verifier's merlin differs from the record"
        elif tag == PLONK:
            vkb, pubb, proofb, chb, ok = blobs
            assert ok == b"\x01", "the reference's verifier rejected its own proof"
            k = [int.from_bytes(vkb[32 * i:32 * (i + 1)], "little") for i in range(5)]
            pts = [_point(vkb[160 + 97 * i:160 + 97 * (i + 1)]) for i in range((len(vkb) - 160) // 97)]
            assert len(pts) == 18, "13 selector + 5 sigma commitments"
            vk = SimpleNamespace(n=a, num_inputs=b, k=k, selector_comms=pts[:13], sigma_comms=pts[13:])
            pub = [int.from_bytes(pubb[i:i + 32], "little") for i in range(0, len(pubb), 32)]
            assert len(pub) == b
            proof = pv.proof_from_bytes(proofb)
            fields = [getattr(proof, f) for f in ("wires_poly_comms", "prod_perm_poly_comm", "split_quot_poly_comms", "opening_proof",
                                                   "shifted_opening_proof", "wires_evals", "wire_sigma_evals", "perm_next_eval")]
            assert Proof(*fields).to_bytes() == proofb, "Proof.to_bytes differs from ark-serialize"
            want = {name: int.from_bytes(chb[32 * i:32 * (i + 1)], "little") for i, name in enumerate(CHALLENGES)}
            assert pv.challenges(vk, pub, proof) == want, "the test verifier derives other challenges"
            tr = T.PlonkTranscript()
            tr.append_vk_and_pub_input(vk, pub)
            tr.append_commitments(b"witness_poly_comms", proof.wires_poly_comms)
            got = {"beta": tr.get_and_append_challenge(b"beta"), "gamma": tr.get_and_append_challenge(b"gamma")}
            tr.append_commitment(b"perm_poly_comms", proof.prod_perm_poly_comm)
            got["alpha"] = tr.get_and_append_challenge(b"alpha")
            tr.append_commitments(b"quot_poly_comms", proof.split_quot_poly_comms)
            got["zeta"] = tr.get_and_append_challenge(b"zeta")
            tr.append_proof_evaluations(proof.wires_evals, proof.wire_sigma_evals, proof.perm_next_eval)
            got["v"] = tr.get_and_append_challenge(b"v")
            assert got == {name: want[name] for name in CHALLENGES[:5]}, "PlonkTranscript derives other challenges"
        else:
            raise AssertionError(f"unknown record tag {tag}")
        n += 1
    return n


def make_from_repo(orc, proof, vk, pub):
    """the record set of rust/dump_fixtures.rs with this repository as the producer: the TRANSCRIPT op sequences, and a
    PLONK record of a proof made by the resident prover (proof, vk, pub as prove_circuit / verifying_key give them)"""
    rec = []
    for msg_lens, ch_lens in (((0, 1, 32, 97), (1, 32, 64)), ((165, 166, 167, 500), (1, 2, 63, 64, 65, 165, 166, 167, 200)),
                              (tuple(range(170)), (3,))):
        ops = [(OP_NEW, b"dump_fixtures", None)]
        for i, ln in enumerate(msg_lens):
            ops += [(OP_APPEND, b"m", bytes((j * 7 + i) & 255 for j in range(ln))), (OP_CHALLENGE, b"c", 64)]
        ops += [(OP_CHALLENGE, b"k", k) for k in ch_lens]
        rec.append((TRANSCRIPT, (len(ops), 0, 0, 0), [encode_ops(ops), replay(ops, T.Transcript)]))
    vkb = b"".join(T.fr_bytes(k) for k in vk.k) + b"".join(T.g1_bytes(p) for p in list(vk.selector_comms) + list(vk.sigma_comms))
    ch = pv.challenges(vk, pub, proof)
    rec.append((PLONK, (vk.n, vk.num_inputs, 0, 0), [vkb, b"".join(T.fr_bytes(v) for v in pub), proof.to_bytes(),
                                                      b"".join(T.fr_bytes(ch[name]) for name in CHALLENGES), b"\x01"]))
    return rec
