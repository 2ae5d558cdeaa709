"""The Fiat-Shamir transcript (distributed_plonk_b200/transcript.py): both Keccak-f[1600] transcriptions - the package's
lane-based one and tests/plonk_verifier.py's byte-array one - inside SHA3 / SHAKE sponges against hashlib; the two merlin
transcriptions against each other on random operation sequences and on every rate boundary; PlonkTranscript's framing
through a recording stub; the challenge reduction against Python integers."""
import hashlib
import random
import struct

import pytest

from distributed_plonk_b200 import transcript as T
from tests import plonk_verifier as pv


def package_f(st: bytearray):
    T.keccak_f(st)


def sponge(f, msg: bytes, rate: int, pad: int, out_len: int) -> bytes:
    """FIPS 202 sponge over the permutation f (200-byte state)"""
    st = bytearray(200)
    m = bytearray(msg) + bytes([pad])
    m += bytes(-len(m) % rate)
    m[-1] |= 0x80
    for i in range(0, len(m), rate):
        for j in range(rate):
            st[j] ^= m[i + j]
        f(st)
    out = bytearray()
    while len(out) < out_len:
        out += st[:rate]
        if len(out) < out_len:
            f(st)
    return bytes(out[:out_len])


def lengths(rate):
    """0 to 3 rates: the first few, every multiple of the rate and its neighbours, a sample in between"""
    rng = random.Random(rate)
    ls = set(range(0, 4)) | {k * rate + d for k in (1, 2, 3) for d in (-2, -1, 0, 1)} | {rng.randrange(3 * rate) for _ in range(8)}
    return sorted(x for x in ls if 0 <= x <= 3 * rate)


@pytest.mark.parametrize("impl", ["package", "verifier"])
def test_keccak_f1600_in_sha3_and_shake_sponges_matches_hashlib(impl):
    f = package_f if impl == "package" else pv.keccak_f
    rng = random.Random(7)
    for name, rate, pad, out_len, ref in (("sha3_256", 136, 0x06, 32, lambda m: hashlib.sha3_256(m).digest()),
                                           ("sha3_512", 72, 0x06, 64, lambda m: hashlib.sha3_512(m).digest()),
                                           ("shake_128", 168, 0x1F, 400, lambda m: hashlib.shake_128(m).digest(400))):
        for ln in lengths(rate):
            m = bytes(rng.randrange(256) for _ in range(ln))
            assert sponge(f, m, rate, pad, out_len) == ref(m), f"{impl} {name}, {ln}-byte message"


def test_keccak_constants_agree():
    """the package's tabulated round constants and rotations = the verifier's LFSR / (t+1)(t+2)/2 derivation"""
    assert list(T._RC) == pv.ROUND_CONSTANTS
    assert [T._ROT[x + 5 * y] for x in range(5) for y in range(5)] == [pv.RHO[x][y] for x in range(5) for y in range(5)]


def replay(ops, make):
    """run (op, label, arg) on a fresh transcript from make(label); returns every challenge's bytes"""
    t, out = None, []
    for op, label, arg in ops:
        if op == "new":
            t = make(label)
        elif op == "msg":
            t.append_message(label, arg)
        elif op == "ch":
            out.append(t.challenge_bytes(label, arg))
        elif op == "clone":
            t = t.clone()
    return out


def random_ops(rng, count):
    ops = [("new", bytes(rng.randrange(256) for _ in range(rng.randrange(0, 20))), None)]
    for _ in range(count):
        label = bytes(rng.randrange(256) for _ in range(rng.randrange(0, 40)))
        r = rng.random()
        if r < 0.55:
            ops.append(("msg", label, bytes(rng.randrange(256) for _ in range(rng.choice([0, 1, 31, 32, 97, 165, 166, 167, 300, 500])))))
        elif r < 0.9:
            ops.append(("ch", label, rng.randrange(1, 201)))
        else:
            ops.append(("clone", b"", None))
    return ops


@pytest.mark.parametrize("seed", range(6))
def test_the_two_merlin_transcriptions_agree_on_random_sequences(seed):
    ops = random_ops(random.Random(seed), 40)
    assert replay(ops, T.Transcript) == replay(ops, pv.Merlin)


def test_the_two_merlin_transcriptions_agree_on_the_boundaries():
    ops = [("new", b"boundaries", None)]
    for ln in (0, 165, 166, 167, 500):
        ops += [("msg", b"m", bytes((i * 7) & 255 for i in range(ln))), ("ch", b"c", 64)]
    ops += [("ch", b"k", k) for k in (1, 2, 63, 64, 65, 165, 166, 167, 200)]
    assert replay(ops, T.Transcript) == replay(ops, pv.Merlin)
    # a begin_op at every position of the rate, R - 1 included: pad with a message whose length walks the position
    for pad in range(0, 170):
        ops = [("new", b"pos", None), ("msg", b"", bytes(pad)), ("ch", b"", 3), ("msg", b"x", b"y"), ("ch", b"z", 40)]
        assert replay(ops, T.Transcript) == replay(ops, pv.Merlin), f"pad {pad}"
    t = T.Transcript(b"pos")
    t.append_message(b"", bytes(0))
    seen = set()
    for _ in range(170):                                      # 9 bytes per call: a begin_op meets every position, R - 1 too
        seen.add(t.strobe.pos)
        t.append_message(b"", b"\x01")
    assert T.STROBE_R - 1 in seen


def test_clone_equals_a_replay():
    rng = random.Random(99)
    a = T.Transcript(b"clone")
    for _ in range(5):
        a.append_message(b"m", bytes(rng.randrange(256) for _ in range(rng.randrange(300))))
    b = a.clone()
    tail = [(b"x", bytes(range(200))), (b"y", b"")]
    for label, m in tail:
        a.append_message(label, m)
        b.append_message(label, m)
    ca, cb = a.challenge_bytes(b"c", 100), b.challenge_bytes(b"c", 100)
    assert ca == cb
    a.append_message(b"after", b"1")                           # the clone is independent of the original
    assert a.challenge_bytes(b"d", 32) != b.challenge_bytes(b"d", 32)


def test_known_first_bytes_are_stable():
    """the same label, message and challenge give the same bytes in a fresh transcript (no hidden state)"""
    f = lambda: T.Transcript(b"test protocol")
    a, b = f(), f()
    for t in (a, b):
        t.append_message(b"some label", b"some data")
    assert a.challenge_bytes(b"challenge", 32) == b.challenge_bytes(b"challenge", 32)


class Recorder:
    """a stub in place of merlin: records every call; clone() shares the record"""

    def __init__(self, log=None, reply=b""):
        self.log = [] if log is None else log
        self.reply = reply

    def append_message(self, label, message):
        self.log.append((bytes(label), bytes(message)))

    def challenge_bytes(self, label, k):
        self.log.append((bytes(label), k))
        return (self.reply * k)[:k]

    def clone(self):
        return Recorder(self.log, self.reply)


def test_challenge_reduction_and_append():
    for reply in (b"\xff", b"\x01\x02\x03", b"\x00"):
        rec = Recorder(reply=reply)
        c = T.PlonkTranscript(rec).get_and_append_challenge(b"beta")
        want = int.from_bytes((reply * 64)[:64], "little") % T.R_MOD
        assert c == want
        assert rec.log == [(b"beta", 64), (b"beta", want.to_bytes(32, "little"))]


def test_encodings():
    assert T.fr_bytes(5) == (5).to_bytes(32, "little") and len(T.fr_bytes(T.R_MOD - 1)) == 32
    ident = T.g1_bytes(None)
    assert len(ident) == 97 and ident[:48] == bytes(48) and ident[48:96] == (1).to_bytes(48, "little") and ident[96] == 1
    p = (0x1234, 0x5678)
    assert T.g1_bytes(p) == (0x1234).to_bytes(48, "little") + (0x5678).to_bytes(48, "little") + b"\x00"
    assert T.g1_bytes(p) == pv._pt(p) and ident == pv._pt(None)


def test_vk_and_pub_input_framing():
    class VK:
        n, num_inputs = 64, 2
        k = [1, 7, 13, 17, 23]
        selector_comms = [(i + 1, i + 2) for i in range(12)] + [None]
        sigma_comms = [(100 + i, 200 + i) for i in range(5)]

    rec = Recorder()
    T.PlonkTranscript(rec).append_vk_and_pub_input(VK, [3, 4])
    want = [(b"field size in bits", struct.pack("<Q", 255)), (b"domain size", struct.pack("<Q", 64)), (b"input size", struct.pack("<Q", 2))]
    want += [(b"wire subsets separators", k.to_bytes(32, "little")) for k in VK.k]
    want += [(b"selector commitments", T.g1_bytes(c)) for c in VK.selector_comms]
    want += [(b"sigma commitments", T.g1_bytes(c)) for c in VK.sigma_comms]
    want += [(b"public input", v.to_bytes(32, "little")) for v in (3, 4)]
    assert rec.log == want
