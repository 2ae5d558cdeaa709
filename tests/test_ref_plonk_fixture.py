"""Reference-side pin of the transcript and the proof format (rust/README.md): when `tests/golden/ref_plonk_v1.bin` -
written by rust/dump_fixtures.rs through the merlin crate and jf-plonk - is present, both merlin transcriptions, the
PlonkTranscript framing and Proof.to_bytes must reproduce it byte for byte.  Without the file that test skips; the
reader and checker are exercised either way on a file of the same format written from this repository."""
import os

import pytest

from tests import ref_fixture as rf
from tests import ref_plonk_fixture as rpf
from tests import test_proof as tp

REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_plonk_v1.bin")
needs_ref = pytest.mark.skipif(not os.path.exists(REF), reason="tests/golden/ref_plonk_v1.bin absent: produce it with rust/dump_fixtures.rs (needs cargo)")


def test_format_round_trip_and_checker(orc, emul_lib, tmp_path):
    c, pr, witness, _ = tp.setup(orc, emul_lib, 6, 13000, "cpu")
    proof, pub = pr.prove_circuit(tp.tc.witness_host(witness, "cpu"))
    recs = rpf.make_from_repo(orc, proof, pr.verifying_key(), pub)
    c.close()
    path = str(tmp_path / "repo_made.bin")
    rf.write(path, recs)
    back = rf.read(path)
    assert [r[0] for r in back] == [rpf.TRANSCRIPT] * 3 + [rpf.PLONK]
    assert rpf.check(back) == len(recs)
    # a flipped bit in a challenge output, in a proof byte, and in an expected challenge must each be caught
    for idx, blob, pos in ((0, 1, 0), (3, 2, 300), (3, 3, 5)):
        tag, p, blobs = back[idx]
        bad = bytearray(blobs[blob])
        bad[pos] ^= 1
        broken = list(back)
        broken[idx] = (tag, p, blobs[:blob] + [bytes(bad)] + blobs[blob + 1:])
        with pytest.raises((AssertionError, ValueError)):
            rpf.check(broken)


@needs_ref
def test_reference_fixture_pins_the_transcript_and_the_proof_format():
    assert rpf.check(rf.read(REF)) > 0
