"""Batch proofs on the GPU (tests/test_batch_proof.py on the emulator): the accumulating quotient equals
dp_poly_lincomb_dev([out0, Q], [1, s]) byte for byte at 2^22 gates over the whole coset and at 2^23 slice by slice; at
2^16 a batch of 4 over universal_setup is accepted by verify_batch_proof and by the trapdoor check, and a batch of one is
prove_circuit's proof; at 2^22 a batch of min(4, max_batch()) is accepted."""
import os

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context
from distributed_plonk_b200.resident import N_BLIND
from distributed_plonk_b200.srs import open_key, universal_setup
from distributed_plonk_b200.verifier import batch_proof_from_bytes, verify_batch_proof
from tests import plonk_batch_verifier as pbv
from tests import plonk_verifier as pv
from tests import test_circuit as tc

pytestmark = pytest.mark.gpu
DRY = os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1"     # tests/conftest.py: the test code itself, on the emulator, tiny sizes
DEV = "cpu" if DRY else "cuda"
TAU = 0x3C6EF372FE94F82BA54FF53A5F1D36F1510E527FADE682D19B05688C2B3E6C1F


def rand_fr(count, gen):
    """count canonical raw Fr on the device (top limb below 2^62 < r's)"""
    x = torch.randint(-(1 << 63), (1 << 63) - 1, (count, 4), dtype=torch.int64, device=DEV, generator=gen)
    x[:, 3] &= (1 << 62) - 1
    return x


def check_accumulate(orc, lib, log_n, sliced):
    n = 1 << log_n
    m = 8 * n
    c = Context(lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, m)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(0xACC + log_n)
    arrays = [rand_fr(n if sliced else m, gen) for _ in range(25)]
    tail_bufs = [rand_fr(3, gen) for _ in range(6)]
    k = orc.gen_fr(0xACC, 5)
    al, be, ga, s = (orc.gen_fr(0xACD + i, 1)[0] for i in range(4))
    P = [a.data_ptr() for a in arrays]
    args = (P[:13], P[13:18], P[18:23], P[23], P[24], k, al, be, ga)
    out0 = rand_fr(m, gen)
    plain, acc, want = torch.empty_like(out0), torch.empty_like(out0), torch.empty_like(out0)
    for tails in (None, [(t.data_ptr(), 2) for t in tail_bufs[:5]] + [(tail_bufs[5].data_ptr(), 3)]):
        acc.copy_(out0)
        if not DRY:
            torch.cuda.synchronize()                          # torch's stream -> the library's
        for sl in (range(8) if sliced else [None]):
            if sl is None:
                (c.quotient_evals_tail_dev(*args, tails, plain.data_ptr()) if tails else c.quotient_evals_dev(*args, plain.data_ptr()))
            elif tails:
                c.quotient_evals_slice_tail_dev(*args, tails, sl, plain.data_ptr())
            else:
                c.quotient_evals_slice_dev(*args, sl, plain.data_ptr())
            c.quotient_evals_acc_dev(*args, tails, s, acc.data_ptr(), sl)
        one = np.frombuffer(((1 << 256) % pv.R).to_bytes(32, "little"), dtype=np.uint64)
        c.poly_lincomb([out0.data_ptr(), plain.data_ptr()], np.stack([one, s]), out_len=m, lens=[m, m], out_ptr=want.data_ptr())
        assert torch.equal(acc, want), f"2^{log_n}, sliced={sliced}, tails={tails is not None}"
    c.close()


def test_accumulate_whole_at_2p22(orc, gpu_lib):
    check_accumulate(orc, gpu_lib, 6 if DRY else 22, False)


def test_accumulate_slices_at_2p23(orc, gpu_lib):
    if not DRY:
        torch.cuda.empty_cache()
    check_accumulate(orc, gpu_lib, 7 if DRY else 23, True)


def test_batch_at_2p16(orc, gpu_lib):
    log_n = 6 if DRY else 16
    n = 1 << log_n
    c = Context(gpu_lib, 0, 0, 1)
    universal_setup(c, torch, n + 2, n, 8 * n, tau=TAU, device=DEV)
    ok = open_key(c, TAU)
    pr, vk, (_, _, witness, _) = tc.prover_from_circuit(orc, c, log_n, 0xB16, DEV)
    vk = pr.verifying_key()
    wit = tc.witness_host(witness, DEV)
    bl = orc.gen_fr(0xB17, N_BLIND)
    proof, _ = pr.prove_circuit(wit, blind=bl)
    one, _ = pr.prove_batch([wit], blind=[bl])
    assert one.instance(0) == proof
    bp, pubs = pr.prove_batch([wit] * 4)
    assert verify_batch_proof(c, vk, ok, pubs, bp)
    assert verify_batch_proof(c, vk, ok, pubs, batch_proof_from_bytes(c, bp.to_bytes()))
    assert pbv.verify_batch(orc, vk, pubs, bp, TAU)
    assert not verify_batch_proof(c, vk, ok, [[(pubs[2][0] + 1) % pv.R] + pubs[2][1:] if i == 2 else p for i, p in enumerate(pubs)], bp)
    c.close()


def test_batch_at_2p22(orc, gpu_lib):
    log_n = 7 if DRY else 22
    n = 1 << log_n
    if not DRY:
        torch.cuda.empty_cache()
    c = Context(gpu_lib, 0, 0, 1)
    tau = universal_setup(c, torch, n + 2, n, 8 * n, device=DEV)
    ok = open_key(c, tau)
    pr, vk, (_, _, witness, _) = tc.prover_from_circuit(orc, c, log_n, 0xB22, DEV)
    k = min(4, pr.max_batch())
    if k < 2:
        c.close()
        pytest.skip(f"a batch at 2^{log_n} needs {pr.instance_bytes() / 2**30:.1f} GiB per instance: max_batch() = {k}")
    bp, pubs = pr.prove_batch([tc.witness_host(witness, DEV)] * k)
    assert len(bp) == k and verify_batch_proof(c, pr.verifying_key(), ok, pubs, bp)
    c.close()
