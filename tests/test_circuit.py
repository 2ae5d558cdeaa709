"""Circuit preprocessing and the witness gather on the kernel-logic emulator: the wire permutation (dp_wire_permutation_dev)
against two restatements of jf-relation's compute_wire_permutation for many variable maps, the identity / sigma
evaluations, the gather of the wire and public-input evaluations, every error code, ResidentProver.load_circuit against
the oracle's iNTT and commitments, prove_witness against prove, and the quotient degree of a satisfied circuit built from
variables - also under adversarial asynchronous stream schedules."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from distributed_plonk_b200._binding import Context, DpError
from distributed_plonk_b200.resident import N_BLIND, N_SEL, N_WIRE, NumpyField, ResidentProver
from tests import common

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def code(f):
    with pytest.raises(DpError) as e:
        f()
    return e.value.code


# ------------------------------------------------------------------ oracle restatements
def succ_literal(wire_vars, nw, n):
    """compute_wire_permutation as jf-relation writes it: variable -> its (wire, gate) slots, wire-major, then each slot's
    successor is the next one of its variable (windows(2) over the list with its first element re-appended)"""
    variable_wires_map = {}
    for wire in range(nw):
        for gate in range(n):
            variable_wires_map.setdefault(int(wire_vars[wire * n + gate]), []).append((wire, gate))
    succ = np.empty(nw * n, dtype=np.uint32)
    for slots in variable_wires_map.values():
        cycle = slots + [slots[0]]
        for (w0, g0), (w1, g1) in zip(cycle, cycle[1:]):
            succ[w0 * n + g0] = w1 * n + g1
    return succ


def succ_argsort(wire_vars):
    """the same by a stable argsort (large sizes): slots sorted by variable, each to the next of its group, the last of
    a group to the group's first"""
    v = np.asarray(wire_vars, dtype=np.uint32)
    order = np.argsort(v, kind="stable").astype(np.uint32)
    keys = v[order]
    cnt = v.shape[0]
    head = np.ones(cnt, dtype=bool)
    head[1:] = keys[1:] != keys[:-1]
    first = np.maximum.accumulate(np.where(head, np.arange(cnt), 0))
    same_next = np.zeros(cnt, dtype=bool)
    same_next[:-1] = ~head[1:]
    succ = np.empty(cnt, dtype=np.uint32)
    succ[order] = np.where(same_next, np.roll(order, -1), order[first])
    return succ


def variable_maps(nw, n, seed):
    """name -> (wire_vars [nw*n] u32, num_vars): the distributions the sort must get right"""
    rng = np.random.default_rng(seed)
    cnt = nw * n
    maps = {
        "uniform": (rng.integers(0, 3 * n, cnt, dtype=np.uint32), 3 * n),
        "one variable of many": (np.full(cnt, 5, dtype=np.uint32), 9),
        "num_vars = 1": (np.zeros(cnt, dtype=np.uint32), 1),
        "sparse near 2^32": (np.uint32(0xFFFFFFFF) - rng.integers(0, 1000, cnt, dtype=np.uint32), 1 << 32),
        "few variables": (rng.integers(0, 7, cnt, dtype=np.uint32), 7),
    }
    padded = rng.integers(1, n, cnt, dtype=np.uint32)
    padded[rng.random(cnt) < 0.85] = 0                       # padding: most slots on one variable
    maps["padded"] = (padded, n)
    sp = maps["sparse near 2^32"][0]
    sp[::17] = rng.integers(0, 300, sp[::17].shape[0], dtype=np.uint32)   # every byte of the key differs somewhere
    return maps


def device_succ(ctx, wire_vars, nw, n, num_vars, as_dev, to_host):
    """dp_wire_permutation_dev on device copies (as_dev: numpy -> buffer with .ptr; to_host: buffer -> numpy)"""
    v = as_dev(np.ascontiguousarray(wire_vars, dtype=np.uint32))
    nbytes = ctx.wire_permutation_scratch_bytes(nw, n, num_vars)
    scratch = as_dev(np.zeros(nbytes, dtype=np.uint8))
    succ = as_dev(np.zeros(nw * n, dtype=np.uint32))
    ctx.wire_permutation_dev(v.ptr, nw, n, num_vars, scratch.ptr, nbytes, succ.ptr)
    return to_host(succ).view(np.uint32)


class HostBuf:
    """emulator 'device' memory is host memory"""
    def __init__(self, a):
        self.a = a
        self.ptr = a.ctypes.data


def host_dev(a):
    return HostBuf(np.ascontiguousarray(a).copy())


def host_read(b):
    return b.a


def check_cycles(succ, wire_vars):
    """following succ from a slot visits exactly its variable's slots, in increasing order, and returns"""
    v = np.asarray(wire_vars)
    for var in np.unique(v)[:50]:
        slots = np.nonzero(v == var)[0]
        s, seen = int(slots[0]), []
        for _ in range(slots.shape[0]):
            seen.append(s)
            s = int(succ[s])
        assert s == slots[0] and seen == sorted(seen) and np.array_equal(np.array(seen), slots), f"cycle of variable {var}"


@pytest.mark.parametrize("log_n", [6, 10])
def test_wire_permutation_matches_both_restatements(emul_lib, log_n):
    n = 1 << log_n
    c = Context(emul_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, 8 * n)
    for name, (wv, num_vars) in variable_maps(N_WIRE, n, 900 + log_n).items():
        want = succ_argsort(wv)
        assert np.array_equal(succ_literal(wv, N_WIRE, n), want), f"the two restatements disagree on {name}"
        got = device_succ(c, wv, N_WIRE, n, num_vars, host_dev, host_read)
        assert np.array_equal(got, want), f"wire permutation, {name}, n = {n}"
        check_cycles(got, wv)
    c.close()


@pytest.mark.parametrize("nw", [1, 2, 3, 4, 5])
def test_wire_permutation_every_wire_count(emul_lib, nw):
    n = 1 << 8
    c = Context(emul_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, 8 * n)
    rng = np.random.default_rng(nw)
    wv = rng.integers(0, 300, nw * n, dtype=np.uint32)
    got = device_succ(c, wv, nw, n, 300, host_dev, host_read)
    assert np.array_equal(got, succ_literal(wv, nw, n))
    c.close()


# ------------------------------------------------------------------ identity / sigma evaluations and the gather
def perm_evals_oracle(succ, nw, n, k):
    F = NumpyField(n.bit_length() - 1)
    w = [F.pow_u64(F.omega, j) for j in range(n)]
    ident = np.stack([F.mul(k[i], w[j]) for i in range(nw) for j in range(n)])
    sigma = ident[np.asarray(succ, dtype=np.int64)] if succ is not None else ident
    return ident, sigma


def test_perm_evals_match_the_oracle(orc, emul_lib):
    log_n = 6
    n = 1 << log_n
    c = Context(emul_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, 8 * n)
    k = orc.gen_fr(9100, N_WIRE)
    wv, num_vars = variable_maps(N_WIRE, n, 9101)["uniform"]
    succ = succ_argsort(wv)
    want_id, want_sig = perm_evals_oracle(succ, N_WIRE, n, k)
    idv, sig = np.zeros((N_WIRE * n, 4), dtype=np.uint64), np.zeros((N_WIRE * n, 4), dtype=np.uint64)
    c.perm_evals_dev(succ.ctypes.data, N_WIRE, n, k, idv.ctypes.data, sig.ctypes.data)
    assert np.array_equal(idv, want_id) and np.array_equal(sig, want_sig)
    c.perm_evals_dev(None, N_WIRE, n, k, idv.ctypes.data, sig.ctypes.data)
    assert np.array_equal(sig, want_id) and np.array_equal(idv, want_id), "without succ, sigma = id"
    c.perm_evals_dev(None, 2, n, k[:2], idv.ctypes.data, sig.ctypes.data)
    assert np.array_equal(idv[:2 * n], want_id[:2 * n])
    c.close()


def gather_oracle(witness, wire_vars, nw, n, num_inputs):
    wires = witness[np.asarray(wire_vars, dtype=np.int64)]
    pub = np.zeros((n, 4), dtype=np.uint64)
    pub[:num_inputs] = wires[(nw - 1) * n:(nw - 1) * n + num_inputs]
    return wires, pub


@pytest.mark.parametrize("nw,num_inputs", [(5, 0), (5, 7), (3, 64), (1, 1)])
def test_witness_gather_matches_fancy_indexing(orc, emul_lib, nw, num_inputs):
    n = 64
    c = Context(emul_lib, 0, 0, 1)
    c.init(np.zeros(0, dtype=np.uint8), n, 8 * n)
    num_vars = 150
    witness = orc.gen_fr(9200 + nw, num_vars)
    wv = np.random.default_rng(nw).integers(0, num_vars, nw * n, dtype=np.uint32)
    wires, pub = np.zeros((nw * n, 4), dtype=np.uint64), np.ones((n, 4), dtype=np.uint64)
    c.witness_gather_dev(witness.ctypes.data, num_vars, wv.ctypes.data, nw, n, num_inputs, wires.ctypes.data, pub.ctypes.data)
    want_w, want_p = gather_oracle(witness, wv, nw, n, num_inputs)
    assert np.array_equal(wires, want_w) and np.array_equal(pub, want_p)
    c.close()


def test_circuit_errors(orc, emul_lib):
    n = 64
    cnt = N_WIRE * n
    c = Context(emul_lib, 0, 0, 1)
    wv = np.arange(cnt, dtype=np.uint32) % 100
    nbytes = c.wire_permutation_scratch_bytes(N_WIRE, n, 100)
    scratch = np.zeros(nbytes, dtype=np.uint8)
    succ = np.zeros(cnt, dtype=np.uint32)
    k = orc.gen_fr(9300, N_WIRE)
    idv, sig = np.zeros((cnt, 4), dtype=np.uint64), np.zeros((cnt, 4), dtype=np.uint64)
    witness = orc.gen_fr(9301, 100)
    wires, pub = np.zeros((cnt, 4), dtype=np.uint64), np.zeros((n, 4), dtype=np.uint64)

    def perm(v=wv, nw=N_WIRE, nn=n, nv=100, s=scratch.ctypes.data, sb=nbytes, out=succ.ctypes.data, vp=None):
        c.wire_permutation_dev(v.ctypes.data if vp is None else vp, nw, nn, nv, s, sb, out)

    def evals(sp=succ.ctypes.data, nw=N_WIRE, nn=n, i=idv.ctypes.data, s=sig.ctypes.data):
        c.perm_evals_dev(sp, nw, nn, k[:max(1, min(nw, 5))], i, s)

    def gather(v=wv, nv=100, nw=N_WIRE, nn=n, ni=3, w=wires.ctypes.data, p=pub.ctypes.data, wit=witness.ctypes.data):
        c.witness_gather_dev(wit, nv, v.ctypes.data, nw, nn, ni, w, p)

    for f in (perm, evals, gather):
        assert code(f) == -2                                                          # before dp_init
    c.init(np.zeros(0, dtype=np.uint8), n, 8 * n)
    perm(), evals(), gather()
    for f in (perm, evals, gather):
        assert code(lambda: f(nn=2 * n)) == -1                                         # n is not the gate domain
        assert code(lambda: f(nw=0)) == -1 and code(lambda: f(nw=6)) == -1             # wire types outside 1..5
    bad = wv.copy()
    bad[cnt - 1] = 100
    assert code(lambda: perm(v=bad)) == -1                                            # an id >= num_vars
    assert code(lambda: gather(v=bad)) == -1
    assert code(lambda: perm(nv=0)) == -1 and code(lambda: gather(nv=0)) == -1        # num_vars == 0
    assert code(lambda: gather(ni=n + 1)) == -1                                       # num_inputs > n
    assert code(lambda: perm(sb=nbytes - 1)) == -1                                    # scratch too small
    assert code(lambda: perm(s=None)) == -1 and code(lambda: perm(out=None)) == -1    # NULL buffers
    assert code(lambda: perm(vp=0)) == -1
    assert code(lambda: evals(i=None)) == -1 and code(lambda: gather(w=None)) == -1 and code(lambda: gather(wit=None)) == -1
    assert code(lambda: perm(out=scratch.ctypes.data + 64)) == -1                     # overlapping buffers
    assert code(lambda: evals(s=idv.ctypes.data + 32)) == -1
    assert code(lambda: gather(p=wires.ctypes.data + 32 * n)) == -1
    assert code(lambda: gather(w=witness.ctypes.data)) == -1
    oob = succ.copy()
    oob[7] = cnt                                                                      # a successor slot out of range
    assert code(lambda: evals(sp=oob.ctypes.data)) == -1
    with pytest.raises(DpError):
        c.wire_permutation_scratch_bytes(0, n, 10)
    assert c.commit_dev_batch([], []) == []
    c.close()


# ------------------------------------------------------------------ the prover from a circuit
def satisfied_circuit(orc, log_n, seed, num_inputs=3):
    """a TurboPlonk circuit built from variables whose gates and copy constraints hold.  Variable 0 is zero and fills
    the a..d wires of the IO gates and every wire of the padding gates (the last quarter, all selectors zero): one huge
    variable class.  IO gates come first (q_o = 1, output = the public input).  The other gates draw a..d from a small
    pool of free variables and the IO outputs - long cycles across all five wire types - and their output e is a fresh
    variable that satisfies the gate.  Returns (selector evals [13][n], wire_vars [5n], witness [num_vars], k)"""
    n = 1 << log_n
    rng = np.random.default_rng(seed)
    V = orc.vec_op
    one = common._fr_one(orc)
    pool = 12
    io_vars = 1 + np.arange(num_inputs)
    free_vars = 1 + num_inputs + np.arange(pool)
    gen = np.arange(num_inputs, n - n // 4)                # general gates
    num_vars = 1 + num_inputs + pool + gen.shape[0]
    witness = np.zeros((num_vars, 4), dtype=np.uint64)
    witness[1:1 + num_inputs + pool] = orc.gen_fr(seed, num_inputs + pool)
    wv = np.zeros((N_WIRE, n), dtype=np.uint32)
    wv[4, :num_inputs] = io_vars
    wv[:4, gen] = rng.choice(np.concatenate([io_vars, free_vars]), size=(4, gen.shape[0]))
    e_vars = 1 + num_inputs + pool + np.arange(gen.shape[0])
    wv[4, gen] = e_vars
    sel = [np.zeros((n, 4), dtype=np.uint64) for _ in range(N_SEL)]
    sel[10][:num_inputs] = one                                 # q_o of the IO gates
    for i in range(N_SEL):
        sel[i][gen] = orc.gen_fr(seed + 1 + i, gen.shape[0])
    a, b, cc, d = (witness[wv[i, gen].astype(np.int64)] for i in range(4))
    g = [s[gen] for s in sel]
    ab, cd = V("mul", a, b), V("mul", cc, d)
    p5 = lambda v: V("mul", V("mul", V("mul", v, v), V("mul", v, v)), v)
    rest = g[11]
    for q, v in ((g[0], a), (g[1], b), (g[2], cc), (g[3], d), (g[4], ab), (g[5], cd), (g[6], p5(a)), (g[7], p5(b)), (g[8], p5(cc)), (g[9], p5(d))):
        rest = V("add", rest, V("mul", q, v))
    witness[e_vars] = V("mul", rest, V("inv", V("sub", g[10], V("mul", g[12], V("mul", ab, cd)))))
    F = NumpyField(log_n)
    k = np.stack([F.from_u64(v) for v in (1, 7, 13, 17, 23)])
    return sel, wv.reshape(-1), witness, k


def prover_from_circuit(orc, ctx, log_n, seed, device, quotient="auto"):
    sel, wv, witness, k = satisfied_circuit(orc, log_n, seed)
    pr = ResidentProver(ctx, torch, log_n, device, NumpyField(log_n), quotient=quotient)
    vk, _ = pr.load_circuit(sel, wv, witness.shape[0], k, 3)
    return pr, vk, (sel, wv, witness, k)


def check_load_circuit(orc, ctx, bases, log_n, seed, device):
    """coefficient forms = the oracle's iNTT of the selector and sigma evaluations; the 18 commitments = orc.commit; the
    identity / sigma evaluations = the oracle restatement of the circuit's permutation"""
    n = 1 << log_n
    pr, vk, (sel, wv, witness, k) = prover_from_circuit(orc, ctx, log_n, seed, device)
    host = lambda t: t.cpu().numpy().view(np.uint64)
    want_id, want_sig = perm_evals_oracle(succ_argsort(wv), N_WIRE, n, k)
    assert np.array_equal(host(pr.id_eval), want_id) and np.array_equal(host(pr.sig_eval), want_sig)
    coefs = [orc.fft(s, True, False) for s in sel] + [orc.fft(want_sig[i * n:(i + 1) * n], True, False) for i in range(N_WIRE)]
    for j, (t, want) in enumerate(zip(pr.sel_coef + pr.sig_coef, coefs)):
        assert np.array_equal(host(t), want), f"coefficient form {j}"
    assert len(vk) == N_SEL + N_WIRE
    for j, (got, want) in enumerate(zip(vk, coefs)):
        common.assert_point_eq(orc, got, orc.commit(bases, want), f"verifying-key commitment {j}")
    return pr, witness


def test_load_circuit_matches_the_oracle(orc, emul_lib):
    log_n = 6
    n = 1 << log_n
    bases = orc.gen_bases(5, n + 3, 64, True)
    c = Context(emul_lib, 0, 0, 1)
    c.init(bases, n, 8 * n)
    check_load_circuit(orc, c, bases, log_n, 9400, "cpu")
    c.close()


def witness_host(witness, device):
    t = torch.as_tensor(witness.view(np.int64))
    return t.pin_memory() if device != "cpu" else t


def check_prove_witness(orc, ctx, log_n, seed, device, quotient):
    """prove_witness == prove(gathered wire evaluations, public input), unblinded and with fixed blinders; the public
    inputs it returns are the IO gates' outputs"""
    n = 1 << log_n
    pr, _, (sel, wv, witness, k) = prover_from_circuit(orc, ctx, log_n, seed, device, quotient)
    wires, pub = gather_oracle(witness, wv, N_WIRE, n, 3)
    F = pr.F
    ch = {name: orc.gen_fr(seed + 60 + j, 1)[0] for j, name in enumerate(("beta", "gamma", "alpha", "zeta", "v"))}
    w_host, p_host = witness_host(wires, device), witness_host(pub, device)
    wit = witness_host(witness, device)
    for blind in (False, orc.gen_fr(seed + 70, N_BLIND)):
        com, ev, pi = pr.prove_witness(wit, ch, blind=blind)
        assert np.array_equal(pi, pub[:3])
        com2, ev2 = pr.prove(w_host, p_host, ch, blind=blind)
        assert len(com) == 13 and len(ev) == 10
        for j, (a, b) in enumerate(zip(com + ev, com2 + ev2)):
            assert np.array_equal(np.asarray(a), np.asarray(b)), f"output {j} ({quotient}, blinded={blind is not False})"
    return pr


@pytest.mark.parametrize("quotient", ["whole", "sliced"])
def test_prove_witness_equals_prove(orc, emul_lib, quotient):
    log_n = 6
    n = 1 << log_n
    c = Context(emul_lib, 0, 0, 1)
    c.init(orc.gen_bases(5, n + 3, 64, True), n, 8 * n)
    check_prove_witness(orc, c, log_n, 9500, "cpu", quotient)
    c.close()


def grand_product_closes(wires, idv, sig, beta, gamma, n):
    """prod over every slot of (w + beta id + gamma) / (w + beta sigma + gamma) == 1 (Python integers)"""
    D, R = NumpyField._dec, NumpyField.R_MOD
    be, ga = D(beta), D(gamma)
    num = den = 1
    for s in range(wires.shape[0]):
        w = D(wires[s])
        num = num * (w + be * D(idv[s]) + ga) % R
        den = den * (w + be * D(sig[s]) + ga) % R
    return num == den


def check_satisfied_circuit_degree(orc, ctx, log_n, seed, device):
    """on the satisfied circuit: the permutation product closes, the quotient divides exactly (degree <= 5(n+1)+2,
    exactly that when blinded); sigma from a map that merges two differently valued variables: degree > 7n"""
    n = 1 << log_n
    pr, _, (sel, wv, witness, k) = prover_from_circuit(orc, ctx, log_n, seed, device)
    ch = {name: orc.gen_fr(seed + 60 + j, 1)[0] for j, name in enumerate(("beta", "gamma", "alpha", "zeta", "v"))}
    wit = witness_host(witness, device)
    host = lambda t: t.cpu().numpy().view(np.uint64)

    def degree():
        q = host(pr.quot)
        nz = np.nonzero(q.any(axis=1))[0]
        return int(nz[-1]) if nz.size else -1

    pr.prove_witness(wit, ch)
    assert grand_product_closes(host(pr.wire_eval), host(pr.id_eval), host(pr.sig_eval), ch["beta"], ch["gamma"], n)
    assert degree() <= 5 * (n + 1) + 2
    pr.prove_witness(wit, ch, blind=orc.gen_fr(seed + 90, N_BLIND))
    assert degree() == 5 * (n + 1) + 2
    # one slot of a free variable relabelled to another, differently valued one: a wrong copy constraint
    merged = wv.copy()
    slot = int(np.nonzero((wv >= 4) & (wv < 16))[0][0])
    other = 4 + (int(wv[slot]) - 4 + 1) % 12
    assert not np.array_equal(witness[wv[slot]], witness[other])
    merged[slot] = other
    pr.load_circuit(sel, merged, witness.shape[0], k, 3)
    wires, pub = gather_oracle(witness, wv, N_WIRE, n, 3)
    pr.prove(witness_host(wires, device), witness_host(pub, device), ch, blind=True)
    assert degree() > 7 * n


def test_quotient_degree_on_a_satisfied_circuit_from_variables(orc, emul_lib):
    log_n = 6
    n = 1 << log_n
    c = Context(emul_lib, 0, 0, 1)
    c.init(orc.gen_bases(5, n + 3, 64, True), n, 8 * n)
    check_satisfied_circuit_degree(orc, c, log_n, 9600, "cpu")
    c.close()


@pytest.mark.timeout(1500)
@pytest.mark.skipif(os.environ.get("DP_TEST_EMUL_ASYNC", "0") == "1", reason="this test starts the asynchronous runs itself")
def test_circuit_under_adversarial_stream_schedules():
    """load_circuit and prove_witness on the asynchronous-stream emulator build, with the compute, copy-in and MSM tail
    streams in turn made pathologically slow (tests/test_emul_async.py)"""
    from tests.emul import build as emul_build
    emul_build.build(async_streams=True)
    select = "load_circuit_matches or (prove_witness_equals_prove and sliced) or (matches_both_restatements and 10)"
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
