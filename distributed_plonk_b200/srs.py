"""KZG setup on the GPU: jf-plonk's PlonkKzgSnark::universal_setup (dispatcher2.rs:1279) - the G1 powers of tau, and
the open key (g, h, beta h) a verifier needs - and a powers-of-tau update ceremony, in which no party ever holds tau."""
from __future__ import annotations

import os
import secrets
import struct
from dataclasses import dataclass

import numpy as np

from ._binding import DP_E_ARG, DpError
from .proof import (_DECOMPRESS_WHY, _Reader, decompress_points, g1_compress, g2_compress, g2_from_raw, g2_to_raw,
                    point_from_raw)
from .transcript import R_MOD

SAVE_CHUNK = 1 << 20            # points per dp_get_bases_compressed call of save_srs (48 MiB of host memory)

# the standard G1 generator (ark-bls12-381 G1Affine::prime_subgroup_generator), affine canonical
G1_GEN = (0x17F1D3A73197D7942695638C4FA9AC0FC3688C4F9774B905A14E3A3F171BAC586C55E83FF97A1AEFFB3AF00ADB22C6BB,
          0x08B3F481E3AAA0F1A09E30ED741D8AE4FCF5E095D5D00AF600DB18CB2C04B3EDD03CC744A2888AE40CAA232946C5E7E1)
# the standard G2 generator (ark-bls12-381 G2Affine::prime_subgroup_generator): ((x.c0, x.c1), (y.c0, y.c1)), canonical
G2_GEN = ((0x024AA2B2F08F0A91260805272DC51051C6E47AD4FA403B02B4510B647AE3D1770BAC0326A805BBEFD48056C8C121BDB8,
           0x13E02B6052719F607DACD3A088274F65596BD0D09920B61AB5DA61BBDC7F5049334CF11213945D57E5AC7D055D042B7E),
          (0x0CE5D527727D6E118CC9CDC6DA2E351AADFD9BAA8CBDD3A76D429A695160D12C923AC9CC3BACA289E193548608B82801,
           0x0606C4A02EA734CC32ACD2B02BC28B99CB3E287E85A763AF267492AB572E99AB3F370D275CEC1DA1AAA9075FF05F79BE))


@dataclass(frozen=True)
class OpenKey:
    """jf-plonk's KZG OpenKey: g the G1 generator, h the G2 generator, beta_h = tau h.  g is affine (x, y), h and
    beta_h are ((x.c0, x.c1), (y.c0, y.c1)), canonical ints.  It holds no secret: a verifier needs nothing else."""
    g: tuple
    h: tuple
    beta_h: tuple

    def to_bytes(self) -> bytes:
        """g (48 B), h (96 B), beta_h (96 B) as ark-serialize 0.3 compressed points: 240 bytes"""
        return g1_compress(self.g) + g2_compress(self.h) + g2_compress(self.beta_h)


def universal_setup(ctx, torch, max_degree: int, domain_size: int, quot_domain_size: int, tau: int | None = None,
                    device: str = "cuda") -> int:
    """Generate the powers-of-tau SRS [tau^i] G1, i <= max_degree, on the context's GPU and dp_init the context with it.

    This is a single-party TEST setup, as jf-plonk's universal_setup is: whoever holds tau can forge proofs for every
    circuit proved over this SRS.  tau: a canonical integer in 1..r-1, or None to draw one with `secrets`.  The points
    go device to device into dp_init; the generated buffer is freed and torch's cache returned before this returns, so
    the memory is free for the prover.  A prover of n gates whose proofs are blinded needs max_degree = n + 2
    (ResidentProver._check_srs: n + 3 bases).  Returns tau."""
    if tau is None:
        tau = 1 + secrets.randbelow(R_MOD - 1)
    n = max_degree + 1
    buf = torch.empty((n, 104), dtype=torch.uint8, device=device)
    try:
        ctx.srs_powers_of_tau_into(tau, n, buf.data_ptr())
        ctx.init_ptr(buf.data_ptr(), n, domain_size, quot_domain_size)
    finally:
        del buf
        if device != "cpu":
            torch.cuda.empty_cache()
    return int(tau)


def open_key(ctx, tau: int) -> OpenKey:
    """The G2 half of the setup of `tau` (the tau given to, or returned by, universal_setup), computed on the GPU
    (dp_srs_open_key); needs no init.  Publish it with the SRS and forget tau."""
    h, beta_h = ctx.srs_open_key(tau)
    return OpenKey(G1_GEN, g2_from_raw(h), g2_from_raw(beta_h))


def _g2_pair_from_bytes(ctx, b: bytes, what: str) -> tuple:
    """h, beta_h from 2 x 96 compressed bytes, decoded and subgroup-checked on the GPU (dp_g2_decompress)"""
    try:
        raw = ctx.g2_decompress(np.frombuffer(b, dtype=np.uint8).reshape(2, 96), check_subgroup=True)
    except DpError as e:
        if e.code != DP_E_ARG:
            raise
        raise ValueError(f"{('h', 'beta_h')[e.index]} of {what}: {_DECOMPRESS_WHY.get(e.why, e.msg)}") from e
    return g2_from_raw(raw[0]), g2_from_raw(raw[1])


def open_key_from_bytes(ctx, b) -> OpenKey:
    """The inverse of OpenKey.to_bytes; the three points are decoded and subgroup-checked on the GPU (ctx needs no init).
    ValueError on a length other than 240 or a rejected point."""
    r = _Reader(b, "open key")
    g, g2 = r.take(48), r.take(192)
    r.end()
    h, beta_h = _g2_pair_from_bytes(ctx, g2, "the open key")
    return OpenKey(decompress_points(ctx, [g], "the open key")[0], h, beta_h)


def _n_bases(ctx) -> int:
    """how many bases the initialised context holds: the largest start an empty range may have (an empty
    dp_get_bases_compressed returns before it touches the device)"""
    lo, hi = 0, 1 << 32
    while lo < hi:
        mid = (lo + hi + 1) // 2
        try:
            ctx.get_bases_compressed(mid, 0)
            lo = mid
        except DpError as e:
            if e.code != DP_E_ARG:
                raise
            hi = mid - 1
    return lo


def save_srs(ctx, path, open_key: OpenKey) -> int:
    """Write the context's SRS and the G2 half of `open_key` as jf-plonk's UniversalSrs under ark-serialize 0.3
    CanonicalSerialize: the number of G1 points (u64 LE), the points compressed (48 B each), then h and beta_h (96 B each).
    The points are encoded on the GPU from the resident bases (dp_get_bases_compressed), SAVE_CHUNK at a time.  Returns
    the number of points.  The file holds no secret."""
    n = _n_bases(ctx)
    if n == 0:
        raise ValueError("the context holds no bases to save")
    g2 = ctx.g2_compress(np.frombuffer(g2_to_raw(open_key.h) + g2_to_raw(open_key.beta_h), dtype=np.uint8).reshape(2, 200))
    buf = np.empty((min(n, SAVE_CHUNK), 48), dtype=np.uint8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", n))
        for first in range(0, n, SAVE_CHUNK):
            m = min(SAVE_CHUNK, n - first)
            f.write(ctx.get_bases_compressed(first, m, buf[:m]).data)
        f.write(g2.tobytes())
    return n


def load_srs(ctx, path, domain_size: int, quot_domain_size: int, check_subgroup: bool = True, check: bool = True) -> OpenKey:
    """dp_init the context from a file save_srs wrote (or jf-plonk's UniversalSrs::serialize) and return its open key.

    Every point is decompressed on the GPU; with check_subgroup (the default) every G1 point is also tested to lie in the
    r-torsion subgroup, as the two G2 points always are.  With check (the default) dp_srs_check then tests that the G1
    points are consecutive powers of the tau of (h, beta_h), starting at the generator - whoever wrote the file cannot
    predict the test's random scalars.  The two checks cover different faults: keep both for a file from somebody else.
    ValueError names what failed: a truncated or over-long file, a count of 0 or above 2^32, the first rejected point
    and why, or the failed consistency check.  A file that fails its format or point checks leaves the context
    uninitialised; one that fails the consistency check leaves it initialised with no bases (the refused points are
    dropped from the device)."""
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        head = f.read(8)
    if len(head) < 8:
        raise ValueError(f"truncated SRS file: {size} bytes")
    n = struct.unpack("<Q", head)[0]
    if n == 0 or n > 1 << 32:
        raise ValueError(f"SRS file: a count of {n} points (1 .. 2^32 are accepted)")
    want = 8 + 48 * n + 192
    if size != want:
        raise ValueError(f"{'truncated' if size < want else 'over-long'} SRS file: {size} bytes, {n} points need {want}")
    g2 = np.fromfile(path, dtype=np.uint8, count=192, offset=8 + 48 * n)
    h, beta_h = _g2_pair_from_bytes(ctx, g2.tobytes(), "the SRS file")
    points = np.memmap(path, dtype=np.uint8, mode="r", offset=8, shape=(n, 48))
    try:
        ctx.init_compressed(points, domain_size, quot_domain_size, check_subgroup)
    except DpError as e:
        if e.code != DP_E_ARG or "rejected" not in e.msg:
            raise
        raise ValueError(f"SRS file: {e.msg.split(': ', 1)[1]}") from e
    finally:
        del points
    key = OpenKey(G1_GEN, h, beta_h)
    if check and not ctx.srs_check(np.frombuffer(g2_to_raw(h) + g2_to_raw(beta_h), dtype=np.uint8).reshape(2, 200)):
        ctx.init(np.zeros((0, 104), dtype=np.uint8), domain_size, quot_domain_size)
        raise ValueError("SRS file: the G1 points are not the consecutive powers g, tau g, tau^2 g, ... of the tau of (h, beta_h)")
    return key


# ------------------------------------------------------------------ the update ceremony (DESIGN.md section 3.10)
def ceremony_start(path, n_points: int) -> None:
    """Write the SRS of tau = 1 that a ceremony starts from, in the UniversalSrs layout of save_srs: n_points copies of
    the G1 generator g, then h and beta h = h.  It is public: nobody has to be trusted for it.  Host only, no context."""
    if not 2 <= n_points <= 1 << 32:
        raise ValueError(f"a ceremony SRS of {n_points} points (2 .. 2^32 are accepted: a receipt needs P_1)")
    g, h = g1_compress(G1_GEN), g2_compress(G2_GEN)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", n_points))
        for first in range(0, n_points, SAVE_CHUNK):
            f.write(g * min(SAVE_CHUNK, n_points - first))
        f.write(h + h)


@dataclass(frozen=True)
class Contribution:
    """The public receipt of one contribution with secret s: old = P_1 = tau g of the SRS it started from, new = Q_1 =
    tau s g of the SRS it wrote, pubkey = s h.  G1 points are affine (x, y), pubkey is ((x.c0, x.c1), (y.c0, y.c1)),
    canonical ints.  load_ceremony_srs checks e(new, h) = e(old, pubkey) for each receipt and that they chain."""
    old: tuple
    new: tuple
    pubkey: tuple

    def to_bytes(self) -> bytes:
        """old (48 B), new (48 B), pubkey (96 B) as ark-serialize 0.3 compressed points: 192 bytes.  This is the library's
        own record; no compatibility with the receipts of other ceremonies is claimed."""
        return g1_compress(self.old) + g1_compress(self.new) + g2_compress(self.pubkey)


def contribution_from_bytes(ctx, b) -> Contribution:
    """The inverse of Contribution.to_bytes; the three points are decoded and subgroup-checked on the GPU (ctx needs no
    init).  ValueError on a length other than 192, a rejected point or an identity pubkey."""
    r = _Reader(b, "contribution")
    g1, pk = r.take(96), r.take(96)
    r.end()
    old, new = decompress_points(ctx, [g1[:48], g1[48:]], "the contribution")
    try:
        raw = ctx.g2_decompress(np.frombuffer(pk, dtype=np.uint8).reshape(1, 96), check_subgroup=True)
    except DpError as e:
        if e.code != DP_E_ARG:
            raise
        raise ValueError(f"pubkey of the contribution: {_DECOMPRESS_WHY.get(e.why, e.msg)}") from e
    pubkey = g2_from_raw(raw[0])
    if pubkey is None:
        raise ValueError("pubkey of the contribution: the identity")
    return Contribution(old, new, pubkey)


def contribute(ctx, in_path, out_path, domain_size: int, quot_domain_size: int, secret: int | None = None) -> Contribution:
    """Add secret randomness to the SRS file in_path and write the result to out_path: Q_i = s^i P_i, the same h and
    s beta h, so the new file is the SRS of tau s.  Returns the receipt to publish with it.

    in_path is first loaded with every check of load_srs (a contributor must not build on a bad file), which leaves ctx
    initialised with it.  The points are computed on the GPU (dp_srs_update) and written straight into a memory map of
    out_path.  With secret None (the only use outside tests) the library draws s inside the call and zeroes every copy
    before it returns, so s never reaches Python; `secret` (a canonical 0 < s < r) exists for reproducible tests.
    ValueError for an SRS of fewer than 2 points: the receipt needs P_1."""
    key = load_srs(ctx, in_path, domain_size, quot_domain_size)
    with open(in_path, "rb") as f:
        n = struct.unpack("<Q", f.read(8))[0]
    if n < 2:
        raise ValueError(f"contribute needs an SRS of at least 2 points, the file holds {n}")
    old = point_from_raw(ctx.get_bases(1, 1)[0])
    with open(out_path, "wb") as f:
        f.write(struct.pack("<Q", n))
        f.truncate(8 + 48 * n + 192)
    points = np.memmap(out_path, dtype=np.uint8, mode="r+", offset=8, shape=(n, 48))
    try:
        _, g2 = ctx.srs_update(np.frombuffer(g2_to_raw(key.h) + g2_to_raw(key.beta_h), dtype=np.uint8).reshape(2, 200), n,
                               secret, out48=points)
        new_bytes = points[1].tobytes()
        points.flush()
    finally:
        del points
    with open(out_path, "r+b") as f:
        f.seek(8 + 48 * n)
        f.write(g2_compress(key.h) + ctx.g2_compress(g2[1:]).tobytes())
    new = decompress_points(ctx, [new_bytes], "the new SRS")[0]
    return Contribution(old, new, g2_from_raw(g2[0]))


def _receipt_holds(ctx, h, items, weights) -> bool:
    """e(sum w_j new_j, h) * prod_j e(-w_j old_j, pubkey_j) == 1, one multi-pairing of len(items) + 1 pairs"""
    from .verifier import _FQ12_ONE, _jacobian_to_raw, _raw_points, _scalars
    g1 = [_jacobian_to_raw(ctx.msm_points(_raw_points([c.new for c in items]), _scalars(weights)))]
    g1 += [_jacobian_to_raw(ctx.msm_points(_raw_points([c.old]), _scalars([-w]))) for c, w in zip(items, weights)]
    g2 = [g2_to_raw(h)] + [g2_to_raw(c.pubkey) for c in items]
    return ctx.multi_pairing(np.frombuffer(b"".join(g1), dtype=np.uint8).reshape(-1, 104),
                             np.frombuffer(b"".join(g2), dtype=np.uint8).reshape(-1, 200)).tobytes() == _FQ12_ONE


def load_ceremony_srs(ctx, path, contributions, domain_size: int, quot_domain_size: int) -> OpenKey:
    """load_srs(path) with all its checks, then check that the file is the end of this chain of contributions from the
    tau = 1 start of ceremony_start: h is the standard generator; every receipt's points pass the checks of
    contribution_from_bytes; receipt 0's old is g, receipt j's old is receipt j - 1's new, and the last new is P_1 of the
    file; and e(new_j, h) = e(old_j, pubkey_j) for every j (so tau_j = tau_(j-1) s_j), tested for all j with one
    multi-pairing under random weights from `secrets`, then receipt by receipt when that fails, to name the first bad one.
    The final tau is the product of the secrets: the SRS is sound if one contributor deleted theirs.  Returns the open
    key.  ValueError names what failed; every refusal after load_srs leaves the context initialised with no bases, as
    load_srs's failed consistency check does."""
    key = load_srs(ctx, path, domain_size, quot_domain_size)
    try:
        if not contributions:
            raise ValueError("ceremony: the chain of contributions is empty")
        if key.h != G2_GEN:
            raise ValueError("ceremony: h of the SRS file is not the standard G2 generator the ceremony starts from")
        if _n_bases(ctx) < 2:
            raise ValueError("ceremony: the SRS file has fewer than 2 points")
        chain = []
        for j, c in enumerate(contributions):
            try:
                chain.append(contribution_from_bytes(ctx, c.to_bytes()))
            except ValueError as e:
                raise ValueError(f"ceremony: contribution {j}: {e}") from e
        for j, c in enumerate(chain):
            if c.old != (G1_GEN if j == 0 else chain[j - 1].new):
                raise ValueError(f"ceremony: contribution {j} does not start from "
                                 f"{'the generator g (tau = 1)' if j == 0 else f'the new point of contribution {j - 1}'}")
        if chain[-1].new != point_from_raw(ctx.get_bases(1, 1)[0]):
            raise ValueError(f"ceremony: the new point of the last contribution ({len(chain) - 1}) is not P_1 of the SRS file")
        if not _receipt_holds(ctx, key.h, chain, [1 + secrets.randbelow(R_MOD - 1) for _ in chain]):
            bad = next((j for j, c in enumerate(chain) if not _receipt_holds(ctx, key.h, [c], [1])), None)
            raise ValueError(f"ceremony: contribution {bad if bad is not None else '?'} fails e(new, h) = e(old, pubkey)")
    except ValueError:
        ctx.init(np.zeros((0, 104), dtype=np.uint8), domain_size, quot_domain_size)
        raise
    return key
