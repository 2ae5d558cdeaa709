"""KZG setup on the GPU: jf-plonk's PlonkKzgSnark::universal_setup (dispatcher2.rs:1279) - the G1 powers of tau, and
the open key (g, h, beta h) a verifier needs."""
from __future__ import annotations

import secrets
from dataclasses import dataclass

from .proof import g2_from_raw
from .transcript import R_MOD

# the standard G1 generator (ark-bls12-381 G1Affine::prime_subgroup_generator), affine canonical
G1_GEN = (0x17F1D3A73197D7942695638C4FA9AC0FC3688C4F9774B905A14E3A3F171BAC586C55E83FF97A1AEFFB3AF00ADB22C6BB,
          0x08B3F481E3AAA0F1A09E30ED741D8AE4FCF5E095D5D00AF600DB18CB2C04B3EDD03CC744A2888AE40CAA232946C5E7E1)


@dataclass(frozen=True)
class OpenKey:
    """jf-plonk's KZG OpenKey: g the G1 generator, h the G2 generator, beta_h = tau h.  g is affine (x, y), h and
    beta_h are ((x.c0, x.c1), (y.c0, y.c1)), canonical ints.  It holds no secret: a verifier needs nothing else."""
    g: tuple
    h: tuple
    beta_h: tuple


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
