"""KZG setup on the GPU: jf-plonk's PlonkKzgSnark::universal_setup (dispatcher2.rs:1279), G1 half."""
from __future__ import annotations

import secrets

from .transcript import R_MOD


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
