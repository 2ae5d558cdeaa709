/*
 * dplonk.h - C ABI of the H100-native worker hot path of MengLing-L/distributed_plonk.
 *
 * The reference worker (Rust) has no FFI today: its RPC method bodies call arkworks directly
 * (SURVEY.md §8b).  Each entry point below is what the body of one `PlonkSlave` / `PlonkPeer`
 * method (src/hello_world.capnp:15-52, implemented in src/worker.rs:125-439) binds instead of the
 * arkworks call it makes today; INTEGRATION.md shows the Rust `extern "C"` block and the patched
 * method bodies.  Wire formats are exactly what the reference puts in its `Data` blobs
 * (src/utils.rs:27-43 = raw in-memory Rust structs):
 *
 *   Fr            32 B  ark-ff Fp256, Montgomery form (R = 2^256), 4 x u64 little-endian
 *   BigInteger256 32 B  canonical scalar (Fr::into_repr), 4 x u64 little-endian
 *   G1Affine     104 B  x (48 B Fq Montgomery) | y (48 B) | infinity flag (1 B) | 7 B padding
 *   G1Projective 144 B  Jacobian X | Y | Z, each 48 B Fq Montgomery; identity has Z = 0
 *
 * Conventions: every function returns DP_OK (0) or a negative DP_E_* code and never throws or
 * aborts across the boundary; dp_last_error() gives the text.  All buffers are caller-owned,
 * borrowed only for the duration of the call, may be unaligned, and are HOST memory unless a
 * parameter says "dev".  One exception, for page-locked (cudaHostAlloc / cudaHostRegister) row
 * buffers handed to dp_fft1 / dp_fft1_rows: their copy-in is truly asynchronous, so they must stay
 * unchanged until dp_fft2 of that task (or dp_sync) returns; ordinary pageable memory - what a
 * Cap'n Proto message gives the reference worker - is staged before the call returns.  A context is bound to one CUDA device and must be used from one thread
 * at a time (the reference worker is single-threaded: worker.rs:441,453).  There is no CPU
 * fallback: dp_create fails with DP_E_CUDA when no sm_90 (H100) device is usable.
 */
#ifndef DPLONK_H
#define DPLONK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DP_OK 0
#define DP_E_ARG (-1)   /* bad argument (size mismatch, non-canonical scalar, unknown id ...) */
#define DP_E_STATE (-2) /* call out of order (fft2 before fft2_prepare, rows missing ...)      */
#define DP_E_OOM (-3)   /* device or host allocation failed                                   */
#define DP_E_CUDA (-4)  /* CUDA runtime / kernel error                                        */
#define DP_E_COMM (-5)  /* exchange needed but no peer transport attached                     */

#define DP_FR_BYTES 32
#define DP_G1_AFFINE_BYTES 104
#define DP_G1_COMPRESSED_BYTES 48 /* ark-serialize 0.3.0 compressed GroupAffine */
#define DP_G1_PROJECTIVE_BYTES 144
#define DP_G2_AFFINE_BYTES 200     /* raw ark 0.3 GroupAffine<g2::Parameters>: x.c0, x.c1, y.c0, y.c1, infinity, padding */
#define DP_G2_COMPRESSED_BYTES 96  /* ark-serialize 0.3 compressed GroupAffine<g2::Parameters>                            */
#define DP_FQ12_BYTES 576         /* 12 Montgomery Fq in the order of the tower Fq2 -> Fq6 -> Fq12 (DESIGN.md 3.8)      */

typedef struct dp_ctx dp_ctx;

/* src/utils.rs:3-19 FftWorkload (src/hello_world.capnp:8-13) */
typedef struct dp_fft_workload {
    uint64_t row_start, row_end, col_start, col_end;
} dp_fft_workload;

/* ---- lifetime -------------------------------------------------------------------------------
 * Replaces the `State` construction in worker main (src/worker.rs:455-472).  `me` is the worker
 * index (argv[1], worker.rs:443-449), `n_workers` the number of workers sharing distributed NTTs. */
int dp_create(int cuda_device, uint64_t me, uint64_t n_workers, dp_ctx **out);
int dp_destroy(dp_ctx *ctx);
const char *dp_last_error(const dp_ctx *ctx); /* valid until the next call on ctx; ctx may be NULL */
const char *dp_version(void);

/* ---- PlonkSlave.init (src/worker.rs:126-157) -------------------------------------------------
 * Stores the SRS bases on the device and builds the (r, c) split domains for `domain_size` and
 * `quot_domain_size` (Radix2EvaluationDomain::new rounds both up to powers of two).
 * bases: n_bases raw G1Affine (104 B each), the concatenation of the `bases` Data chunks; host memory, or
 * device memory of the context's GPU (a resident SRS: the copy is then device-to-device). */
int dp_init(dp_ctx *ctx, const void *bases, size_t n_bases, uint64_t domain_size, uint64_t quot_domain_size);

/* "next" row (SURVEY.md §8f-4): the same, from the canonical encoding SRS files hold - what the
 * reference's dispatcher deserialises on the CPU before shipping raw structs (ark-serialize 0.3.0
 * `GroupAffine::deserialize` / `deserialize_unchecked`; jellyfish `UnivariateUniversalParams`).
 * bases48: n_bases x 48 B = canonical x little-endian, bit 7 of the last byte = (y > -y), bit 6 =
 * infinity.  Decompression (a 381-bit square root per point) and, when check_subgroup != 0, the
 * r-torsion check run on the GPU.  A rejected point (x >= p, both flags, no such point, outside the
 * subgroup) returns DP_E_ARG naming the first bad index and leaves the context uninitialised.     */
int dp_init_compressed(dp_ctx *ctx, const void *bases48, size_t n_bases, uint64_t domain_size, uint64_t quot_domain_size,
                       int check_subgroup);
/* bases [start, start + n) back as raw G1Affine (104 B each; identity = (0, 1, true))             */
int dp_get_bases(dp_ctx *ctx, uint64_t start, size_t n, void *out104);

/* KZG powers of tau for a test setup (jf-plonk PlonkKzgSnark::universal_setup, dispatcher2.rs:1279):
 * out104[i] = tau^i * G1 for i < n, raw G1Affine (104 B, the layout dp_init reads).  tau32: 32 B canonical,
 * 0 < tau < r, else DP_E_ARG.  out104: host memory or device memory of the context's GPU.  Needs no dp_init
 * and leaves an initialised context's state as it was; its first call builds a 48 MiB fixed-base table that
 * the context keeps until the next dp_init.  Returns when the points are written.  n = 0 writes nothing;
 * n > 2^32 is DP_E_ARG.  Whoever knows tau can forge proofs against this SRS.                             */
int dp_srs_powers_of_tau(dp_ctx *ctx, const void *tau32, size_t n, void *out104);

/* ---- verifier (DESIGN.md section 3.8): none of these needs dp_init; all read and write host memory ------------
 * ark-serialize 0.3 compressed points (48 B each, the proof's encoding) -> raw G1Affine (104 B each), on the GPU.
 * check_subgroup != 0 also runs the r-torsion check.  A rejected point returns DP_E_ARG, writes nothing to out104,
 * and sets *bad_index to its index and *why to 1 (x >= p), 2 (both flag bits), 3 (no such point) or 4 (outside the
 * subgroup); on success *bad_index = n and *why = 0 (either pointer may be NULL).                                  */
int dp_g1_decompress(dp_ctx *ctx, const void *in48, size_t n, int check_subgroup, void *out104, size_t *bad_index, int *why);
/* out144 = sum_i scalars32[i] * points104[i] over n caller-given raw G1Affine points (not validated; the identity
 * flag is honoured).  Scalars: canonical BigInteger256 as in dp_msm.  out144: 144 B raw G1Projective, normalised
 * (Z = 1) or the identity.  n = 0 writes the identity.                                                            */
int dp_msm_points(dp_ctx *ctx, const void *points104, const void *scalars32, size_t n, void *out144);
/* The G2 half of jf-plonk's KZG test setup: out400 = H, tau * H (two raw G2Affine, 200 B each), H the standard G2
 * generator.  tau32: 32 B canonical, 0 < tau < r, else DP_E_ARG.                                                  */
int dp_srs_open_key(dp_ctx *ctx, const void *tau32, void *out400);
/* out576 = prod_i e(g1_104[i], g2_200[i]) as an Fq12 (DP_FQ12_BYTES), one final exponentiation for all k pairs.
 * e(P, Q) = f^(3 (p^12 - 1) / r) for the optimal-ate Miller value f: the cube of the textbook reduced pairing
 * (DESIGN.md section 3.8).  A pair with a point at infinity contributes 1; k = 0 gives 1.  A G1 point off the curve,
 * a G2 point off the twist or outside the r-torsion, or a coordinate >= p is DP_E_ARG naming the first bad pair.   */
int dp_multi_pairing(dp_ctx *ctx, const void *g1_104, const void *g2_200, size_t k, void *out576);

/* ---- setup files (DESIGN.md section 3.9): the encodings an SRS, open-key or verifying-key file holds.  Only
 * dp_get_bases_compressed and dp_srs_check need dp_init.  Buffers: host memory, or device memory of the context's GPU.
 * The inverse of dp_g1_decompress: n raw G1Affine (104 B each, not validated; the identity flag is honoured) -> ark-serialize
 * 0.3 compressed points (48 B each: canonical x little-endian, bit 7 of the last byte = (y > -y), bit 6 = identity).      */
int dp_g1_compress(dp_ctx *ctx, const void *in104, size_t n, void *out48);
/* bases [start, start + n) of an initialised context in that encoding, straight from the resident points               */
int dp_get_bases_compressed(dp_ctx *ctx, uint64_t start, size_t n, void *out48);
/* n raw G2Affine (200 B each) -> ark-serialize 0.3 compressed points (96 B each: canonical x.c0 then x.c1, 48 little-endian
 * bytes each; bit 7 of the last byte = (y > -y) with Fq2 ordered by c1 first, then c0; bit 6 = identity).  n <= 2^20.    */
int dp_g2_compress(dp_ctx *ctx, const void *in200, size_t n, void *out96);
/* The inverse, with the reason codes of dp_g1_decompress: *why = 1 (a coordinate >= p), 2 (both flag bits), 3 (no such point
 * on the twist y^2 = x^3 + 4 (u + 1)) or 4 (outside the r-torsion, checked when check_subgroup != 0).  A rejected point
 * returns DP_E_ARG, writes nothing to out200 and sets *bad_index; on success *bad_index = n, *why = 0.  n <= 2^20.       */
int dp_g2_decompress(dp_ctx *ctx, const void *in96, size_t n, int check_subgroup, void *out200, size_t *bad_index, int *why);
/* Are the context's bases P_0 .. P_(N-1) the powers g, tau g, tau^2 g, ... of the tau of this open key?  g2_400 = h, beta h
 * (two raw G2Affine, host).  *ok = 1 iff P_0 is the G1 generator and e(A, beta h) = e(B, h) for A = sum rho_i P_i and
 * B = sum rho_i P_(i+1), i < N - 1, with 128-bit rho_i from ChaCha20 blocks (RFC 8439) keyed by seed32 (32 B; NULL: drawn
 * from getrandom(2), DP_E_STATE if unavailable): an SRS that is not such a sequence passes with probability about 2^-128
 * over the seed, so a seed the producer of the SRS could predict proves nothing.  Two MSMs over all N bases and one 2-pair
 * pairing.  It does NOT replace the per-point subgroup check of dp_init_compressed: a component of a G1 point in the
 * cofactor subgroup is invisible to the pairing.  A G2 point off the twist or outside the r-torsion is DP_E_ARG, as in
 * dp_multi_pairing.  DP_E_STATE before dp_init or without bases; the context's state stays as it was.                    */
int dp_srs_check(dp_ctx *ctx, const void *g2_400, const void *seed32, int *ok);
/* the last dp_srs_check on ctx: host-clock ms of its scalar generation, its two MSMs and its pairing (each ends in a
 * device synchronise; 0 for a phase that did not run), and A, B (2 x 144 B normalised G1Projective).  NULL = not wanted */
int dp_last_srs_check(const dp_ctx *ctx, float *scalars_ms, float *msm_ms, float *pairing_ms, void *ab288);

/* ---- setup ceremony (DESIGN.md section 3.10): one contribution to a powers-of-tau SRS.  For the N resident bases P_i of
 * an initialised context and g2_400 = h, beta h (two raw G2Affine): out48[i] = s^i P_i as 48-byte compressed points
 * (the encoding of dp_g1_compress), and out400 = s h, s beta h (two raw G2Affine).  If P_i = tau^i g and beta h = tau h,
 * the output is the SRS of tau s.  s32: 32 B canonical, 0 < s < r, else DP_E_ARG; NULL draws s from getrandom(2)
 * (DP_E_STATE if unavailable).  s lives only inside the call: its host copies and the device power tables are zeroed
 * before it returns.  A G2 input off the twist, outside the r-torsion or with a coordinate >= p is DP_E_ARG, before any
 * G1 work.  The bases must lie in the r-torsion (dp_init_compressed with check_subgroup guarantees it).  out48, out400:
 * host memory or device memory of the context's GPU.  DP_E_STATE before dp_init or without bases; the context's state
 * (bases, MSM tables and tuning) stays as it was.                                                                        */
int dp_srs_update(dp_ctx *ctx, const void *s32, const void *g2_400, void *out48, void *out400);

/* ---- PlonkSlave.varMsm (src/worker.rs:159-185) -----------------------------------------------
 * out = sum_{k < min(end-start, n_scalars)} scalars[k] * bases[start + k]
 * (VariableBaseMSM::multi_scalar_mul(&bases[start..end], &scalars) truncates to the shorter).
 * scalars: canonical BigInteger256.  out: 144 B raw G1Projective, normalised (Z = 1) or identity. */
int dp_msm(dp_ctx *ctx, uint64_t start, uint64_t end, const void *scalars, size_t n_scalars, void *out);

/* Several varMsm requests issued together (the dispatcher joins the commitments of a round,
 * dispatcher2.rs:316-321, 526-532): scalars of request k+1 are copied in under the kernels of
 * request k, and the narrow tail kernels of k overlap the wide head kernels of k+1.  Arrays of
 * n_jobs entries, each with the semantics of dp_msm. */
int dp_msm_batch(dp_ctx *ctx, size_t n_jobs, const uint64_t *starts, const uint64_t *ends, const void *const *scalars,
                 const size_t *n_scalars, void *const *outs);

/* varMsm answered asynchronously (the Rust worker returns a Promise, as it already does for
 * fft2Prepare, src/worker.rs:293): dp_msm_submit queues the copy-in and the kernels behind whatever
 * the context is doing and returns; dp_msm_collect blocks until THAT job is done and writes the
 * 144-byte G1Projective.  `id` is the caller's (unique among pending jobs; at most 64 pending).
 * `scalars` must stay valid until the copy-in has run (dp_msm_collect, or dp_sync).  Lets
 * commitments share the GPU with transforms whose time goes into PCIe transfers.                 */
int dp_msm_submit(dp_ctx *ctx, uint64_t id, uint64_t start, uint64_t end, const void *scalars, size_t n_scalars);
int dp_msm_collect(dp_ctx *ctx, uint64_t id, void *out144);

/* ---- commit_polynomial (src/worker.rs:117-123) -----------------------------------------------
 * Fr::into_repr on every coefficient, zero-pad to bases.len(), MSM over all bases.
 * coeffs: n raw Fr (Montgomery), n <= n_bases. */
int dp_commit(dp_ctx *ctx, const void *coeffs, size_t n, void *out);

/* ---- PlonkSlave.fftInit (src/worker.rs:187-233) ----------------------------------------------
 * Opens task `id` (an open task with the same id is replaced, as `fft_tasks.insert` does).
 * workloads[w] is worker w's row / column range; n_workloads must equal n_workers and the ranges
 * must tile [0,r) x [0,c) in equal power-of-two blocks. */
int dp_fft_init(dp_ctx *ctx, uint64_t id, const dp_fft_workload *workloads, size_t n_workloads, int is_quot,
                int is_inv, int is_coset);

/* ---- PlonkSlave.fft1 (src/worker.rs:235-278) -------------------------------------------------
 * Hands in local row `i` (global row i + row_start).  len is normally c; a shorter row is zero-extended
 * and a longer one cut to c, which is what `c_domain.fft_in_place(&mut v)` does to `v` in the reference
 * (it resizes to the domain size) - a dispatcher may therefore leave out the zero tail of a padded
 * polynomial's rows.  The row transform (fft1_helper, worker.rs:66-94) runs on the device, at the latest
 * in dp_fft2_prepare. */
int dp_fft1(dp_ctx *ctx, uint64_t id, uint64_t i, const void *row, size_t len);
/* n_rows consecutive local rows in one call (rows = n_rows * c Fr, row-major) */
int dp_fft1_rows(dp_ctx *ctx, uint64_t id, uint64_t i_first, uint64_t n_rows, const void *rows);
/* the same for rows that are all cut after their first row_len <= c entries (rows = n_rows * row_len Fr,
 * compact): only the non-zero part of a padded polynomial's rows crosses PCIe, and the row kernel neither
 * reads the zero tail nor spends multiplications on it */
int dp_fft1_rows_short(dp_ctx *ctx, uint64_t id, uint64_t i_first, uint64_t n_rows, const void *rows, size_t row_len);

/* ---- PlonkSlave.fft2Prepare + PlonkPeer.fftExchange (src/worker.rs:280-345, 412-438) ---------
 * Finishes the row phase and moves every (rows_p x cols_q) block to its owner.  n_workers == 1:
 * purely local.  n_workers > 1: either peers were attached with dp_peer_attach (the blocks are
 * written straight into the owners' memory over NVLink by the row kernel), or the caller drives
 * the split API below around its own all-to-all (NCCL / torch.distributed). */
int dp_fft2_prepare(dp_ctx *ctx, uint64_t id);

/* split exchange: after _begin, *send_dev / *recv_dev are DEVICE pointers to n_workers blocks of
 * *block_elems Fr each (block q of send = my rows x q's columns, row-major = the payload of
 * fftExchange, worker.rs:327-330; block p of recv = p's rows x my columns).  The caller performs
 * the all-to-all (block q of send -> rank q, into block `me` of its recv) and calls _end. */
int dp_fft_exchange_begin(dp_ctx *ctx, uint64_t id, void **send_dev, void **recv_dev, uint64_t *block_elems);
int dp_fft_exchange_end(dp_ctx *ctx, uint64_t id);
/* Stream-ordered form of the same step, for a host that issues the exchange with its own NCCL
 * communicator: dp_fft_exchange_begin_async returns without waiting for the row phase; the two buffers
 * are then valid only for work enqueued on the context's compute stream (dp_compute_stream gives the
 * cudaStream_t), i.e. ncclGroupStart(); ncclSend / ncclRecv(..., stream) x W; ncclGroupEnd(); followed
 * by dp_fft_exchange_end.  Nothing blocks the host: copy-in, row kernels, all-to-all and column
 * kernels of consecutive tasks pipeline as they do for a single worker.                             */
int dp_fft_exchange_begin_async(dp_ctx *ctx, uint64_t id, void **send_dev, void **recv_dev, uint64_t *block_elems);
int dp_compute_stream(dp_ctx *ctx, void **stream);

/* ---- PlonkSlave.fft2 (src/worker.rs:347-381) -------------------------------------------------
 * Column transforms (fft2_helper, worker.rs:96-115); writes the local columns back to back
 * (n_cols * r Fr, column k at out + k*r*32 = the k-th `Data` of the reply) and drops the task. */
int dp_fft2(dp_ctx *ctx, uint64_t id, void *out, size_t out_bytes);

/* ---- whole-domain transform ------------------------------------------------------------------
 * Radix2EvaluationDomain::{fft,ifft,coset_fft,coset_ifft} on one device (round1's
 * ifft_in_place, worker.rs:398; the dispatcher-local coset_ifft, dispatcher2.rs:507).
 * data: n Fr in, 2^log_n Fr out (n <= 2^log_n, zero-padded like ark's resize); capacity of the
 * buffer must be 2^log_n elements. */
int dp_ntt(dp_ctx *ctx, void *data, size_t n, uint32_t log_n, int is_inv, int is_coset);

/* ---- PlonkSlave.round1 (src/worker.rs:383-408) -----------------------------------------------
 * evals (n Fr) -> ifft -> wire = (b0 + b1*X) * (X^n - 1) + poly -> commitment.  The reference
 * draws b0,b1 from the worker's ThreadRng (a CSPRNG): pass two secret, uniformly random Fr from the
 * host's own RNG in `blind` (2 raw Fr; also what makes the call reproducible in tests), or NULL to let
 * the library draw them from the operating system's entropy pool (getrandom(2), rejection-sampled
 * below r; DP_E_STATE if that source is unavailable).  The blinded polynomial stays resident
 * (state.wire, worker.rs:58) and can be read back with dp_get_wire. */
int dp_round1(dp_ctx *ctx, const void *evals, size_t n, const void *blind, void *out);
int dp_get_wire(dp_ctx *ctx, void *out, size_t out_bytes, size_t *n_coeffs);

/* ---- "next" row (SURVEY.md §8f-3): the round-2 permutation grand product -----------------------
 * What the dispatcher computes serially with one field division per row (src/dispatcher2.rs:
 * 329-345): z[0] = 1, z[j+1] = z[j] * prod_i (w_i[j] + gamma + beta*id_i[j])
 *                                     / prod_i (w_i[j] + gamma + beta*sigma_i[j]),  j < n-1.
 * wires[i][j] = circuit.witness[wire_variables[i][j]], id_perm[i][j] = extended_id_permutation[i*n+j],
 * sigma_perm[i][j] = extended_id_permutation[perm_i*n+perm_j]; all [num_wire_types][n] raw Fr, as are
 * beta, gamma (one Fr each) and out (n Fr).  DP_E_ARG when a denominator is zero. */
int dp_perm_product(dp_ctx *ctx, const void *wires, const void *id_perm, const void *sigma_perm, size_t num_wire_types, size_t n,
                    const void *beta, const void *gamma, void *out);
/* same with device-resident inputs and output (beta, gamma stay host pointers to one Fr each) */
int dp_perm_product_dev(dp_ctx *ctx, const void *wires_dev, const void *id_dev, const void *sigma_dev, size_t num_wire_types, size_t n,
                        const void *beta, const void *gamma, void *out_dev);

/* ---- circuit preprocessing and the witness gather, on the device --------------------------------
 * What jf-plonk's preprocessing and the dispatcher build on the CPU before round 1 (dispatcher2.rs:299, 337-342, 382-403).
 * A slot is s = i*n + j (wire type i, gate j), the indexing of wire_permutation[i*n + j].  vars_dev: num_wire_types*n u32
 * variable ids, slot order.  n must be the gate domain given to dp_init, num_wire_types 1..5.  Every entry returns
 * DP_E_STATE before dp_init and DP_E_ARG for n != the gate domain, num_wire_types outside 1..5, num_vars == 0, a variable
 * id >= num_vars, NULL or overlapping buffers; out-of-range ids are found by a check kernel, never read.               */
/* size of the scratch dp_wire_permutation_dev needs (about 16.5 B per slot when num_vars > 256)                     */
int dp_wire_permutation_scratch_bytes(size_t num_wire_types, size_t n, uint64_t num_vars, size_t *bytes);
/* succ_out_dev[s] = the next slot, in increasing slot order, holding the same variable as s; the last slot of a variable
 * maps to its first (the cycles of jf-relation's compute_wire_permutation).  A stable radix sort of the slots by
 * variable, ceil(bits(num_vars - 1) / 8) passes, in the caller's scratch (DP_E_ARG when smaller than
 * dp_wire_permutation_scratch_bytes says).                                                                          */
int dp_wire_permutation_dev(dp_ctx *ctx, const uint32_t *vars_dev, size_t num_wire_types, size_t n, uint64_t num_vars, void *scratch_dev,
                            size_t scratch_bytes, uint32_t *succ_out_dev);
/* id_out_dev[i*n + j] = k[i] * omega_n^j and sigma_out_dev[s] = id[succ_dev[s]] (dispatcher2.rs:340-342), both
 * num_wire_types*n raw Fr; succ_dev NULL: sigma = id.  k: num_wire_types raw Fr, host.  A host that already holds
 * jf-plonk's wire_permutation passes it here as flat slots (wire * n + gate).  DP_E_ARG for a slot >= num_wire_types*n.
 * The permutation argument is sound only when succ_dev is a permutation; that is not checked.                       */
int dp_perm_evals_dev(dp_ctx *ctx, const uint32_t *succ_dev, size_t num_wire_types, size_t n, const void *k, void *id_out_dev,
                      void *sigma_out_dev);
/* wires_out_dev[s] = witness_dev[vars_dev[s]] (num_wire_types*n raw Fr) and pub_out_dev[j] = the last wire type's value
 * at gate j for j < num_inputs, 0 up to n (the public input: the output wire of the first num_inputs gates, zero-padded
 * to n as the prover's pub_input).  witness_dev: num_vars raw Fr.  DP_E_ARG also for num_inputs > n.               */
int dp_witness_gather_dev(dp_ctx *ctx, const void *witness_dev, uint64_t num_vars, const uint32_t *vars_dev, size_t num_wire_types,
                          size_t n, size_t num_inputs, void *wires_out_dev, void *pub_out_dev);
/* dp_commit_dev of n_jobs device polynomials as one MSM batch (the joined commitments of a verifying key): outs144 =
 * n_jobs x 144 B, host.  Each coefficient buffer is converted to canonical form in place for the MSM and restored
 * before the call returns, so no n-sized scratch is needed per job.  DP_E_ARG for lens[j] > the number of bases.    */
int dp_commit_dev_batch(dp_ctx *ctx, size_t n_jobs, void *const *coeffs_dev, const size_t *lens, void *outs144);

/* ---- "next" row (SURVEY.md §8f-1): rounds 3-5 of Prover::prove on polynomials resident on the worker
 *
 * The reference declares round3 / round4 / round5 RPCs (hello_world.capnp:26-44) but never implements
 * them: the dispatcher pulls every polynomial back and does this arithmetic serially
 * (src/dispatcher2.rs:363-690).  These entries are the bodies those RPCs would call.  The plain
 * entries take host buffers (copied in and out); the *_dev entries take device pointers for the
 * polynomial-sized arrays (challenges and points stay host-side, 32 B each).  All values raw
 * Montgomery Fr; results byte-identical to the reference's sequential code.                        */

typedef struct dp_quotient_args {
    const void *selectors[13]; /* q_lc[4], q_mul[2], q_hash[4], q_o, q_c, q_ecc (dispatcher2.rs:437-450) */
    const void *sigmas[5];
    const void *wires[5];
    const void *perm;      /* permutation product polynomial z                                          */
    const void *pub_input;
    /* ^ 25 arrays of quot_domain_size Fr: coset evaluations over the quotient domain (lines 381-432)  */
    const void *k;         /* vk.k, 5 Fr, host                                                          */
    const void *alpha, *beta, *gamma; /* 1 Fr each, host                                                */
} dp_quotient_args;

/* Round 3, src/dispatcher2.rs:434-504: out[i] = 1/Z_H(x_i) * (gate(i) + alpha * permutation(i)) +
 * alpha^2/n * (z[i] - 1)/(x_i - 1), x_i = g * omega_m^i, over the quotient domain given to dp_init
 * (GATE_WIDTH 4, five wire types); the input of the final coset iFFT (line 507, dp_ntt).          */
int dp_quotient_evals(dp_ctx *ctx, const dp_quotient_args *host_arrays, void *out);
int dp_quotient_evals_dev(dp_ctx *ctx, const dp_quotient_args *dev_arrays, void *out_dev);

/* Round 3 one slice at a time, with n-sized instead of m-sized evaluation buffers (n, m = the two domains given to
 * dp_init, m/n slices).  The quotient coset is the disjoint union of m/n cosets of the gate domain:
 * g * omega_m^(slice + (m/n) i) = s * omega_n^i, s = g * omega_m^slice, i < n.
 * p(s * omega_n^i), i < n: slice `slice` of the coset evaluation on the quotient domain.  coeffs_dev: n_valid <= n
 * coefficients, not modified (entries past n_valid are not read); out_dev: n Fr, must not overlap coeffs_dev.
 * wait = 0 returns once queued (dp_sync waits).  DP_E_STATE before dp_init; DP_E_ARG for slice >= m/n, n_valid > n,
 * NULL pointers or overlapping buffers.                                                                            */
int dp_ntt_dev_quot_slice(dp_ctx *ctx, const void *coeffs_dev, size_t n_valid, uint32_t slice, void *out_dev, int wait);
/* dp_quotient_evals_dev for one slice: the 25 arrays hold n Fr each (slice `slice` of the coset evaluations, as
 * dp_ntt_dev_quot_slice writes them); writes out_dev[slice + (m/n) i], i < n, of the m-entry output and nothing else.
 * All m/n slices = dp_quotient_evals_dev, byte for byte.  Same errors as dp_ntt_dev_quot_slice.                    */
int dp_quotient_evals_slice_dev(dp_ctx *ctx, const dp_quotient_args *slice_arrays, uint32_t slice, void *out_dev);

/* Round 3 with blinded wires and z (dispatcher2.rs:294-361: each wire + rand(1)*Z_H, z + rand(2)*Z_H).  A blinded
 * polynomial has n + t coefficients (t <= 3); split it as p = head + X^n * tail, head = its first n coefficients.
 * The 25 arrays of dp_quotient_args hold the coset evaluations of the heads only (the usual n-coefficient transforms);
 * the tails are coefficients n, n+1, ... of each wire and of z, device pointers, t of them (0 = not blinded).  The
 * output is the quotient of the full polynomials.  With every length 0 it equals dp_quotient_evals[_slice]_dev byte
 * for byte.  DP_E_ARG for a length > 3, a NULL pointer with a length > 0, or a tail that overlaps the output; else the
 * errors of the entry without tails.                                                                               */
typedef struct dp_quotient_tails {
    const void *wires[5];
    size_t wire_len[5];
    const void *perm;
    size_t perm_len;
} dp_quotient_tails;
int dp_quotient_evals_tail_dev(dp_ctx *ctx, const dp_quotient_args *dev_arrays, const dp_quotient_tails *tails, void *out_dev);
int dp_quotient_evals_slice_tail_dev(dp_ctx *ctx, const dp_quotient_args *slice_arrays, const dp_quotient_tails *tails,
                                     uint32_t slice, void *out_dev);

/* Round 3 of a batch proof (DESIGN.md 3.11): out_dev[pt] += scale * Q(pt), Q the quotient value the entries above write,
 * over the whole coset (dev_arrays: 25 arrays of m Fr) or over the points of one slice (slice_arrays: n Fr each; only
 * out_dev[slice + (m/n) i] is read and written).  The batch quotient sum_i alpha^(3i) Q_i is one call per instance into
 * the same output, instance 0 through the non-accumulating entries.  tails: as above, or NULL for unblinded wires and z.
 * scale32: 1 raw Fr below r, host.  The result is byte for byte dp_poly_lincomb_dev([out, Q], [1, scale]).  DP_E_ARG
 * for a scale not below r, an output that overlaps any of the 25 inputs or a tail; else the errors of the entries above. */
int dp_quotient_evals_acc_dev(dp_ctx *ctx, const dp_quotient_args *dev_arrays, const dp_quotient_tails *tails, const void *scale32,
                              void *out_dev);
int dp_quotient_evals_slice_acc_dev(dp_ctx *ctx, const dp_quotient_args *slice_arrays, const dp_quotient_tails *tails,
                                    uint32_t slice, const void *scale32, void *out_dev);

/* Blinding, as the reference prover does it to every wire (k = 2) and to z (k = 3): coeffs += b(X) * (X^n - 1),
 * b(X) = b_0 + b_1 X + ... + b_(k-1) X^(k-1), in place on a device buffer of at least n + k Fr (b_j is subtracted
 * from coefficient j and added to coefficient n + j).  blind: k raw Fr below r on the host (reproducible, for
 * tests), or NULL: the library draws k secret scalars uniformly below r from the operating system's entropy pool
 * (getrandom(2)) and they never leave it.  DP_E_ARG for k > 3 or a scalar not below r; DP_E_STATE if the entropy
 * source is unavailable.                                                                                          */
int dp_poly_blind_dev(dp_ctx *ctx, void *coeffs_dev, size_t n, uint32_t k, const void *blind);

/* Round 4, DensePolynomial::evaluate (src/dispatcher2.rs:535-548): out32 = sum_j coeffs[j] * point^j */
int dp_poly_eval(dp_ctx *ctx, const void *coeffs, size_t n, const void *point, void *out32);
int dp_poly_eval_dev(dp_ctx *ctx, const void *coeffs_dev, size_t n, const void *point, void *out32);

/* Round 5, the folds of src/dispatcher2.rs:566-649 (lin_poly, r_quot, batch_poly):
 * out[j] = sum_{i<k} coeffs[i] * polys[i][j], polys[i] zero-extended past lens[i]; k <= 32.
 * polys / lens / coeffs are host arrays; polys[i] points to host (plain) or device (_dev) memory.
 * The combination is element-wise, so out_dev may be one of the operands (the same pointer, read at j before out[j] is
 * written): more than 32 operands are chained, out = lincomb(first 32), then out = lincomb([out] + next 31, [1, ...]). */
int dp_poly_lincomb(dp_ctx *ctx, const void *const *polys, const size_t *lens, const void *coeffs, size_t k, void *out, size_t out_len);
int dp_poly_lincomb_dev(dp_ctx *ctx, const void *const *polys_dev, const size_t *lens, const void *coeffs, size_t k, void *out_dev,
                        size_t out_len);

/* Round 5, the opening witnesses (src/dispatcher2.rs:651-666, 672-688): the n-1 coefficients of
 * p(X) / (X - point) into out, and the remainder p(point) into rem32 when it is not NULL.
 * out_dev must not overlap coeffs_dev (DP_E_ARG): the division is not done in place.              */
int dp_poly_div_linear(dp_ctx *ctx, const void *coeffs, size_t n, const void *point, void *out, void *rem32);
int dp_poly_div_linear_dev(dp_ctx *ctx, const void *coeffs_dev, size_t n, const void *point, void *out_dev, void *rem32);

/* ---- worker-resident polynomials ---------------------------------------------------------------
 * `state.wire` of the reference (src/worker.rs:58,400-405) generalised: named device buffers the
 * *_dev entries above, dp_ntt_dev, dp_perm_product_dev and dp_commit_dev work on, so a polynomial
 * crosses PCIe once (or never: outputs of one step are inputs of the next).  A Rust worker has no
 * device allocator of its own; this is it.                                                          */
/* create / overwrite polynomial `poly_id`: `capacity` Fr on the device (>= n; e.g. the quotient domain
 * size for a polynomial that will be transformed in place), coefficients [0, n) copied from the host,
 * the rest zero.  Re-putting with the same capacity reuses the buffer.                              */
int dp_poly_put(dp_ctx *ctx, uint64_t poly_id, const void *coeffs, size_t n, size_t capacity);
int dp_poly_ptr(dp_ctx *ctx, uint64_t poly_id, void **dev, size_t *capacity); /* the device address         */
int dp_poly_get(dp_ctx *ctx, uint64_t poly_id, size_t offset, size_t n, void *out);    /* copy back        */
int dp_poly_free(dp_ctx *ctx, uint64_t poly_id);
/* commit_polynomial (src/worker.rs:117-123) of n coefficients already on the device -> 144 B        */
int dp_commit_dev(dp_ctx *ctx, const void *coeffs_dev, size_t n, void *out144);

/* ---- peer transport for n_workers > 1 ---------------------------------------------------------
 * Exchange arena shared between the GPUs of one box through CUDA IPC: every rank exports a
 * handle, the ranks swap them out of band (torch.distributed / the capnp control plane) and attach
 * the others'.  Afterwards dp_fft2_prepare stores the row-phase output straight into the owners'
 * arenas over NVLink and returns when its stores are complete; the caller provides the barrier across
 * ranks between fft2Prepare and fft2 - the dispatcher's join over the fft2Prepare replies is one.
 * Slots: the arena holds as many receive matrices ([r][c/n_workers] Fr of the LARGER domain given to dp_init) as fit
 * into arena_bytes, at least two are required; exchange number k uses slot k mod n_slots on every rank, so every rank
 * must issue its exchanges in the same order (as for a collective) and at most n_slots tasks per context may sit
 * between dp_fft2_prepare and dp_fft2: one more dp_fft2_prepare returns DP_E_STATE (nothing is consumed: call dp_fft2
 * on an earlier task, then retry - or use dp_fft_exchange_begin/_end, which has per-task buffers and no limit).
 * The slot sequence only advances on success.  A worker behind the reference dispatcher (up to 26 transforms in
 * flight, dispatcher2.rs:382-414) creates 32 slots; two are enough for one transform at a time.
 * arena_bytes >= n_slots * (r * c / n_workers) * 32 for the largest domain; the same on every rank. */
#define DP_IPC_HANDLE_BYTES 64
int dp_peer_arena_create(dp_ctx *ctx, uint64_t arena_bytes, void *handle_out /* DP_IPC_HANDLE_BYTES */);
int dp_peer_attach(dp_ctx *ctx, uint64_t peer, const void *handle /* DP_IPC_HANDLE_BYTES */);
int dp_peer_ready(const dp_ctx *ctx); /* 1 when the arena exists and every peer is attached */

/* ---- instrumentation --------------------------------------------------------------------------*/
/* device-side time (ms, CUDA events on the context stream) and kernel launches of the last call */
int dp_last_timing(const dp_ctx *ctx, float *kernel_ms, uint64_t *launches);
/* total kernel launches since dp_create */
uint64_t dp_launch_count(const dp_ctx *ctx);
/* block until everything queued on the context stream has finished */
int dp_sync(dp_ctx *ctx);

/* device-side ms of the three phases of the last MSM on ctx: digit sort (count/scan/scatter/tasks),
 * bucket accumulation (the dominant kernel), bucket reduction + window combine + normalise */
int dp_last_msm_breakdown(const dp_ctx *ctx, float *sort_ms, float *accumulate_ms, float *reduce_ms);

/* what dp_init's MSM tuning found: one MSM over the context's own window-multiple table with the plain pipeline
 * (XYZZ chunks) and one with 2 batched-affine tree levels in front of it (1, 2 and 3 with DP_MSM_TUNE=2; *affine_ms = the best);
 * *equal = all results were the same 144 bytes (1), some differed (0: the plain pipeline is kept), or the tuning did not
 * run (-1: DP_MSM_TUNE=0, small SRS, or DP_MSM_AFFINE set); *levels = what MSMs of this context use (0 = plain).  Replaces nothing in the reference: ark-ec has one algorithm. */
int dp_msm_tuning(const dp_ctx *ctx, float *plain_ms, float *affine_ms, int *levels, int *equal);
/* the same experiment in full: ms of one MSM with 0 (plain), 1, 2 and 3 tree levels (0 = not measured) */
int dp_msm_tuning_all(const dp_ctx *ctx, float ms_by_levels[4]);

/* synthetic SRS: n distinct points k_i*G (k_i = SplitMix64(seed, i)), raw 104-byte G1Affine each,
 * computed on the device and written to `out` (host memory, or device memory of the same GPU); feeds
 * dp_init in benches and tests */
int dp_debug_gen_bases(dp_ctx *ctx, uint64_t seed, size_t n, void *out);

/* dp_srs_update computed with the plain 255-bit double-and-add per point instead of the endomorphism split: the same
 * bytes, slower; the reference dp_srs_update is measured and tested against                                   */
int dp_debug_srs_update_plain(dp_ctx *ctx, const void *s32, const void *g2_400, void *out48, void *out400);

/* test hook: lower the pass-planning limits (sub-transform sizes 2^k handled by one kernel pass;
 * defaults 11 / 9) and/or steer the MSM (0 = automatic: precomputed window multiples when the SRS is
 * large enough; 1 = per-window bucket sets with automatic width; c >= 2 = per-window sets of width c)
 * so that small inputs exercise the multi-pass NTT plans and every MSM geometry. */
int dp_debug_set_limits(dp_ctx *ctx, uint32_t max_contig_log_k, uint32_t max_strided_log_k, int msm_window_bits);
/* test hook: the single-worker three-pass transform plan (DESIGN.md section 3.1) is used for domains of at least
 * 2^min_log_n points (default 20); 0 switches it off (the 2-D row / column plan is used everywhere). */
int dp_debug_set_three_pass(dp_ctx *ctx, uint32_t min_log_n);

/* device-resident variants used by bench.py to time the kernels with inputs already in HBM.
 * All pointers are DEVICE pointers owned by the caller (e.g. torch tensors). */
int dp_msm_dev(dp_ctx *ctx, uint64_t start, uint64_t end, const void *scalars_dev, size_t n_scalars, void *out_dev);
/* several MSMs issued together (the commitments of one prover round, join_all in dispatcher2.rs:
 * 316-321, 526-532): the narrow tail kernels of MSM k overlap the wide head kernels of MSM k+1.
 * Arrays of n_jobs entries; same semantics per job as dp_msm_dev. */
int dp_msm_dev_batch(dp_ctx *ctx, size_t n_jobs, const uint64_t *starts, const uint64_t *ends, const void *const *scalars_dev,
                     const size_t *n_scalars, void *const *outs_dev);
int dp_ntt_dev(dp_ctx *ctx, void *data_dev, uint32_t log_n, int is_inv, int is_coset);
/* the same on a buffer whose entries from n_valid on are ZERO (a resident coefficient vector shorter than the
 * domain: n coefficients evaluated on the 8n-point coset, dispatcher2.rs:386-388): the forward transform neither
 * reads nor multiplies the zero tail.  wait = 0 returns once the kernels are queued (dp_sync waits).        */
int dp_ntt_dev_padded(dp_ctx *ctx, void *data_dev, size_t n_valid, uint32_t log_n, int is_inv, int is_coset, int wait);
/* full 2-D pipeline of one worker on device-resident rows: rows_dev = my rows (n_rows*c Fr),
 * cols_dev receives my columns (n_cols*r Fr); n_workers must be 1 or peers attached. */
int dp_fft_dev(dp_ctx *ctx, const void *rows_dev, void *cols_dev, int is_quot, int is_inv, int is_coset);
/* Promise about the rows given to the dp_fft_dev* entries of one domain (is_quot) from now on: every row is
 * zero from column valid_cols on - the shape of n coefficients on the 8n-point quotient domain, where
 * valid_cols = c/8 (dispatcher2.rs:386-388).  Forward transforms then neither read nor multiply the zero
 * tail (same effect as short rows through dp_fft1); inverse transforms ignore the promise.  0 = no promise. */
int dp_fft_dev_hint_valid_cols(dp_ctx *ctx, int is_quot, uint64_t valid_cols);
/* the same split around the caller's all-to-all for n_workers > 1 (one transform in flight per ctx):
 * _rows runs the row phase on my row block (rows_dev: r/W x c Fr) and returns the exchange buffers
 * exactly like dp_fft_exchange_begin; after the all-to-all _cols runs the column phase into
 * cols_dev (c/W x r Fr).  With n_workers == 1 recv == send and no exchange is needed. */
int dp_fft_dev_rows(dp_ctx *ctx, const void *rows_dev, int is_quot, int is_inv, int is_coset, void **send_dev,
                    void **recv_dev, uint64_t *block_elems);
int dp_fft_dev_cols(dp_ctx *ctx, void *cols_dev);
/* fused variant of _rows for attached peers: the row kernel stores into the owners' arenas; the
 * caller then only needs a barrier across ranks before dp_fft_dev_cols */
int dp_fft_dev_rows_p2p(dp_ctx *ctx, const void *rows_dev, int is_quot, int is_inv, int is_coset);
/* the whole distributed transform of one worker without host involvement: row kernels (stores into
 * the owners' arenas), a device-side barrier kernel (system-scope arrival counters in the arenas,
 * over NVLink), column kernels, queued back to back on the context stream; returns when done.
 * Every rank must call it for the same transforms in the same order (it blocks like a collective). */
int dp_fft_dev_p2p(dp_ctx *ctx, const void *rows_dev, void *cols_dev, int is_quot, int is_inv, int is_coset);
/* the same, returning as soon as the kernels are queued (rows_dev / cols_dev must stay valid until dp_sync,
 * which also reports a barrier time-out as DP_E_COMM).  Any number of transforms may be queued back to back:
 * the two arena slots are recycled in stream order behind the device-side barriers.                      */
int dp_fft_dev_p2p_async(dp_ctx *ctx, const void *rows_dev, void *cols_dev, int is_quot, int is_inv, int is_coset);

#ifdef __cplusplus
}
#endif
#endif /* DPLONK_H */
