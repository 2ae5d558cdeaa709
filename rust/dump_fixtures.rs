//! dump_fixtures: golden vectors for the MSM + NTT hot path produced by the REFERENCE's own code - arkworks 0.3.0 as
//! pinned by the reference's Cargo.lock, the helper bodies of src/worker.rs:66-123, src/utils.rs `serialize`.
//!
//!   cp rust/dump_fixtures.rs <reference>/src/bin/dump_fixtures.rs
//!   (Cargo.toml: rand_chacha = "0.3" next to `rand`; nothing else)
//!   cargo run --release --bin dump_fixtures -- ref_v1.bin ref_plonk_v1.bin && cp ref_v1.bin ref_plonk_v1.bin <this repo>/tests/golden/
//!
//! ref_plonk_v1.bin (same format) pins the Fiat-Shamir side: merlin 3.0.0 op sequences and the challenge bytes they give
//! (TRANSCRIPT), and one small jf-plonk proof with its verifying key, public inputs, the six challenges jf-plonk's
//! verifier derives, and the verify result (PLONK).  Consumer: tests/test_ref_plonk_fixture.py.
//!
//! Format: rust/README.md ("ref_v1.bin format").  Consumer: tests/test_ref_fixture.py (oracle on the CPU, the CUDA
//! library with -m gpu), byte for byte.  NOT COMPILED in this repository (no Rust toolchain in the build image).
use ark_bls12_381::{Fr, G1Affine, G1Projective};
use ark_ec::{msm::VariableBaseMSM, AffineCurve, ProjectiveCurve};
use ark_ff::{BigInteger256, FftField, Field, PrimeField, UniformRand, Zero, One};
use ark_poly::{EvaluationDomain, Radix2EvaluationDomain};
use ark_serialize::CanonicalSerialize;
use hello_world::utils::serialize;
use rand_chacha::{rand_core::SeedableRng, ChaCha20Rng};
use std::{fs::File, io::Write};
use ark_bls12_381::Bls12_381;
use jf_plonk::prelude::*;
use jf_plonk::proof_system::{PlonkKzgSnark, Snark};
use jf_utils::to_bytes;
use merlin::Transcript;

const SEED: u64 = 0xD15791B07E5EED;

struct Out {
    f: File,
    count: u32,
    body: Vec<u8>,
}
impl Out {
    fn record(&mut self, tag: u32, p: [u64; 4], blobs: &[&[u8]]) {
        self.body.extend_from_slice(&tag.to_le_bytes());
        for v in p.iter() {
            self.body.extend_from_slice(&v.to_le_bytes());
        }
        self.body.extend_from_slice(&(blobs.len() as u32).to_le_bytes());
        for b in blobs {
            self.body.extend_from_slice(&(b.len() as u64).to_le_bytes());
            self.body.extend_from_slice(b);
        }
        self.count += 1;
    }
    fn finish(mut self) {
        self.f.write_all(b"DPREFv1\0").unwrap();
        self.f.write_all(&self.count.to_le_bytes()).unwrap();
        self.f.write_all(&self.body).unwrap();
    }
    fn rng(&self) -> ChaCha20Rng {
        ChaCha20Rng::seed_from_u64(SEED ^ self.count as u64)
    }
}

// ---- src/worker.rs:66-115, verbatim semantics (the functions are private to the worker binary)
fn fft1_helper(v: &mut Vec<Fr>, i: u64, is_coset: bool, is_inv: bool, domain: &Radix2EvaluationDomain<Fr>,
               c_domain: &Radix2EvaluationDomain<Fr>, r_domain: &Radix2EvaluationDomain<Fr>) {
    if is_coset && !is_inv {
        let g = Fr::multiplicative_generator();
        v.iter_mut().enumerate().for_each(|(j, u)| *u *= g.pow([i + j as u64 * r_domain.size]));
    }
    if is_inv { c_domain.ifft_in_place(v) } else { c_domain.fft_in_place(v) }
    let w = if is_inv { domain.group_gen_inv } else { domain.group_gen };
    v.iter_mut().enumerate().for_each(|(j, u)| *u *= w.pow([i * j as u64]));
}
fn fft2_helper(v: &mut Vec<Fr>, i: u64, is_coset: bool, is_inv: bool, c_domain: &Radix2EvaluationDomain<Fr>,
               r_domain: &Radix2EvaluationDomain<Fr>) {
    if is_inv { r_domain.ifft_in_place(v) } else { r_domain.fft_in_place(v) }
    if is_coset && is_inv {
        let g = Fr::multiplicative_generator().inverse().unwrap();
        v.iter_mut().enumerate().for_each(|(j, u)| *u *= g.pow([i + j as u64 * c_domain.size]));
    }
}
fn split(domain: &Radix2EvaluationDomain<Fr>) -> (Radix2EvaluationDomain<Fr>, Radix2EvaluationDomain<Fr>) {
    let r = 1 << (domain.log_size_of_group >> 1); // worker.rs:144-147
    let c = domain.size() / r;
    (Radix2EvaluationDomain::new(r).unwrap(), Radix2EvaluationDomain::new(c).unwrap())
}
/// the distributed transform as the dispatcher drives it (dispatcher2.rs:731-787) with the worker helpers above
fn dist_fft(x: &[Fr], log: u32, is_inv: bool, is_coset: bool) -> Vec<Fr> {
    let domain = Radix2EvaluationDomain::<Fr>::new(1 << log).unwrap();
    let (r_domain, c_domain) = split(&domain);
    let (r, c) = (r_domain.size(), c_domain.size());
    let mut x = x.to_vec();
    x.resize(domain.size(), Fr::zero());
    let mut rows = (0..r).map(|i| (0..c).map(|j| x[i + r * j]).collect::<Vec<_>>()).collect::<Vec<_>>();
    for (i, row) in rows.iter_mut().enumerate() {
        fft1_helper(row, i as u64, is_coset, is_inv, &domain, &c_domain, &r_domain);
    }
    let mut cols = (0..c).map(|k| (0..r).map(|i| rows[i][k]).collect::<Vec<_>>()).collect::<Vec<_>>();
    for (k, col) in cols.iter_mut().enumerate() {
        fft2_helper(col, k as u64, is_coset, is_inv, &c_domain, &r_domain);
    }
    let mut out = vec![Fr::zero(); r * c];
    for k in 0..c {
        for j in 0..r {
            out[j * c + k] = cols[k][j]; // dispatcher2.rs:780-786
        }
    }
    out
}

// ---- ref_plonk_v1.bin: the transcript and one jf-plonk proof
const OP_NEW: u8 = 0;
const OP_APPEND: u8 = 1;
const OP_CHALLENGE: u8 = 2;

/// one op of a TRANSCRIPT record: kind u8, label (u32 LE length + bytes), then the message (u32 LE length + bytes) of
/// an append or the u32 LE byte count of a challenge
fn op(ops: &mut Vec<u8>, kind: u8, label: &[u8], payload: &[u8]) {
    ops.push(kind);
    ops.extend_from_slice(&(label.len() as u32).to_le_bytes());
    ops.extend_from_slice(label);
    if kind == OP_APPEND {
        ops.extend_from_slice(&(payload.len() as u32).to_le_bytes());
    }
    ops.extend_from_slice(payload);
}

fn transcript_record(o: &mut Out, msg_lens: &[usize], challenge_lens: &[usize]) {
    let (mut ops, mut out, mut count) = (vec![], vec![], 0u64);
    let mut t = Transcript::new(b"dump_fixtures");
    op(&mut ops, OP_NEW, b"dump_fixtures", &[]);
    count += 1;
    for (i, &ln) in msg_lens.iter().enumerate() {
        let m = (0..ln).map(|j| ((j * 7 + i) & 255) as u8).collect::<Vec<_>>();
        t.append_message(b"m", &m);
        op(&mut ops, OP_APPEND, b"m", &m);
        let mut buf = vec![0u8; 64];
        t.challenge_bytes(b"c", &mut buf);
        op(&mut ops, OP_CHALLENGE, b"c", &64u32.to_le_bytes());
        out.extend_from_slice(&buf);
        count += 2;
    }
    for &k in challenge_lens {
        let mut buf = vec![0u8; k];
        t.challenge_bytes(b"k", &mut buf);
        op(&mut ops, OP_CHALLENGE, b"k", &(k as u32).to_le_bytes());
        out.extend_from_slice(&buf);
        count += 1;
    }
    o.record(9, [count, 0, 0, 0], &[&ops, &out]);
}

/// get_and_append_challenge of dispatcher2.rs:144-153
fn challenge(t: &mut Transcript, label: &'static [u8]) -> Fr {
    let mut buf = [0u8; 64];
    t.challenge_bytes(label, &mut buf);
    let c = Fr::from_le_bytes_mod_order(&buf);
    t.append_message(label, &to_bytes!(&c).unwrap());
    c
}

fn plonk_record(o: &mut Out) {
    let mut rng = o.rng();
    let mut circuit = PlonkCircuit::<Fr>::new();
    let x = circuit.create_public_variable(Fr::from(3u64)).unwrap();
    let y = circuit.create_variable(Fr::from(4u64)).unwrap();
    let s = circuit.add(x, y).unwrap();
    let p = circuit.mul(s, y).unwrap();
    let out = circuit.create_public_variable(Fr::from(28u64)).unwrap();
    circuit.equal_gate(p, out).unwrap();
    circuit.finalize_for_arithmetization().unwrap();
    let srs = PlonkKzgSnark::<Bls12_381>::universal_setup(circuit.srs_size().unwrap(), &mut rng).unwrap();
    let (pk, vk) = PlonkKzgSnark::<Bls12_381>::preprocess(&srs, &circuit).unwrap();
    let proof = PlonkKzgSnark::<Bls12_381>::prove::<_, _, StandardTranscript>(&mut rng, &circuit, &pk).unwrap();
    let pub_input = circuit.public_input().unwrap();
    let ok = PlonkKzgSnark::<Bls12_381>::verify::<StandardTranscript>(&vk, &pub_input, &proof).is_ok();
    // the verifier's transcript, as FakeStandardTranscript (dispatcher2.rs:44-154) and jf-plonk's verifier feed it
    let mut t = Transcript::new(b"PlonkProof");
    t.append_message(b"field size in bits", &Fr::size_in_bits().to_le_bytes());
    t.append_message(b"domain size", &vk.domain_size.to_le_bytes());
    t.append_message(b"input size", &vk.num_inputs.to_le_bytes());
    let mut vk_bytes = vec![];
    for k in vk.k.iter() {
        vk_bytes.extend(to_bytes!(k).unwrap());
        t.append_message(b"wire subsets separators", &to_bytes!(k).unwrap());
    }
    for c in vk.selector_comms.iter() {
        vk_bytes.extend(to_bytes!(c).unwrap());
        t.append_message(b"selector commitments", &to_bytes!(c).unwrap());
    }
    for c in vk.sigma_comms.iter() {
        vk_bytes.extend(to_bytes!(c).unwrap());
        t.append_message(b"sigma commitments", &to_bytes!(c).unwrap());
    }
    let mut pub_bytes = vec![];
    for v in pub_input.iter() {
        pub_bytes.extend(to_bytes!(v).unwrap());
        t.append_message(b"public input", &to_bytes!(v).unwrap());
    }
    for c in proof.wires_poly_comms.iter() {
        t.append_message(b"witness_poly_comms", &to_bytes!(c).unwrap());
    }
    let beta = challenge(&mut t, b"beta");
    let gamma = challenge(&mut t, b"gamma");
    t.append_message(b"perm_poly_comms", &to_bytes!(&proof.prod_perm_poly_comm).unwrap());
    let alpha = challenge(&mut t, b"alpha");
    for c in proof.split_quot_poly_comms.iter() {
        t.append_message(b"quot_poly_comms", &to_bytes!(c).unwrap());
    }
    let zeta = challenge(&mut t, b"zeta");
    for v in proof.poly_evals.wires_evals.iter() {
        t.append_message(b"wire_evals", &to_bytes!(v).unwrap());
    }
    for v in proof.poly_evals.wire_sigma_evals.iter() {
        t.append_message(b"wire_sigma_evals", &to_bytes!(v).unwrap());
    }
    t.append_message(b"perm_next_eval", &to_bytes!(&proof.poly_evals.perm_next_eval).unwrap());
    let v = challenge(&mut t, b"v");
    t.append_message(b"open_proof", &to_bytes!(&proof.opening_proof).unwrap());
    t.append_message(b"shifted_open_proof", &to_bytes!(&proof.shifted_opening_proof).unwrap());
    let u = challenge(&mut t, b"u");
    let mut ch = vec![];
    for c in [beta, gamma, alpha, zeta, v, u].iter() {
        ch.extend(to_bytes!(c).unwrap());
    }
    let mut proof_bytes = vec![];
    proof.serialize(&mut proof_bytes).unwrap();
    o.record(10, [vk.domain_size as u64, vk.num_inputs as u64, 0, 0], &[&vk_bytes, &pub_bytes, &proof_bytes, &ch, &[ok as u8]]);
}

fn main() {
    let path = std::env::args().nth(1).unwrap_or_else(|| "ref_v1.bin".to_string());
    let mut o = Out { f: File::create(&path).unwrap(), count: 0, body: vec![] };

    // 1 LAYOUT
    let seven = Fr::from(7u64);
    o.record(1,
        [std::mem::size_of::<Fr>() as u64, std::mem::size_of::<G1Affine>() as u64, std::mem::size_of::<G1Projective>() as u64,
         std::mem::size_of::<BigInteger256>() as u64],
        &[serialize(&[Fr::one()]), serialize(&[seven]), serialize(&[G1Affine::prime_subgroup_generator()]),
          serialize(&[G1Affine::zero()]), serialize(&[G1Projective::zero()]), serialize(&[seven.into_repr()])]);

    // 2 NTT: every flag combination, full and short inputs, sizes around the library's pass-plan boundaries
    for &log in &[0u32, 1, 3, 6, 9, 11, 12, 15, 16] {
        for &(inv, coset) in &[(false, false), (true, false), (false, true), (true, true)] {
            for &n_in in &[1usize << log, ((1usize << log) / 8).max(1)] {
                let mut rng = o.rng();
                let x = (0..n_in).map(|_| Fr::rand(&mut rng)).collect::<Vec<_>>();
                let domain = Radix2EvaluationDomain::<Fr>::new(1 << log).unwrap();
                let mut y = x.clone();
                match (inv, coset) {
                    (false, false) => domain.fft_in_place(&mut y),
                    (true, false) => domain.ifft_in_place(&mut y),
                    (false, true) => domain.coset_fft_in_place(&mut y),
                    (true, true) => domain.coset_ifft_in_place(&mut y),
                }
                o.record(2, [log as u64, inv as u64, coset as u64, n_in as u64], &[serialize(&x), serialize(&y)]);
                if log >= 3 {
                    let z = dist_fft(&x, log, inv, coset);
                    o.record(7, [log as u64, inv as u64, coset as u64, n_in as u64], &[serialize(&x), serialize(&z)]);
                }
            }
        }
    }
    // 3 / 4: single rows and columns through the worker's helpers
    for &log in &[6u32, 9, 13] {
        let domain = Radix2EvaluationDomain::<Fr>::new(1 << log).unwrap();
        let (r_domain, c_domain) = split(&domain);
        for &(inv, coset) in &[(false, false), (true, false), (false, true), (true, true)] {
            for &i in &[0u64, 1, (r_domain.size() - 1) as u64] {
                let mut rng = o.rng();
                let row = (0..c_domain.size()).map(|_| Fr::rand(&mut rng)).collect::<Vec<_>>();
                let mut out = row.clone();
                fft1_helper(&mut out, i, coset, inv, &domain, &c_domain, &r_domain);
                o.record(3, [log as u64, i, inv as u64, coset as u64], &[serialize(&row), serialize(&out)]);
            }
            for &i in &[0u64, 2, (c_domain.size() - 1) as u64] {
                let mut rng = o.rng();
                let col = (0..r_domain.size()).map(|_| Fr::rand(&mut rng)).collect::<Vec<_>>();
                let mut out = col.clone();
                fft2_helper(&mut out, i, coset, inv, &c_domain, &r_domain);
                o.record(4, [log as u64, i, inv as u64, coset as u64], &[serialize(&col), serialize(&out)]);
            }
        }
    }
    // 5 MSM / 6 COMMIT: bases in the style of dispatcher.rs:190-196 (distinct points tiled by doubling, one infinity)
    for &n in &[1usize, 33, 600, (1 << 12) + 32] {
        let mut rng = o.rng();
        let distinct = n.min(64);
        let mut bases = (0..distinct).map(|_| G1Projective::rand(&mut rng).into_affine()).collect::<Vec<_>>();
        if distinct > 3 {
            bases[3] = G1Affine::zero();
        }
        while bases.len() < n {
            let take = (n - bases.len()).min(bases.len());
            let more = bases[..take].to_vec();
            bases.extend(more);
        }
        let mut scalars = (0..n).map(|_| Fr::rand(&mut rng).into_repr()).collect::<Vec<_>>();
        if n > 8 {
            scalars[1] = Fr::zero().into_repr();
            scalars[2] = Fr::one().into_repr();
            scalars[5] = (-Fr::one()).into_repr();
        }
        for &(a, b) in &[(0usize, n), (n / 3, n - n / 4)] {
            let s = &scalars[..b - a];
            let res = VariableBaseMSM::multi_scalar_mul(&bases[a..b], s);
            o.record(5, [a as u64, b as u64, 0, 0],
                &[serialize(&bases), serialize(s), serialize(&[res]), serialize(&[res.into_affine()])]);
        }
        let coeffs = (0..n.saturating_sub(n / 5).max(1)).map(|_| Fr::rand(&mut rng)).collect::<Vec<_>>();
        let mut sc = coeffs.iter().map(|s| s.into_repr()).collect::<Vec<_>>(); // worker.rs:117-123
        sc.resize(bases.len(), Fr::zero().into_repr());
        let res = VariableBaseMSM::multi_scalar_mul(&bases, &sc);
        o.record(6, [coeffs.len() as u64, 0, 0, 0], &[serialize(&bases), serialize(&coeffs), serialize(&[res.into_affine()])]);
    }
    // 8 COMPRESSED: canonical encoding (what SRS files hold) next to the raw structs
    {
        let mut rng = o.rng();
        let mut pts = (0..40).map(|_| G1Projective::rand(&mut rng).into_affine()).collect::<Vec<_>>();
        pts[7] = G1Affine::zero();
        let mut comp = vec![];
        for p in &pts {
            p.serialize(&mut comp).unwrap();
        }
        o.record(8, [pts.len() as u64, 0, 0, 0], &[serialize(&pts), &comp]);
    }
    let n = o.count;
    o.finish();
    println!("{}: {} records", path, n);

    // ref_plonk_v1.bin: 9 TRANSCRIPT, 10 PLONK
    let path = std::env::args().nth(2).unwrap_or_else(|| "ref_plonk_v1.bin".to_string());
    let mut o = Out { f: File::create(&path).unwrap(), count: 0, body: vec![] };
    transcript_record(&mut o, &[0, 1, 32, 97], &[1, 32, 64]);
    transcript_record(&mut o, &[165, 166, 167, 500], &[1, 2, 63, 64, 65, 165, 166, 167, 200]);
    transcript_record(&mut o, &(0..170).collect::<Vec<_>>(), &[3]);
    plonk_record(&mut o);
    let n = o.count;
    o.finish();
    println!("{}: {} records", path, n);
}
