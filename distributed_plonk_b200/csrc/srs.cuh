// KZG powers of tau on the device: out[i] = tau^i * G1, the SRS of jf-plonk's PlonkKzgSnark::universal_setup
// (dispatcher2.rs:1279) without its G2 half.
//
//   srs_multiples_kernel M[q][k] = k * P_q, k < 2^(c/2), of the points P_2w = 2^(c*w) * G and P_2w+1 = 2^(c*w + c/2) * G
//                      the host computes (248 doublings of G in all); one thread per entry: <= c/2 doublings and additions
//   srs_table_kernel   T[w][j] = (j + 1) * 2^(c*w) * G, j < 2^(c-1), as M[2w][(j+1) mod 2^(c/2)] + M[2w+1][(j+1) >> c/2]: one
//                      mixed addition per entry, 16 entries per thread normalised with one inversion
//   srs_powers_kernel  one thread per point: tau^i = A[i mod 2^h] * B[i >> h] (the two-factor power tables), canonical,
//                      recoded into signed c-bit digits (for_each_digit, msm.cuh), one mixed XYZZ addition of +-T[w][|d|-1]
//                      per non-zero digit: ceil(256/c) additions, no doublings
// The other two end in srs_block_to_affine: one field inversion per block of AFF_TPB points (Montgomery's trick over a
// product tree in shared memory), so no point ever leaves the block in XYZZ form and the kernels need no scratch.
#pragma once
#include "msm.cuh"
#include "pairing.cuh"

namespace dp {

// window width of the fixed-base table: 16 additions per point from a 48 MiB table gathered from HBM and L2 (c = 8: 32
// additions from a 384 KiB table that stays in L2 took 1.9x as long on the H100, DESIGN.md section 3.7)
constexpr uint32_t SRS_C = 16;
constexpr uint32_t SRS_WINDOWS = (256 + SRS_C - 1) / SRS_C;
constexpr uint32_t SRS_ROW = 1u << (SRS_C - 1);            // entries per window: digit magnitudes 1 .. 2^(c-1)
constexpr uint32_t SRS_HALF = SRS_C / 2;                    // bits of a digit magnitude per multiples table
constexpr uint32_t SRS_MULTIPLES = 2 * SRS_WINDOWS << SRS_HALF;
constexpr uint32_t SRS_TABLE_GROUP = 16;                    // table entries per thread of srs_table_kernel
static_assert((SRS_ROW % SRS_TABLE_GROUP) == 0, "the table is a whole number of groups");
constexpr uint64_t SRS_CHUNK = (uint64_t)1 << 20;           // points per launch (104 MiB of staging for the output)

// The affine form of each thread's point, with one inversion of the product of the block's zz * zzz.  Every thread of the
// block calls it (blockDim.x == AFF_TPB); a thread without a point passes infinity, which contributes a factor 1.
DP_D G1Affine srs_block_to_affine(const G1XYZZ &p, Fq *tree) {
    const uint32_t t = threadIdx.x;
    aff_tree_up(tree, p.is_inf() ? Fq::one() : p.zz * p.zzz);
    if (t == 0) tree[1] = tree[1].inverse_vartime();  // the points have order r: no factor is zero
    __syncthreads();
    for (uint32_t w = 1; w < AFF_TPB; w <<= 1) {  // push the inverse down: each child gets 1 / (its subtree's product)
        if (t < w) {
            const uint32_t node = w + t;
            const Fq iv = tree[node], l = tree[2 * node], r = tree[2 * node + 1];
            tree[2 * node] = iv * r;
            tree[2 * node + 1] = iv * l;
        }
        __syncthreads();
    }
    if (p.is_inf()) return G1Affine::inf();
    const Fq inv = tree[AFF_TPB + t];
    return G1Affine{p.x * (inv * p.zzz), p.y * (inv * p.zz)};
}

__global__ void __launch_bounds__(AFF_TPB) srs_multiples_kernel(const G1Affine *base, G1Affine *mult) {
    __shared__ Fq tree[2 * AFF_TPB];
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    G1XYZZ acc = G1XYZZ::inf();
    const uint32_t k = e & ((1u << SRS_HALF) - 1);
    if (e < SRS_MULTIPLES && k) {
        const G1Affine b = base[e >> SRS_HALF];
        for (int bit = 31 - __clz((int)k); bit >= 0; bit--) {
            acc = acc.dbl();
            if ((k >> bit) & 1) acc = acc.add_mixed(b);
        }
    }
    const G1Affine a = srs_block_to_affine(acc, tree);
    if (e < SRS_MULTIPLES) mult[e] = a;
}

// T[w][j] = M[2w][k mod 2^(c/2)] + M[2w+1][k >> c/2], k = j + 1 <= 2^(c-1) (so k >> c/2 < 2^(c/2)); never infinity
DP_D G1XYZZ srs_table_entry(const G1Affine *mult, uint32_t e) {
    const uint32_t w = e / SRS_ROW, k = e % SRS_ROW + 1;
    const G1Affine *m = mult + ((2 * w) << SRS_HALF);
    const G1Affine lo = load_affine(m + (k & ((1u << SRS_HALF) - 1))), hi = load_affine(m + (1u << SRS_HALF) + (k >> SRS_HALF));
    return G1XYZZ::from_affine(lo).add_mixed(hi);
}

// SRS_TABLE_GROUP consecutive entries per thread, normalised with one inversion (Montgomery's trick; the prefix products
// wait in the x slots of the output, and the second pass recomputes each entry's single addition): no block barriers
__global__ void __launch_bounds__(128) srs_table_kernel(const G1Affine *mult, G1Affine *table) {
    const uint32_t e0 = (blockIdx.x * blockDim.x + threadIdx.x) * SRS_TABLE_GROUP;
    if (e0 >= SRS_WINDOWS * SRS_ROW) return;
    Fq run = Fq::one();
    for (uint32_t k = 0; k < SRS_TABLE_GROUP; k++) {
        const G1XYZZ p = srs_table_entry(mult, e0 + k);
        store_fq(&table[e0 + k].x, run);
        run = run * (p.zz * p.zzz);
    }
    Fq inv = run.inverse_vartime();
    for (int k = SRS_TABLE_GROUP - 1; k >= 0; k--) {
        const G1XYZZ p = srs_table_entry(mult, e0 + k);
        const Fq t = inv * load_fq(&table[e0 + k].x);
        inv = inv * (p.zz * p.zzz);
        table[e0 + k] = G1Affine{p.x * (t * p.zzz), p.y * (t * p.zz)};
    }
}

// points [first, end) of the SRS, written as raw ark GroupAffine (104 B) to ark_out[(i - first) * 13]
__global__ void __launch_bounds__(AFF_TPB) srs_powers_kernel(const Fr *pow_a, const Fr *pow_b, uint32_t log_a, uint64_t first,
                                                             uint64_t end, MsmGeom g, const G1Affine *table, uint64_t *ark_out) {
    __shared__ Fq tree[2 * AFF_TPB];
    const uint64_t i = first + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    G1XYZZ acc = G1XYZZ::inf();
    if (i < end) {
        const Fr s = (pow_a[i & (((uint64_t)1 << log_a) - 1)] * pow_b[i >> log_a]).from_mont();
        Scalar256 sc;
#pragma unroll
        for (int k = 0; k < 8; k++) sc.w[k] = s.l[k];
        // s < r < 2^255: the top digit never carries out
        for_each_digit(sc, g, [&](uint32_t w, uint32_t key, uint32_t neg) {
            G1Affine q = load_affine(table + w * SRS_ROW + key);
            if (neg) q = q.neg();
            acc = acc.add_mixed(q);
        });
    }
    const G1Affine a = srs_block_to_affine(acc, tree);
    if (i >= end) return;
    uint64_t *dst = ark_out + (i - first) * 13;
#pragma unroll
    for (int k = 0; k < 6; k++) {
        dst[k] = (uint64_t)a.x.l[2 * k] | ((uint64_t)a.x.l[2 * k + 1] << 32);
        dst[6 + k] = (uint64_t)a.y.l[2 * k] | ((uint64_t)a.y.l[2 * k + 1] << 32);
    }
    dst[12] = 0;  // infinity flag + padding
}

// ---- one contribution to a powers-of-tau ceremony (DESIGN.md section 3.10): Q_i = s^i P_i over the resident bases
// The endomorphism phi(x, y) = (beta x, y) of G1 acts on the r-torsion as multiplication by lambda = x^2 - 1 (x the
// curve parameter), and r = lambda^2 + lambda + 1, so every canonical k < r is k1 + lambda k2 with k2 = floor(k / lambda)
// <= lambda + 1 < 2^128 and k1 < lambda: k P = k1 P + k2 phi(P) is 128 joint doublings instead of 255.
DP_HD constexpr uint32_t glv_lambda(int i) {  // lambda = 0xac45a4010001a40200000000ffffffff, little-endian limbs
    constexpr uint32_t m[4] = {0xffffffffu, 0x00000000u, 0x0001a402u, 0xac45a401u};
    return m[i];
}
DP_HD Fq glv_beta() {  // the cube root of unity in Fq with phi = lambda on G1 (canonical, converted to Montgomery form)
    const uint32_t b[12] = {0x0000aaacu, 0x8bfd0000u, 0x4f49fffdu, 0x409427ebu, 0x0fb85f9bu, 0x897d2965u,
                            0x89759ad4u, 0xaa0d857du, 0x63d4de85u, 0xec024086u, 0x397fe699u, 0x1a0111eau};
    Fq z;
#pragma unroll
    for (int k = 0; k < 12; k++) z.l[k] = b[k];
    return z.to_mont();
}

// k (8 limbs, canonical) -> k1, k2 (4 limbs each) with k = k1 + lambda k2, by restoring division: 255 shift-subtract steps
DP_D void glv_split(const uint32_t *k, uint32_t *k1, uint32_t *k2) {
    uint32_t rem[5] = {0, 0, 0, 0, 0};  // < 2 lambda < 2^129 before each subtraction
#pragma unroll
    for (int w = 0; w < 4; w++) k2[w] = 0;
    for (int bit = 254; bit >= 0; bit--) {
#pragma unroll
        for (int w = 4; w > 0; w--) rem[w] = (rem[w] << 1) | (rem[w - 1] >> 31);
        rem[0] = (rem[0] << 1) | ((k[bit >> 5] >> (bit & 31)) & 1);
        bool ge = rem[4] != 0, decided = ge;
#pragma unroll
        for (int w = 3; w >= 0; w--)
            if (!decided && rem[w] != glv_lambda(w)) {
                ge = rem[w] > glv_lambda(w);
                decided = true;
            }
        if (!decided) ge = true;  // equal
        if (ge) {
            uint32_t borrow = 0;
#pragma unroll
            for (int w = 0; w < 5; w++) {
                const uint64_t d = (uint64_t)rem[w] - (w < 4 ? glv_lambda(w) : 0u) - borrow;
                rem[w] = (uint32_t)d;
                borrow = (uint32_t)(d >> 63);
            }
            if (bit < 128) k2[bit >> 5] |= 1u << (bit & 31);  // the quotient is below 2^128
        }
    }
    for (int w = 0; w < 4; w++) k1[w] = rem[w];
}

// Points [first, end) of the update, as 48-byte compressed points at out48[(i - first) * 12].  s^i = A[i mod 2^h] B[i >> h],
// as in srs_powers_kernel.  GLV: the joint double-and-add of k1 on P and k2 on phi(P), whose third addend P + phi(P) is
// normalised per block (srs_block_to_affine), so every addition is mixed.  !GLV: the plain 255-bit double-and-add of
// g1_decompress_kernel's subgroup check, kept as the reference the GLV kernel was measured and tested against.  The bases
// must lie in the r-torsion (dp_init_compressed and load_srs check it): only there is phi(P) = lambda P.
template <bool GLV>
__global__ void __launch_bounds__(AFF_TPB) srs_update_kernel(const G1Affine *bases, const Fr *pow_a, const Fr *pow_b, uint32_t log_a,
                                                             uint64_t first, uint64_t end, Fq beta, uint32_t *out48) {
    __shared__ Fq tree[2 * AFF_TPB];
    const uint64_t i = first + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    G1XYZZ acc = G1XYZZ::inf();
    G1Affine p = G1Affine::inf();
    uint32_t k[8] = {};
    if (i < end) {
        const Fr s = (pow_a[i & (((uint64_t)1 << log_a) - 1)] * pow_b[i >> log_a]).from_mont();
        for (int w = 0; w < 8; w++) k[w] = s.l[w];
        p = load_affine(bases + i);
    }
    if constexpr (GLV) {
        const G1Affine phi = p.is_inf() ? p : G1Affine{p.x * beta, p.y};
        const G1Affine both = srs_block_to_affine(G1XYZZ::from_affine(p).add_mixed(phi), tree);
        __syncthreads();  // the tree is reused below
        if (i < end) {
            uint32_t k1[4], k2[4];
            glv_split(k, k1, k2);
            for (int bit = 127; bit >= 0; bit--) {
                acc = acc.dbl();
                const uint32_t sel = ((k1[bit >> 5] >> (bit & 31)) & 1) | (((k2[bit >> 5] >> (bit & 31)) & 1) << 1);
                if (sel) acc = acc.add_mixed(sel == 1 ? p : sel == 2 ? phi : both);
            }
        }
    } else {
        if (i < end)
            for (int w = 7; w >= 0; w--)
                for (int b = 31; b >= 0; b--) {
                    acc = acc.dbl();
                    if ((k[w] >> b) & 1) acc = acc.add_mixed(p);
                }
    }
    const G1Affine a = srs_block_to_affine(acc, tree);
    if (i < end) g1_compress_store(a, out48 + (i - first) * 12);
}

// The G2 half of the update: out[t] = s q_t for the raw 200-byte points in[0] = h, in[1] = beta h, one thread each, with
// the input checks of pairing_check_pair (*bad = min((t + 1) << 8 | why)).  s is read from the device power table
// (pow_a[1] = s, Montgomery form), so it never travels as a kernel parameter.
__global__ void __launch_bounds__(32) srs_update_g2_kernel(const Fr *pow_a, const uint64_t *in, uint64_t *out, unsigned long long *bad) {
    const uint32_t t = threadIdx.x;
    if (t >= 2) return;
    const G2Affine q = load_g2_ark(in + 25 * t);
    uint32_t why = 0;
    if (!q.inf) {
        uint32_t r[8];
#pragma unroll
        for (int k = 0; k < 8; k++) r[k] = FrParams::mod(k);
        if (!q.x.c0.canon_is_reduced() || !q.x.c1.canon_is_reduced() || !q.y.c0.canon_is_reduced() || !q.y.c1.canon_is_reduced())
            why = PAIR_G2_NOT_FQ;
        else if (!q.on_twist())
            why = PAIR_G2_OFF_TWIST;
        else if (!g2_mul(q, r).is_inf())
            why = PAIR_G2_NOT_TORSION;
    }
    if (why) {
        atomicMin(bad, ((unsigned long long)(t + 1) << 8) | why);
        return;
    }
    const Fr s = pow_a[1].from_mont();
    store_g2_ark(out + 25 * t, g2_mul(q, s.l).to_affine());
}

}  // namespace dp
