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

}  // namespace dp
