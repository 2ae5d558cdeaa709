// Pippenger-bucket multi-scalar multiplication over BLS12-381 G1 for sm_90a.
//
// Replaces ark-ec 0.3.0 VariableBaseMSM::multi_scalar_mul as called by the reference worker
// (src/worker.rs:117-123 commit_polynomial, 159-185 var_msm; twin call sites
// src/dispatcher.rs:1042-1060, src/dispatcher2.rs:834-843).  Same function (sum_i s_i * P_i over
// canonical 256-bit scalars and affine bases, zero scalars and infinity bases contribute nothing),
// different schedule - chosen for a GPU, which is legal because the result is a unique group
// element (SURVEY.md §8c):
//
//   1. msm_count      signed-digit recode (digits in [-2^(c-1), 2^(c-1)]), histogram of
//                     (window, |digit|) keys with L2 atomics; 128-bit coalesced scalar loads
//   2. scan (3 kernels) exclusive prefix sums -> bucket offsets
//   3. msm_scatter    counting-sort the point indices by key (sign kept in bit 31)
//   4. msm_accumulate one thread per CHUNK of 64 sorted digits (chunks ignore bucket boundaries, so
//                     every lane does the same number of additions whatever the scalars look
//                     like): XYZZ accumulator in registers, mixed additions of the gathered affine
//                     bases (96 B = 6 x 128-bit loads each), one partial sum per bucket touched
//   5. msm_collapse   buckets spread over many chunks (witness vectors are full of 0/1/small
//                     values): one warp per bucket, lanes stride over its partial sums,
//                     warp-shuffle butterfly reduction
//   6. msm_reduce     per window, per segment of buckets: running-sum reduction
//                     sum_k k*B_k (+ small scalar multiple for the segment offset)
//   7. msm_window_sum block per window: tree reduction of the segment sums
//   8. msm_final      Horner over windows (c doublings each), normalise, emit 144-byte Jacobian
// With the precomputed table of window multiples (built at dp_init, msm_precompute_kernel) steps
// 1-7 run over ONE shared bucket set and step 8 has nothing to combine.
//
// Work: N*ceil(256/c) mixed additions (10 Fq mul) dominate; HBM traffic is ~96 B gathered per
// addition plus 32 B per scalar per pass - the kernel set is bound by the INT32 multiply pipe,
// not by HBM (DESIGN.md).
#pragma once
#include "g1.cuh"
#include "rt.cuh"

namespace dp {

constexpr uint32_t MSM_CHUNK = 64;      // sorted digits per accumulate thread (chunks ignore bucket boundaries)
constexpr uint32_t MSM_BIG_SPAN = 8;    // buckets spread over more chunks than this are folded by a warp first
constexpr uint32_t MSM_SEG = 16;        // buckets per reduce segment
constexpr int MSM_TPB = 128;

constexpr uint32_t MSM_SLICES = 32;     // partial sums per window in the two-level window sum

struct MsmGeom {
    uint32_t c;            // window bits
    uint32_t n_windows;    // digit windows = ceil(256 / c)
    uint32_t bpw;          // buckets per window = 2^(c-1)
    uint32_t n_keys;       // bucket sets * bpw
    uint32_t seg;          // buckets per reduce segment
    uint32_t segs_per_window;
    uint32_t red_windows;  // bucket sets to reduce: n_windows, or 1 with precomputed window multiples
    uint32_t pre;          // 1: bases come from the table T[w][i] = 2^(c*w) * P_i, one shared bucket set
    uint32_t stride;       // table row length (points)
    uint32_t slices;       // partial sums per bucket set in the two-level window sum (<= 32)
    uint32_t chunk;        // sorted digits per accumulate thread
};

// cost in Fq multiplications of an n-point MSM with window c
inline double msm_cost(uint64_t n, uint32_t c, bool pre) {
    const double w = (double)((256 + c - 1) / c), buckets = (double)(1u << (c - 1)) * (pre ? 1.0 : w);
    // n*W mixed adds (10) + 2 full adds (14) per bucket, the latter at much lower parallelism (x2);
    // without precomputation also 256 serial doublings at single-thread speed (~ x400)
    return (double)n * w * 10.0 + 2.0 * 2.0 * buckets * 14.0 + (pre ? 0.0 : 256.0 * 9.0 * 400.0);
}

inline MsmGeom msm_make_geom(uint32_t c, bool pre, uint64_t stride) {
    MsmGeom g;
    g.c = c;
    g.n_windows = (256 + c - 1) / c;
    g.bpw = 1u << (c - 1);
    g.pre = pre ? 1 : 0;
    g.stride = (uint32_t)stride;
    g.red_windows = pre ? 1 : g.n_windows;
    g.n_keys = g.red_windows * g.bpw;
    // buckets per reduce thread: 16 while the bucket set is large (throughput-bound: 3.4 point operations per bucket);
    // small sets - a worker's shard of a multi-GPU MSM gets a narrower window - are latency-bound (a thread's chain of
    // 2*seg additions + a ~1.5*log2(buckets/seg)-step scalar multiple), so
    // they get more, shorter threads
    uint32_t seg = g.bpw >= (1u << 18) ? 16 : g.bpw >= (1u << 17) ? 8 : g.bpw >= (1u << 16) ? 4 : 2;
    if (seg > MSM_SEG) seg = MSM_SEG;
    g.seg = g.bpw < seg ? g.bpw : seg;
    g.segs_per_window = g.bpw / g.seg;
    g.slices = g.segs_per_window / 64;  // >= 64 segment sums per slice block
    if (g.slices < 1) g.slices = 1;
    if (g.slices > MSM_SLICES) g.slices = MSM_SLICES;
    g.chunk = MSM_CHUNK;
    return g;
}

inline MsmGeom msm_geometry(uint64_t n, int force_c = 0) {
    uint32_t best_c = 4;
    double best = 1e300;
    for (uint32_t c = 4; c <= 18; c++) {
        const double cost = msm_cost(n, c, false);
        if (cost < best) {
            best = cost;
            best_c = c;
        }
    }
    return msm_make_geom(force_c ? (uint32_t)force_c : best_c, false, 0);
}

// window width for the precomputed table of an n-base context, limited by the table size
inline uint32_t msm_pick_pre_c(uint64_t n_bases, uint64_t max_table_bytes) {
    uint32_t best_c = 0;
    double best = 1e300;
    for (uint32_t c = 8; c <= 22; c++) {
        const uint64_t w = (256 + c - 1) / c;
        if (w * n_bases * 96ull > max_table_bytes || w * n_bases >= (1ull << 31)) continue;
        const double cost = msm_cost(n_bases, c, true);
        if (cost < best) {
            best = cost;
            best_c = c;
        }
    }
    return best_c;
}

// ------------------------------------------------------------------ bases import (init time)
// raw ark GroupAffine<G1> (104 B: x@0, y@48 Fq Montgomery, infinity flag @96; utils.rs:27-43)
// -> device affine (96 B, infinity = (0,0))
__global__ void g1_import_ark_kernel(const uint64_t *ark, G1Affine *out, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t *src = ark + i * 13;  // 104 B = 13 u64
    G1Affine p;
    const bool inf = (src[12] & 0xff) != 0;
#pragma unroll
    for (int k = 0; k < 6; k++) {
        uint64_t a = inf ? 0 : src[k], b = inf ? 0 : src[6 + k];
        p.x.l[2 * k] = (uint32_t)a;
        p.x.l[2 * k + 1] = (uint32_t)(a >> 32);
        p.y.l[2 * k] = (uint32_t)b;
        p.y.l[2 * k + 1] = (uint32_t)(b >> 32);
    }
    out[i] = p;
}

// device affine -> raw ark GroupAffine (104 B; identity = (0, 1, true) like GroupAffine::zero())
__global__ void g1_export_ark_kernel(const G1Affine *in, uint64_t *ark, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    G1Affine p = in[i];
    const bool inf = p.is_inf();
    if (inf) p.y = Fq::one();
    uint64_t *dst = ark + i * 13;
#pragma unroll
    for (int k = 0; k < 6; k++) {
        dst[k] = (uint64_t)p.x.l[2 * k] | ((uint64_t)p.x.l[2 * k + 1] << 32);
        dst[6 + k] = (uint64_t)p.y.l[2 * k] | ((uint64_t)p.y.l[2 * k + 1] << 32);
    }
    dst[12] = inf ? 1 : 0;
}

// Canonical SRS ingest ("next" row 4 of SURVEY.md 8f): ark-serialize 0.3.0 compressed GroupAffine,
// 48 B per point = canonical x little-endian, bit 7 of the last byte = (y > -y), bit 6 = infinity.
// One thread per point: y = (x^3 + 4)^((p+1)/4) (p = 3 mod 4), the root whose order matches the flag;
// optional r-torsion check by double-and-add with the scalar r.  *err = 1 + index of the first
// rejected point, err[1] = why (1 x >= p, 2 both flags, 3 not on the curve, 4 not in the subgroup).
__global__ void __launch_bounds__(128) g1_decompress_kernel(const uint32_t *in, G1Affine *out, uint64_t n, uint32_t check_subgroup,
                                                            unsigned long long *err) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fq xc;
#pragma unroll
    for (int k = 0; k < 12; k++) xc.l[k] = in[i * 12 + k];
    const bool positive = (xc.l[11] >> 31) & 1, infinity = (xc.l[11] >> 30) & 1;
    xc.l[11] &= 0x3fffffffu;
    uint32_t why = 0;
    G1Affine p = G1Affine::inf();
    if (positive && infinity) {
        why = 2;
    } else if (!infinity) {
        if (!xc.canon_is_reduced()) {
            why = 1;
        } else {
            const Fq x = xc.to_mont();
            const Fq rhs = x.sqr() * x + fq_from_u32(4);
            uint32_t e[12];  // (p + 1) / 4: the low limb ...aaab + 1 does not carry
#pragma unroll
            for (int k = 0; k < 12; k++) e[k] = FqParams::mod(k);
            e[0] += 1;
#pragma unroll
            for (int k = 0; k < 12; k++) e[k] = (e[k] >> 2) | (k < 11 ? e[k + 1] << 30 : 0);
            Fq y = rhs.pow_limbs(e, 12);
            if (y.sqr() != rhs) {
                why = 3;
            } else {
                const Fq ny = y.neg();
                const bool y_is_larger = Fq::canon_gt(y.from_mont(), ny.from_mont());
                p = G1Affine{x, y_is_larger == positive ? y : ny};
                if (check_subgroup) {
                    G1XYZZ acc = G1XYZZ::inf();
                    for (int k = 7; k >= 0; k--)
                        for (int b = 31; b >= 0; b--) {
                            acc = acc.dbl();
                            if ((FrParams::mod(k) >> b) & 1) acc = acc.add_mixed(p);
                        }
                    if (!acc.is_inf()) why = 4;
                }
            }
        }
    }
    if (why) {
        const unsigned long long mine = ((unsigned long long)(i + 1) << 8) | why;
        atomicMin(err, mine);
        p = G1Affine::inf();
    }
    out[i] = p;
}

// The inverse of g1_decompress_kernel: device affine -> the 48 compressed bytes (12 u32).  Two Montgomery reductions
// per point (x and y leave Montgomery form; -y is then p - y on the canonical integer), so 96 or 104 B read and 48 B
// written per point against ~300 multiply-adds: the kernels below are meant to run at the speed of their memory traffic.
DP_D void g1_compress_store(const G1Affine &p, uint32_t *out) {
    Fq x = Fq::zero();
    uint32_t flags = 1u << 30;
    if (!p.is_inf()) {
        x = p.x.from_mont();
        const Fq y = p.y.from_mont();
        flags = Fq::canon_gt(y, y.neg()) ? 1u << 31 : 0u;
    }
#pragma unroll
    for (int k = 0; k < 12; k++) out[k] = x.l[k] | (k == 11 ? flags : 0u);
}
// from the context's resident bases (96 B each)
__global__ void __launch_bounds__(256) g1_compress_kernel(const G1Affine *in, uint32_t *out, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) g1_compress_store(in[i], out + i * 12);
}
// from raw ark GroupAffine structs (104 B each, the layout g1_import_ark_kernel reads; not validated)
__global__ void __launch_bounds__(256) g1_compress_ark_kernel(const uint64_t *ark, uint32_t *out, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t *src = ark + i * 13;
    G1Affine p = G1Affine::inf();
    if ((src[12] & 0xff) == 0) {
#pragma unroll
        for (int k = 0; k < 6; k++) {
            p.x.l[2 * k] = (uint32_t)src[k];
            p.x.l[2 * k + 1] = (uint32_t)(src[k] >> 32);
            p.y.l[2 * k] = (uint32_t)src[6 + k];
            p.y.l[2 * k + 1] = (uint32_t)(src[6 + k] >> 32);
        }
    }
    g1_compress_store(p, out + i * 12);
}

// The random scalars of dp_srs_check: rho_i = 128 bits, words 4 (i mod 4) .. 4 (i mod 4) + 3 (little-endian) of the
// ChaCha20 block (RFC 8439 section 2.3) with the 256-bit key `key`, block counter i div 4 and an all-zero nonce.
DP_D void chacha20_block(const uint32_t *key, uint32_t counter, uint32_t *out) {
    uint32_t s[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key[0], key[1], key[2], key[3],
                      key[4],      key[5],      key[6],      key[7],      counter, 0u,     0u,     0u};
    uint32_t x[16];
#pragma unroll
    for (int k = 0; k < 16; k++) x[k] = s[k];
    auto rotl = [](uint32_t v, int c) { return (v << c) | (v >> (32 - c)); };
    auto quarter = [&](int a, int b, int c, int d) {
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 16);
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 12);
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 8);
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 7);
    };
    for (int round = 0; round < 10; round++) {
        quarter(0, 4, 8, 12); quarter(1, 5, 9, 13); quarter(2, 6, 10, 14); quarter(3, 7, 11, 15);
        quarter(0, 5, 10, 15); quarter(1, 6, 11, 12); quarter(2, 7, 8, 13); quarter(3, 4, 9, 14);
    }
#pragma unroll
    for (int k = 0; k < 16; k++) out[k] = x[k] + s[k];
}
struct ChaChaKey {
    uint32_t w[8];
};
// One thread per block = four scalars.  a[i] = rho_i and b[i + 1] = rho_i for i < n - 1, a[n - 1] = b[0] = 0: canonical
// 256-bit MSM scalars (two uint4 each), so that sum a[i] P_i and sum b[i] P_i pair rho_i with P_i and with P_(i+1).
__global__ void __launch_bounds__(128) srs_check_scalars_kernel(ChaChaKey key, uint64_t n, uint4 *a, uint4 *b) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint4 zero = make_uint4(0, 0, 0, 0);
    if (t == 0) {
        a[2 * (n - 1)] = a[2 * (n - 1) + 1] = zero;
        b[0] = b[1] = zero;
    }
    if (4 * t >= n - 1) return;
    uint32_t ks[16];
    chacha20_block(key.w, (uint32_t)t, ks);
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const uint64_t i = 4 * t + j;
        if (i >= n - 1) break;
        const uint4 rho = make_uint4(ks[4 * j], ks[4 * j + 1], ks[4 * j + 2], ks[4 * j + 3]);
        a[2 * i] = rho;
        a[2 * i + 1] = zero;
        b[2 * (i + 1)] = rho;
        b[2 * (i + 1) + 1] = zero;
    }
}

// Synthetic SRS for benchmarks / tests: out[i] = k_i * G with k_i = SplitMix64(seed, i) (64-bit,
// distinct points), written in the raw ark GroupAffine layout (104 B) that dp_init ingests.
DP_HD G1Affine g1_generator() {
    const uint32_t gx[12] = {0xfd530c16u, 0x5cb38790u, 0x9976fff5u, 0x7817fc67u, 0x143ba1c1u, 0x154f95c7u,
                             0xf3d0e747u, 0xf0ae6acdu, 0x21dbf440u, 0xedce6eccu, 0x9e0bfb75u, 0x12017741u};
    const uint32_t gy[12] = {0x0ce72271u, 0xbaac93d5u, 0x7918fd8eu, 0x8c22631au, 0x570725ceu, 0xdd595f13u,
                             0x50405194u, 0x51ac5829u, 0xad0059c0u, 0x0e1c8c3fu, 0x5008a26au, 0x0bbc3efcu};
    G1Affine g;
    for (int i = 0; i < 12; i++) {
        g.x.l[i] = gx[i];
        g.y.l[i] = gy[i];
    }
    return g;
}
__global__ void g1_gen_bases_kernel(uint64_t *ark_out, uint64_t n, uint64_t seed) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t z = seed + (i + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    z |= 1;
    const G1Affine g = g1_generator();
    G1XYZZ acc = G1XYZZ::inf();
    for (int b = 63; b >= 0; b--) {
        acc = acc.dbl();
        if ((z >> b) & 1) acc = acc.add_mixed(g);
    }
    const G1Affine a = acc.to_affine();
    uint64_t *dst = ark_out + i * 13;
    for (int k = 0; k < 6; k++) {
        dst[k] = (uint64_t)a.x.l[2 * k] | ((uint64_t)a.x.l[2 * k + 1] << 32);
        dst[6 + k] = (uint64_t)a.y.l[2 * k] | ((uint64_t)a.y.l[2 * k + 1] << 32);
    }
    dst[12] = 0;  // infinity flag + padding
}

// ------------------------------------------------------------------ digit recode
struct Scalar256 {
    uint32_t w[8];
};
DP_D Scalar256 load_scalar(const uint4 *scalars, uint64_t i) {
    const uint4 a = scalars[2 * i], b = scalars[2 * i + 1];
    Scalar256 s;
    s.w[0] = a.x; s.w[1] = a.y; s.w[2] = a.z; s.w[3] = a.w;
    s.w[4] = b.x; s.w[5] = b.y; s.w[6] = b.z; s.w[7] = b.w;
    return s;
}
// c raw bits of the scalar starting at bit position `pos`
DP_D uint32_t scalar_bits(const Scalar256 &s, uint32_t pos, uint32_t c) {
    const uint32_t word = pos >> 5, sh = pos & 31;
    if (word >= 8) return 0;
    uint32_t v = s.w[word] >> sh;
    if (sh && word + 1 < 8) v |= s.w[word + 1] << (32 - sh);
    return v & ((1u << c) - 1);
}

// Calls f(window, key, negative) for every non-zero signed digit; returns the carry out of the top
// window (non-zero only for scalars >= 2^255 or so: not canonical Fr, reported as DP_E_ARG).
template <class F>
DP_D uint32_t for_each_digit(const Scalar256 &s, const MsmGeom &g, F f) {
    uint32_t carry = 0;
    for (uint32_t w = 0; w < g.n_windows; w++) {
        uint32_t raw = scalar_bits(s, w * g.c, g.c) + carry;
        carry = 0;
        const uint32_t set = g.pre ? 0u : w * g.bpw;
        if (raw > g.bpw) {  // digit = raw - 2^c  (negative)
            const uint32_t mag = (1u << g.c) - raw;
            carry = 1;
            if (mag) f(w, set + (mag - 1), 1u);
        } else if (raw) {
            f(w, set + (raw - 1), 0u);
        }
    }
    return carry;
}

__global__ void msm_count_kernel(const uint4 *scalars, uint64_t n, MsmGeom g, uint32_t *counts, uint32_t *err) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Scalar256 s = load_scalar(scalars, i);
    const uint32_t carry = for_each_digit(s, g, [&](uint32_t, uint32_t key, uint32_t) { atomicAdd(&counts[key], 1u); });
    if (carry) atomicOr(err, 1u);
}

__global__ void msm_scatter_kernel(const uint4 *scalars, uint64_t n, MsmGeom g, uint32_t *cursor, uint32_t *sorted) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Scalar256 s = load_scalar(scalars, i);
    for_each_digit(s, g, [&](uint32_t w, uint32_t key, uint32_t neg) {
        const uint32_t pos = atomicAdd(&cursor[key], 1u);
        sorted[pos] = ((uint32_t)i + (g.pre ? w * g.stride : 0u)) | (neg << 31);
    });
}

// ------------------------------------------------------------------ exclusive scan (3 phases)
// offsets[i] = sum_{k<i} counts[k]  (bucket start in sorted[]) for i <= n; offsets[n] = number of digits
constexpr int SCAN_TPB = 256;
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_BLOCK = SCAN_TPB * SCAN_ITEMS;

// block-wide exclusive scan of one value per thread (Hillis-Steele in shared memory); returns the
// exclusive prefix of this thread and the block total
DP_D uint32_t block_exclusive_scan(uint32_t v, uint32_t *sh, uint32_t &total) {
    const uint32_t tid = threadIdx.x, nt = blockDim.x;
    sh[tid] = v;
    __syncthreads();
    for (uint32_t off = 1; off < nt; off <<= 1) {
        uint32_t add = tid >= off ? sh[tid - off] : 0;
        __syncthreads();
        sh[tid] += add;
        __syncthreads();
    }
    total = sh[nt - 1];
    const uint32_t excl = tid ? sh[tid - 1] : 0;
    __syncthreads();
    return excl;
}

__global__ void __launch_bounds__(SCAN_TPB) scan_block_sums_kernel(const uint32_t *counts, uint32_t n, uint32_t *block_sums) {
    __shared__ uint32_t sh[SCAN_TPB];
    const uint32_t base = blockIdx.x * SCAN_BLOCK + threadIdx.x * SCAN_ITEMS;
    uint32_t a = 0;
    for (int k = 0; k < SCAN_ITEMS; k++)
        if (base + k < n) a += counts[base + k];
    uint32_t ta;
    block_exclusive_scan(a, sh, ta);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = ta;
}

// single block: exclusive scan of the per-block sums in place; grand total -> offsets[n]
__global__ void __launch_bounds__(SCAN_TPB) scan_block_offsets_kernel(uint32_t *block_sums, uint32_t n_blocks, uint32_t *offsets,
                                                                       uint32_t n) {
    __shared__ uint32_t sh[SCAN_TPB];
    uint32_t run = 0;
    for (uint32_t base = 0; base < n_blocks; base += SCAN_TPB) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < n_blocks ? block_sums[i] : 0;
        uint32_t total;
        const uint32_t e = block_exclusive_scan(v, sh, total);
        if (i < n_blocks) block_sums[i] = run + e;
        run += total;
    }
    if (threadIdx.x == 0) offsets[n] = run;
}

__global__ void __launch_bounds__(SCAN_TPB) scan_write_kernel(const uint32_t *counts, uint32_t n, const uint32_t *block_sums,
                                                               uint32_t *offsets) {
    __shared__ uint32_t sh[SCAN_TPB];
    const uint32_t base = blockIdx.x * SCAN_BLOCK + threadIdx.x * SCAN_ITEMS;
    uint32_t c[SCAN_ITEMS];
    uint32_t a = 0;
    for (int k = 0; k < SCAN_ITEMS; k++) {
        c[k] = base + k < n ? counts[base + k] : 0;
        a += c[k];
    }
    uint32_t total;
    uint32_t e = block_exclusive_scan(a, sh, total) + block_sums[blockIdx.x];
    for (int k = 0; k < SCAN_ITEMS; k++)
        if (base + k < n) {
            offsets[base + k] = e;
            e += c[k];
        }
}

// ------------------------------------------------------------------ chunks
// The sorted digit array is cut into chunks of MSM_CHUNK entries regardless of bucket boundaries, one
// thread per chunk: every thread does the same number of additions (with one thread per bucket
// the Poisson spread of bucket sizes left 18 % of the lanes idle, ncu: 26.1 active threads per
// warp instruction).  A chunk that crosses bucket boundaries emits one partial sum per bucket it
// touches; the partial of (chunk j, bucket b) lives in slot j + b, which is unique and dense along
// the staircase of (chunk, bucket) pairs.  Bucket b therefore owns slots j0+b .. j1+b with
// j0 = offsets[b] / CHUNK, j1 = (offsets[b+1]-1) / CHUNK.
DP_D void bucket_span(const uint32_t *offsets, uint32_t key, uint32_t chunk, uint32_t &j0, uint32_t &j1, bool &empty) {
    const uint32_t lo = offsets[key], hi = offsets[key + 1];
    empty = lo == hi;
    j0 = lo / chunk;
    j1 = empty ? j0 : (hi - 1) / chunk;
}

// buckets spread over many chunks (skewed scalars) are listed for msm_collapse
__global__ void msm_find_big_kernel(const uint32_t *offsets, uint32_t n_keys, uint32_t chunk, uint32_t *multi_keys, uint32_t *n_multi) {
    const uint32_t key = blockIdx.x * blockDim.x + threadIdx.x;
    if (key >= n_keys) return;
    uint32_t j0, j1;
    bool empty;
    bucket_span(offsets, key, chunk, j0, j1, empty);
    if (!empty && j1 - j0 + 1 > MSM_BIG_SPAN) multi_keys[atomicAdd(n_multi, 1u)] = key;
}

DP_D G1Affine load_affine(const G1Affine *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    G1Affine r;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        uint4 a = q[k], b = q[3 + k];
        r.x.l[4 * k] = a.x; r.x.l[4 * k + 1] = a.y; r.x.l[4 * k + 2] = a.z; r.x.l[4 * k + 3] = a.w;
        r.y.l[4 * k] = b.x; r.y.l[4 * k + 1] = b.y; r.y.l[4 * k + 2] = b.z; r.y.l[4 * k + 3] = b.w;
    }
    return r;
}

// MINB: resident blocks per SM the register allocation aims for (3: 152 registers, no spills; 4: 128 registers and a
// few hundred bytes of spills around the outlined multiplications).  The kernel is bound by the dependent carry
// chains of the Fq products (ncu r02a: 52 % of the warp samples are fixed-latency waits at 3 warps per scheduler).
// DIRECT: the points to add are bases[e] themselves, in bucket order (the output of the batched-affine tree levels below)
// instead of bases[sorted[e]] with the sign in bit 31.
template <int MINB, bool DIRECT = false>
__global__ void __launch_bounds__(MSM_TPB, MINB) msm_accumulate_kernel(const uint32_t *offsets, uint32_t n_keys, uint32_t chunk,
                                                                        const uint32_t *sorted, const G1Affine *bases, G1XYZZ *partials) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n_digits = offsets[n_keys];  // the grid is sized for the worst case
    const uint64_t pos0 = (uint64_t)j * chunk;
    if (pos0 >= n_digits) return;
    const uint32_t pos1 = pos0 + chunk < n_digits ? (uint32_t)pos0 + chunk : n_digits;
    // bucket holding the first digit: largest b with offsets[b] <= pos0 (skips empty buckets)
    uint32_t lo = 0, hi = n_keys;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (offsets[mid] <= (uint32_t)pos0) lo = mid; else hi = mid;
    }
    uint32_t b = lo, next = offsets[b + 1];
    G1XYZZ acc = G1XYZZ::inf();
    for (uint32_t e = (uint32_t)pos0; e < pos1; e++) {
        if (e == next) {  // leaving bucket b: emit its partial, move to the bucket that holds digit e
            partials[j + b] = acc;
            acc = G1XYZZ::inf();
            do {
                b++;
                next = offsets[b + 1];
            } while (next == e);
        }
        G1Affine p;
        if (DIRECT) {
            p = load_affine(bases + e);
        } else {
            const uint32_t v = sorted[e];
            p = load_affine(bases + (v & 0x7fffffffu));
            if (v >> 31) p = p.neg();
        }
        acc = acc.add_mixed(p);
    }
    partials[j + b] = acc;
}

// ------------------------------------------------------------------ batched-affine tree levels
// Before the XYZZ chunks, L levels of a pairwise tree inside every bucket: level l replaces the elements (2k, 2k+1) of
// the bucket-ordered sequence by their sum, an AFFINE addition whose field inversion is shared by a whole thread block
// (Montgomery's trick): 6.4 field products per addition at 16 pairs per thread against 10 for the XYZZ mixed addition
// (tools/microbench6.cu times one level of each).  For pairs never to straddle two buckets every bucket's slice of the sorted index
// array is padded to a multiple of 2^L entries (msm_pad_counts_kernel; the holes keep the 0xffffffff the array was
// filled with = the point at infinity), so all levels are plain strided passes and bucket b's survivors sit at
// offsets[b] >> L afterwards.  One level = three kernels:
//   aff_k1  per pair the denominator d (x2 - x1; 2y for a doubling; 1 when a partner is infinity or the sum is), each
//           thread chains the products of its KP pairs (exclusive prefixes -> global), block tree over the thread totals
//   aff_k2  one inversion per block (binary extended Euclid per lane)
//   aff_k3  the tree again, inverses pushed down to the threads, then per pair 1/d = inv_run * prefix, lambda, x3, y3
constexpr int AFF_TPB = 128;
constexpr int AFF_KP = 16;                                  // pairs per thread
constexpr uint32_t AFF_BLOCK_PAIRS = AFF_TPB * AFF_KP;
constexpr uint32_t AFF_HOLE = 0xffffffffu;                  // padding entry of the sorted index array

DP_D Fq load_fq(const Fq *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    Fq r;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const uint4 v = q[k];
        r.l[4 * k] = v.x; r.l[4 * k + 1] = v.y; r.l[4 * k + 2] = v.z; r.l[4 * k + 3] = v.w;
    }
    return r;
}
DP_D void store_fq(Fq *p, const Fq &v) {
    uint4 *q = reinterpret_cast<uint4 *>(p);
#pragma unroll
    for (int k = 0; k < 3; k++) q[k] = make_uint4(v.l[4 * k], v.l[4 * k + 1], v.l[4 * k + 2], v.l[4 * k + 3]);
}

// counts[key] rounded up to a multiple of 2^log_pad (before the scan turns them into offsets)
__global__ void msm_pad_counts_kernel(uint32_t *counts, uint32_t n_keys, uint32_t log_pad) {
    const uint32_t key = blockIdx.x * blockDim.x + threadIdx.x;
    if (key >= n_keys) return;
    const uint32_t m = (1u << log_pad) - 1;
    counts[key] = (counts[key] + m) & ~m;
}
// out[i] = offsets[i] >> shift, i <= n_keys: where the buckets start after `shift` tree levels
__global__ void msm_shift_offsets_kernel(const uint32_t *offsets, uint32_t n_keys, uint32_t shift, uint32_t *out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n_keys) out[i] = offsets[i] >> shift;
}

// where a level reads its operands: GATHER = the window-multiple table through the sorted index array, else the previous level
struct AffSrc {
    const uint32_t *sorted;
    const G1Affine *pts;
};
// element e of the level's input; `hole` = padding entry.  x only: the y coordinate is fetched by aff_y when needed.
template <bool GATHER>
DP_D Fq aff_x(const AffSrc &s, uint64_t e, uint32_t &v, bool &hole) {
    if (GATHER) {
        v = s.sorted[e];
        hole = v == AFF_HOLE;
        return hole ? Fq::zero() : load_fq(&s.pts[v & 0x7fffffffu].x);
    }
    v = 0;
    hole = false;
    return load_fq(&s.pts[e].x);
}
template <bool GATHER>
DP_D Fq aff_y(const AffSrc &s, uint64_t e, uint32_t v, bool hole) {
    if (GATHER) {
        if (hole) return Fq::zero();
        const Fq y = load_fq(&s.pts[v & 0x7fffffffu].y);
        return (v >> 31) && !y.is_zero() ? y.neg() : y;   // (x, 0) only when x = 0 too: infinity stays (0, 0)
    }
    return load_fq(&s.pts[e].y);
}

// What pair k = elements (2k, 2k+1) needs: kind 0 = chord addition (d = x2 - x1), 1 = doubling (d = 2 y1), 2 = the sum is the
// first point, 3 = the second, 4 = infinity (kinds 2-4: d = 1).  d is never zero.  With LAZY the y coordinates are loaded
// only when x1 = x2 or an x is zero (a hole, infinity, or one of the two curve points with x = 0); the classification
// does not depend on LAZY, so aff_k1 (LAZY) and aff_k3 compute the same d for the same pair.
struct AffPair {
    Fq x1, y1, x2, y2, d;
    uint32_t kind;
};
template <bool GATHER, bool LAZY>
DP_D void aff_pair(const AffSrc &s, uint64_t k, AffPair &p) {
    uint32_t v1, v2;
    bool h1, h2;
    p.x1 = aff_x<GATHER>(s, 2 * k, v1, h1);
    p.x2 = aff_x<GATHER>(s, 2 * k + 1, v2, h2);
    const bool plain = !h1 && !h2 && !p.x1.is_zero() && !p.x2.is_zero() && p.x1 != p.x2;
    if (!(LAZY && plain)) {
        p.y1 = aff_y<GATHER>(s, 2 * k, v1, h1);
        p.y2 = aff_y<GATHER>(s, 2 * k + 1, v2, h2);
    }
    if (plain) {
        p.kind = 0;
        p.d = p.x2 - p.x1;
        return;
    }
    const bool inf1 = h1 || (p.x1.is_zero() && p.y1.is_zero()), inf2 = h2 || (p.x2.is_zero() && p.y2.is_zero());
    p.d = Fq::one();
    if (inf1 && inf2) {
        p.kind = 4;
    } else if (inf2) {
        p.kind = 2;
    } else if (inf1) {
        p.kind = 3;
    } else if (p.x1 != p.x2) {
        p.kind = 0;
        p.d = p.x2 - p.x1;
    } else if (p.y1 == p.y2 && !p.y1.is_zero()) {
        p.kind = 1;
        p.d = p.y1.dbl();
    } else {
        p.kind = 4;   // P + (-P), or the doubling of a point of order two
    }
}

// product of the block's thread totals -> tree[1]; leaves at tree[AFF_TPB + t]
DP_D void aff_tree_up(Fq *tree, const Fq &mine) {
    const uint32_t t = threadIdx.x;
    tree[AFF_TPB + t] = mine;
    __syncthreads();
    for (uint32_t w = AFF_TPB >> 1; w >= 1; w >>= 1) {
        if (t < w) tree[w + t] = tree[2 * (w + t)] * tree[2 * (w + t) + 1];
        __syncthreads();
    }
}

// number of pairs of this level: (*n_elems >> level_shift) / 2, n_elems = total entries of the padded sorted array
DP_D uint64_t aff_pairs(const uint32_t *n_elems, uint32_t level_shift) { return ((uint64_t)*n_elems >> level_shift) >> 1; }

template <bool GATHER>
__global__ void __launch_bounds__(AFF_TPB) aff_k1_kernel(AffSrc src, const uint32_t *n_elems, uint32_t level_shift, Fq *pre, Fq *root) {
    __shared__ Fq tree[2 * AFF_TPB];
    const uint32_t t = threadIdx.x;
    const uint64_t m = aff_pairs(n_elems, level_shift), first = (uint64_t)blockIdx.x * AFF_BLOCK_PAIRS;
    if (first >= m) {  // (block-uniform) nothing here: the inversion kernel still reads this block's root
        if (t == 0) store_fq(root + blockIdx.x, Fq::one());
        return;
    }
    Fq run = Fq::one();
    for (int j = 0; j < AFF_KP; j++) {
        const uint64_t k = first + (uint64_t)j * AFF_TPB + t;
        if (k < m) {
            AffPair p;
            aff_pair<GATHER, true>(src, k, p);
            store_fq(pre + k, run);  // product of this thread's earlier denominators
            run = run * p.d;
        }
    }
    aff_tree_up(tree, run);
    if (t == 0) store_fq(root + blockIdx.x, tree[1]);
}

// inv[i] = 1 / root[i]; one root per lane, data-dependent iteration counts (the warp takes the slowest lane's)
__global__ void __launch_bounds__(32) aff_k2_kernel(const Fq *root, Fq *inv, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fq r = load_fq(root + i);
    store_fq(inv + i, r.is_zero() ? r : r.inverse_vartime());  // (a root is never zero; zero would not terminate)
}

template <bool GATHER>
__global__ void __launch_bounds__(AFF_TPB) aff_k3_kernel(AffSrc src, const uint32_t *n_elems, uint32_t level_shift, const Fq *pre,
                                                         const Fq *root_inv, G1Affine *out) {
    __shared__ Fq tree[2 * AFF_TPB];
    const uint32_t t = threadIdx.x;
    const uint64_t m = aff_pairs(n_elems, level_shift), first = (uint64_t)blockIdx.x * AFF_BLOCK_PAIRS;
    if (first >= m) return;  // block-uniform
    // this thread's total again: the prefix of its last pair times that pair's denominator
    int last = -1;
    for (int j = AFF_KP - 1; j >= 0 && last < 0; j--)
        if (first + (uint64_t)j * AFF_TPB + t < m) last = j;
    Fq total = Fq::one();
    if (last >= 0) {
        const uint64_t k = first + (uint64_t)last * AFF_TPB + t;
        AffPair p;
        aff_pair<GATHER, true>(src, k, p);
        total = load_fq(pre + k) * p.d;
    }
    aff_tree_up(tree, total);
    if (t == 0) tree[1] = load_fq(root_inv + blockIdx.x);
    __syncthreads();
    for (uint32_t w = 1; w < AFF_TPB; w <<= 1) {
        if (t < w) {
            const uint32_t node = w + t;
            const Fq iv = tree[node], l = tree[2 * node], r = tree[2 * node + 1];
            tree[2 * node] = iv * r;
            tree[2 * node + 1] = iv * l;
        }
        __syncthreads();
    }
    Fq inv_run = tree[AFF_TPB + t];  // 1 / (product of this thread's denominators)
    for (int j = last; j >= 0; j--) {
        const uint64_t k = first + (uint64_t)j * AFF_TPB + t;
        AffPair p;
        aff_pair<GATHER, false>(src, k, p);
        const Fq inv_d = inv_run * load_fq(pre + k);
        inv_run = inv_run * p.d;
        G1Affine r;
        if (p.kind <= 1) {
            Fq num;
            if (p.kind == 0) {
                num = p.y2 - p.y1;
            } else {
                const Fq xx = p.x1.sqr();
                num = xx.dbl() + xx;  // 3 x^2 (a = 0)
                p.x2 = p.x1;
            }
            const Fq lambda = num * inv_d;
            r.x = lambda.sqr() - p.x1 - p.x2;
            r.y = lambda * (p.x1 - r.x) - p.y1;
        } else if (p.kind == 2) {
            r.x = p.x1;
            r.y = p.y1;
        } else if (p.kind == 3) {
            r.x = p.x2;
            r.y = p.y2;
        } else {
            r = G1Affine::inf();
        }
        store_fq(&out[k].x, r.x);
        store_fq(&out[k].y, r.y);
    }
}

// Buckets cut into several tasks (skewed scalars: one bucket can hold a large share of all points)
// are folded by ONE WARP each: lanes stride over the bucket's partial sums, then a warp-shuffle
// butterfly adds the 32 lane sums; the result replaces the bucket's first partial.
DP_D G1XYZZ shfl_xor_point(const G1XYZZ &p, int mask) {
#if defined(DP_EMUL)
    return dp_emul_shfl_struct(p, dp_emul::t_lane ^ (unsigned)mask);
#endif
    G1XYZZ r;
#pragma unroll
    for (int i = 0; i < 12; i++) {
        r.x.l[i] = __shfl_xor_sync(0xffffffffu, p.x.l[i], mask);
        r.y.l[i] = __shfl_xor_sync(0xffffffffu, p.y.l[i], mask);
        r.zz.l[i] = __shfl_xor_sync(0xffffffffu, p.zz.l[i], mask);
        r.zzz.l[i] = __shfl_xor_sync(0xffffffffu, p.zzz.l[i], mask);
    }
    return r;
}
__global__ void __launch_bounds__(MSM_TPB) msm_collapse_kernel(const uint32_t *multi_keys, const uint32_t *n_multi,
                                                                const uint32_t *offsets, uint32_t chunk, G1XYZZ *partials) {
    // fixed-size grid, warps loop over the (usually empty) list: the count is only known on the device
    const uint32_t n_warps = (gridDim.x * blockDim.x) >> 5, lane = threadIdx.x & 31;
    for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < *n_multi; w += n_warps) {  // warp-uniform
        const uint32_t key = multi_keys[w];
        uint32_t j0, j1;
        bool empty;
        bucket_span(offsets, key, chunk, j0, j1, empty);
        G1XYZZ acc = G1XYZZ::inf();
        for (uint32_t j = j0 + lane; j <= j1; j += 32) acc = acc.add(partials[j + key]);
        for (int m = 16; m >= 1; m >>= 1) acc = acc.add(shfl_xor_point(acc, m));
        if (lane == 0) partials[j0 + key] = acc;
    }
}

// sum of one bucket: its few partial sums, or the folded one when msm_collapse handled it
DP_D G1XYZZ bucket_sum(const G1XYZZ *partials, const uint32_t *offsets, uint32_t chunk, uint32_t key) {
    uint32_t j0, j1;
    bool empty;
    bucket_span(offsets, key, chunk, j0, j1, empty);
    if (empty) return G1XYZZ::inf();
    G1XYZZ b = partials[j0 + key];
    if (j1 - j0 + 1 <= MSM_BIG_SPAN)
        for (uint32_t j = j0 + 1; j <= j1; j++) b = b.add(partials[j + key]);
    return b;
}

// k * P for a small non-negative integer k
DP_D G1XYZZ small_mul(const G1XYZZ &p, uint32_t k) {
    G1XYZZ acc = G1XYZZ::inf();
    for (int b = 31 - __clz((int)(k | 1)); b >= 0; b--) {
        acc = acc.dbl();
        if ((k >> b) & 1) acc = acc.add(p);
    }
    return k ? acc : G1XYZZ::inf();
}

// one thread per (window, segment): sum_{k in segment} k * B_k with the running-sum trick
__global__ void __launch_bounds__(MSM_TPB) msm_reduce_kernel(const G1XYZZ *partials, const uint32_t *offsets, MsmGeom g,
                                                              G1XYZZ *seg_sums) {
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= g.red_windows * g.segs_per_window) return;
    const uint32_t w = idx / g.segs_per_window, sgm = idx % g.segs_per_window;
    const uint32_t lo = sgm * g.seg;  // buckets lo+1 .. lo+seg of this window (bucket k <-> digit k)
    G1XYZZ running = G1XYZZ::inf(), acc = G1XYZZ::inf();
    for (uint32_t k = g.seg; k >= 1; k--) {
        running = running.add(bucket_sum(partials, offsets, g.chunk, w * g.bpw + lo + k - 1));
        acc = acc.add(running);
    }
    if (lo) acc = acc.add(small_mul(running, lo));
    seg_sums[idx] = acc;
}

// two-level sum of the segment sums: block (w, slice) folds its share into slice_sums[w*SLICES+slice]
__global__ void __launch_bounds__(MSM_TPB) msm_window_sum_kernel(const G1XYZZ *seg_sums, MsmGeom g, G1XYZZ *slice_sums) {
    __shared__ G1XYZZ red[MSM_TPB];
    const uint32_t w = blockIdx.x / g.slices, slice = blockIdx.x % g.slices, tid = threadIdx.x;
    const uint32_t per = (g.segs_per_window + g.slices - 1) / g.slices;
    const uint32_t lo = slice * per, hi = lo + per < g.segs_per_window ? lo + per : g.segs_per_window;
    G1XYZZ acc = G1XYZZ::inf();
    for (uint32_t s = lo + tid; s < hi; s += MSM_TPB) acc = acc.add(seg_sums[w * g.segs_per_window + s]);
    red[tid] = acc;
    __syncthreads();
    for (uint32_t off = MSM_TPB / 2; off >= 1; off >>= 1) {
        if (tid < off) red[tid] = red[tid].add(red[tid + off]);
        __syncthreads();
    }
    if (tid == 0) slice_sums[blockIdx.x] = red[0];
}

// one warp: per bucket set fold the SLICES partial sums (warp-shuffle butterfly), Horner over the
// windows when the bases were not premultiplied, normalise, write the raw 144-byte GroupProjective
__global__ void msm_final_kernel(const G1XYZZ *slice_sums, MsmGeom g, G1JacobianOut *out) {
    const uint32_t lane = threadIdx.x & 31;
    G1XYZZ total = G1XYZZ::inf();
    for (int w = (int)g.red_windows - 1; w >= 0; w--) {
        G1XYZZ part = lane < g.slices ? slice_sums[w * g.slices + lane] : G1XYZZ::inf();
        for (int m = 16; m >= 1; m >>= 1) part = part.add(shfl_xor_point(part, m));
        if (w != (int)g.red_windows - 1)
            for (uint32_t k = 0; k < g.c; k++) total = total.dbl();
        total = total.add(part);
    }
    if (lane == 0) *out = G1JacobianOut::from_affine(total.to_affine(true));
}

// pseudo-random canonical scalars below 2^254 (< r) for msm_tune(): SplitMix64 per limb
__global__ void msm_tune_scalars_kernel(uint4 *scalars, uint64_t n, uint64_t seed) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t w[8];
    for (int k = 0; k < 4; k++) {
        uint64_t z = seed + (4 * i + k + 1) * 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        z ^= z >> 31;
        w[2 * k] = (uint32_t)z;
        w[2 * k + 1] = (uint32_t)(z >> 32);
    }
    w[7] &= 0x3fffffffu;
    scalars[2 * i] = make_uint4(w[0], w[1], w[2], w[3]);
    scalars[2 * i + 1] = make_uint4(w[4], w[5], w[6], w[7]);
}

// ------------------------------------------------------------------ precomputed window multiples
// table[w * stride + i] = 2^(c*w) * P_i  (affine), w < n_windows.  With it every digit of every
// window lands in ONE shared set of 2^(c-1) buckets: no per-window bucket sets, no Horner pass
// (256 serial doublings), and a wider window for the same bucket count.  Built once per SRS.
constexpr int MSM_PRE_MAX_WINDOWS = 32;
__global__ void __launch_bounds__(128) msm_precompute_kernel(const G1Affine *bases, G1Affine *table, uint64_t n,
                                                              uint64_t stride, uint32_t c, uint32_t n_windows) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const G1Affine b = load_affine(bases + i);
    table[i] = b;
    if (b.is_inf()) {
        for (uint32_t w = 1; w < n_windows; w++) table[w * stride + i] = G1Affine::inf();
        return;
    }
    // doublings never reach infinity (prime-order subgroup); normalise all rows with one inversion
    G1XYZZ pts[MSM_PRE_MAX_WINDOWS];
    Fq prefix[MSM_PRE_MAX_WINDOWS];
    G1XYZZ p = G1XYZZ::from_affine(b);
    Fq run = Fq::one();
    for (uint32_t w = 1; w < n_windows; w++) {
        for (uint32_t k = 0; k < c; k++) p = p.dbl();
        pts[w] = p;
        prefix[w] = run;  // product of t_1 .. t_{w-1}
        run = run * (p.zz * p.zzz);
    }
    Fq inv = run.inverse();
    for (uint32_t w = n_windows - 1; w >= 1; w--) {
        const Fq t_inv = inv * prefix[w];  // (zz*zzz)^-1 of row w
        inv = inv * (pts[w].zz * pts[w].zzz);
        G1Affine a;
        a.x = pts[w].x * (t_inv * pts[w].zzz);
        a.y = pts[w].y * (t_inv * pts[w].zz);
        table[w * stride + i] = a;
    }
}

}  // namespace dp
