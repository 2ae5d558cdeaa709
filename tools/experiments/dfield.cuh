// EXPERIMENT: Montgomery multiplication in BLS12-381 Fr / Fq on the FP64 pipe (DFMA), 52-bit limbs.
//
// Why: the 32-bit carry-chain product of field.cuh is bound by IMAD.WIDE.U32.X, which issues at a
// lower rate than the plain form: 128 of them per Fr product.  The FP64 pipe (on H100 at half the
// FP32 rate) is otherwise untouched by the prover.  A double holds a 52-bit limb exactly, and two fused multiply-adds with round-to-zero
// split an exact 104-bit limb product into its high and low 52 bits:
//      hi = fma_rz(a, b, 2^104)            = 2^104 + floor(a*b / 2^52) * 2^52
//      lo = fma_rz(a, b, 2^104 + 2^52 - hi) = 2^52  + (a*b mod 2^52)
// The bit patterns of hi / lo are (constant exponent | 52-bit payload), so summing them as 64-bit
// integers (IADD3 with two carry-outs adds two of them per instruction pair) accumulates product
// columns; the exponent constants are subtracted once per column.  Fr = 5 limbs (R' = 2^260),
// Fq = 8 limbs (R' = 2^416).  As for the unsaturated-limb experiment the Montgomery radix differs
// from arkworks' 2^256 / 2^384: the NTT only multiplies data by table entries, so tables stored as
// w * R' mod r keep the data in arkworks' own form.
//
// Host build (tests): the caller sets fesetround(FE_TOWARDZERO); fma() is then exactly __fma_rz.
#pragma once
#include <math.h>
#include <stdint.h>
#if !defined(__CUDACC__)
#define DF_HD inline
#else
#define DF_HD __host__ __device__ __forceinline__
#endif

namespace dpd {

DF_HD double fma_rz(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
    return __fma_rz(a, b, c);
#else
    return fma(a, b, c);
#endif
}
DF_HD uint64_t d2b(double x) {
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double_as_longlong(x);
#else
    uint64_t u;
    __builtin_memcpy(&u, &x, 8);
    return u;
#endif
}
DF_HD double b2d(uint64_t u) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)u);
#else
    double x;
    __builtin_memcpy(&x, &u, 8);
    return x;
#endif
}

constexpr uint64_t MASK52 = (1ull << 52) - 1;
constexpr uint64_t EXP_LO = 0x4330000000000000ull;  // bits of 2^52
constexpr uint64_t EXP_HI = 0x4670000000000000ull;  // bits of 2^104
#define DF_C1 0x1p104
#define DF_C2 (0x1p104 + 0x1p52)

// integer < 2^52 -> double (exact)
DF_HD double u52_to_double(uint64_t t) { return b2d(t | EXP_LO) - 0x1p52; }

struct FrDParams {
    static constexpr int L = 5;
    DF_HD static constexpr uint64_t mod(int i) {
        constexpr uint64_t m[5] = {0xfffff00000001ull, 0x2fffe5bfefffull, 0x9a1d80553bda4ull, 0x7d483339d8080ull, 0x73eda753299dull};
        return m[i];
    }
    // -r^-1 mod 2^52 = 2^52 - 2^32 - 1  (r = 1 - 2^32 mod 2^64): q = -(t + t*2^32) mod 2^52, integer ops only
    DF_HD static uint64_t q_of(uint64_t t) { return (0 - (t + (t << 32))) & MASK52; }
};
struct FqDParams {
    static constexpr int L = 8;
    DF_HD static constexpr uint64_t mod(int i) {
        constexpr uint64_t m[8] = {0xeffffffffaaabull, 0xfeb153ffffb9full, 0x6b0f6241eabffull, 0x12bf6730d2a0full,
                                   0x764774b84f385ull, 0x1ba7b6434bacdull, 0x1ea397fe69a4bull, 0x1a011ull};
        return m[i];
    }
    // -p^-1 mod 2^52 = 0x3fffcfffcfffd: one low product on the FP64 pipe
    DF_HD static uint64_t q_of(uint64_t t) {
        const double td = u52_to_double(t);
        const double ninv = (double)0x3fffcfffcfffdull;
        const double hi = fma_rz(td, ninv, DF_C1);
        const double lo = fma_rz(td, ninv, DF_C2 - hi);
        return d2b(lo) & MASK52;
    }
};

// out = a * b / 2^(52 L) mod m, limbs < 2^52, value < 2m  (inputs: limbs < 2^52, a*b < m * 2^(52 L))
template <class P>
DF_HD void mont_mul_dfma(const double *a, const double *b, uint64_t *out) {
    constexpr int L = P::L;
    uint64_t col[2 * L];
#pragma unroll
    for (int k = 0; k < 2 * L; k++) col[k] = 0;
#pragma unroll
    for (int i = 0; i < L; i++)
#pragma unroll
        for (int j = 0; j < L; j++) {
            const double hi = fma_rz(a[i], b[j], DF_C1);
            const double lo = fma_rz(a[i], b[j], DF_C2 - hi);
            col[i + j + 1] += d2b(hi);
            col[i + j] += d2b(lo);
        }
    // remove the exponent constants: column k holds n_lo(k) low halves and n_hi(k) = n_lo(k-1) high halves
#pragma unroll
    for (int k = 0; k < 2 * L; k++) {
        const int nlo = k < L ? k + 1 : 2 * L - 1 - k;
        const int nhi = k == 0 ? 0 : (k - 1 < L ? k : 2 * L - k);
        col[k] -= (uint64_t)nlo * EXP_LO + (uint64_t)nhi * EXP_HI;
    }
    // word-serial reduction, one 52-bit limb per round
#pragma unroll
    for (int k = 0; k < L; k++) {
        const uint64_t q = P::q_of(col[k] & MASK52);
        const double qd = u52_to_double(q);
#pragma unroll
        for (int j = 0; j < L; j++) {
            const double hi = fma_rz(qd, (double)P::mod(j), DF_C1);
            const double lo = fma_rz(qd, (double)P::mod(j), DF_C2 - hi);
            col[k + j + 1] += d2b(hi) - EXP_HI;
            col[k + j] += d2b(lo) - EXP_LO;
        }
        col[k + 1] += col[k] >> 52;  // col[k] is now a multiple of 2^52
    }
#pragma unroll
    for (int k = L; k < 2 * L - 1; k++) {
        col[k + 1] += col[k] >> 52;
        out[k - L] = col[k] & MASK52;
    }
    out[L - 1] = col[2 * L - 1];
}

// 8 x u32 (256-bit little-endian) <-> 5 x 52-bit limbs
DF_HD void fr_words_to_limbs(const uint32_t *w, uint64_t *l) {
    const uint64_t w01 = (uint64_t)w[0] | ((uint64_t)w[1] << 32), w23 = (uint64_t)w[2] | ((uint64_t)w[3] << 32);
    const uint64_t w45 = (uint64_t)w[4] | ((uint64_t)w[5] << 32), w67 = (uint64_t)w[6] | ((uint64_t)w[7] << 32);
    l[0] = w01 & MASK52;
    l[1] = ((w01 >> 52) | (w23 << 12)) & MASK52;
    l[2] = ((w23 >> 40) | (w45 << 24)) & MASK52;
    l[3] = ((w45 >> 28) | (w67 << 36)) & MASK52;
    l[4] = w67 >> 16;
}
DF_HD void fr_limbs_to_words(const uint64_t *l, uint32_t *w) {
    const uint64_t w01 = l[0] | (l[1] << 52), w23 = (l[1] >> 12) | (l[2] << 40);
    const uint64_t w45 = (l[2] >> 24) | (l[3] << 28), w67 = (l[3] >> 36) | (l[4] << 16);
    w[0] = (uint32_t)w01; w[1] = (uint32_t)(w01 >> 32);
    w[2] = (uint32_t)w23; w[3] = (uint32_t)(w23 >> 32);
    w[4] = (uint32_t)w45; w[5] = (uint32_t)(w45 >> 32);
    w[6] = (uint32_t)w67; w[7] = (uint32_t)(w67 >> 32);
}

}  // namespace dpd
