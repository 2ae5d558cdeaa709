// Prime-field arithmetic for BLS12-381 Fr (8 x u32) and Fq (12 x u32), Montgomery form.
//
// Replaces ark-ff 0.3.0 Fp256<FrParameters> / Fp384<FqParameters> (4 / 6 x u64 Montgomery,
// R = 2^256 / 2^384) that every arithmetic line of the reference hot path goes through
// (src/worker.rs:76-93,104-114,118,179; Cargo.toml:31-36).  The in-memory bytes are identical:
// 8 (12) little-endian u32 limbs == 4 (6) little-endian u64 limbs, same R, fully reduced.
//
// Multiplication is word-serial Montgomery with the products split into two accumulators of
// non-overlapping 64-bit columns ("even" columns start at even word positions, "odd" ones at odd
// positions) so each row a[*]*b[i] and m*p[*] is two straight carry chains of fused
// multiply-adds (IMAD.WIDE.U32 + carry) with no per-product carry fix-up.
#pragma once
#include "ptx_arith.cuh"

namespace dp {

template <int N>
struct alignas(16) Limbs {
    uint32_t l[N];
};

// ------------------------------------------------------------------------------ parameters
struct FrParams {
    static constexpr int N = 8;
    DP_HD static constexpr uint32_t mod(int i) {
        constexpr uint32_t m[8] = {0x00000001u, 0xffffffffu, 0xfffe5bfeu, 0x53bda402u,
                                   0x09a1d805u, 0x3339d808u, 0x299d7d48u, 0x73eda753u};
        return m[i];
    }
    // R mod r (Montgomery one)
    DP_HD static constexpr uint32_t one(int i) {
        constexpr uint32_t m[8] = {0xfffffffeu, 0x00000001u, 0x00034802u, 0x5884b7fau,
                                   0xecbc4ff5u, 0x998c4fefu, 0xacc5056fu, 0x1824b159u};
        return m[i];
    }
    // R^2 mod r
    DP_HD static constexpr uint32_t r2(int i) {
        constexpr uint32_t m[8] = {0xf3f29c6du, 0xc999e990u, 0x87925c23u, 0x2b6cedcbu,
                                   0x7254398fu, 0x05d31496u, 0x9f59ff11u, 0x0748d9d9u};
        return m[i];
    }
    static constexpr uint32_t INV = 0xffffffffu;  // -r^-1 mod 2^32
    static constexpr bool OUTLINE_MUL = false;    // NTT butterflies: a handful of call sites, keep inline
    // r = 1 - 2^32 (mod 2^64): the two lowest modulus limbs are 1 and 2^32 - 1, so m * r[0] = m and
    // m * r[1] = (m << 32) - m need no multiplier: 16 of the 128 multiply-accumulates of a product become
    // additions on the ALU pipe (the multiplier pipe is what bounds the NTT, DESIGN.md section 3.3)
    static constexpr bool LOW_LIMBS_ARE_1_AND_FFFFFFFF = true;
    static constexpr bool DEDICATED_SQR = false;
};

struct FqParams {
    static constexpr int N = 12;
    DP_HD static constexpr uint32_t mod(int i) {
        constexpr uint32_t m[12] = {0xffffaaabu, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu,
                                    0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u,
                                    0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau};
        return m[i];
    }
    DP_HD static constexpr uint32_t one(int i) {
        constexpr uint32_t m[12] = {0x0002fffdu, 0x76090000u, 0xc40c0002u, 0xebf4000bu,
                                    0x53c758bau, 0x5f489857u, 0x70525745u, 0x77ce5853u,
                                    0xa256ec6du, 0x5c071a97u, 0xfa80e493u, 0x15f65ec3u};
        return m[i];
    }
    DP_HD static constexpr uint32_t r2(int i) {
        constexpr uint32_t m[12] = {0x1c341746u, 0xf4df1f34u, 0x09d104f1u, 0x0a76e6a6u,
                                    0x4c95b6d5u, 0x8de5476cu, 0x939d83c0u, 0x67eb88a9u,
                                    0xb519952du, 0x9a793e85u, 0x92cae3aau, 0x11988fe5u};
        return m[i];
    }
    static constexpr uint32_t INV = 0xfffcfffdu;  // -p^-1 mod 2^32
    // One Fq product is ~380 SASS instructions (6 KB).  The curve formulas use 10-16 of them per
    // point operation; inlining every site made the MSM kernels 60-400 KB of straight-line code that
    // thrashed the instruction cache (ncu: 14% "no instruction" stalls in msm_accumulate, 30x
    // slowdown of msm_reduce).  A real call costs ~30 register moves (args travel in registers).
    static constexpr bool OUTLINE_MUL = true;
    static constexpr bool LOW_LIMBS_ARE_1_AND_FFFFFFFF = false;
    static constexpr bool DEDICATED_SQR = false;   // see Field::sqr()
};

// ------------------------------------------------------------------------------ field
template <class P>
struct Field : Limbs<P::N> {
    static constexpr int N = P::N;
    using Limbs<P::N>::l;

    DP_HD static Field zero() {
        Field z;
#pragma unroll
        for (int i = 0; i < N; i++) z.l[i] = 0;
        return z;
    }
    DP_HD static Field one() {
        Field z;
#pragma unroll
        for (int i = 0; i < N; i++) z.l[i] = P::one(i);
        return z;
    }
    DP_HD static Field r2() {
        Field z;
#pragma unroll
        for (int i = 0; i < N; i++) z.l[i] = P::r2(i);
        return z;
    }
    DP_HD bool is_zero() const {
        uint32_t o = 0;
#pragma unroll
        for (int i = 0; i < N; i++) o |= l[i];
        return o == 0;
    }
    DP_HD bool operator==(const Field &b) const {
        uint32_t o = 0;
#pragma unroll
        for (int i = 0; i < N; i++) o |= l[i] ^ b.l[i];
        return o == 0;
    }
    DP_HD bool operator!=(const Field &b) const { return !(*this == b); }

    // t in [0, 2p) -> [0, p)
    DP_HD static void final_sub(uint32_t *t) {
        uint32_t d[N];
        d[0] = ptx::sub_cc(t[0], P::mod(0));
#pragma unroll
        for (int i = 1; i < N; i++) d[i] = ptx::subc_cc(t[i], P::mod(i));
        uint32_t borrow = ptx::subc(0u, 0u);  // 0 or 0xffffffff
#pragma unroll
        for (int i = 0; i < N; i++) t[i] = borrow ? t[i] : d[i];
    }

    DP_HD friend Field operator+(const Field &a, const Field &b) {
        Field z;
        z.l[0] = ptx::add_cc(a.l[0], b.l[0]);
#pragma unroll
        for (int i = 1; i < N; i++) z.l[i] = ptx::addc_cc(a.l[i], b.l[i]);
        // p < 2^(32N-1): no carry out of the top limb
        final_sub(z.l);
        return z;
    }
    DP_HD friend Field operator-(const Field &a, const Field &b) {
        Field z;
        z.l[0] = ptx::sub_cc(a.l[0], b.l[0]);
#pragma unroll
        for (int i = 1; i < N; i++) z.l[i] = ptx::subc_cc(a.l[i], b.l[i]);
        uint32_t borrow = ptx::subc(0u, 0u);  // 0 or 0xffffffff
        z.l[0] = ptx::add_cc(z.l[0], P::mod(0) & borrow);
#pragma unroll
        for (int i = 1; i < N - 1; i++) z.l[i] = ptx::addc_cc(z.l[i], P::mod(i) & borrow);
        z.l[N - 1] = ptx::addc(z.l[N - 1], P::mod(N - 1) & borrow);
        return z;
    }
    DP_HD Field neg() const { return zero() - *this; }
    DP_HD Field dbl() const { return *this + *this; }

    // ---- Montgomery product building blocks ------------------------------------------------
    // acc[0..N) (64-bit columns at word 0,2,4..)  =  {a[0],a[2],...} * bi          (no carries)
    DP_HD static void mul_row(uint32_t *acc, const uint32_t *a, uint32_t bi) {
#pragma unroll
        for (int j = 0; j < N; j += 2) ptx::mul_wide(acc[j], acc[j + 1], a[j], bi);
    }
    // acc += {a[0],a[2],...} * bi as one carry chain; carry-out left in CC
    DP_HD static void mad_row(uint32_t *acc, const uint32_t *a, uint32_t bi) {
        ptx::mad_wide_cc(acc[0], acc[1], a[0], bi);
#pragma unroll
        for (int j = 2; j < N; j += 2) ptx::madc_wide_cc(acc[j], acc[j + 1], a[j], bi);
    }
    // constant-operand variant with the modulus limbs {p[off], p[off+2], ...}
    template <int OFF>
    DP_HD static void mad_row_mod(uint32_t *acc, uint32_t mi) {
        if (P::LOW_LIMBS_ARE_1_AND_FFFFFFFF) {
            static_assert(!P::LOW_LIMBS_ARE_1_AND_FFFFFFFF || (P::mod(0) == 1u && P::mod(1) == 0xffffffffu), "modulus shape");
            if (OFF == 0) {  // + mi * 1
                acc[0] = ptx::add_cc(acc[0], mi);
                acc[1] = ptx::addc_cc(acc[1], 0u);
            } else {         // + mi * (2^32 - 1) = {hi: mi - (mi != 0), lo: -mi}
                const uint32_t xlo = ptx::sub_cc(0u, mi);
                const uint32_t xhi = ptx::subc(mi, 0u);
                acc[0] = ptx::add_cc(acc[0], xlo);
                acc[1] = ptx::addc_cc(acc[1], xhi);
            }
#pragma unroll
            for (int j = 2; j < N; j += 2) ptx::madc_wide_cc(acc[j], acc[j + 1], P::mod(OFF + j), mi);
            return;
        }
        ptx::mad_wide_cc(acc[0], acc[1], P::mod(OFF), mi);
#pragma unroll
        for (int j = 2; j < N; j += 2) ptx::madc_wide_cc(acc[j], acc[j + 1], P::mod(OFF + j), mi);
    }
    // acc = (acc >> 64) + {a[0],a[2],...} * bi, continuing the carry in CC (carry-in consumed)
    DP_HD static void mad_row_shift(uint32_t *acc, const uint32_t *a, uint32_t bi) {
#pragma unroll
        for (int j = 0; j < N - 2; j += 2) ptx::madc_wide_cc(acc[j], acc[j + 1], a[j], bi, acc[j + 2], acc[j + 3]);
        ptx::madc_wide_last(acc[N - 2], acc[N - 1], a[N - 2], bi);
    }
    // One word-serial step.  `lo` holds the columns starting at the current word 0, `hi` those
    // starting at word 1 (from the previous step `hi` still holds the old `lo`-role array, whose
    // words 1.. are pending).  Adds a*bi, then m*p with m chosen to clear word 0.
    DP_HD static void mont_step(uint32_t *lo, uint32_t *hi, const uint32_t *a, uint32_t bi, bool first) {
        if (first) {
            mul_row(hi, a + 1, bi);
            mul_row(lo, a, bi);
        } else {
            lo[0] = ptx::add_cc(lo[0], hi[1]);      // pending word of the old array
            mad_row_shift(hi, a + 1, bi);           // hi = (old >> 64) + a_odd*bi (+carry)
            mad_row(lo, a, bi);
            hi[N - 1] = ptx::addc(hi[N - 1], 0u);
        }
        uint32_t mi = lo[0] * P::INV;
        mad_row_mod<1>(hi, mi);
        // p < 2^(32N-2) and the running value < 2p*2^32: the hi chain cannot carry out
        mad_row_mod<0>(lo, mi);
        hi[N - 1] = ptx::addc(hi[N - 1], 0u);
    }

#if defined(__CUDACC__)
    __device__ __noinline__ static Field mul_outlined(Field a, Field b) { return mul_inline(a, b); }
#endif
    DP_HD friend Field operator*(const Field &a, const Field &b) {
#if defined(__CUDA_ARCH__)
        if (P::OUTLINE_MUL) return mul_outlined(a, b);
#endif
        return mul_inline(a, b);
    }
    DP_HD static Field mul_inline(const Field &a, const Field &b) {
        uint32_t even[N], odd[N];
#pragma unroll
        for (int i = 0; i < N; i += 2) {
            mont_step(even, odd, a.l, b.l[i], i == 0);
            mont_step(odd, even, a.l, b.l[i + 1], false);
        }
        // after an even number of steps: value/2^32 = even (word 0..) + odd[1..] pending
        Field z;
        z.l[0] = ptx::add_cc(even[0], odd[1]);
#pragma unroll
        for (int i = 1; i < N - 1; i++) z.l[i] = ptx::addc_cc(even[i], odd[i + 1]);
        z.l[N - 1] = ptx::addc(even[N - 1], 0u);
        final_sub(z.l);
        return z;
    }
    // a^2.  The products a_i * a_j with i != j come in pairs: they are formed once and doubled, then the squares a_i^2
    // are added and the 2N-word result goes through a word-serial Montgomery reduction.  2N^2 + N(N+1) multiply
    // instructions of the single-result kind (IMAD / IMAD.HI with carry) instead of N^2 wide ones with carry plus 2N^2
    // single ones: at Fq size 444 against 576 pipe-equivalents, 27 % less than a general product (two of the ten
    // products of a mixed addition and three of the nine of a doubling are squarings).
    DP_HD static Field sqr_inline(const Field &x) {
        const uint32_t *a = x.l;
        uint32_t t[2 * N];
        // ---- sum_{i<j} a_i a_j 2^(32(i+j)): row i holds a_i * (a_{i+1} .. a_{N-1}) at word 2i+1; after row i the partial
        // sum is below 2^(32(i+N+1)), so a row never carries out of its own top word i+N
        t[0] = 0;
#pragma unroll
        for (int j = 1; j < N; j++) t[j] = ptx::mul_lo(a[0], a[j]);
        t[N] = 0;
        t[2] = ptx::mad_hi_cc(a[0], a[1], t[2]);
#pragma unroll
        for (int j = 2; j < N - 1; j++) t[j + 1] = ptx::madc_hi_cc(a[0], a[j], t[j + 1]);
        t[N] = ptx::madc_hi(a[0], a[N - 1], t[N]);
#pragma unroll
        for (int i = 1; i < N - 1; i++) {
            t[2 * i + 1] = ptx::mad_lo_cc(a[i], a[i + 1], t[2 * i + 1]);
#pragma unroll
            for (int j = i + 2; j < N; j++) t[i + j] = ptx::madc_lo_cc(a[i], a[j], t[i + j]);
            t[i + N] = ptx::addc(0u, 0u);
            if (i + 2 < N) {
                t[2 * i + 2] = ptx::mad_hi_cc(a[i], a[i + 1], t[2 * i + 2]);
#pragma unroll
                for (int j = i + 2; j < N - 1; j++) t[i + j + 1] = ptx::madc_hi_cc(a[i], a[j], t[i + j + 1]);
                t[i + N] = ptx::madc_hi(a[i], a[N - 1], t[i + N]);
            } else {  // last row: the single product a_{N-2} * a_{N-1}
                t[2 * i + 2] = ptx::mad_hi_cc(a[i], a[i + 1], t[2 * i + 2]);  // (the carry flag it sets is not used)
            }
        }
        // ---- double, add the squares a_i^2 at word 2i (one carry chain over all 2N words)
        t[2 * N - 1] = t[2 * N - 2] >> 31;
#pragma unroll
        for (int k = 2 * N - 2; k >= 1; k--) t[k] = (t[k] << 1) | (t[k - 1] >> 31);
        t[0] = ptx::mad_lo_cc(a[0], a[0], 0u);
        t[1] = ptx::madc_hi_cc(a[0], a[0], t[1]);
#pragma unroll
        for (int i = 1; i < N - 1; i++) {
            t[2 * i] = ptx::madc_lo_cc(a[i], a[i], t[2 * i]);
            t[2 * i + 1] = ptx::madc_hi_cc(a[i], a[i], t[2 * i + 1]);
        }
        t[2 * N - 2] = ptx::madc_lo_cc(a[N - 1], a[N - 1], t[2 * N - 2]);
        t[2 * N - 1] = ptx::madc_hi(a[N - 1], a[N - 1], t[2 * N - 1]);
        // ---- word-serial reduction: step i clears word i with m * p; the carries out of the low and the high chain go
        // into word i+N+1 at the next step (value 0..2)
        uint32_t pending = 0;
#pragma unroll
        for (int i = 0; i < N; i++) {
            const uint32_t m = t[i] * P::INV;
            t[i] = ptx::mad_lo_cc(m, P::mod(0), t[i]);
#pragma unroll
            for (int j = 1; j < N; j++) t[i + j] = ptx::madc_lo_cc(m, P::mod(j), t[i + j]);
            t[i + N] = ptx::addc_cc(t[i + N], pending);
            const uint32_t c_lo = ptx::addc(0u, 0u);
            t[i + 1] = ptx::mad_hi_cc(m, P::mod(0), t[i + 1]);
#pragma unroll
            for (int j = 1; j < N; j++) t[i + j + 1] = ptx::madc_hi_cc(m, P::mod(j), t[i + j + 1]);
            pending = c_lo + ptx::addc(0u, 0u);
        }
        Field z;
#pragma unroll
        for (int i = 0; i < N; i++) z.l[i] = t[N + i];
        final_sub(z.l);
        return z;
    }
#if defined(__CUDACC__)
    __device__ __noinline__ static Field sqr_outlined(Field a) { return sqr_inline(a); }
#endif
    // NOT ADOPTED: ptxas splits the single-result multiply-adds with carry into IMAD + IADD3.X pairs, the additions land
    // on the ALU pipe next to the carry work that is already there, and msm_accumulate got slower although 13 % of its
    // multiplier work is gone.
    // sqr() therefore stays the general product; sqr_inline() is kept, tested bit for bit (tests/test_emul_field.py).
    DP_HD Field sqr() const {
        if (P::DEDICATED_SQR) {
#if defined(__CUDA_ARCH__)
            if (P::OUTLINE_MUL) return sqr_outlined(*this);
#endif
            return sqr_inline(*this);
        }
        return (*this) * (*this);
    }

    DP_HD Field &operator+=(const Field &b) { return *this = *this + b; }
    DP_HD Field &operator-=(const Field &b) { return *this = *this - b; }
    DP_HD Field &operator*=(const Field &b) { return *this = *this * b; }

    // canonical integer <-> Montgomery (ark: from_repr / into_repr)
    DP_HD Field to_mont() const { return (*this) * r2(); }
    DP_HD Field from_mont() const {
        Field o = zero();
        o.l[0] = 1;
        return (*this) * o;
    }

    // x^e for a 64-bit exponent (Fr::pow([e]); worker.rs:79,93,113)
    DP_HD Field pow(uint64_t e) const {
        Field acc = one();
        bool started = false;
        for (int b = 63; b >= 0; b--) {
            if (started) acc = acc.sqr();
            if ((e >> b) & 1) {
                acc = started ? acc * (*this) : *this;
                started = true;
            }
        }
        return acc;
    }
    // x^e, e = n_limbs 32-bit little-endian limbs
    DP_HD Field pow_limbs(const uint32_t *e, int n_limbs) const {
        Field acc = one();
        bool started = false;
        for (int i = n_limbs - 1; i >= 0; i--) {
            for (int b = 31; b >= 0; b--) {
                if (started) acc = acc.sqr();
                if ((e[i] >> b) & 1) {
                    acc = started ? acc * (*this) : *this;
                    started = true;
                }
            }
        }
        return acc;
    }
    // canonical integers (NOT Montgomery form): a > b
    DP_HD static bool canon_gt(const Field &a, const Field &b) {
        for (int i = N - 1; i >= 0; i--)
            if (a.l[i] != b.l[i]) return a.l[i] > b.l[i];
        return false;
    }
    // canonical integer < modulus
    DP_HD bool canon_is_reduced() const {
        for (int i = N - 1; i >= 0; i--)
            if (l[i] != P::mod(i)) return l[i] < P::mod(i);
        return false;
    }
    // 1/x for ONE thread on the critical path (msm_final: a single lane normalises the result): binary extended
    // Euclid on the limbs - shifts, additions and comparisons only, ~1.5 * bits iterations with data-dependent
    // branches - instead of the ~1.5 * bits dependent Montgomery products of Fermat's exponentiation (a long
    // serial chain for a lone warp at Fq size; this is ~10x shorter).  Divergent across a warp: keep inverse() for full warps.
    // x != 0, Montgomery form in and out.
    DP_HD Field inverse_vartime() const {
        uint32_t u[N], v[N], x1[N], x2[N];
#pragma unroll
        for (int i = 0; i < N; i++) {
            u[i] = l[i];
            v[i] = P::mod(i);
            x1[i] = i == 0 ? 1u : 0u;
            x2[i] = 0u;
        }
        auto is_one = [](const uint32_t *a) {
            uint32_t o = a[0] ^ 1u;
#pragma unroll
            for (int i = 1; i < N; i++) o |= a[i];
            return o == 0;
        };
        auto halve = [](uint32_t *a, uint32_t top) {  // (top:a) >> 1
#pragma unroll
            for (int i = 0; i < N - 1; i++) a[i] = (a[i] >> 1) | (a[i + 1] << 31);
            a[N - 1] = (a[N - 1] >> 1) | (top << 31);
        };
        auto halve_mod = [&](uint32_t *a) {  // a / 2 mod p, a < p
            uint32_t top = 0;
            if (a[0] & 1u) {
                a[0] = ptx::add_cc(a[0], P::mod(0));
#pragma unroll
                for (int i = 1; i < N; i++) a[i] = ptx::addc_cc(a[i], P::mod(i));
                top = ptx::addc(0u, 0u);
            }
            halve(a, top);
        };
        auto geq = [](const uint32_t *a, const uint32_t *b) {
            for (int i = N - 1; i >= 0; i--)
                if (a[i] != b[i]) return a[i] > b[i];
            return true;
        };
        auto sub = [](uint32_t *a, const uint32_t *b) {  // a -= b, a >= b
            a[0] = ptx::sub_cc(a[0], b[0]);
#pragma unroll
            for (int i = 1; i < N; i++) a[i] = ptx::subc_cc(a[i], b[i]);
        };
        auto sub_mod = [&](uint32_t *a, const uint32_t *b) {  // a = a - b mod p, both < p
            a[0] = ptx::sub_cc(a[0], b[0]);
#pragma unroll
            for (int i = 1; i < N; i++) a[i] = ptx::subc_cc(a[i], b[i]);
            const uint32_t borrow = ptx::subc(0u, 0u);
            if (borrow) {
                a[0] = ptx::add_cc(a[0], P::mod(0));
#pragma unroll
                for (int i = 1; i < N; i++) a[i] = ptx::addc_cc(a[i], P::mod(i));
            }
        };
        while (!is_one(u) && !is_one(v)) {
            while (!(u[0] & 1u)) {
                halve(u, 0u);
                halve_mod(x1);
            }
            while (!(v[0] & 1u)) {
                halve(v, 0u);
                halve_mod(x2);
            }
            if (geq(u, v)) {
                sub(u, v);
                sub_mod(x1, x2);
            } else {
                sub(v, u);
                sub_mod(x2, x1);
            }
        }
        // (x R)^-1 = x^-1 R^-1 as a plain residue; times R^3 (Montgomery product) = x^-1 R
        Field r;
#pragma unroll
        for (int i = 0; i < N; i++) r.l[i] = is_one(u) ? x1[i] : x2[i];
        return r * (r2() * r2());
    }

    // x^(p-2) (Fermat); x != 0
    DP_HD Field inverse() const {
        uint32_t e[N];
        uint32_t borrow = 2;
#pragma unroll
        for (int i = 0; i < N; i++) {
            uint32_t m = P::mod(i);
            e[i] = m - borrow;
            borrow = m < borrow ? 1u : 0u;
        }
        Field acc = one();
        bool started = false;
        for (int i = N - 1; i >= 0; i--) {
            for (int b = 31; b >= 0; b--) {
                if (started) acc = acc.sqr();
                if ((e[i] >> b) & 1) {
                    acc = started ? acc * (*this) : *this;
                    started = true;
                }
            }
        }
        return acc;
    }
};

using Fr = Field<FrParams>;
using Fq = Field<FqParams>;

}  // namespace dp
