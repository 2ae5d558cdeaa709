// EXPERIMENT (negative result, not part of the product): carry-free ("unsaturated limb") Montgomery
// arithmetic.  It was measured slower than the carry-chain form of field.cuh (tools/microbench5.cu
// times both) - the extra partial products and the 64-bit accumulator register traffic cost more
// than the slower carry forms save.
//
// Carry-free ("unsaturated limb") Montgomery arithmetic.
//
// Why: the carry forms of the integer multiply-add (IMAD.WIDE.U32.X) issue at a lower rate than the
// plain IMAD.WIDE.U32 (tools/microbench.cu measures both) - so the classic 32-bit-limb Montgomery product of field.cuh, which is one long carry chain per row,
// runs at less than half of the multiplier's throughput.  Here a field element is L limbs of
// W < 32 bits held in 32-bit registers; partial products are accumulated in 64-bit columns with
// plain IMAD.WIDE.U32 (no carry in or out: W is chosen so that a column never overflows 64 bits)
// and carries are resolved once per product with shifts.  Additions and subtractions are limb-wise
// and lazy (no carry propagation, no conditional subtraction): values may exceed p by a bounded
// factor, limbs may exceed 2^W by a few bits; `normalize()` restores limbs < 2^W and every
// Montgomery product brings the value back below 2p.
//
//   Fr : L = 10, W = 27  (270 bits; capacity 2^15.1 * r; 100 + 100 MACs per product)
//   Fq : L = 14, W = 28  (392 bits; capacity 2^11.3 * p; 196 + 196 MACs per product)
//
// Montgomery radix is R' = 2^(L*W), NOT arkworks' 2^256 / 2^384.  Data that crosses the ABI stays
// in arkworks' form: the NTT only ever multiplies data by table entries, so the tables are stored
// in R' form (w * R' mod r) and data * table * R'^-1 keeps the data's own form; the MSM converts
// the bases once at import and the result once at the end.
//
// Bounds (B = 2^W): mul(a, b) needs a.limbs < 2^32, b.limbs <= B ("normalized") and
// value(a) * value(b) < p * R'; then column sums stay below L*(2^32*B + B*B) < 2^64 and the
// result is normalized with value < p * (value(a)*value(b)/(p*R') + 1) <= 2p.
#pragma once
#include "../../distributed_plonk_b200/csrc/ptx_arith.cuh"

namespace dp {

struct FrUParams {
    static constexpr int L = 10, W = 27, NW = 8;  // NW = packed 32-bit words
    DP_HD static constexpr uint32_t mod(int i) {
        constexpr uint32_t m[10] = {0x00000001u, 0x07ffffe0u, 0x016ffbffu, 0x02017fffu, 0x00553bdau,
                                    0x001343b0u, 0x04ce7602u, 0x04ebea41u, 0x05a75329u, 0x00000e7du};
        return m[i];
    }
    static constexpr uint32_t INV = 0x07ffffffu;  // -r^-1 mod 2^27
};

struct FqUParams {
    static constexpr int L = 14, W = 28, NW = 12;
    DP_HD static constexpr uint32_t mod(int i) {
        constexpr uint32_t m[14] = {0x0fffaaabu, 0x0fefffffu, 0x03ffffb9u, 0x0fffeb15u, 0x06241eabu,
                                    0x0a0f6b0fu, 0x0f6730d2u, 0x0f38512bu, 0x04774b84u, 0x04bacd76u,
                                    0x0ba7b643u, 0x0e69a4b1u, 0x01ea397fu, 0x0001a011u};
        return m[i];
    }
    static constexpr uint32_t INV = 0x0ffcfffdu;  // -p^-1 mod 2^28
};

template <class P>
struct UField {
    static constexpr int L = P::L, W = P::W, NW = P::NW;
    static constexpr uint32_t MASK = (1u << W) - 1;
    uint32_t l[L];

    DP_HD static UField zero() {
        UField z;
#pragma unroll
        for (int i = 0; i < L; i++) z.l[i] = 0;
        return z;
    }
    DP_HD static UField modulus() {
        UField z;
#pragma unroll
        for (int i = 0; i < L; i++) z.l[i] = P::mod(i);
        return z;
    }

    // ---- packed little-endian 32-bit words (the ABI / HBM format) <-> limbs
    DP_HD static UField unpack(const uint32_t *w) {
        UField z;
#pragma unroll
        for (int i = 0; i < L; i++) {
            const int bit = i * W, wi = bit >> 5, sh = bit & 31;
            uint32_t v = wi < NW ? (w[wi] >> sh) : 0u;
            if (sh + W > 32 && wi + 1 < NW) v |= w[wi + 1] << (32 - sh);
            z.l[i] = v & MASK;
        }
        return z;
    }
    // requires normalized limbs and value < 2^(32*NW)
    DP_HD void pack(uint32_t *w) const {
#pragma unroll
        for (int k = 0; k < NW; k++) {
            const int bit = 32 * k, i0 = bit / W, o = bit - i0 * W;
            uint32_t v = l[i0] >> o;
            int have = W - o;
#pragma unroll
            for (int i = i0 + 1; i < L && i < i0 + 3; i++) {
                if (have < 32) v |= l[i] << have;
                have += W;
            }
            w[k] = v;
        }
    }

    // ---- lazy arithmetic
    DP_HD friend UField operator+(const UField &a, const UField &b) {
        UField z;
#pragma unroll
        for (int i = 0; i < L; i++) z.l[i] = a.l[i] + b.l[i];
        return z;
    }
    // a - b + bias, where bias is a multiple of p whose limbs dominate b's limb by limb
    DP_HD static UField sub(const UField &a, const UField &b, const UField &bias) {
        UField z;
#pragma unroll
        for (int i = 0; i < L; i++) z.l[i] = a.l[i] + bias.l[i] - b.l[i];
        return z;
    }
    DP_HD UField shl(int k) const {  // 2^k * this, limb-wise
        UField z;
#pragma unroll
        for (int i = 0; i < L; i++) z.l[i] = l[i] << k;
        return z;
    }
    // limbs -> < 2^W (the top limb absorbs the rest; value unchanged)
    DP_HD UField normalized() const {
        UField z;
        uint32_t c = 0;
#pragma unroll
        for (int i = 0; i < L - 1; i++) {
            const uint32_t v = l[i] + c;  // limbs are far below 2^32 - 2^(32-W): no wrap
            z.l[i] = v & MASK;
            c = v >> W;
        }
        z.l[L - 1] = l[L - 1] + c;
        return z;
    }

    // Montgomery product a * b / 2^(L*W) mod p;  a lazy (limbs < 2^32), b normalized
    DP_HD static UField mul(const UField &a, const UField &b) {
        uint64_t acc[L];
#pragma unroll
        for (int j = 0; j < L; j++) acc[j] = 0;
#pragma unroll
        for (int i = 0; i < L; i++) {
#pragma unroll
            for (int j = 0; j < L; j++) acc[j] += (uint64_t)a.l[j] * b.l[i];
            const uint32_t m = ((uint32_t)acc[0] * P::INV) & MASK;
#pragma unroll
            for (int j = 0; j < L; j++) acc[j] += (uint64_t)m * P::mod(j);
            const uint64_t carry = acc[0] >> W;  // low W bits are zero now
#pragma unroll
            for (int j = 0; j < L - 1; j++) acc[j] = acc[j + 1];
            acc[L - 1] = 0;
            acc[0] += carry;
        }
        UField z;
#pragma unroll
        for (int j = 0; j < L - 1; j++) {
            z.l[j] = (uint32_t)acc[j] & MASK;
            acc[j + 1] += acc[j] >> W;
        }
        z.l[L - 1] = (uint32_t)acc[L - 1];
        return z;
    }
    DP_HD friend UField operator*(const UField &a, const UField &b) { return mul(a, b); }

    // value < 2p, normalized  ->  the canonical representative in [0, p), normalized
    DP_HD UField canonical_from_2p() const {
        // d = this - p with signed limb-wise borrow propagation
        uint32_t d[L];
        int32_t borrow = 0;
#pragma unroll
        for (int i = 0; i < L; i++) {
            const int32_t v = (int32_t)l[i] - (int32_t)P::mod(i) + borrow;
            d[i] = (uint32_t)v & MASK;
            borrow = v >> W;  // arithmetic shift: 0 or -1 (top limb: sign of the whole difference)
        }
        UField z;
#pragma unroll
        for (int i = 0; i < L; i++) z.l[i] = borrow < 0 ? l[i] : d[i];
        return z;
    }

    DP_HD bool is_zero_canonical() const {
        uint32_t o = 0;
#pragma unroll
        for (int i = 0; i < L; i++) o |= l[i];
        return o == 0;
    }
};

using FrU = UField<FrUParams>;
using FqU = UField<FqUParams>;

// bias for lazy subtraction: K*p written with limbs i < L-1 in [floor, 2*floor + 2^W) and the top limb
// taking the rest, so that (a - b + bias) is limb-wise non-negative for every b whose lower limbs are
// < floor and whose top limb is <= the bias' top limb.  Computed once on the host (init time).
template <class P>
inline bool make_sub_bias(uint32_t k_log2, uint32_t limb_floor_log2, UField<P> &out) {
    constexpr int L = P::L, W = P::W;
    // v = 2^k_log2 * p as (L+1) limbs of W bits, little endian
    uint64_t v[L + 1] = {0};
    for (int i = 0; i < L; i++) v[i] = P::mod(i);
    for (uint32_t s = 0; s < k_log2; s++) {
        uint64_t c = 0;
        for (int i = 0; i <= L; i++) {
            uint64_t t = v[i] * 2 + c;
            v[i] = t & ((1ull << W) - 1);
            c = t >> W;
        }
        if (c) return false;
    }
    if (v[L]) return false;  // exceeds the L*W-bit capacity
    // move `borrow_units` = 2^(floor-W) units from limb i+1 into limb i (worth 2^floor there)
    const uint64_t fl = 1ull << limb_floor_log2;
    if (limb_floor_log2 < (uint32_t)W) return false;
    const uint64_t units = fl >> W;
    for (int i = 0; i < L - 1; i++) {
        v[i] += fl;
        // take `units` from the next limb, borrowing further up when needed
        int j = i + 1;
        uint64_t need = units;
        while (true) {
            if (v[j] >= need) {
                v[j] -= need;
                break;
            }
            if (j == L - 1) return false;  // top limb exhausted: bias value too small for this floor
            v[j] += (1ull << W) - need;
            need = 1;
            j++;
        }
    }
    for (int i = 0; i < L; i++) {
        if (v[i] >> 32) return false;
        out.l[i] = (uint32_t)v[i];
    }
    return true;
}

}  // namespace dp
