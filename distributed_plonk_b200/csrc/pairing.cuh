// BLS12-381 optimal-ate pairing, G2 and the open key of the KZG setup, for a verifier that holds no trapdoor.
//
// Tower (ark-bls12-381's):  Fq2 = Fq[u]/(u^2 + 1),  Fq6 = Fq2[v]/(v^3 - xi) with xi = u + 1,  Fq12 = Fq6[w]/(w^2 - v).
// G2 is the M-type sextic twist E': y^2 = x^3 + 4 xi; psi(x, y) = (x / w^2, y / w^3) maps it into E(Fq12).
//
// Pairing: e(P, Q) = f^(3 (p^12 - 1) / r) with f = conj(f_{|x|,Q}(P)), x = -0xd201000000010000 - the CUBE of the
// textbook reduced pairing f^((p^12 - 1) / r): the hard part of the final exponentiation uses
//   3 (p^4 - p^2 + 1) / r = (x - 1)^2 (x + p) (x^2 + p^2 - 1) + 3
// (DESIGN.md section 3.8).  gcd(3, r) = 1, so e is a non-degenerate bilinear pairing all the same.
//
// The Miller loop keeps T in Jacobian coordinates on the twist; each line through T (and Q) evaluated at P is scaled by
// a factor of Fq2 and by w^3 (in Fq4), both killed by the final exponentiation, which leaves the sparse Fq12 element
//   l0 + l1 v + l2 v w     (l0, l1, l2 in Fq2; l1 and l2 linear in x_P and y_P)
// and costs 13 Fq2 products to multiply in.  Vertical lines are dropped for the same reason.
//
// One thread computes a whole pairing (latency-bound, DESIGN.md section 3.8): the tower products are outlined like the
// Fq product (field.cuh), so the kernels stay small enough for the instruction cache.
#pragma once
#include "g1.cuh"

namespace dp {

#if defined(__CUDACC__)
#define DP_PAIR_FN __device__ __noinline__
#else
#define DP_PAIR_FN inline
#endif

DP_D Fq fq_lit(const uint32_t (&v)[12]) {
    Fq z;
#pragma unroll
    for (int i = 0; i < 12; i++) z.l[i] = v[i];
    return z;
}

// ------------------------------------------------------------------------------------------------ Fq2
struct alignas(16) Fq2 {
    Fq c0, c1;
    DP_D static Fq2 zero() { return Fq2{Fq::zero(), Fq::zero()}; }
    DP_D static Fq2 one() { return Fq2{Fq::one(), Fq::zero()}; }
    DP_D bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    DP_D bool operator==(const Fq2 &b) const { return c0 == b.c0 && c1 == b.c1; }
    DP_D Fq2 neg() const { return Fq2{c0.neg(), c1.neg()}; }
    DP_D Fq2 dbl() const { return Fq2{c0.dbl(), c1.dbl()}; }
    DP_D Fq2 conj() const { return Fq2{c0, c1.neg()}; }
    DP_D Fq2 mul_by_xi() const { return Fq2{c0 - c1, c0 + c1}; }  // (c0 + c1 u)(1 + u)
    DP_D Fq2 mul_fq(const Fq &s) const { return Fq2{c0 * s, c1 * s}; }
};
DP_D Fq2 operator+(const Fq2 &a, const Fq2 &b) { return Fq2{a.c0 + b.c0, a.c1 + b.c1}; }
DP_D Fq2 operator-(const Fq2 &a, const Fq2 &b) { return Fq2{a.c0 - b.c0, a.c1 - b.c1}; }

DP_PAIR_FN Fq2 fq2_mul(Fq2 a, Fq2 b) {  // Karatsuba: 3 Fq products
    const Fq t0 = a.c0 * b.c0, t1 = a.c1 * b.c1;
    return Fq2{t0 - t1, (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1};
}
DP_PAIR_FN Fq2 fq2_sqr(Fq2 a) {  // (c0 + c1)(c0 - c1) + 2 c0 c1 u
    const Fq t = a.c0 * a.c1;
    return Fq2{(a.c0 + a.c1) * (a.c0 - a.c1), t.dbl()};
}
DP_D Fq2 operator*(const Fq2 &a, const Fq2 &b) { return fq2_mul(a, b); }
// a != 0; one lane (the binary extended Euclid of Field::inverse_vartime)
DP_D Fq2 fq2_inv(const Fq2 &a) {
    const Fq t = (a.c0 * a.c0 + a.c1 * a.c1).inverse_vartime();
    return Fq2{a.c0 * t, (a.c1 * t).neg()};
}

// ------------------------------------------------------------------------------------------------ Fq6
struct alignas(16) Fq6 {
    Fq2 b0, b1, b2;
    DP_D static Fq6 zero() { return Fq6{Fq2::zero(), Fq2::zero(), Fq2::zero()}; }
    DP_D static Fq6 one() { return Fq6{Fq2::one(), Fq2::zero(), Fq2::zero()}; }
    DP_D Fq6 neg() const { return Fq6{b0.neg(), b1.neg(), b2.neg()}; }
    DP_D Fq6 mul_by_v() const { return Fq6{b2.mul_by_xi(), b0, b1}; }  // v^3 = xi
};
DP_D Fq6 operator+(const Fq6 &a, const Fq6 &b) { return Fq6{a.b0 + b.b0, a.b1 + b.b1, a.b2 + b.b2}; }
DP_D Fq6 operator-(const Fq6 &a, const Fq6 &b) { return Fq6{a.b0 - b.b0, a.b1 - b.b1, a.b2 - b.b2}; }

DP_PAIR_FN Fq6 fq6_mul(Fq6 a, Fq6 b) {  // 6 Fq2 products
    const Fq2 t0 = a.b0 * b.b0, t1 = a.b1 * b.b1, t2 = a.b2 * b.b2;
    Fq6 z;
    z.b0 = t0 + ((a.b1 + a.b2) * (b.b1 + b.b2) - t1 - t2).mul_by_xi();
    z.b1 = (a.b0 + a.b1) * (b.b0 + b.b1) - t0 - t1 + t2.mul_by_xi();
    z.b2 = (a.b0 + a.b2) * (b.b0 + b.b2) - t0 - t2 + t1;
    return z;
}
DP_D Fq6 operator*(const Fq6 &a, const Fq6 &b) { return fq6_mul(a, b); }
// a * (s0 + s1 v): 5 Fq2 products
DP_PAIR_FN Fq6 fq6_mul_by_01(Fq6 a, Fq2 s0, Fq2 s1) {
    return Fq6{a.b0 * s0 + (a.b2 * s1).mul_by_xi(), a.b0 * s1 + a.b1 * s0, a.b1 * s1 + a.b2 * s0};
}
// a * s1 v: 3 Fq2 products
DP_D Fq6 fq6_mul_by_1(const Fq6 &a, const Fq2 &s1) { return Fq6{(a.b2 * s1).mul_by_xi(), a.b0 * s1, a.b1 * s1}; }
DP_D Fq6 fq6_inv(const Fq6 &a) {
    const Fq2 A = fq2_sqr(a.b0) - (a.b1 * a.b2).mul_by_xi();
    const Fq2 B = fq2_sqr(a.b2).mul_by_xi() - a.b0 * a.b1;
    const Fq2 C = fq2_sqr(a.b1) - a.b0 * a.b2;
    const Fq2 F = fq2_inv(a.b0 * A + (a.b2 * B + a.b1 * C).mul_by_xi());
    return Fq6{A * F, B * F, C * F};
}

// ------------------------------------------------------------------------------------------------ Fq12
struct alignas(16) Fq12 {
    Fq6 c0, c1;
    DP_D static Fq12 one() { return Fq12{Fq6::one(), Fq6::zero()}; }
    DP_D Fq12 conj() const { return Fq12{c0, c1.neg()}; }  // x^(p^6); the inverse in the cyclotomic subgroup
};
DP_PAIR_FN Fq12 fq12_mul(Fq12 a, Fq12 b) {  // 3 Fq6 products
    const Fq6 t0 = a.c0 * b.c0, t1 = a.c1 * b.c1;
    return Fq12{t0 + t1.mul_by_v(), (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1};
}
DP_D Fq12 operator*(const Fq12 &a, const Fq12 &b) { return fq12_mul(a, b); }
DP_PAIR_FN Fq12 fq12_sqr(Fq12 a) {  // 2 Fq6 products: c0^2 + v c1^2 = (c0 + c1)(c0 + v c1) - t - v t, t = c0 c1
    const Fq6 t = a.c0 * a.c1;
    return Fq12{(a.c0 + a.c1) * (a.c0 + a.c1.mul_by_v()) - t - t.mul_by_v(), t + t};
}
DP_D Fq12 fq12_inv(const Fq12 &a) {
    const Fq6 t = fq6_inv(a.c0 * a.c0 - (a.c1 * a.c1).mul_by_v());
    return Fq12{a.c0 * t, (a.c1 * t).neg()};
}
// f * (l0 + l1 v + l2 v w), the sparse value of a line: 13 Fq2 products
DP_PAIR_FN Fq12 fq12_mul_by_line(Fq12 f, Fq2 l0, Fq2 l1, Fq2 l2) {
    const Fq6 t0 = fq6_mul_by_01(f.c0, l0, l1), t1 = fq6_mul_by_1(f.c1, l2);
    return Fq12{t0 + t1.mul_by_v(), fq6_mul_by_01(f.c0 + f.c1, l0, l1 + l2) - t0 - t1};
}

// Frobenius x -> x^(p^K), K = 1, 2: v^(p^K) = xi^((p^K - 1) / 3) v, w^(p^K) = xi^((p^K - 1) / 6) w
template <int K>
DP_D Fq2 frob_v(int power) {  // xi^(power (p^K - 1) / 3), power = 1, 2 (Montgomery form)
    if (K == 1) {
        if (power == 1)
            return Fq2{Fq::zero(), fq_lit({0x8671f071u, 0xcd03c9e4u, 0x1fcda5d2u, 0x5dab2246u, 0xd3851b95u, 0x587042afu,
                                           0x01bacb9eu, 0x8eb60ebeu, 0x83d050d2u, 0x03f97d6eu, 0x54638741u, 0x18f02065u})};
        return Fq2{fq_lit({0x867545c3u, 0x890dc9e4u, 0x3285a5d5u, 0x2af32253u, 0x309b7e2cu, 0x50880866u, 0x7e881024u,
                           0xa20d1b8cu, 0xe2db9068u, 0x14e4f04fu, 0x1564853au, 0x14e56d3fu}),
                   Fq::zero()};
    }
    if (power == 1)
        return Fq2{fq_lit({0x798a64e8u, 0x30f1361bu, 0x7ece5a2au, 0xf3b8ddabu, 0xc61577f7u, 0x16a8ca3au, 0x74fd029bu,
                           0xc26a2ff8u, 0x60701c6eu, 0x3636b766u, 0x241b6160u, 0x051ba4abu}),
                   Fq::zero()};
    return Fq2{fq_lit({0x8671f071u, 0xcd03c9e4u, 0x1fcda5d2u, 0x5dab2246u, 0xd3851b95u, 0x587042afu, 0x01bacb9eu,
                       0x8eb60ebeu, 0x83d050d2u, 0x03f97d6eu, 0x54638741u, 0x18f02065u}),
               Fq::zero()};
}
template <int K>
DP_D Fq2 frob_w() {  // xi^((p^K - 1) / 6)
    if (K == 1)
        return Fq2{fq_lit({0xb319d465u, 0x07089552u, 0xb50a8313u, 0xc6695f92u, 0xd117228fu, 0x97e83cccu, 0xb2dc29eeu,
                           0xa35baecau, 0x5daace4du, 0x1ce393eau, 0xb0fb66ebu, 0x08f2220fu}),
                   fq_lit({0x4ce5d646u, 0xb2f66aadu, 0xfc497cecu, 0x5842a06bu, 0x2599d394u, 0xcf4895d4u, 0x40a8e8d0u,
                           0xc11b9cbau, 0xe5a0de89u, 0x2e3813cbu, 0x88847fafu, 0x110eefdau})};
    return Fq2{fq_lit({0x798dba3au, 0xecfb361bu, 0x91865a2cu, 0xc100ddb8u, 0x232bda8eu, 0x0ec08ff1u, 0xf1ca4721u,
                       0xd5c13cc6u, 0xbf7b5c04u, 0x47222a47u, 0xe51c5f59u, 0x0110f184u}),
               Fq::zero()};
}
template <int K>
DP_D Fq2 frob2(const Fq2 &a) { return (K & 1) ? a.conj() : a; }  // u^p = -u
template <int K>
DP_D Fq6 frob6(const Fq6 &a) {
    return Fq6{frob2<K>(a.b0), frob2<K>(a.b1) * frob_v<K>(1), frob2<K>(a.b2) * frob_v<K>(2)};
}
template <int K>
DP_PAIR_FN Fq12 fq12_frob(Fq12 a) {
    const Fq6 c1 = frob6<K>(a.c1);
    const Fq2 g = frob_w<K>();
    return Fq12{frob6<K>(a.c0), Fq6{c1.b0 * g, c1.b1 * g, c1.b2 * g}};
}

// Squaring in the cyclotomic subgroup (Granger-Scott): f = A + B w + C w^2 over Fq4 = Fq2[W]/(W^2 - xi), W = w^3, with
// A = c0.b0 + c1.b1 W, B = c1.b0 + c0.b2 W, C = c0.b1 + c1.b2 W;  f^2 = (3A^2 - 2 conj A) + (3 W C^2 + 2 conj B) w
// + (3 B^2 - 2 conj C) w^2, conj(a + b W) = a - b W.  Valid only for f^(p^4 - p^2 + 1) = 1 (after the easy part).
DP_D void fq4_sqr(const Fq2 &a, const Fq2 &b, Fq2 &s0, Fq2 &s1) {  // (a + b W)^2 = a^2 + xi b^2 + 2ab W
    const Fq2 t0 = fq2_sqr(a), t1 = fq2_sqr(b);
    s0 = t0 + t1.mul_by_xi();
    s1 = fq2_sqr(a + b) - t0 - t1;
}
DP_PAIR_FN Fq12 fq12_cyclotomic_sqr(Fq12 f) {
    Fq2 a0, a1, b0, b1, c0, c1;
    fq4_sqr(f.c0.b0, f.c1.b1, a0, a1);  // A^2
    fq4_sqr(f.c1.b0, f.c0.b2, b0, b1);  // B^2
    fq4_sqr(f.c0.b1, f.c1.b2, c0, c1);  // C^2
    auto three = [](const Fq2 &x) { return x.dbl() + x; };
    Fq12 z;
    z.c0.b0 = three(a0) - f.c0.b0.dbl();
    z.c1.b1 = three(a1) + f.c1.b1.dbl();
    z.c1.b0 = three(c1.mul_by_xi()) + f.c1.b0.dbl();  // W C^2 = xi c1 + c0 W
    z.c0.b2 = three(c0) - f.c0.b2.dbl();
    z.c0.b1 = three(b0) - f.c0.b1.dbl();
    z.c1.b2 = three(b1) + f.c1.b2.dbl();
    return z;
}

// ------------------------------------------------------------------------------------------------ G2 on the twist
constexpr uint64_t PAIRING_ABS_X = 0xd201000000010000ull;  // |x|, x < 0

DP_D Fq2 g2_b() {  // 4 (u + 1)
    const Fq four = fq_lit({0x000cfff3u, 0xaa270000u, 0xfc34000au, 0x53cc0032u, 0x6b0a807fu, 0x478fe97au, 0xe6ba24d7u,
                            0xb1d37ebeu, 0xbf78ab2fu, 0x8ec9733bu, 0x3d83de7eu, 0x09d64551u});
    return Fq2{four, four};
}

struct alignas(16) G2Affine {
    Fq2 x, y;
    bool inf;
    DP_D static G2Affine generator() {  // ark-bls12-381 G2Affine::prime_subgroup_generator (Montgomery form)
        G2Affine h;
        h.x = Fq2{fq_lit({0x02940a10u, 0xf5f28fa2u, 0x87b4961au, 0xb3f5fb26u, 0x3e2ae580u, 0xa1a893b5u, 0x1a3caee9u,
                          0x9894999du, 0x1863366bu, 0x6f67b763u, 0x4350bcd7u, 0x05819192u}),
                  fq_lit({0x9e23f606u, 0xa5a9c075u, 0xbccd60c3u, 0xaaa0c59du, 0xe2867806u, 0x3bb17e18u, 0x8541b367u,
                          0x1b1ab6ccu, 0xf2158547u, 0xc2b6ed0eu, 0x7360edf3u, 0x11922a09u})};
        h.y = Fq2{fq_lit({0x60494c4au, 0x4c730af8u, 0x5e369c5au, 0x597cfa1fu, 0xaa0a635au, 0xe7e6856cu, 0x6e0d495fu,
                          0xbbefb5e9u, 0xf0ef25a2u, 0x07d3a975u, 0x7e80dae5u, 0x0083fd8eu}),
                  fq_lit({0xdf64b05du, 0xadc0fc92u, 0x2b1461dcu, 0x18aa270au, 0x3be4eba0u, 0x86adac6au, 0xc93da33au,
                          0x79495c4eu, 0xa43ccaedu, 0xe7175850u, 0x63de1bf2u, 0x0b2bc2a1u})};
        h.inf = false;
        return h;
    }
    DP_D bool on_twist() const { return inf || fq2_sqr(y) == fq2_sqr(x) * x + g2_b(); }
};

struct alignas(16) G2Jac {  // x = X / Z^2, y = Y / Z^3; Z = 0 is the point at infinity
    Fq2 X, Y, Z;
    DP_D bool is_inf() const { return Z.is_zero(); }
    DP_D static G2Jac from_affine(const G2Affine &q) {
        return q.inf ? G2Jac{Fq2::one(), Fq2::one(), Fq2::zero()} : G2Jac{q.x, q.y, Fq2::one()};
    }
    DP_D G2Jac dbl() const {  // dbl-2009-l (a = 0)
        if (is_inf()) return *this;
        const Fq2 A = fq2_sqr(X), B = fq2_sqr(Y), C = fq2_sqr(B);
        const Fq2 D = (fq2_sqr(X + B) - A - C).dbl(), E = A.dbl() + A, F = fq2_sqr(E);
        G2Jac r;
        r.X = F - D.dbl();
        r.Y = E * (D - r.X) - C.dbl().dbl().dbl();
        r.Z = (Y * Z).dbl();
        return r;
    }
    DP_D G2Jac add_mixed(const G2Affine &q) const {  // handles infinity, doubling and T + (-T)
        if (q.inf) return *this;
        if (is_inf()) return from_affine(q);
        const Fq2 ZZ = fq2_sqr(Z), H = q.x * ZZ - X, R = q.y * Z * ZZ - Y;
        if (H.is_zero()) return R.is_zero() ? from_affine(q).dbl() : G2Jac{Fq2::one(), Fq2::one(), Fq2::zero()};
        const Fq2 HH = fq2_sqr(H), HHH = H * HH, V = X * HH;
        G2Jac o;
        o.X = fq2_sqr(R) - HHH - V.dbl();
        o.Y = R * (V - o.X) - Y * HHH;
        o.Z = Z * H;
        return o;
    }
    DP_D G2Affine to_affine() const {  // one lane
        if (is_inf()) return G2Affine{Fq2::zero(), Fq2::one(), true};
        const Fq2 zi = fq2_inv(Z), zi2 = fq2_sqr(zi);
        return G2Affine{X * zi2, Y * zi2 * zi, false};
    }
};

// k * q for a 256-bit integer k (8 little-endian limbs), double-and-add from the top bit
DP_D G2Jac g2_mul(const G2Affine &q, const uint32_t *k) {
    G2Jac acc = G2Jac::from_affine(G2Affine{Fq2::zero(), Fq2::one(), true});
    for (int i = 7; i >= 0; i--)
        for (int b = 31; b >= 0; b--) {
            acc = acc.dbl();
            if ((k[i] >> b) & 1) acc = acc.add_mixed(q);
        }
    return acc;
}

// ------------------------------------------------------------------------------------------------ Miller loop
// f <- f * l_{T,T}(P), T <- 2T.  Line scaled by 2 Y Z^3:  l0 = 3X^3 - 2Y^2,  l1 = -3X^2 Z^2 x_P,  l2 = 2Y Z^3 y_P
DP_D void miller_dbl_step(G2Jac &T, const G1Affine &P, Fq12 &f) {
    const Fq2 A = fq2_sqr(T.X), B = fq2_sqr(T.Y), C = fq2_sqr(B), ZZ = fq2_sqr(T.Z);
    const Fq2 D = (fq2_sqr(T.X + B) - A - C).dbl(), E = A.dbl() + A, F = fq2_sqr(E);
    const Fq2 Z3 = (T.Y * T.Z).dbl();
    f = fq12_mul_by_line(f, E * T.X - B.dbl(), (E * ZZ).mul_fq(P.x).neg(), (Z3 * ZZ).mul_fq(P.y));
    const Fq2 X3 = F - D.dbl();
    T.Y = E * (D - X3) - C.dbl().dbl().dbl();
    T.X = X3;
    T.Z = Z3;
}
// f <- f * l_{T,Q}(P), T <- T + Q (T != +-Q in the loop).  Line through Q scaled by Z H (R = y_Q Z^3 - Y, H = x_Q Z^2 - X):
// l0 = R x_Q - y_Q Z H,  l1 = -R x_P,  l2 = Z H y_P
DP_D void miller_add_step(G2Jac &T, const G2Affine &Q, const G1Affine &P, Fq12 &f) {
    const Fq2 ZZ = fq2_sqr(T.Z), H = Q.x * ZZ - T.X, R = Q.y * T.Z * ZZ - T.Y, Z3 = T.Z * H;
    f = fq12_mul_by_line(f, R * Q.x - Q.y * Z3, R.mul_fq(P.x).neg(), Z3.mul_fq(P.y));
    const Fq2 HH = fq2_sqr(H), HHH = H * HH, V = T.X * HH;
    const Fq2 X3 = fq2_sqr(R) - HHH - V.dbl();
    T.Y = R * (V - X3) - T.Y * HHH;
    T.X = X3;
    T.Z = Z3;
}
// f_{|x|,Q}(P) without the final conjugation; P and Q finite
DP_D Fq12 miller_loop(const G1Affine &P, const G2Affine &Q) {
    G2Jac T{Q.x, Q.y, Fq2::one()};
    Fq12 f = Fq12::one();
    for (int bit = 62; bit >= 0; bit--) {  // bit 63 of |x| is the leading one
        f = fq12_sqr(f);
        miller_dbl_step(T, P, f);
        if ((PAIRING_ABS_X >> bit) & 1) miller_add_step(T, Q, P, f);
    }
    return f;
}

// ------------------------------------------------------------------------------------------------ final exponentiation
DP_D Fq12 cyclotomic_exp_abs_x(const Fq12 &g) {  // g^|x|
    Fq12 acc = g;
    for (int bit = 62; bit >= 0; bit--) {
        acc = fq12_cyclotomic_sqr(acc);
        if ((PAIRING_ABS_X >> bit) & 1) acc = acc * g;
    }
    return acc;
}
DP_D Fq12 cyclotomic_exp_x(const Fq12 &g) { return cyclotomic_exp_abs_x(g).conj(); }  // g^x, x < 0

// f^(3 (p^12 - 1) / r)
DP_D Fq12 final_exponentiation(const Fq12 &f) {
    const Fq12 t = f.conj() * fq12_inv(f);                          // f^(p^6 - 1)
    const Fq12 m = fq12_frob<2>(t) * t;                              // f^((p^6 - 1)(p^2 + 1)): cyclotomic from here
    Fq12 a = cyclotomic_exp_x(m) * m.conj();                         // m^(x - 1)
    a = cyclotomic_exp_x(a) * a.conj();                              // m^((x - 1)^2)
    const Fq12 b = cyclotomic_exp_x(a) * fq12_frob<1>(a);            // ... (x + p)
    const Fq12 c = cyclotomic_exp_x(cyclotomic_exp_x(b)) * fq12_frob<2>(b) * b.conj();  // ... (x^2 + p^2 - 1)
    return c * fq12_cyclotomic_sqr(m) * m;                           // ... + 3
}

// ------------------------------------------------------------------------------------------------ raw layouts and kernels
// raw ark 0.3 GroupAffine<g1::Parameters> (104 B = 13 u64) / GroupAffine<g2::Parameters> (200 B = 25 u64: x.c0, x.c1,
// y.c0, y.c1 in Montgomery Fq, the infinity flag in the low byte of word 24)
DP_D Fq load_fq_u64(const uint64_t *w) {
    Fq z;
#pragma unroll
    for (int k = 0; k < 6; k++) {
        z.l[2 * k] = (uint32_t)w[k];
        z.l[2 * k + 1] = (uint32_t)(w[k] >> 32);
    }
    return z;
}
DP_D void store_fq_u64(uint64_t *w, const Fq &a) {
#pragma unroll
    for (int k = 0; k < 6; k++) w[k] = (uint64_t)a.l[2 * k] | ((uint64_t)a.l[2 * k + 1] << 32);
}
DP_D G2Affine load_g2_ark(const uint64_t *w) {
    return G2Affine{Fq2{load_fq_u64(w), load_fq_u64(w + 6)}, Fq2{load_fq_u64(w + 12), load_fq_u64(w + 18)}, (w[24] & 0xff) != 0};
}
DP_D void store_g2_ark(uint64_t *w, const G2Affine &q) {  // identity = (0, 1, true), like GroupAffine::zero()
    const G2Affine o = q.inf ? G2Affine{Fq2::zero(), Fq2::one(), true} : q;
    store_fq_u64(w, o.x.c0);
    store_fq_u64(w + 6, o.x.c1);
    store_fq_u64(w + 12, o.y.c0);
    store_fq_u64(w + 18, o.y.c1);
    w[24] = o.inf ? 1 : 0;
}

// why a pair is rejected (dp_multi_pairing reports the first bad pair): 0 = fine
enum : uint32_t { PAIR_G1_NOT_FQ = 1, PAIR_G1_OFF_CURVE = 2, PAIR_G2_NOT_FQ = 3, PAIR_G2_OFF_TWIST = 4, PAIR_G2_NOT_TORSION = 5 };

DP_D uint32_t pairing_check_pair(const uint64_t *g1, const uint64_t *g2) {
    if ((g1[12] & 0xff) == 0) {
        const Fq x = load_fq_u64(g1), y = load_fq_u64(g1 + 6);
        if (!x.canon_is_reduced() || !y.canon_is_reduced()) return PAIR_G1_NOT_FQ;
        if (y.sqr() != x.sqr() * x + fq_from_u32(4)) return PAIR_G1_OFF_CURVE;
    }
    const G2Affine q = load_g2_ark(g2);
    if (!q.inf) {
        if (!q.x.c0.canon_is_reduced() || !q.x.c1.canon_is_reduced() || !q.y.c0.canon_is_reduced() || !q.y.c1.canon_is_reduced())
            return PAIR_G2_NOT_FQ;
        if (!q.on_twist()) return PAIR_G2_OFF_TWIST;
        uint32_t r[8];
#pragma unroll
        for (int k = 0; k < 8; k++) r[k] = FrParams::mod(k);
        if (!g2_mul(q, r).is_inf()) return PAIR_G2_NOT_TORSION;
    }
    return 0;
}

// Threads [0, k): the Miller value of pair t (1 when either point is the identity).  Threads [k, 2k): the input checks of
// pair t - k, at the same time; *bad = min((index + 1) << 8 | why) over the rejected pairs (~0 when none is).
__global__ void __launch_bounds__(64) pairing_miller_kernel(const uint64_t *g1, const uint64_t *g2, uint32_t k, Fq12 *f,
                                                            unsigned long long *bad) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < k) {
        const uint64_t *p = g1 + (uint64_t)t * 13;
        const G2Affine q = load_g2_ark(g2 + (uint64_t)t * 25);
        const bool trivial = (p[12] & 0xff) != 0 || q.inf;
        f[t] = trivial ? Fq12::one() : miller_loop(G1Affine{load_fq_u64(p), load_fq_u64(p + 6)}, q);
    } else if (t < 2 * k) {
        const uint32_t i = t - k;
        const uint32_t why = pairing_check_pair(g1 + (uint64_t)i * 13, g2 + (uint64_t)i * 25);
        if (why) atomicMin(bad, ((unsigned long long)(i + 1) << 8) | why);
    }
}

// One thread: the product of the k Miller values, conjugated (x < 0), to the power 3 (p^12 - 1) / r
__global__ void __launch_bounds__(32) pairing_final_kernel(const Fq12 *f, uint32_t k, const unsigned long long *bad, Fq12 *out) {
    if (threadIdx.x != 0 || *bad != ~0ull) return;
    Fq12 acc = Fq12::one();
    for (uint32_t i = 0; i < k; i++) acc = acc * f[i];
    *out = final_exponentiation(acc.conj());
}

// The G2 half of the KZG setup: out = H, tau H (raw 200-byte points); tau canonical, 0 < tau < r.  One thread.
__global__ void __launch_bounds__(32) g2_open_key_kernel(Fr tau, uint64_t *out) {
    if (threadIdx.x != 0) return;
    const G2Affine h = G2Affine::generator();
    store_g2_ark(out, h);
    store_g2_ark(out + 25, g2_mul(h, tau.l).to_affine());
}

// ------------------------------------------------------------------------------------------------ compressed G2 points
// ark-serialize 0.3 of GroupAffine<g2::Parameters>, 96 B = 24 u32: canonical x.c0 then x.c1, 48 little-endian bytes each;
// bit 7 of the last byte = (y > -y), bit 6 = infinity.  Fq2 is ordered by c1 first, then c0 (canonical integers).
DP_D bool fq2_is_larger_than_neg(const Fq2 &y) {  // Montgomery form; false for y = 0
    const Fq c1 = y.c1.from_mont();
    if (!c1.is_zero()) return Fq::canon_gt(c1, c1.neg());  // p is odd: c1 != -c1
    const Fq c0 = y.c0.from_mont();
    return Fq::canon_gt(c0, c0.neg());
}

// One thread per point; a file holds two of them.
__global__ void __launch_bounds__(32) g2_compress_kernel(const uint64_t *in, uint32_t *out, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const G2Affine q = load_g2_ark(in + i * 25);
    Fq x0 = Fq::zero(), x1 = Fq::zero();
    uint32_t flags = 1u << 30;
    if (!q.inf) {
        x0 = q.x.c0.from_mont();
        x1 = q.x.c1.from_mont();
        flags = fq2_is_larger_than_neg(q.y) ? 1u << 31 : 0u;
    }
    uint32_t *o = out + i * 24;
#pragma unroll
    for (int k = 0; k < 12; k++) {
        o[k] = x0.l[k];
        o[12 + k] = x1.l[k] | (k == 11 ? flags : 0u);
    }
}

// a^((p + 1) / 4): a square root of a when a is a square, of -a otherwise (p = 3 mod 4; g1_decompress_kernel's exponent)
DP_D Fq fq_sqrt_candidate(const Fq &a) {
    uint32_t e[12];  // the low limb ...aaab + 1 does not carry
#pragma unroll
    for (int k = 0; k < 12; k++) e[k] = FqParams::mod(k);
    e[0] += 1;
#pragma unroll
    for (int k = 0; k < 12; k++) e[k] = (e[k] >> 2) | (k < 11 ? e[k + 1] << 30 : 0);
    return a.pow_limbs(e, 12);
}
// A square root of a in Fq2 = Fq[u]/(u^2 + 1), if there is one.  a = (x0 + x1 u)^2 means x0^2 - x1^2 = a0 and 2 x0 x1 = a1,
// so x0^2 = (a0 +- alpha) / 2 with alpha^2 = a0^2 + a1^2, the norm.  With d = (a0 + alpha) / 2 and c = d^((p + 1) / 4):
// c^2 = d gives x0 = c, x1 = a1 / (2c); c^2 = -d (d is not a square, so the other sign is: their product is -a1^2 / 4)
// gives x1 = c, x0 = a1 / (2c).  Two exponentiations and one inversion; the caller squares the result to find out
// whether a was a square at all.  a1 = 0: c = a0^((p + 1) / 4) is the root itself, or u times it.
DP_D Fq2 fq2_sqrt_candidate(const Fq2 &a) {
    if (a.c1.is_zero()) {
        const Fq c = fq_sqrt_candidate(a.c0);
        return c.sqr() == a.c0 ? Fq2{c, Fq::zero()} : Fq2{Fq::zero(), c};
    }
    const Fq alpha = fq_sqrt_candidate(a.c0.sqr() + a.c1.sqr());
    Fq half = Fq::zero();  // (p + 1) / 2 = 1 / 2
#pragma unroll
    for (int k = 0; k < 12; k++) half.l[k] = FqParams::mod(k);
    half.l[0] += 1;
#pragma unroll
    for (int k = 0; k < 12; k++) half.l[k] = (half.l[k] >> 1) | (k < 11 ? half.l[k + 1] << 31 : 0);
    const Fq d = (a.c0 + alpha) * half.to_mont();
    const Fq c = fq_sqrt_candidate(d);
    if (c.is_zero()) return Fq2::zero();  // only when the norm is no square (then a is none either): d = 0 needs alpha = -a0
    const Fq other = a.c1 * c.dbl().inverse_vartime();
    return c.sqr() == d ? Fq2{c, other} : Fq2{other, c};
}

// One lane per point.  Reason codes as g1_decompress_kernel's: 1 a coordinate >= p, 2 both flags, 3 x^3 + 4 (u + 1) is not
// a square, 4 outside the r-torsion; *err = min((index + 1) << 8 | why).  Writes the raw 200-byte struct.
__global__ void __launch_bounds__(32) g2_decompress_kernel(const uint32_t *in, uint64_t *out, uint64_t n, uint32_t check_subgroup,
                                                           unsigned long long *err) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fq x0, x1;
#pragma unroll
    for (int k = 0; k < 12; k++) {
        x0.l[k] = in[i * 24 + k];
        x1.l[k] = in[i * 24 + 12 + k];
    }
    const bool positive = (x1.l[11] >> 31) & 1, infinity = (x1.l[11] >> 30) & 1;
    x1.l[11] &= 0x3fffffffu;
    uint32_t why = 0;
    G2Affine q{Fq2::zero(), Fq2::one(), true};
    if (positive && infinity) {
        why = 2;
    } else if (!infinity) {
        if (!x0.canon_is_reduced() || !x1.canon_is_reduced()) {
            why = 1;
        } else {
            const Fq2 x{x0.to_mont(), x1.to_mont()};
            const Fq2 rhs = fq2_sqr(x) * x + g2_b();
            const Fq2 y = fq2_sqrt_candidate(rhs);
            if (!(fq2_sqr(y) == rhs)) {
                why = 3;
            } else {
                q = G2Affine{x, fq2_is_larger_than_neg(y) == positive ? y : y.neg(), false};
                if (check_subgroup) {
                    uint32_t r[8];
#pragma unroll
                    for (int k = 0; k < 8; k++) r[k] = FrParams::mod(k);
                    if (!g2_mul(q, r).is_inf()) why = 4;
                }
            }
        }
    }
    if (why) {
        atomicMin(err, ((unsigned long long)(i + 1) << 8) | why);
        q = G2Affine{Fq2::zero(), Fq2::one(), true};
    }
    store_g2_ark(out + i * 25, q);
}

}  // namespace dp
