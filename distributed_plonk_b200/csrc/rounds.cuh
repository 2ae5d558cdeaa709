// Rounds 3-5 of Prover::prove on the GPU: the Fr arithmetic the dispatcher does between the transforms.
//
// "Next" row 1 of SURVEY.md §8(f).  The reference computes all of it serially on the dispatcher
// (src/dispatcher2.rs): the quotient's coset evaluations (363-504, one field division per element),
// polynomial evaluations at zeta (535-548), the linear combinations lin_poly / batch_poly (566-649)
// and the two divisions by (X - point) that give the opening witnesses (651-690).  With the
// polynomials resident on the worker these are four small families of kernels:
//   * quotient_kernel        one thread per point of the quotient domain, or of one n-point slice of it
//                            (DESIGN.md 3.4); the 1/(x_i - 1) of the L_1 term come from a cached table or
//                            from ONE inversion per block (product tree in shared memory); the tail variant
//                            adds the blinding coefficients of the wires and z as it loads them
//   * poly_fold_kernel       p(z): Horner per thread, tree per block, recursion over block results
//   * poly_suffix_kernel     E_j = sum_{k>=j} p_k z^(k-j): the quotient by (X - z) is E shifted by one,
//                            E_0 is the remainder p(z); same chunking, carries from a recursive scan
//   * poly_lincomb_kernel    sum_k c_k * p_k with zero extension
// Every result is a canonical Montgomery Fr, so equal values are equal bytes: parity with the
// reference's sequential code is bit-exact by construction, whatever the order of operations.
#pragma once
#include <type_traits>

#include "ntt.cuh"

namespace dp {

constexpr int RND_TPB = 256;
constexpr int QUO_TPB = 128;                                   // quotient kernel: ~150 registers per thread
constexpr int RND_LOG_ITEMS = 3;
constexpr int RND_ITEMS = 1 << RND_LOG_ITEMS;                  // coefficients per thread
constexpr int RND_LOG_CHUNK = 8 + RND_LOG_ITEMS;               // coefficients per block (2048)
constexpr uint64_t RND_CHUNK = (uint64_t)1 << RND_LOG_CHUNK;
constexpr int RND_MAX_POLYS = 32;
constexpr int RND_MAX_RATIO = 16;                              // quotient domain / gate domain (8 in the reference)
constexpr int RND_POW_TABLE = 80;                              // z^(2^j), j < 80

// ------------------------------------------------------------------ batch inversion inside a block
// Returns 1/d for every thread of a TPB-thread block (d != 0).  Up-sweep builds the product tree
// (tree[1] = product of all), the root is inverted, the down-sweep hands each child
// inv(parent) * sibling: ~3 multiplications per element.  The inverse of the root comes from
// *root_inv when the caller has it (computed for all blocks at once by a pre-pass, so that no block
// sits behind one thread's 380-multiplication exponentiation), else thread 0 computes it.
template <int TPB>
DP_D Fr block_batch_invert(const Fr &d, Fr *tree /* 2 * TPB */, const Fr *root_inv) {
    const uint32_t t = threadIdx.x;
    tree[TPB + t] = d;
    __syncthreads();
    for (uint32_t s = TPB >> 1; s >= 1; s >>= 1) {
        if (t < s) tree[s + t] = tree[2 * (s + t)] * tree[2 * (s + t) + 1];
        __syncthreads();
    }
    if (t == 0) tree[1] = root_inv ? gmem_ld(root_inv) : tree[1].inverse();
    __syncthreads();
    for (uint32_t s = 1; s < TPB; s <<= 1) {
        if (t < s) {
            const uint32_t node = s + t;
            const Fr iv = tree[node], l = tree[2 * node], r = tree[2 * node + 1];
            tree[2 * node] = iv * r;
            tree[2 * node + 1] = iv * l;
        }
        __syncthreads();
    }
    const Fr out = tree[TPB + t];
    __syncthreads();
    return out;
}

__global__ void fr_invert_kernel(Fr *x, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) gmem_st(x + i, gmem_ld(x + i).inverse());
}

// ------------------------------------------------------------------ round 3: quotient evaluations
// The quotient kernel is ~60 field multiplications of straight-line code per thread; inlined that is
// > 120 KB of instructions streamed through the instruction cache by every warp.  Calling the
// out-of-line multiplication keeps the kernel a few KB (the lesson of msm_reduce, which ran two orders of magnitude slower inlined).
DP_D Fr qmul(const Fr &a, const Fr &b) {
#if defined(__CUDA_ARCH__)
    return Fr::mul_outlined(a, b);
#else
    return a * b;
#endif
}

struct QuotientArgs {
    const Fr *sel[13];  // q_lc[4], q_mul[2], q_hash[4], q_o, q_c, q_ecc   (dispatcher2.rs:437-450)
    const Fr *sig[5];
    const Fr *w[5];
    const Fr *z;        // permutation product polynomial
    const Fr *pi;       // public input polynomial
    Fr k_beta[5];       // vk.k[j] * beta
    Fr alpha, beta, gamma, alpha_sq_div_n, gen;
    Fr zh_inv[RND_MAX_RATIO];  // 1 / (x_i^n - 1), i < ratio
    const Fr *H;        // omega_m^e, e < m/2
    const Fr *prod_inv; // per block: 1 / product of (x_i - 1), from the pre-pass
    const Fr *inv_xm1;  // TABLE variant: 1 / (x_i - 1) for every point of the coset (cached per quotient domain)
    uint64_t m;
    uint32_t log_m, ratio;
    // The points this launch covers: thread i < pts handles point pt = first + step * i of the quotient coset, reads the 25
    // inputs at i and z(omega x) at (i + z_next) mod pts, and writes out[pt].  The whole coset: first 0, step 1, pts m,
    // z_next = ratio.  Slice k (x = s_k omega_n^i, s_k = g omega_m^k): first k, step ratio, pts n, z_next 1.
    uint64_t pts;
    uint32_t first, step, z_next;
    Fr *out;
};

// Point set of one quotient launch (see QuotientArgs::pts)
struct QuotPts {
    uint64_t pts;
    uint32_t first, step;
};

// x_i - 1, x_i = g * omega_m^(first + step * i) (lines 366-369); 1 past the end of the point set.  g*H never meets 1.
DP_D Fr quotient_xm1(const Fr &gen, const Fr *H, uint32_t log_m, const QuotPts &s, uint64_t i, Fr &x) {
    x = i < s.pts ? gen * tw_lookup(H, s.first + (uint64_t)s.step * i, log_m, 0) : Fr::one() + Fr::one();
    return x - Fr::one();
}

// pre-pass: prod[b] = product of (x_i - 1) over the points of quotient block b
__global__ void __launch_bounds__(QUO_TPB) quotient_xm1_products_kernel(Fr gen, const Fr *H, uint32_t log_m, QuotPts ps, Fr *prod) {
    __shared__ Fr sh[QUO_TPB];
    const uint32_t t = threadIdx.x;
    Fr x;
    sh[t] = quotient_xm1(gen, H, log_m, ps, (uint64_t)blockIdx.x * QUO_TPB + t, x);
    __syncthreads();
    for (uint32_t s = QUO_TPB >> 1; s >= 1; s >>= 1) {
        if (t < s) sh[t] = sh[t] * sh[t + s];
        __syncthreads();
    }
    if (t == 0) gmem_st(prod + blockIdx.x, sh[0]);
}

// The 1/(x_i - 1) depend on the quotient domain only, not on the proof: with a worker that keeps its polynomials
// resident they are computed ONCE per dp_init (first quotient call) into a table of m Fr - the per-block product
// tree, its 14 block-wide barriers and the pre-pass (one inversion per block) leave the per-proof path, which
// becomes straight-line code without shared memory (r02 ncu: 25 % of the warp samples of the tree variant sat at
// those barriers).  dplonk.cu falls back to the tree variant when the table (32 B per point) does not fit.
__global__ void __launch_bounds__(QUO_TPB) quotient_inv_table_kernel(Fr gen, const Fr *H, uint32_t log_m, uint64_t m, const Fr *prod_inv,
                                                                     Fr *table) {
    __shared__ Fr tree[2 * QUO_TPB];
    const uint64_t i = (uint64_t)blockIdx.x * QUO_TPB + threadIdx.x;
    Fr x;
    const Fr xm1 = quotient_xm1(gen, H, log_m, QuotPts{m, 0, 1}, i, x);
    const Fr inv = block_batch_invert<QUO_TPB>(xm1, tree, prod_inv + blockIdx.x);
    if (i < m) gmem_st(table + i, inv);
}

// Blinded inputs (DESIGN.md 3.4): a wire or z with n + t coefficients (t <= 3) is p = head + X^n tail.  The 25 arrays hold
// the evaluations of the heads (n coefficients, the usual coset transforms); the kernel adds x^n tail(x) to each blinded
// input as it loads it, and x^n tail(omega_n x) to z(omega x), since (omega_n x)^n = x^n.  x^n takes one value per slice
// class pt mod ratio: the same constants whose inverses zh_inv holds shifted by one.
constexpr uint32_t RND_MAX_TAIL = 3;
struct QuotientTailArgs : QuotientArgs {
    const Fr *w_tail[5];   // coefficients n, n+1, ... of each wire (device; read by every thread)
    const Fr *z_tail;
    uint32_t w_tail_len[5], z_tail_len;
    Fr xn[RND_MAX_RATIO];  // x_i^n, i < ratio
    Fr omega_n;
};

// t[0] + t[1] y + ... + t[len - 1] y^(len - 1), len <= RND_MAX_TAIL (uniform across the launch): len - 1 products
DP_D Fr quotient_tail_at(const Fr *t, uint32_t len, const Fr &y) {
    Fr acc = Fr::zero();
#pragma unroll
    for (int j = (int)RND_MAX_TAIL - 1; j >= 0; j--) {
        if ((uint32_t)j + 1 < len) acc = qmul(acc, y) + gmem_ld(t + j);
        else if ((uint32_t)j + 1 == len) acc = gmem_ld(t + j);
    }
    return acc;
}

// Accumulating form (batch proofs, DESIGN.md 3.11): out[pt] += scale * quotient(pt).  The host folds the scale into zh_inv[]
// and alpha_sq_div_n, so the kernel's extra work is one load and one addition.  A distinct argument type rather than a
// template flag, so the plain and tail instantiations keep their names and their code.
template <typename Base>
struct QuotientAcc : Base {};

template <bool TABLE, typename Args = QuotientArgs>
__global__ void __launch_bounds__(QUO_TPB) quotient_kernel(Args q) {
    constexpr bool TAIL = std::is_base_of<QuotientTailArgs, Args>::value;
    constexpr bool ACC = std::is_same<Args, QuotientAcc<QuotientArgs>>::value || std::is_same<Args, QuotientAcc<QuotientTailArgs>>::value;
    const uint64_t i = (uint64_t)blockIdx.x * QUO_TPB + threadIdx.x;
    const bool live = i < q.pts;
    const uint64_t pt = q.first + (uint64_t)q.step * i;  // the point's index in the quotient coset
    const Fr one = Fr::one();
    Fr x, inv_xm1;
    if (TABLE) {
        if (!live) return;
        x = q.gen * tw_lookup(q.H, pt, q.log_m, 0);
        inv_xm1 = gmem_ld(q.inv_xm1 + pt);
    } else {
        __shared__ Fr tree[2 * QUO_TPB];
        const Fr xm1 = quotient_xm1(q.gen, q.H, q.log_m, QuotPts{q.pts, q.first, q.step}, i, x);
        inv_xm1 = block_batch_invert<QUO_TPB>(xm1, tree, q.prod_inv ? q.prod_inv + blockIdx.x : nullptr);
        if (!live) return;
    }
    Fr a = gmem_ld(q.w[0] + i), b = gmem_ld(q.w[1] + i), c = gmem_ld(q.w[2] + i), d = gmem_ld(q.w[3] + i), e = gmem_ld(q.w[4] + i);
    if constexpr (TAIL) {
        const Fr xn = q.xn[pt % q.ratio];
        auto blind = [&](Fr &w, int j) {
            if (q.w_tail_len[j]) w = w + qmul(xn, quotient_tail_at(q.w_tail[j], q.w_tail_len[j], x));
        };
        blind(a, 0), blind(b, 1), blind(c, 2), blind(d, 3), blind(e, 4);
    }
    const Fr ab = qmul(a, b), cd = qmul(c, d);
    // gate constraint (lines 451-472)
    Fr gate = gmem_ld(q.sel[11] + i) + gmem_ld(q.pi + i);
    gate = gate + qmul(gmem_ld(q.sel[0] + i), a) + qmul(gmem_ld(q.sel[1] + i), b) + qmul(gmem_ld(q.sel[2] + i), c) + qmul(gmem_ld(q.sel[3] + i), d);
    gate = gate + qmul(gmem_ld(q.sel[4] + i), ab) + qmul(gmem_ld(q.sel[5] + i), cd);
    gate = gate + qmul(gmem_ld(q.sel[12] + i), qmul(qmul(ab, cd), e));
    const Fr wv[5] = {a, b, c, d, e};
#pragma unroll
    for (int j = 0; j < 4; j++) {  // q_hash[j] * w_j^5
        const Fr w2 = qmul(wv[j], wv[j]);
        gate = gate + qmul(gmem_ld(q.sel[6 + j] + i), qmul(qmul(w2, w2), wv[j]));
    }
    gate = gate - qmul(gmem_ld(q.sel[10] + i), e);
    // permutation constraint (lines 473-491): z(X) prod(w + beta k X + gamma) - z(omega X) prod(w + beta sigma + gamma)
    Fr zi = gmem_ld(q.z + i), zw = gmem_ld(q.z + ((i + q.z_next) & (q.pts - 1)));
    if constexpr (TAIL) {
        if (q.z_tail_len) {
            const Fr xn = q.xn[pt % q.ratio];
            zi = zi + qmul(xn, quotient_tail_at(q.z_tail, q.z_tail_len, x));
            zw = zw + qmul(xn, quotient_tail_at(q.z_tail, q.z_tail_len, qmul(q.omega_n, x)));
        }
    }
    Fr acc1 = zi, acc2 = zw;
#pragma unroll
    for (int j = 0; j < 5; j++) {
        const Fr t = wv[j] + q.gamma;
        acc1 = qmul(acc1, t + qmul(q.k_beta[j], x));
        acc2 = qmul(acc2, t + qmul(gmem_ld(q.sig[j] + i), q.beta));
    }
    Fr r = qmul(q.zh_inv[pt % q.ratio], gate + qmul(q.alpha, acc1 - acc2));
    // (z - 1) L_1 alpha^2 / Z_H = alpha^2/n (z - 1) / (x - 1)   (lines 493-499)
    r = r + qmul(qmul(q.alpha_sq_div_n, zi - one), inv_xm1);
    if constexpr (ACC) r = r + gmem_ld(q.out + pt);
    gmem_st(q.out + pt, r);
}

// ------------------------------------------------------------------ p(z) and the suffix Horner scan
// pw[j] = z^(2^j).  A call at exponent e works with the point y = pw[e] (the recursion levels use
// y = z^(2048^level)): threads step with y, thread blocks combine with y^(8 * 2^l) = pw[e + 3 + l].

// Horner over this thread's RND_ITEMS coefficients (zero beyond n)
DP_D Fr thread_fold(const Fr *in, uint64_t n, uint64_t base, const Fr &y) {
    Fr acc = Fr::zero();
    for (int k = RND_ITEMS - 1; k >= 0; k--) {
        acc = acc * y;
        if (base + k < n) acc = acc + gmem_ld(in + base + k);
    }
    return acc;
}

// out[b] = sum_{k in chunk b} in[k] * y^(k - 2048 b)
__global__ void __launch_bounds__(RND_TPB) poly_fold_kernel(const Fr *in, uint64_t n, const Fr *pw, uint32_t e, Fr *out) {
    __shared__ Fr sh[RND_TPB];
    const uint32_t t = threadIdx.x;
    const uint64_t base = (uint64_t)blockIdx.x * RND_CHUNK + (uint64_t)t * RND_ITEMS;
    sh[t] = thread_fold(in, n, base, gmem_ld(pw + e));
    __syncthreads();
    uint32_t lvl = 0;
    for (uint32_t s = 1; s < RND_TPB; s <<= 1, lvl++) {
        if ((t & (2 * s - 1)) == 0) sh[t] = sh[t] + sh[t + s] * gmem_ld(pw + e + RND_LOG_ITEMS + lvl);
        __syncthreads();
    }
    if (t == 0) gmem_st(out + blockIdx.x, sh[0]);
}

// E_j = in[j] + y * E_(j+1), E_n = 0.  carry[b + 1] = E at the first coefficient of chunk b + 1 (from the
// recursive scan of the fold results; nullptr when there is a single chunk).  E_j is stored at
// out[j - shift] (shift = 1 drops E_0, which goes to *rem when rem != nullptr).
__global__ void __launch_bounds__(RND_TPB) poly_suffix_kernel(const Fr *in, uint64_t n, const Fr *pw, uint32_t e, const Fr *carry,
                                                               uint64_t n_chunks, Fr *out, uint32_t shift, Fr *rem) {
    __shared__ Fr sh[RND_TPB];
    const uint32_t t = threadIdx.x;
    const uint64_t base = (uint64_t)blockIdx.x * RND_CHUNK + (uint64_t)t * RND_ITEMS;
    const Fr y = gmem_ld(pw + e);
    const Fr block_carry = (carry && blockIdx.x + 1 < n_chunks) ? gmem_ld(carry + blockIdx.x + 1) : Fr::zero();
    Fr f = thread_fold(in, n, base, y);
    if (t == RND_TPB - 1) f = f + block_carry * gmem_ld(pw + e + RND_LOG_ITEMS);  // the carry enters above the last thread
    sh[t] = f;
    __syncthreads();
    // inclusive suffix scan over the threads: sh[t] = sum_{u >= t} f_u y^(8 (u - t))
    uint32_t lvl = 0;
    for (uint32_t off = 1; off < RND_TPB; off <<= 1, lvl++) {
        Fr v = sh[t];
        if (t + off < RND_TPB) v = v + sh[t + off] * gmem_ld(pw + e + RND_LOG_ITEMS + lvl);
        __syncthreads();
        sh[t] = v;
        __syncthreads();
    }
    Fr E = t + 1 < RND_TPB ? sh[t + 1] : block_carry;  // E just above this thread's coefficients
    for (int k = RND_ITEMS - 1; k >= 0; k--) {
        const uint64_t j = base + k;
        if (j >= n) continue;  // E stays 0 above the top coefficient
        E = gmem_ld(in + j) + y * E;
        if (j >= shift) gmem_st(out + j - shift, E);
        else if (rem) gmem_st(rem, E);
    }
}

// ------------------------------------------------------------------ round 5: linear combinations
struct LincombArgs {
    const Fr *poly[RND_MAX_POLYS];
    uint64_t len[RND_MAX_POLYS];
    Fr coeff[RND_MAX_POLYS];
    uint32_t k;
    uint64_t out_len;
    Fr *out;
};

__global__ void poly_lincomb_kernel(LincombArgs a) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= a.out_len) return;
    Fr acc = Fr::zero();
    for (uint32_t i = 0; i < a.k; i++)
        if (j < a.len[i]) acc = acc + gmem_ld(a.poly[i] + j) * a.coeff[i];
    gmem_st(a.out + j, acc);
}

}  // namespace dp
