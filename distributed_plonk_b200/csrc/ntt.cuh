// NTT / iNTT over BLS12-381 Fr for sm_90a.
//
// Replaces ark-poly 0.3.0 Radix2EvaluationDomain::{fft,ifft}_in_place and the per-element
// Fr::pow coset / twiddle loops around it in the reference worker:
//   src/worker.rs:66-94   fft1_helper  (coset pre-scale, size-c (i)NTT, omega^(i*j) twiddle)
//   src/worker.rs:96-115  fft2_helper  (size-r (i)NTT, inverse-coset post-scale)
//   src/worker.rs:398     whole-domain ifft_in_place (round1)
//   src/playground.rs:21-80 the 2-D decomposition these implement
//
// One kernel does all of it: `ntt_tile_kernel` runs a batch of K-point sub-DFTs (K = 2^log_k) for
// G "lanes" at a time out of a (K x G)-element shared-memory tile (K*G = 2048 elements = 64 KiB),
// radix-4 decimation-in-frequency butterflies in registers, natural-order in / natural-order out
// (the bit reversal is done in the shared-memory read-out addressing), with fused
//   * input scaling   v *= A[..] * B[..]        (forward coset  g^(i + j*r))
//   * output twiddle  v *= omega_N^(+-e(o,lane,f))  from the per-domain half table
//   * output scaling  v *= A[..] * B[..] * const  (inverse coset g^-(i+j*c), 1/size)
// Every transform is a short list of such passes with explicit element strides (NttPass), so the
// same kernel serves the worker's row phase, column phase, the four-step split of long rows and
// the whole-domain transform.  The per-stage butterfly twiddles (omega_{2^(s+1)}^j, stage-major,
// K entries) are staged into shared memory by a 1-D bulk TMA copy (cp.async.bulk + mbarrier)
// that overlaps the tile load.
//
// HBM traffic per pass: 64 B per element (32 B read + 32 B written) + 32 B twiddle-table read
// when a pass applies the omega_N twiddle; no tensor cores (modular arithmetic, not a contraction).
#pragma once
#include "rt.cuh"

namespace dp {

constexpr int NTT_TPB = 256;
constexpr uint32_t NTT_TILE_LOG = 11;  // elements per tile (K * G)
constexpr uint32_t NTT_WTAB_LOG = 11;  // largest K the level table covers
constexpr uint32_t NTT_MAX_STRIDED_LOG_K = 9;   // keep G >= 4 lanes (128 B) when lanes are the contiguous axis

// 2^32-th root of unity 7^((r-1)/2^32), Montgomery form (ark FrParameters::TWO_ADIC_ROOT_OF_UNITY)
DP_HD Fr fr_two_adic_root() {
    Fr w;
    const uint32_t c[8] = {0x5f0e466au, 0xb9b58d8cu, 0x1819d7ecu, 0x5b1b4c80u,
                           0x52a31e64u, 0x0af53ae3u, 0x19e9b27bu, 0x5bf3addau};
    for (int i = 0; i < 8; i++) w.l[i] = c[i];
    return w;
}
// Radix2EvaluationDomain::new(2^log_size).group_gen
DP_HD Fr fr_domain_gen(uint32_t log_size) {
    Fr w = fr_two_adic_root();
    for (uint32_t i = log_size; i < 32; i++) w = w.sqr();
    return w;
}
DP_HD Fr fr_from_u64(uint64_t v) {
    Fr x = Fr::zero();
    x.l[0] = (uint32_t)v;
    x.l[1] = (uint32_t)(v >> 32);
    return x.to_mont();
}

struct NttPass {
    const Fr *in;
    Fr *out;
    uint32_t log_k, log_g;   // sub-DFT size, lanes per tile
    uint32_t lane_tiles;     // n_lanes / G   (grid = n_outer * lane_tiles)
    uint32_t n_outer;
    uint64_t in_os, in_ls, in_ps;     // element strides: outer, lane, point
    uint64_t out_os, out_ls, out_ps;
    // output element address = out + o*out_os + lane*out_ls + S(lane*out_lc + f*out_ps) where S is the
    // identity, or (exchange layout, W blocks of [rows][cols/W]) S(k) = (k >> split_log)*split_stride
    // + (k & (2^split_log - 1)):  the pack step of worker.rs:327-330 fused into the store
    uint64_t out_lc, split_stride;
    uint32_t split_on, split_log;
    // fused exchange over peer memory: block q of the exchange layout is not a slice of `out` but
    // the receive matrix of worker q, mapped into this process through CUDA IPC (NVLink stores):
    //   address = peer_base[k >> split_log] + peer_row_off + o*out_os + lane*out_ls + (k & mask)
    // This is PlonkPeer.fftExchange (worker.rs:327-330 send side + 432-435 scatter side) done by the
    // row kernel's own epilogue, tile by tile, while other tiles are still computing.
    uint32_t peer_on;
    uint64_t peer_row_off;
    Fr *peer_base[8];
    const uint4 *w_lo, *w_hi;         // stage-major butterfly twiddles, plane-split, >= K entries
    // output twiddle omega_N^(+-e),  e = (tw_la*lane + tw_oa*o + tw_c0) * (tw_fb*f + tw_lb*lane)
    const Fr *tw_tab;                 // omega_N^e, e < N/2   (nullptr = no twiddle)
    uint32_t tw_log_n, tw_inverse;
    uint64_t tw_la, tw_oa, tw_c0, tw_fb, tw_lb;
    // input scaling  v *= pre_a[pa_o*o + pa_l*lane] * pre_b[pb_m*m + pb_l*lane]   (nullptr = none)
    const Fr *pre_a, *pre_b;
    uint64_t pa_o, pa_l, pb_m, pb_l;
    // output scaling v *= post_a[qa_o*o + qa_l*lane] * post_b[qb_o*o + qb_f*f + qb_l*lane] (nullptr = none)
    const Fr *post_a, *post_b;
    uint64_t qa_o, qa_l, qb_o, qb_f, qb_l;
    uint32_t post_const_on;           // v *= post_const
    Fr post_const;
    // Zero-padded input: only points m < 2^(log_k - in_zlog) of every lane are read, the rest are implicit zeros
    // (in_zlog == 0: everything is read).  This is the shape of 25 of the 33 transforms of a proof:
    // n coefficients on the 8n-point quotient domain (dispatcher2.rs:386-388).  The first in_zlog
    // butterfly stages then have a zero upper input each and collapse into ONE product per element,
    // out[j + V*t] = x[j] * omega_K^(j * bitrev(t)), instead of a load and up to three products.
    uint32_t in_zlog;
    // Order in which the threads of a block walk the tile when it is loaded / stored, and the element address that goes
    // with it: work item = a + A * (lane + G * b) with A = 2^a_log "fast" point values and the rest "slow" ones;
    //   point index  = a + A * b                      (a_hi == 0)      or   b + (points / A) * a      (a_hi == 1)
    //   address      = o * os + lane * ls + a * ps_a + b * ps_b
    // Threads with consecutive a (then consecutive lanes) touch consecutive addresses when ps_a = 1 and ls = A.
    // a_log = log2(points): points contiguous (ps_a = 1);  a_log = 0: lanes contiguous, points strided by ps_b;
    // 0 < a_log < log2(points), a_hi = 1: the point index is made of two digit groups that are contiguous runs of
    // A elements strided by ps_b - the middle pass of the three-pass single-worker plan.  Filled in by launch_pass()
    // from in_ps / out_ps unless map_set.
    uint32_t map_set, in_a_log, in_a_hi, out_a_log, out_a_hi;
    uint64_t in_ps_a, in_ps_b, out_ps_a, out_ps_b;
    uint32_t tw_prefetch;             // experiment knob: pull the epilogue's omega_N twiddles towards L2 while the tile is transformed
};

// ------------------------------------------------------------------ shared-memory element access
// An Fr is kept as two 16-byte halves in separate planes so that consecutive element indices are
// conflict-free for LDS.128 / STS.128.
DP_D Fr smem_ld(const uint4 *lo, const uint4 *hi, uint32_t e) {
    Fr v;
    uint4 a = lo[e], b = hi[e];
    v.l[0] = a.x; v.l[1] = a.y; v.l[2] = a.z; v.l[3] = a.w;
    v.l[4] = b.x; v.l[5] = b.y; v.l[6] = b.z; v.l[7] = b.w;
    return v;
}
DP_D void smem_st(uint4 *lo, uint4 *hi, uint32_t e, const Fr &v) {
    lo[e] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    hi[e] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}
DP_D Fr gmem_ld(const Fr *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    uint4 a = q[0], b = q[1];
    Fr v;
    v.l[0] = a.x; v.l[1] = a.y; v.l[2] = a.z; v.l[3] = a.w;
    v.l[4] = b.x; v.l[5] = b.y; v.l[6] = b.z; v.l[7] = b.w;
    return v;
}
DP_D void gmem_st(Fr *p, const Fr &v) {
    uint4 *q = reinterpret_cast<uint4 *>(p);
    q[0] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    q[1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}

// omega_N^(+-e) from the half table H[e] = omega_N^e, e < N/2  (omega^(N/2) = -1)
DP_D Fr tw_lookup(const Fr *H, uint64_t e, uint32_t log_n, uint32_t inverse) {
    const uint64_t n = (uint64_t)1 << log_n, half = n >> 1;
    e &= n - 1;
    if (inverse) e = (n - e) & (n - 1);
    const bool neg = half != 0 && e >= half;  // (a one-element domain has no -1 half)
    if (neg) e -= half;
    Fr w = gmem_ld(H + e);
    return neg ? w.neg() : w;
}

// ------------------------------------------------------------------ TMA bulk copy of the level table
#if !defined(DP_EMUL)
DP_D uint32_t smem_addr_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
DP_D void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
DP_D void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr_u32(bar)), "r"(bytes)
                 : "memory");
}
DP_D void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_addr_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_addr_u32(bar))
        : "memory");
}
DP_D void mbar_wait(uint64_t *bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_addr_u32(bar)),
        "r"(phase)
        : "memory");
}
// 16-byte asynchronous copy global -> shared (LDGSTS): the tile load needs no registers and every thread's
// copies are in flight together instead of one dependent load-store pair after the other
DP_D void cp_async16(void *dst_smem, const void *src_gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr_u32(dst_smem)), "l"(src_gmem) : "memory");
}
DP_D void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}
DP_D void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
#else
DP_D void cp_async16(void *dst_smem, const void *src_gmem) { memcpy(dst_smem, src_gmem, 16); }
DP_D void cp_async_wait_all() {}
DP_D void prefetch_l2(const void *) {}
#endif

// work item -> (point index, lane, fast digit a, slow digit b) for the tile walk described at NttPass::in_a_log
struct TileIdx {
    uint32_t pt, g, a, b;
};
DP_D TileIdx tile_idx(uint32_t idx, uint32_t a_log, uint32_t a_hi, uint32_t log_g, uint32_t log_pts) {
    TileIdx t;
    t.a = idx & ((1u << a_log) - 1);
    t.g = (idx >> a_log) & ((1u << log_g) - 1);
    t.b = idx >> (a_log + log_g);
    t.pt = a_hi ? t.b + (t.a << (log_pts - a_log)) : t.a + (t.b << a_log);
    return t;
}

// dynamic shared memory: [lo plane | hi plane] of G*(K+1) uint4 each, [w_lo | w_hi] of K uint4 each,
// one 8-byte mbarrier
DP_HD size_t ntt_pass_smem_bytes(uint32_t log_k, uint32_t log_g) {
    size_t K = (size_t)1 << log_k, G = (size_t)1 << log_g;
    return 2 * G * (K + 1) * 16 + 2 * K * 16 + 16;
}

// MINB = resident CTAs per SM the register allocation aims for: 2 (<= 128 registers) or 3 (<= 85; three 64-70 KB tiles
// fit the 227 KB of shared memory): more warps to cover the dependent carry chains and the table loads
template <int MINB>
__global__ void __launch_bounds__(NTT_TPB, MINB) ntt_tile_kernel(NttPass p) {
    DP_DYN_SMEM(smem_raw);
    const uint32_t K = 1u << p.log_k, G = 1u << p.log_g, tile = K * G, pitch = K + 1;
    uint4 *lo = reinterpret_cast<uint4 *>(smem_raw);
    uint4 *hi = lo + (size_t)G * pitch;
    uint4 *wlo = hi + (size_t)G * pitch;
    uint4 *whi = wlo + K;
    uint64_t *bar = reinterpret_cast<uint64_t *>(whi + K);
    const uint32_t tid = threadIdx.x;

    const uint32_t o = blockIdx.x / p.lane_tiles;
    const uint32_t lane0 = (blockIdx.x % p.lane_tiles) * G;

    // ---- stage the butterfly twiddles (TMA bulk copy, overlaps the tile load below)
#if defined(DP_EMUL)
    (void)bar;
    if (tid == 0) {
        memcpy(wlo, p.w_lo, (size_t)K * 16);
        memcpy(whi, p.w_hi, (size_t)K * 16);
    }
#else
    if (tid == 0) mbar_init(bar, 1);
    __syncthreads();  // nobody may wait on the barrier before it is initialised (tiny tiles get here at once)
    if (tid == 0) {
        mbar_expect_tx(bar, 2 * K * 16);
        tma_bulk_g2s(wlo, p.w_lo, K * 16, bar);
        tma_bulk_g2s(whi, p.w_hi, K * 16, bar);
    }
#endif

    // ---- the omega_N twiddles of the epilogue are known now: optionally pull them towards L2 while the tile is loaded
    // and transformed (the table of a 2^25-point domain is 512 MiB; a demand miss in the store loop costs ~1 us).
    // Off by default: the prefetches add DRAM reads of their own to the 2-D twiddle pass.
    if (p.tw_tab && p.tw_prefetch) {
        const uint64_t n_tw = (uint64_t)1 << p.tw_log_n, half_tw = n_tw >> 1;
        for (uint32_t idx = tid; idx < tile; idx += NTT_TPB) {
            const TileIdx ti = tile_idx(idx, p.out_a_log, p.out_a_hi, p.log_g, p.log_k);
            const uint32_t f = ti.pt, g = ti.g;
            const uint64_t lane = lane0 + g;
            uint64_t e = ((p.tw_la * lane + p.tw_oa * o + p.tw_c0) * (p.tw_fb * f + p.tw_lb * lane)) & (n_tw - 1);
            if (p.tw_inverse) e = (n_tw - e) & (n_tw - 1);
            if (half_tw && e >= half_tw) e -= half_tw;
            prefetch_l2(p.tw_tab + e);
        }
    }

    // ---- load the tile (natural point order) with asynchronous 16-byte copies straight into the two planes
    const uint32_t vlog = p.log_k - p.in_zlog, V = 1u << vlog;  // points >= V of every lane are implicit zeros
    {
        const Fr *src = p.in + (uint64_t)o * p.in_os + (uint64_t)lane0 * p.in_ls;
        const uint32_t n_ld = G << vlog;
        for (uint32_t idx = tid; idx < n_ld; idx += NTT_TPB) {
            const TileIdx ti = tile_idx(idx, p.in_a_log, p.in_a_hi, p.log_g, vlog);
            const uint32_t m = ti.pt, g = ti.g;
            const uint4 *q = reinterpret_cast<const uint4 *>(src + (uint64_t)g * p.in_ls + (uint64_t)ti.a * p.in_ps_a + (uint64_t)ti.b * p.in_ps_b);
            cp_async16(lo + g * pitch + m, q);
            cp_async16(hi + g * pitch + m, q + 1);
        }
        cp_async_wait_all();
        // fused input scaling, in place, every thread on the elements it copied itself (no barrier needed).
        // Zero inputs stay zero: whole warps skip both products on padded data.
        if (p.pre_a) {
            for (uint32_t idx = tid; idx < n_ld; idx += NTT_TPB) {
                const TileIdx ti = tile_idx(idx, p.in_a_log, p.in_a_hi, p.log_g, vlog);
                const uint32_t m = ti.pt, g = ti.g;
                Fr v = smem_ld(lo, hi, g * pitch + m);
                if (!v.is_zero()) {
                    const uint64_t lane = lane0 + g;
                    v = v * gmem_ld(p.pre_a + p.pa_o * o + p.pa_l * lane);
                    v = v * gmem_ld(p.pre_b + p.pb_m * m + p.pb_l * lane);
                    smem_st(lo, hi, g * pitch + m, v);
                }
            }
        }
    }
#if !defined(DP_EMUL)
    mbar_wait(bar, 0);
#endif
    __syncthreads();

    // Work-item order of the in-tile stages.  A quarter-warp (8 threads) is conflict-free for 16-byte accesses when its
    // elements fall into 8 different 16-byte bank groups.  With the point index fastest that fails for the short-span
    // stages (elements 4 apart: 4-way conflicts in the last radix-4 pair, 2-way in the one before - 84 % extra
    // shared-memory wavefronts per tile, ncu r02a).  With the LANE index fastest the eight threads sit in eight lanes,
    // pitch K + 1 elements apart, i.e. in eight different bank groups whatever the stage; they also share one twiddle.
    const bool lanes_fast = G >= 8;
    // ---- zero-padded input: the stages whose upper input is zero, as one product per element
    int s = (int)vlog - 1;
    if (p.in_zlog) {
        const uint32_t z = p.in_zlog, halfK = K >> 1;
        for (uint32_t idx = tid; idx < tile; idx += NTT_TPB) {
            const uint32_t g = lanes_fast ? idx & (G - 1) : idx >> p.log_k, mm = lanes_fast ? idx >> p.log_g : idx & (K - 1);
            const uint32_t t = mm >> vlog, j = mm & (V - 1);
            if (t == 0) continue;                                   // x[j] itself stays where it is
            Fr v = smem_ld(lo, hi, g * pitch + j);
            uint32_t e = j * (__brev(t) >> (32 - z));                // < K
            if (e) {
                const bool neg = e >= halfK;
                if (neg) e -= halfK;
                if (e) v = v * smem_ld(wlo, whi, halfK + e);        // W[K/2 + e] = omega_K^(+-e)
                if (neg) v = v.neg();
            }
            smem_st(lo, hi, g * pitch + mm, v);
        }
        __syncthreads();
    }

    // ---- butterflies: decimation in frequency, stages s .. 0
    if ((s + 1) & 1) {  // one radix-2 stage on top so that the rest pairs up
        const uint32_t span = 1u << s, units = tile >> 1, upl = K >> 1;  // units per lane
        for (uint32_t u = tid; u < units; u += NTT_TPB) {
            const uint32_t g = lanes_fast ? u & (G - 1) : u >> (p.log_k - 1), uu = lanes_fast ? u >> p.log_g : u & (upl - 1);
            const uint32_t j = uu & (span - 1);
            const uint32_t m0 = ((uu >> s) << (s + 1)) | j;
            const uint32_t e0 = g * pitch + m0, e1 = e0 + span;
            Fr a = smem_ld(lo, hi, e0), b = smem_ld(lo, hi, e1);
            Fr d = a - b;
            a = a + b;
            if (s > 0) d = d * smem_ld(wlo, whi, span + j);
            smem_st(lo, hi, e0, a);
            smem_st(lo, hi, e1, d);
        }
        __syncthreads();
        s--;
    }
    for (; s >= 1; s -= 2) {  // radix-4: stages s and s-1
        const int sl = s - 1;
        const uint32_t q = 1u << sl, units = tile >> 2, upl = K >> 2;
        for (uint32_t u = tid; u < units; u += NTT_TPB) {
            const uint32_t g = lanes_fast ? u & (G - 1) : u >> (p.log_k - 2), uu = lanes_fast ? u >> p.log_g : u & (upl - 1);
            const uint32_t j = uu & (q - 1);
            const uint32_t m0 = ((uu >> sl) << (sl + 2)) | j;
            const uint32_t e0 = g * pitch + m0;
            Fr x0 = smem_ld(lo, hi, e0), x1 = smem_ld(lo, hi, e0 + q);
            Fr x2 = smem_ld(lo, hi, e0 + 2 * q), x3 = smem_ld(lo, hi, e0 + 3 * q);
            // stage s (span 2q): (x0,x2) with T_s[j], (x1,x3) with T_s[j+q]
            Fr b0 = x0 + x2, b2 = x0 - x2;
            if (sl > 0) b2 = b2 * smem_ld(wlo, whi, 2 * q + j);  // sl == 0: T_1[0] = 1
            Fr b1 = x1 + x3, b3 = (x1 - x3) * smem_ld(wlo, whi, 2 * q + j + q);
            // stage s-1 (span q): (b0,b1), (b2,b3) with T_{s-1}[j]
            Fr c0 = b0 + b1, c1 = b0 - b1, c2 = b2 + b3, c3 = b2 - b3;
            if (sl > 0) {
                const Fr w = smem_ld(wlo, whi, q + j);
                c1 = c1 * w;
                c3 = c3 * w;
            }
            smem_st(lo, hi, e0, c0);
            smem_st(lo, hi, e0 + q, c1);
            smem_st(lo, hi, e0 + 2 * q, c2);
            smem_st(lo, hi, e0 + 3 * q, c3);
        }
        __syncthreads();
    }

    // ---- write out (frequency f sits at bit-reversed position), fused twiddle / scaling
    {
        Fr *dst = p.out + (uint64_t)o * p.out_os;
#pragma unroll 2
        for (uint32_t idx = tid; idx < tile; idx += NTT_TPB) {
            const TileIdx ti = tile_idx(idx, p.out_a_log, p.out_a_hi, p.log_g, p.log_k);
            const uint32_t f = ti.pt, g = ti.g;
            const uint32_t pos = p.log_k ? (__brev(f) >> (32 - p.log_k)) : 0;
            Fr v = smem_ld(lo, hi, g * pitch + pos);
            const uint64_t lane = lane0 + g;
            if (p.tw_tab) {
                const uint64_t e = (p.tw_la * lane + p.tw_oa * o + p.tw_c0) * (p.tw_fb * f + p.tw_lb * lane);
                v = v * tw_lookup(p.tw_tab, e, p.tw_log_n, p.tw_inverse);
            }
            if (p.post_a) {
                v = v * gmem_ld(p.post_a + p.qa_o * o + p.qa_l * lane);
                v = v * gmem_ld(p.post_b + p.qb_o * o + p.qb_f * f + p.qb_l * lane);
            }
            if (p.post_const_on) v = v * p.post_const;
            uint64_t col = lane * p.out_lc + (uint64_t)f * p.out_ps;
            if (p.peer_on) {
                Fr *pd = p.peer_base[col >> p.split_log] + p.peer_row_off + (uint64_t)o * p.out_os + lane * p.out_ls;
                gmem_st(pd + (col & (((uint64_t)1 << p.split_log) - 1)), v);
                continue;
            }
            if (p.split_on) {
                col = (col >> p.split_log) * p.split_stride + (col & (((uint64_t)1 << p.split_log) - 1));
                gmem_st(dst + lane * p.out_ls + col, v);
                continue;
            }
            gmem_st(dst + lane * p.out_ls + lane * p.out_lc + (uint64_t)ti.a * p.out_ps_a + (uint64_t)ti.b * p.out_ps_b, v);
        }
    }
}

// ------------------------------------------------------------------ device-side barrier across GPUs
// Every rank owns a monotonically increasing arrival counter at the head of its peer arena.
// Barrier number k: each rank adds 1 to EVERY rank's counter (system-scope atomics over NVLink)
// after a system fence that orders the row kernel's peer stores before the arrival, then waits
// until its own counter reaches W*k.  Launched between the row and the column kernels on the
// same stream: the exchange needs no host synchronisation and no NCCL call at all.
struct PeerCounters {
    uint32_t *c[8];
};
__global__ void p2p_barrier_kernel(PeerCounters pc, uint32_t n_ranks, uint32_t me, uint32_t target) {
    const uint32_t t = threadIdx.x;
#if defined(DP_EMUL)
    (void)me;
    (void)target;
    if (t < n_ranks) atomicAdd(pc.c[t], 1u);  // contexts run one after another in the emulator: no waiting
#else
    __threadfence_system();
    if (t < n_ranks) atomicAdd_system(pc.c[t], 1u);
    if (t == 0) {
        volatile uint32_t *mine = pc.c[me];
        unsigned long long t0, now;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        while (*mine < target) {
            __nanosleep(100);
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (now - t0 > 20000000000ull) {  // 20 s: a peer is gone; give up instead of hanging the GPU
                pc.c[me][1] = 1u;             // word 1 of my arena header = "barrier timed out" (read by the host)
                break;
            }
        }
        __threadfence_system();
    }
#endif
}

// ------------------------------------------------------------------ table generation (init time)
// stage-major butterfly twiddles: W[2^s + j] = omega_{2^(s+1)}^(+-j), j < 2^s, s < NTT_WTAB_LOG;
// W[0] unused (= 1).  Plane-split (low / high 16 bytes) so one bulk copy per plane stages a prefix.
__global__ void ntt_gen_level_table_kernel(uint4 *w_lo, uint4 *w_hi, uint32_t inverse) {
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (1u << NTT_WTAB_LOG)) return;
    Fr v = Fr::one();
    if (idx >= 1) {
        const uint32_t s = 31 - __clz((int)idx), j = idx - (1u << s);
        Fr g = fr_domain_gen(s + 1);
        if (inverse) g = g.inverse();
        v = g.pow(j);
    }
    w_lo[idx] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    w_hi[idx] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}

// out[i] = mulc * base^(first + i*step) for i < n   (half twiddle tables, coset power tables)
__global__ void fr_gen_powers_kernel(Fr *out, uint64_t n, Fr base, uint64_t first, uint64_t step, Fr mulc) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    gmem_st(out + i, base.pow(first + i * step) * mulc);
}

// x[i] *= base^(i) * c   elementwise (whole-domain coset scaling: distribute_powers)
__global__ void fr_scale_powers_kernel(Fr *x, uint64_t n, Fr base, Fr c) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    gmem_st(x + i, gmem_ld(x + i) * (base.pow(i) * c));
}

// out[i] = in[i] * base^i for i < n_in, 0 for n_in <= i < n_out   (out-of-place coset scaling; `in` is not written)
__global__ void fr_scale_powers_copy_kernel(const Fr *in, Fr *out, uint64_t n_in, uint64_t n_out, Fr base) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    gmem_st(out + i, i < n_in ? gmem_ld(in + i) * base.pow(i) : Fr::zero());
}

// Montgomery -> canonical (Fr::into_repr, worker.rs:118), optionally zero-padding up to n_out
__global__ void fr_into_repr_kernel(const Fr *in, Fr *out, uint64_t n_in, uint64_t n_out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    gmem_st(out + i, i < n_in ? gmem_ld(in + i).from_mont() : Fr::zero());
}

}  // namespace dp
