// C ABI (include/dplonk.h) over the NTT / MSM kernels: device-resident worker state that mirrors
// the reference's `State` / `FftTask` (src/worker.rs:32-59) and the bodies of its RPC methods
// (src/worker.rs:125-439).  Host code only plans launches and moves bytes; every field / curve
// operation that contributes to a result runs in a CUDA kernel.
#include "../../include/dplonk.h"

#include <sys/random.h>

#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "circuit.cuh"
#include "msm.cuh"
#include "ntt.cuh"
#include "perm.cuh"
#include "rounds.cuh"
#include "pairing.cuh"
#include "srs.cuh"

using namespace dp;

namespace {

// ------------------------------------------------------------------ device memory pool
// cudaFree synchronises the device; tasks allocate the same few sizes over and over, so freed
// blocks are kept and handed back by exact size.  Single stream => stream-ordered reuse is safe.
struct DevPool {
    std::multimap<size_t, void *> free_blocks;
    std::unordered_map<void *, size_t> live;
    size_t total = 0;
    void *alloc(size_t bytes) {
        bytes = (bytes + 511) & ~(size_t)511;
        if (bytes == 0) bytes = 512;
        auto it = free_blocks.find(bytes);
        if (it != free_blocks.end()) {
            void *p = it->second;
            free_blocks.erase(it);
            live[p] = bytes;
            return p;
        }
        void *p = nullptr;
        if (cudaMalloc(&p, bytes) != cudaSuccess) {
            purge();  // drop cached blocks and retry once
            if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
        }
        total += bytes;
        live[p] = bytes;
        return p;
    }
    void release(void *p) {
        if (!p) return;
        auto it = live.find(p);
        if (it == live.end()) return;
        free_blocks.emplace(it->second, p);
        live.erase(it);
    }
    void purge() {
        for (auto &kv : free_blocks) {
            cudaFree(kv.second);
            total -= kv.first;
        }
        free_blocks.clear();
    }
    void destroy() {
        purge();
        for (auto &kv : live) cudaFree(kv.first);
        live.clear();
    }
};

// scope guard: pool blocks borrowed for one call go back on every exit path
struct Scratch {
    DevPool &pool;
    std::vector<void *> held;
    explicit Scratch(DevPool &p) : pool(p) {}
    ~Scratch() {
        for (void *p : held) pool.release(p);
    }
    template <class T>
    T *get(size_t count) {
        void *p = pool.alloc((count ? count : 1) * sizeof(T));
        if (p) held.push_back(p);
        return static_cast<T *>(p);
    }
    Scratch(const Scratch &) = delete;
    Scratch &operator=(const Scratch &) = delete;
};

struct DomainDev {
    uint32_t log_n = 0, log_r = 0, log_c = 0;
    Fr *H = nullptr;       // omega_N^e, e < N/2
    Fr *g_row = nullptr;   // g^i, i < r                (forward coset, by global row)
    Fr *g_col = nullptr;   // g^(r*j), j < c
    Fr *gi_col = nullptr;  // g^-i / r, i < c           (inverse coset + 1/r, by global column)
    Fr *gi_pt = nullptr;   // g^-(c*j), j < r
    Fr c_inv, r_inv, n_inv;
    // whole-domain (natural order) coset transforms: x[j] * g^j = wg_a[j mod 2^(L-l1)] * wg_b[j >> (L-l1)] on the way in,
    // X[k] * g^-k / N = wgi_a[k mod 2^(L-ll)] * wgi_b[k >> (L-ll)] on the way out, for the pass split (l1 first, ll last)
    // plan_whole_ntt uses; two small table reads and two products instead of one Fr::pow per element
    Fr *wg_a = nullptr, *wg_b = nullptr, *wgi_a = nullptr, *wgi_b = nullptr;
    uint32_t w_l1 = 0, w_ll = 0;
    // gate domain only: the same pair for each slice shift s_k = g * omega_m^k, k < m/n (the quotient domain's slices,
    // dp_ntt_dev_quot_slice): ws_a[k * 2^(L-l1) + j] = s_k^j, ws_b[k * 2^l1 + j] = s_k^(2^(L-l1) * j)
    Fr *ws_a = nullptr, *ws_b = nullptr;
    uint64_t n() const { return (uint64_t)1 << log_n; }
    uint64_t r() const { return (uint64_t)1 << log_r; }
    uint64_t c() const { return (uint64_t)1 << log_c; }
};

struct FftTask {
    bool is_quot, is_inv, is_coset;
    std::vector<dp_fft_workload> wl;
    uint64_t n_rows, n_cols, row_start, col_start;
    Fr *rows = nullptr;  // [n_rows][c]
    Fr *send = nullptr;  // W blocks of [n_rows][c/W]           (aliases rows when W == 1)
    Fr *recv = nullptr;  // [r][n_cols] = W blocks of [r/W][n_cols] (aliases send when W == 1)
    Fr *cols = nullptr;  // [n_cols][r]  column-phase result, produced asynchronously after the exchange
    uint64_t rows_filled = 0;
    std::vector<uint32_t> row_len;  // 0 = not received; else columns handed in for that row (c: a whole row)
    bool row_phase_done = false, exchanged = false;
    bool p2p = false;  // rows were stored straight into the peers' arenas; column phase waits for fft2
    cudaEvent_t ev_in = nullptr;  // last fft1 H2D copy (copy-in stream)
    cudaEvent_t ev_c = nullptr;   // column phase finished (compute stream)
};

}  // namespace

namespace {
struct MsmPending;  // defined with the MSM driver below
}

struct dp_ctx {
    int device = 0;
    uint32_t n_sms = 0;  // streaming multiprocessors of the device (sizes grids that loop over a device-side count)
    uint64_t me = 0, W = 1;
    // Three streams so that consecutive tasks overlap: rows of task k+1 stream in (s_in) while task k
    // computes (stream) and the columns of task k-1 stream out (s_out); PCIe is full duplex.
    cudaStream_t stream = nullptr, s_in = nullptr, s_out = nullptr, s_tail = nullptr, s_sort = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t ev_msm[4] = {nullptr, nullptr, nullptr, nullptr};  // sort done | accumulate done | tail done
    float msm_ms[3] = {0.f, 0.f, 0.f};
    std::string err;
    uint64_t launches = 0, launches_at_call = 0;
    float last_ms = 0.f;
    DevPool pool;     // everything touched by the compute stream (stream-ordered reuse)
    DevPool pool_io;  // fft1 row buffers: written by s_in, recycled only after their task fully completed
    uint4 *wf_lo = nullptr, *wf_hi = nullptr, *wi_lo = nullptr, *wi_hi = nullptr;
    G1Affine *bases = nullptr;
    uint64_t n_bases = 0;
    // window multiples 2^(c*w) * P_i (msm.cuh) for bases [pre_lo, pre_hi): the whole SRS for a single
    // worker, this worker's MsmWorkload shard (dispatcher.rs:219-229) otherwise; row length pre_hi-pre_lo
    G1Affine *pre_table = nullptr;
    uint32_t pre_c = 0, pre_nw = 0;
    uint64_t pre_lo = 0, pre_hi = 0;
    DomainDev dom[2];
    bool inited = false;
    std::map<uint64_t, FftTask> tasks;
    Fr *wire = nullptr;
    uint64_t wire_len = 0;
    // fused peer-memory exchange (dp_peer_arena_create / dp_peer_attach)
    Fr *arena = nullptr;            // my receive arena: header + n >= 2 receive slots, used round-robin (p2p_slot_geom)
    uint64_t arena_bytes = 0;
    Fr *peer_arena[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    uint64_t p2p_seq = 0;           // exchanges issued so far; must advance identically on every rank
    // receive slots of the arena: as many as fit (one slot = the receive matrix of the larger domain, at least two);
    // busy = written by a row phase whose column phase has not consumed it yet
    static constexpr uint32_t P2P_MAX_SLOTS = 64;
    bool p2p_slot_busy[P2P_MAX_SLOTS] = {};
    uint32_t bar_seq = 0;           // device-side barriers issued so far (p2p_barrier_kernel)
    // worker-resident polynomials (dp_poly_*): id -> device buffer of `cap` Fr, zero beyond what was written
    struct Poly {
        Fr *dev = nullptr;
        size_t cap = 0;
    };
    std::map<uint64_t, Poly> polys;
    // MSMs submitted with dp_msm_submit and not collected yet (keyed by the caller's id)
    std::map<uint64_t, MsmPending *> msm_pending;
    uint8_t *msm_pinned = nullptr;  // MSM_SLOTS x MSM_SLOT_BYTES of pinned host memory: result + error flag per job
    uint64_t msm_slots_used = 0;    // bit mask
    Fr *dev_send = nullptr, *dev_recv = nullptr;  // dp_fft_dev_rows / _cols staging (one transform in flight)
    Fr *dev_p2p_slot = nullptr;                   // receive slot of the last dp_fft_dev_rows_p2p
    int dev_flags = -1;
    uint64_t dev_valid[2] = {0, 0};  // dp_fft_dev_hint_valid_cols: leading non-zero columns of the rows given to dp_fft_dev*
    // pass-planning limits (dp_debug_set_limits lowers them so small tests reach the multi-pass plans)
    uint32_t max_contig_log_k = NTT_WTAB_LOG, max_strided_log_k = NTT_MAX_STRIDED_LOG_K;
    uint32_t three_pass_min_log = 20;  // smallest domain the three-pass single-worker plan is used for (tests lower it)
    bool no_three_pass = false;    // knob (env DP_NTT_NO_3PASS / dp_debug_set_limits): single-worker transforms use the 2-D four-pass plan
    int msm_min_blocks = 3;        // experiment knob (env DP_MSM_BLOCKS): register budget of msm_accumulate_kernel for 3, 4 or 5 blocks per SM
    bool ntt_tw_prefetch = false;  // experiment knob (env DP_NTT_PREFETCH)
    int ntt_min_blocks = 3;    // knob (env DP_NTT_BLOCKS): register budget of ntt_tile_kernel for 2 or 3 CTAs per SM (3: -7 % per transform)
    uint32_t msm_chunk = 0;    // experiment knob (env DP_MSM_CHUNK): digits per accumulate thread, 0 = default
    int msm_force_c = 0;       // 0 auto, 1 = windowed path with automatic c, >= 2 forced c (windowed)
    // knob (env DP_MSM_PRE_C): width of the window-multiple table built by dp_init.  Unset = msm_pick_pre_c's choice within
    // a quarter of the free memory; 0 = no table (pre_disabled: every MSM takes the per-window pipeline); 8..22 = exactly
    // that width or dp_init fails (DP_E_ARG when the width cannot index the shard, DP_E_OOM when the table does not fit)
    int msm_pre_c = -1;        // -1 = unset; a value that does not parse is kept as out of range and refused by dp_init
    bool pre_disabled = false;
    // 1 / (x_i - 1) over the quotient coset (rounds.cuh: quotient_kernel<true>): depends on the domain only, built by the
    // first dp_quotient_evals after dp_init when it fits (32 B per point), dropped by the next dp_init
    Fr *quot_inv = nullptr;
    uint32_t quot_inv_log = 0;
    // fixed-base table of dp_srs_powers_of_tau (srs.cuh, 48 MiB): built by its first call, dropped by the next dp_init
    G1Affine *srs_table = nullptr;
    // the last dp_srs_check: ms of its scalar generation, two MSMs and pairing, and its two MSM results (dp_last_srs_check)
    float srs_check_ms[3] = {0.f, 0.f, 0.f};
    G1JacobianOut srs_check_ab[2] = {};
    // batched-affine tree levels in front of the XYZZ chunks (msm.cuh): 0 = none, else L.  env DP_MSM_AFFINE=L forces L levels;
    // otherwise dp_init chooses by msm_tune() - one MSM over the context's own window table per candidate, results compared
    // byte for byte, levels kept only if identical and faster (an SRS whose hot-path MSM has fewer than msm_affine_min_digits
    // digits is not tuned and stays plain; env DP_MSM_AFFINE_MIN).  bench.py runs the wider search (DP_MSM_TUNE=2) in a child
    // process and forces its answer (distributed_plonk_b200/tune.py).
    uint32_t msm_affine_levels = 0;
    int msm_affine_forced = -1;             // -1 = not forced
    // env DP_MSM_TUNE: 0 = dp_init never tunes (plain pipeline unless forced); 1 (default) = msm_tune() compares the plain
    // pipeline with two tree levels; 2 = it also tries one and three levels (what bench.py's child-process probe asks for)
    int msm_tune_mode = 1;
    uint64_t msm_affine_min_digits = (uint64_t)1 << 22;
    float tune_ms[2] = {0.f, 0.f};          // msm_tune(): plain / best candidate with levels (0 = not measured)
    float tune_all_ms[4] = {0.f, 0.f, 0.f, 0.f};  // msm_tune(): 0, 1, 2, 3 levels
    int tune_equal = -1;                    // msm_tune(): results identical (1), different (0), not run (-1)
    // knob (env DP_MSM_SORT_STREAM=1): the digit sorts of a batch run on their own stream, ahead of / under the accumulations.
    // NOT ADOPTED (tools/ab_sort_stream.py compares the two): the sort's atomics and its blocks taking SM slots cost the
    // accumulation more than the sort time that leaves the critical path.  Default: sorts queue in front of their accumulation.
    bool msm_sort_own_stream = false;
    int quot_table = -1;       // knob (env DP_QUOT_TABLE): -1 auto (table when it is at most 1/8 of the free memory), 0 never, 1 always
};

namespace {

thread_local std::string g_err_noctx;

int fail(dp_ctx *ctx, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (ctx)
        ctx->err = buf;
    else
        g_err_noctx = buf;
    return code;
}

#define DP_CUDA(ctx, expr)                                                                              \
    do {                                                                                                \
        cudaError_t e__ = (expr);                                                                       \
        if (e__ != cudaSuccess)                                                                         \
            return fail(ctx, DP_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

#define DP_TRY(expr)               \
    do {                           \
        int rc__ = (expr);         \
        if (rc__ != DP_OK) return rc__; \
    } while (0)

inline uint32_t log2_ceil_u64(uint64_t n) {
    uint32_t l = 0;
    while (((uint64_t)1 << l) < n) l++;
    return l;
}
inline unsigned blocks_for(uint64_t n, unsigned tpb) { return (unsigned)((n + tpb - 1) / tpb); }

void call_begin(dp_ctx *ctx) {
    ctx->launches_at_call = ctx->launches;
    cudaEventRecord(ctx->ev0, ctx->stream);
}
int call_end(dp_ctx *ctx, bool sync) {
    cudaEventRecord(ctx->ev1, ctx->stream);
    if (sync) {
        DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        DP_CUDA(ctx, cudaGetLastError());
        cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1);
    }
    return DP_OK;
}

// ------------------------------------------------------------------ NTT planning
NttPass pass_base(dp_ctx *ctx, bool inverse) {
    NttPass p;
    memset((void *)&p, 0, sizeof p);
    p.w_lo = inverse ? ctx->wi_lo : ctx->wf_lo;
    p.w_hi = inverse ? ctx->wi_hi : ctx->wf_hi;
    p.n_outer = 1;
    p.lane_tiles = 1;
    p.tw_inverse = inverse ? 1 : 0;
    p.tw_prefetch = ctx->ntt_tw_prefetch ? 1 : 0;
    return p;
}

// lanes per tile: fill the 2048-element tile but never exceed the number of lanes
uint32_t pick_log_g(uint32_t log_k, uint64_t n_lanes) {
    uint32_t lg = NTT_TILE_LOG > log_k ? NTT_TILE_LOG - log_k : 0;
    while (((uint64_t)1 << lg) > n_lanes) lg--;
    return lg;
}

int launch_pass(dp_ctx *ctx, NttPass &p, uint64_t n_lanes) {
    p.lane_tiles = (uint32_t)(n_lanes >> p.log_g);
    if (!p.map_set) {  // the two classic tile walks: points contiguous, or lanes contiguous with strided points
        const bool in_contig = p.in_ps == 1, out_contig = p.out_ps == 1 && !p.out_lc;
        p.in_a_log = in_contig ? p.log_k - p.in_zlog : 0;
        p.out_a_log = out_contig ? p.log_k : 0;
        p.in_a_hi = p.out_a_hi = 0;
        p.in_ps_a = p.in_ps_b = p.in_ps;
        p.out_ps_a = p.out_ps_b = p.out_ps;
    }
    const uint64_t grid = (uint64_t)p.n_outer * p.lane_tiles;
    if (grid == 0 || grid > 0x7fffffffull) return fail(ctx, DP_E_ARG, "ntt pass grid %llu out of range", (unsigned long long)grid);
    const size_t smem = ntt_pass_smem_bytes(p.log_k, p.log_g);
    if (ctx->ntt_min_blocks == 3)
        DP_LAUNCH(ntt_tile_kernel<3>, dim3((unsigned)grid), dim3(NTT_TPB), smem, ctx->stream, p);
    else
        DP_LAUNCH(ntt_tile_kernel<2>, dim3((unsigned)grid), dim3(NTT_TPB), smem, ctx->stream, p);
    ctx->launches++;
    DP_CUDA(ctx, cudaGetLastError());
    return DP_OK;
}

// Row phase of the 2-D transform (fft1_helper, worker.rs:66-94) over all local rows:
//   src  [n_rows][c] row-major;  dst = exchange layout: W blocks of [n_rows][c/W]
// scratch ([n_rows][c]) is used when c > 2^11 (row split into two passes).
struct PeerDst {
    Fr *base[8];
    uint64_t row_off;
};

// Three-pass plan of a single worker (n_workers == 1), for domains of >= 2^20 points.  With every row and every
// column on one device the transform need not stop at the row / column boundary of the 2-D scheme (two passes for the
// rows, two for the columns at 2^25): the index n = i + r*j of rows[i][j] is cut into three digit groups instead,
//   n1 = high a bits of j            pass A: 2^a-point transforms along a row, points 2^lj apart, 2^lj-element runs
//   n2 = (low lj bits of j, high ih bits of i)   pass B: runs of 2^lj contiguous elements from 2^ih row slabs
//   n3 = low il bits of i            pass C: 2^il-point strided transforms, written as the columns cols[k2][k1]
// with the usual twiddles omega_N^(k1' * n_low) after A and omega_N^(2^a * k2' * n3) after B.  Same input and output
// layouts, same values (the transform is unique) - one pass over HBM and one twiddle product per element fewer.
struct Split3 {
    uint32_t a, lj, ih, il;
    bool ok;
};
Split3 single_worker_split(const dp_ctx *ctx, const DomainDev &d) {
    Split3 s{0, 0, 0, 0, false};
    if (ctx->W != 1 || ctx->no_three_pass || d.log_n < ctx->three_pass_min_log || d.log_r < 4 || d.log_c < 5 || ctx->max_strided_log_k != NTT_MAX_STRIDED_LOG_K || ctx->max_contig_log_k != NTT_WTAB_LOG)
        return s;
    const uint32_t lr = d.log_r, lc = d.log_c;
    s.ih = lr <= 12 ? 3 : lr - 9;
    s.il = lr - s.ih;
    s.lj = lc > 11 ? lc - 8 : 3;
    if (s.lj + s.ih > 9) s.lj = lc - 9;
    s.a = lc - s.lj;
    s.ok = s.a <= 9 && s.lj + s.ih <= 9 && s.il <= 9 && s.ih >= 2 && s.ih <= 5 && s.lj >= 2;
    return s;
}

// Columns of a row the row phase reads when only the first `valid` hold data (the rest of the row is an
// implicit zero tail, as for n coefficients on the 8n-point domain): a power-of-two count of whole passes'
// points, so that the kernel can drop the butterfly stages whose upper input is zero (NttPass.in_zlog).
uint64_t row_read_cols(const dp_ctx *ctx, const DomainDev &d, uint64_t valid) {
    const uint64_t c = d.c();
    if (valid >= c) return c;
    if (valid == 0) valid = 1;
    uint64_t unit = 1;  // columns per point of the first pass
    const Split3 s3 = single_worker_split(ctx, d);
    if (s3.ok)
        unit = (uint64_t)1 << s3.lj;
    else if (d.log_c > ctx->max_contig_log_k)
        unit = (uint64_t)1 << (d.log_c - d.log_c / 2);
    uint64_t pts = (valid + unit - 1) / unit, p2 = 1;
    while (p2 < pts) p2 <<= 1;
    return p2 * unit < c ? p2 * unit : c;
}

int plan_single_worker3(dp_ctx *ctx, const DomainDev &d, const Split3 &s3, const Fr *src, Fr *w1, Fr *w2, Fr *dst, bool is_inv,
                        bool is_coset, uint64_t rd_cols) {
    const uint64_t r = d.r(), c = d.c(), N = d.n();
    const uint32_t a = s3.a, lj = s3.lj, ih = s3.ih, il = s3.il, b = lj + ih;
    if (rd_cols == 0 || rd_cols > c) rd_cols = c;
    {   // ---- pass A: o = row i, lanes = low digit of j (contiguous), points = high digit of j
        NttPass p = pass_base(ctx, is_inv);
        p.in = src;
        p.out = w1;
        p.log_k = a;
        p.log_g = pick_log_g(a, (uint64_t)1 << lj);
        p.n_outer = (uint32_t)r;
        p.in_os = p.out_os = c;
        p.in_ls = p.out_ls = 1;
        p.in_ps = p.out_ps = (uint64_t)1 << lj;
        const uint64_t pts = rd_cols >> lj;  // row_read_cols: a power of two of whole points (or the whole row)
        p.in_zlog = pts >= 1 && pts < ((uint64_t)1 << a) ? a - log2_ceil_u64(pts) : (pts == 0 ? a : 0);
        p.tw_tab = d.H;
        p.tw_log_n = d.log_n;
        p.tw_oa = 1;       // omega_N^(+-f * (i + r * j_lo))
        p.tw_la = r;
        p.tw_fb = 1;
        if (is_coset && !is_inv) {  // g^(i + r*j) = g_row[i] * g_col[j]
            p.pre_a = d.g_row;
            p.pa_o = 1;
            p.pre_b = d.g_col;
            p.pb_l = 1;
            p.pb_m = (uint64_t)1 << lj;
        }
        if (is_inv && is_coset) {  // gi_col of pass C carries 1/r
            p.post_const_on = 1;
            p.post_const = d.c_inv;
        }
        DP_TRY(launch_pass(ctx, p, (uint64_t)1 << lj));
    }
    {   // ---- pass B: o = i_lo, lanes = k1' (2^lj apart), points = (i_hi slow, j_lo fast and contiguous)
        NttPass p = pass_base(ctx, is_inv);
        p.in = w1;
        p.out = w2;
        p.log_k = b;
        p.log_g = pick_log_g(b, (uint64_t)1 << a);
        p.n_outer = 1u << il;
        p.in_os = c;
        p.in_ls = (uint64_t)1 << lj;
        p.out_os = c << ih;                    // w2[i_lo][k2'_lo][k1'][k2'_hi]
        p.out_ls = (uint64_t)1 << ih;
        p.map_set = 1;
        p.in_a_log = lj;                       // point m = i_hi + 2^ih * j_lo: j_lo fast
        p.in_a_hi = 1;
        p.in_ps_a = 1;
        p.in_ps_b = c << il;
        p.out_a_log = ih;                      // frequency f = k2'_lo + 2^lj * k2'_hi: k2'_hi fast
        p.out_a_hi = 1;
        p.out_ps_a = 1;
        p.out_ps_b = (uint64_t)1 << (a + ih);
        p.in_ps = p.out_ps = 2;                // (unused with map_set; not 1)
        p.tw_tab = d.H;
        p.tw_log_n = d.log_n;
        p.tw_oa = (uint64_t)1 << a;            // omega_N^(+-2^a * f * i_lo)
        p.tw_fb = 1;
        DP_TRY(launch_pass(ctx, p, (uint64_t)1 << a));
    }
    {   // ---- pass C: o = k2 = k1' + 2^a * k2'_lo, lanes = k2'_hi (contiguous), points = i_lo; out = cols[k2][k1]
        NttPass p = pass_base(ctx, is_inv);
        p.in = w2;
        p.out = dst;
        p.log_k = il;
        p.log_g = pick_log_g(il, (uint64_t)1 << ih);
        p.n_outer = (uint32_t)c;
        p.in_os = (uint64_t)1 << ih;
        p.in_ls = 1;
        p.in_ps = c << ih;
        p.out_os = r;
        p.out_ls = 1;                          // k1 = k2'_hi + 2^ih * k3'
        p.out_ps = (uint64_t)1 << ih;
        if (is_inv && is_coset) {  // g^-(k2 + c*k1) / r
            p.post_a = d.gi_col;
            p.qa_o = 1;
            p.post_b = d.gi_pt;
            p.qb_l = 1;
            p.qb_f = (uint64_t)1 << ih;
        } else if (is_inv) {
            p.post_const_on = 1;
            p.post_const = d.n_inv;
        }
        DP_TRY(launch_pass(ctx, p, (uint64_t)1 << ih));
    }
    (void)N;
    return DP_OK;
}

int plan_row_phase(dp_ctx *ctx, const DomainDev &d, const Fr *src, Fr *dst, Fr *scratch, uint64_t n_rows,
                   uint64_t row_start, bool is_inv, bool is_coset, uint64_t W, const PeerDst *peers = nullptr,
                   uint64_t rd_cols = 0 /* row_read_cols(); 0 = whole rows */) {
    const uint32_t lc = d.log_c;
    if (rd_cols == 0 || rd_cols > d.c()) rd_cols = d.c();
    const uint64_t c = d.c();
    const uint32_t log_ncq = lc - log2_ceil_u64(W);
    const bool pre = is_coset && !is_inv;
    auto finish = [&](NttPass &p) {
        p.tw_tab = d.H;
        p.tw_log_n = d.log_n;
        if (W > 1) {
            p.split_on = 1;
            p.split_log = log_ncq;
            p.split_stride = n_rows << log_ncq;
            if (peers) {
                p.peer_on = 1;
                p.peer_row_off = peers->row_off;
                for (uint64_t q = 0; q < W; q++) p.peer_base[q] = peers->base[q];
            }
        }
        if (is_inv) {
            p.post_const_on = 1;
            p.post_const = d.c_inv;
        }
    };
    if (lc <= ctx->max_contig_log_k) {
        NttPass p = pass_base(ctx, is_inv);
        p.in = src;
        p.out = dst;
        p.log_k = lc;
        p.log_g = pick_log_g(lc, n_rows);
        p.in_zlog = lc - log2_ceil_u64(rd_cols);
        p.in_ls = c;
        p.in_ps = 1;
        p.out_ls = W > 1 ? ((uint64_t)1 << log_ncq) : c;
        p.out_ps = 1;
        // omega_N^(+-(row_start + lane) * f)
        p.tw_la = 1;
        p.tw_c0 = row_start;
        p.tw_fb = 1;
        if (pre) {
            p.pre_a = d.g_row + row_start;
            p.pa_l = 1;
            p.pre_b = d.g_col;
            p.pb_m = 1;
        }
        finish(p);
        return launch_pass(ctx, p, n_rows);
    }
    // c = L1 * L2: pass 1 strided (points L2 apart, lanes = p2 contiguous), pass 2 contiguous chunks
    const uint32_t l1 = lc / 2, l2 = lc - l1;
    const uint64_t L1 = (uint64_t)1 << l1, L2 = (uint64_t)1 << l2;
    {
        NttPass p = pass_base(ctx, is_inv);
        p.in = src;
        p.out = scratch;
        p.log_k = l1;
        p.log_g = pick_log_g(l1, L2);
        p.in_zlog = rd_cols >= L2 ? l1 - log2_ceil_u64(rd_cols / L2) : l1;
        p.n_outer = (uint32_t)n_rows;
        p.in_os = p.out_os = c;
        p.in_ls = p.out_ls = 1;
        p.in_ps = p.out_ps = L2;
        // omega_c^(+-f*lane) = omega_N^(+-(N/c)*lane*f)
        p.tw_tab = d.H;
        p.tw_log_n = d.log_n;
        p.tw_la = d.n() >> lc;
        p.tw_fb = 1;
        if (pre) {
            p.pre_a = d.g_row + row_start;
            p.pa_o = 1;
            p.pre_b = d.g_col;
            p.pb_m = L2;
            p.pb_l = 1;
        }
        DP_TRY(launch_pass(ctx, p, L2));
    }
    {
        NttPass p = pass_base(ctx, is_inv);
        p.in = scratch;
        p.out = dst;
        p.log_k = l2;
        p.log_g = pick_log_g(l2, L1);
        p.n_outer = (uint32_t)n_rows;
        p.in_os = c;
        p.in_ls = L2;
        p.in_ps = 1;
        // output column index = lane + L1 * f
        p.out_os = W > 1 ? ((uint64_t)1 << log_ncq) : c;
        p.out_ls = 0;
        p.out_lc = 1;
        p.out_ps = L1;
        // omega_N^(+-(row_start + o) * (lane + L1*f))
        p.tw_oa = 1;
        p.tw_c0 = row_start;
        p.tw_lb = 1;
        p.tw_fb = L1;
        finish(p);
        return launch_pass(ctx, p, L1);
    }
}

// Column phase (fft2_helper, worker.rs:96-115): src = [r][ncq] row-major (column k = src[j*ncq+k]),
// dst = [ncq][r] (column k contiguous).  src is overwritten when r > 2^9 (two passes).
int plan_col_phase(dp_ctx *ctx, const DomainDev &d, Fr *src, Fr *dst, uint64_t ncq, uint64_t col_start, bool is_inv,
                   bool is_coset) {
    const uint32_t lr = d.log_r;
    const uint64_t r = d.r();
    const bool post = is_coset && is_inv;
    auto finish = [&](NttPass &p) {
        if (post) {
            p.post_a = d.gi_col + col_start;  // carries the 1/r of the inverse transform
            p.qa_l = 1;
            p.post_b = d.gi_pt;
        } else if (is_inv) {
            p.post_const_on = 1;
            p.post_const = d.r_inv;
        }
    };
    if (lr <= ctx->max_strided_log_k) {
        NttPass p = pass_base(ctx, is_inv);
        p.in = src;
        p.out = dst;
        p.log_k = lr;
        p.log_g = pick_log_g(lr, ncq);
        p.in_ls = 1;
        p.in_ps = ncq;
        p.out_ls = r;
        p.out_ps = 1;
        if (post) p.qb_f = 1;
        finish(p);
        return launch_pass(ctx, p, ncq);
    }
    const uint32_t l1 = lr / 2, l2 = lr - l1;
    const uint64_t R1 = (uint64_t)1 << l1, R2 = (uint64_t)1 << l2;
    {
        NttPass p = pass_base(ctx, is_inv);
        p.in = src;
        p.out = src;
        p.log_k = l1;
        p.log_g = pick_log_g(l1, ncq);
        p.n_outer = (uint32_t)R2;  // o = j2
        p.in_os = p.out_os = ncq;
        p.in_ls = p.out_ls = 1;
        p.in_ps = p.out_ps = R2 * ncq;
        // omega_r^(+-f*j2) = omega_N^(+-(N/r)*o*f)
        p.tw_tab = d.H;
        p.tw_log_n = d.log_n;
        p.tw_oa = d.n() >> lr;
        p.tw_fb = 1;
        DP_TRY(launch_pass(ctx, p, ncq));
    }
    {
        NttPass p = pass_base(ctx, is_inv);
        p.in = src;
        p.out = dst;
        p.log_k = l2;
        p.log_g = pick_log_g(l2, ncq);
        p.n_outer = (uint32_t)R1;  // o = f1
        p.in_os = R2 * ncq;
        p.in_ls = 1;
        p.in_ps = ncq;
        // out[k][f1 + R1*f2]
        p.out_os = 1;
        p.out_ls = r;
        p.out_ps = R1;
        if (post) {
            p.qb_o = 1;
            p.qb_f = R1;
        }
        finish(p);
        return launch_pass(ctx, p, ncq);
    }
}

// pass split of a whole-domain transform of 2^L points: sub-transform sizes (first .. last), 1-3 passes, 0 = too large
int whole_split(const dp_ctx *ctx, uint32_t L, uint32_t l[3]) {
    l[0] = l[1] = l[2] = 0;
    if (L <= ctx->max_contig_log_k) {
        l[0] = L;
        return 1;
    }
    if (L <= 2 * ctx->max_strided_log_k) {
        l[0] = L / 2;
        l[1] = L - l[0];
        return 2;
    }
    if (L > 3 * ctx->max_strided_log_k) return 0;
    l[0] = L / 3;
    l[1] = (L - l[0]) / 2;
    l[2] = L - l[0] - l[1];
    return 3;
}

// The factor tables of domain d serve a whole-domain transform of 2^L points when they were built for its pass split
bool whole_tables_fit(const dp_ctx *ctx, const DomainDev *d, uint32_t L) {
    uint32_t l[3];
    const int np = whole_split(ctx, L, l);
    return d && d->log_n == L && d->wg_a && np >= 2 && d->w_l1 == l[0] && d->w_ll == l[np - 1];
}

// Forward coset factors of a whole-domain transform that replace the domain's own wg_a / wg_b (a shift other than g)
struct CosetTables {
    const Fr *a, *b;
};

// Whole-domain transform of 2^L elements: x (in place) with scratch of the same size.  n_valid: x[n_valid..) is
// zero (a coefficient vector shorter than the domain): the first pass then reads and multiplies only what is there.
// src != nullptr: out of place, the first pass reads src instead of x (src is never written; only its first n_valid
// entries are read when the first pass's zero-input cut falls exactly on n_valid - the caller checks, see slice_ntt_device).
// shift != nullptr: forward coset with those factor tables instead of the domain's (requires whole_tables_fit).
int plan_whole_ntt(dp_ctx *ctx, const DomainDev *d, Fr *x, Fr *scratch, uint32_t L, bool is_inv, bool is_coset,
                   const Fr *H, uint32_t H_log_n, uint64_t n_valid = 0, const Fr *src = nullptr, const CosetTables *shift = nullptr) {
    const uint64_t N = (uint64_t)1 << L;
    if (n_valid == 0 || n_valid > N) n_valid = N;
    uint32_t l[3];
    const int np = whole_split(ctx, L, l);
    if (np == 0) return fail(ctx, DP_E_ARG, "dp_ntt: log_n %u too large for one device pass plan", L);
    const uint32_t l1 = l[0];
    Fr g = fr_from_u64(7), ninv = fr_from_u64(N).inverse();
    // coset scaling fused into the first load / the last store when this domain's factor tables fit the split
    const bool tabs = whole_tables_fit(ctx, d, L);
    if (shift && !(tabs && is_coset && !is_inv)) return fail(ctx, DP_E_ARG, "coset factor tables do not fit the 2^%u plan", L);
    if (src && is_coset && !tabs) return fail(ctx, DP_E_ARG, "out-of-place coset transform without factor tables");
    const Fr *in0 = src ? src : x;
    if (is_coset && !is_inv && !tabs) {
        DP_LAUNCH(fr_scale_powers_kernel, dim3(blocks_for(n_valid, 256)), dim3(256), 0, ctx->stream, x, n_valid, g, Fr::one());
        ctx->launches++;
    }
    auto set_first = [&](NttPass &p, uint64_t lanes /* 2^(L - l1) */) {
        if (n_valid < N) {  // points m >= ceil(n_valid / lanes) of every lane are zero
            const uint64_t pts = (n_valid + lanes - 1) / lanes;
            const uint32_t vlog = log2_ceil_u64(pts);
            p.in_zlog = vlog < p.log_k ? p.log_k - vlog : 0;
        }
        if (is_coset && !is_inv && tabs) {
            p.pre_a = shift ? shift->a : d->wg_a;
            p.pa_l = 1;
            p.pre_b = shift ? shift->b : d->wg_b;
            p.pb_m = 1;
        }
    };
    auto set_final = [&](NttPass &p) {
        if (is_inv && !is_coset) {
            p.post_const_on = 1;
            p.post_const = ninv;
        }
    };
    const uint64_t tw_mul = (uint64_t)1 << (H_log_n - L);  // omega_N = omega_H^(tw_mul)
    if (np == 1) {
        NttPass p = pass_base(ctx, is_inv);
        p.in = in0;
        p.out = x;
        p.log_k = L;
        p.log_g = 0;
        p.in_ps = p.out_ps = 1;
        if (n_valid < N) p.in_zlog = L - log2_ceil_u64(n_valid);
        set_final(p);
        DP_TRY(launch_pass(ctx, p, 1));
    } else if (np == 2) {
        const uint32_t l2 = l[1];
        const uint64_t N1 = (uint64_t)1 << l1, N2 = (uint64_t)1 << l2;
        NttPass p = pass_base(ctx, is_inv);
        p.in = in0;
        p.out = scratch;
        p.log_k = l1;
        p.log_g = pick_log_g(l1, N2);
        p.in_ls = p.out_ls = 1;
        p.in_ps = p.out_ps = N2;
        p.tw_tab = H;
        p.tw_log_n = H_log_n;
        p.tw_la = tw_mul;
        p.tw_fb = 1;
        set_first(p, N2);
        DP_TRY(launch_pass(ctx, p, N2));
        NttPass q = pass_base(ctx, is_inv);
        q.in = scratch;
        q.out = x;
        q.log_k = l2;
        q.log_g = pick_log_g(l2, N1);
        q.in_ls = N2;
        q.in_ps = 1;
        q.out_ls = 1;
        q.out_ps = N1;
        set_final(q);
        if (is_coset && is_inv && tabs) {  // k = lane + N1 * f
            q.post_a = d->wgi_a;
            q.qa_l = 1;
            q.post_b = d->wgi_b;
            q.qb_f = 1;
        }
        DP_TRY(launch_pass(ctx, q, N1));
    } else {
        const uint32_t l2 = l[1], l3 = l[2];
        const uint64_t N1 = (uint64_t)1 << l1, N2 = (uint64_t)1 << l2, N3 = (uint64_t)1 << l3;
        NttPass a = pass_base(ctx, is_inv);
        a.in = in0;
        a.out = scratch;
        a.log_k = l1;
        a.log_g = pick_log_g(l1, N2 * N3);
        a.in_ls = a.out_ls = 1;
        a.in_ps = a.out_ps = N2 * N3;
        a.tw_tab = H;
        a.tw_log_n = H_log_n;
        a.tw_la = tw_mul;
        a.tw_fb = 1;
        set_first(a, N2 * N3);
        DP_TRY(launch_pass(ctx, a, N2 * N3));
        NttPass b = pass_base(ctx, is_inv);
        b.in = scratch;
        b.out = scratch;
        b.log_k = l2;
        b.log_g = pick_log_g(l2, N3);
        b.n_outer = (uint32_t)N1;
        b.in_os = b.out_os = N2 * N3;
        b.in_ls = b.out_ls = 1;
        b.in_ps = b.out_ps = N3;
        b.tw_tab = H;
        b.tw_log_n = H_log_n;
        b.tw_la = tw_mul * N1;
        b.tw_fb = 1;
        DP_TRY(launch_pass(ctx, b, N3));
        NttPass c3 = pass_base(ctx, is_inv);
        c3.in = scratch;
        c3.out = x;
        c3.log_k = l3;
        c3.log_g = pick_log_g(l3, N1);
        c3.n_outer = (uint32_t)N2;  // o = k2
        c3.in_os = N3;
        c3.out_os = N1;
        c3.in_ls = N2 * N3;  // lane = k1
        c3.out_ls = 1;
        c3.in_ps = 1;
        c3.out_ps = N1 * N2;
        set_final(c3);
        if (is_coset && is_inv && tabs) {  // k = lane + N1 * o + N1 N2 * f
            c3.post_a = d->wgi_a;
            c3.qa_l = 1;
            c3.qa_o = N1;
            c3.post_b = d->wgi_b;
            c3.qb_f = 1;
        }
        DP_TRY(launch_pass(ctx, c3, N1));
    }
    if (is_coset && is_inv && !tabs) {
        DP_LAUNCH(fr_scale_powers_kernel, dim3(blocks_for(N, 256)), dim3(256), 0, ctx->stream, x, N, g.inverse(), ninv);
        ctx->launches++;
    }
    DP_CUDA(ctx, cudaGetLastError());
    return DP_OK;
}

int gen_powers(dp_ctx *ctx, Fr *out, uint64_t n, const Fr &base, uint64_t first, uint64_t step, const Fr &mulc) {
    DP_LAUNCH(fr_gen_powers_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, ctx->stream, out, n, base, first, step, mulc);
    ctx->launches++;
    DP_CUDA(ctx, cudaGetLastError());
    return DP_OK;
}

int build_domain(dp_ctx *ctx, DomainDev &d, uint64_t min_size) {
    d.log_n = log2_ceil_u64(min_size);
    if (d.log_n > 32) return fail(ctx, DP_E_ARG, "domain size 2^%u exceeds the two-adicity of Fr", d.log_n);
    d.log_r = d.log_n >> 1;  // worker.rs:144-147
    d.log_c = d.log_n - d.log_r;
    const uint64_t N = d.n(), r = d.r(), c = d.c();
    const uint64_t half = N >= 2 ? N / 2 : 1;
    d.H = (Fr *)ctx->pool.alloc(half * sizeof(Fr));
    d.g_row = (Fr *)ctx->pool.alloc(r * sizeof(Fr));
    d.g_col = (Fr *)ctx->pool.alloc(c * sizeof(Fr));
    d.gi_col = (Fr *)ctx->pool.alloc(c * sizeof(Fr));
    d.gi_pt = (Fr *)ctx->pool.alloc(r * sizeof(Fr));
    if (!d.H || !d.g_row || !d.g_col || !d.gi_col || !d.gi_pt) return fail(ctx, DP_E_OOM, "domain tables (2^%u)", d.log_n);
    const Fr g = fr_from_u64(7), gi = g.inverse(), one = Fr::one();
    d.c_inv = fr_from_u64(c).inverse();
    d.r_inv = fr_from_u64(r).inverse();
    d.n_inv = fr_from_u64(N).inverse();
    DP_TRY(gen_powers(ctx, d.H, half, fr_domain_gen(d.log_n), 0, 1, one));
    DP_TRY(gen_powers(ctx, d.g_row, r, g, 0, 1, one));
    DP_TRY(gen_powers(ctx, d.g_col, c, g, 0, r, one));
    DP_TRY(gen_powers(ctx, d.gi_col, c, gi, 0, 1, d.r_inv));
    DP_TRY(gen_powers(ctx, d.gi_pt, r, gi, 0, c, one));
    uint32_t l[3];
    const int np = whole_split(ctx, d.log_n, l);
    if (np >= 2) {
        d.w_l1 = l[0];
        d.w_ll = l[np - 1];
        const uint64_t na = N >> d.w_l1, nb = (uint64_t)1 << d.w_l1, nia = N >> d.w_ll, nib = (uint64_t)1 << d.w_ll;
        d.wg_a = (Fr *)ctx->pool.alloc(na * sizeof(Fr));
        d.wg_b = (Fr *)ctx->pool.alloc(nb * sizeof(Fr));
        d.wgi_a = (Fr *)ctx->pool.alloc(nia * sizeof(Fr));
        d.wgi_b = (Fr *)ctx->pool.alloc(nib * sizeof(Fr));
        if (!d.wg_a || !d.wg_b || !d.wgi_a || !d.wgi_b) return fail(ctx, DP_E_OOM, "coset factor tables (2^%u)", d.log_n);
        DP_TRY(gen_powers(ctx, d.wg_a, na, g, 0, 1, one));
        DP_TRY(gen_powers(ctx, d.wg_b, nb, g, 0, na, one));
        DP_TRY(gen_powers(ctx, d.wgi_a, nia, gi, 0, 1, d.n_inv));
        DP_TRY(gen_powers(ctx, d.wgi_b, nib, gi, 0, nia, one));
    }
    return DP_OK;
}

// s_k = g * omega_m^k: the shift of slice k of the quotient coset g*H_m as cosets of the gate domain H_n,
// g * omega_m^(k + (m/n) i) = s_k * omega_n^i
Fr slice_shift(const DomainDev &dq, uint32_t k) { return fr_from_u64(7) * fr_domain_gen(dq.log_n).pow(k); }

// the per-slice factor tables of the gate domain dg (DomainDev::ws_a / ws_b), for the m/n slices of dq; none when the
// gate domain has no fused tables (single-pass split) or the quotient domain is not a multiple of it
int build_slice_tables(dp_ctx *ctx, DomainDev &dg, const DomainDev &dq) {
    if (!dg.wg_a || dq.log_n < dg.log_n || dq.log_n - dg.log_n > 4) return DP_OK;  // (ratios above RND_MAX_RATIO: no quotient)
    const uint32_t ns = 1u << (dq.log_n - dg.log_n);
    const uint64_t na = dg.n() >> dg.w_l1, nb = (uint64_t)1 << dg.w_l1;
    dg.ws_a = (Fr *)ctx->pool.alloc(ns * na * sizeof(Fr));
    dg.ws_b = (Fr *)ctx->pool.alloc(ns * nb * sizeof(Fr));
    if (!dg.ws_a || !dg.ws_b) return fail(ctx, DP_E_OOM, "slice factor tables (%u x 2^%u)", ns, dg.log_n);
    for (uint32_t k = 0; k < ns; k++) {
        const Fr s = slice_shift(dq, k), one = Fr::one();
        DP_TRY(gen_powers(ctx, dg.ws_a + k * na, na, s, 0, 1, one));
        DP_TRY(gen_powers(ctx, dg.ws_b + k * nb, nb, s, 0, na, one));
    }
    return DP_OK;
}

void free_domain(dp_ctx *ctx, DomainDev &d) {
    ctx->pool.release(d.ws_a);
    ctx->pool.release(d.ws_b);
    ctx->pool.release(d.H);
    ctx->pool.release(d.g_row);
    ctx->pool.release(d.g_col);
    ctx->pool.release(d.gi_col);
    ctx->pool.release(d.gi_pt);
    ctx->pool.release(d.wg_a);
    ctx->pool.release(d.wg_b);
    ctx->pool.release(d.wgi_a);
    ctx->pool.release(d.wgi_b);
    d = DomainDev();
}

// only called when every stream is done with the task (after the D2H of dp_fft2, or at dp_init)
void p2p_release_slot(dp_ctx *ctx, const Fr *slot);
void free_task(dp_ctx *ctx, FftTask &t) {
    if (t.p2p) p2p_release_slot(ctx, t.recv);
    if (t.recv && t.recv != t.send && !t.p2p) ctx->pool.release(t.recv);
    if (t.send && t.send != t.rows) ctx->pool.release(t.send);
    ctx->pool.release(t.cols);
    ctx->pool_io.release(t.rows);
    t.rows = t.send = t.recv = t.cols = nullptr;
    if (t.ev_in) cudaEventDestroy(t.ev_in);
    if (t.ev_c) cudaEventDestroy(t.ev_c);
    t.ev_in = t.ev_c = nullptr;
}

// ------------------------------------------------------------------ MSM driver (device pointers)
// One MSM in flight: its scratch lives until msm_finish().  The head (digit sort + bucket
// accumulation: wide kernels) runs on the compute stream, the tail (bucket reduction, window sum,
// normalisation: narrow, latency-bound kernels) on s_tail, so that in a batch the tail of MSM k
// overlaps the head of MSM k+1 - the dispatcher issues the commitments of a round concurrently
// (join_all, dispatcher2.rs:316-321, 526-532).
// The digit sort of a job (histogram, scan, scatter: atomics and memory traffic, no multiplier work) can run on a third
// stream, s_sort, so that in a batch the sort of MSM k+1 runs under the accumulation of MSM k instead of in front of it
// (dp_ctx::msm_sort_own_stream; off by default - measured slower, see there).
struct MsmJob {
    std::vector<void *> scratch;
    uint32_t *err = nullptr;
    cudaEvent_t ev_head = nullptr;    // accumulate + collapse done (compute stream) -> tail stream
    cudaEvent_t ev_ready = nullptr;   // inputs complete and recycled scratch free (compute stream) -> sort stream
    cudaEvent_t ev_sorted = nullptr;  // digits sorted (sort stream) -> compute stream
};
void job_destroy_events(MsmJob &j) {
    if (j.ev_head) cudaEventDestroy(j.ev_head);
    if (j.ev_ready) cudaEventDestroy(j.ev_ready);
    if (j.ev_sorted) cudaEventDestroy(j.ev_sorted);
    j.ev_head = j.ev_ready = j.ev_sorted = nullptr;
}

// an MSM between dp_msm_submit and dp_msm_collect
constexpr uint32_t MSM_SLOTS = 64, MSM_SLOT_BYTES = 256;  // pinned: 144 B result at 0, error flag at 192
struct MsmPending {
    MsmJob job;
    uint4 *scalars = nullptr;         // pool_io
    G1JacobianOut *out = nullptr;     // pool
    cudaEvent_t ev_in = nullptr, ev_done = nullptr;
    uint32_t slot = 0;
};

// `ready`: an event after which the scalars are complete AND every earlier user of the pool blocks this job may be
// handed has finished (a batch records one on the compute stream before it queues anything, so that the sorts of all
// its jobs can run ahead); nullptr = the compute stream as it stands now.
// `points`: the bases are these n device points (dp_msm_points) instead of the context's SRS from `start` on; such an MSM
// always takes the per-window pipeline (no window-multiple table exists for them).
int msm_enqueue(dp_ctx *ctx, uint64_t start, const uint4 *scalars_dev, uint64_t n, G1JacobianOut *out_dev, MsmJob &job,
                bool record_breakdown, cudaEvent_t ready = nullptr, const G1Affine *points = nullptr) {
    cudaStream_t st = ctx->stream, tl = ctx->s_tail, so = ctx->msm_sort_own_stream ? ctx->s_sort : ctx->stream;
    if (n == 0) {
        static const G1JacobianOut id = G1JacobianOut::from_affine(G1Affine::inf());
        DP_CUDA(ctx, cudaMemcpyAsync(out_dev, &id, sizeof id, cudaMemcpyHostToDevice, st));
        return DP_OK;
    }
    if (n >= ((uint64_t)1 << 31)) return fail(ctx, DP_E_ARG, "msm: %llu points exceed 2^31", (unsigned long long)n);
    // precomputed window multiples pay off once the shared bucket set is reasonably filled
    const bool use_pre = !points && ctx->pre_table && ctx->msm_force_c == 0 && start >= ctx->pre_lo && start + n <= ctx->pre_hi &&
                         n * ctx->pre_nw >= 4ull * (1ull << (ctx->pre_c - 1));
    MsmGeom g = use_pre ? msm_make_geom(ctx->pre_c, true, ctx->pre_hi - ctx->pre_lo)
                        : msm_geometry(n, ctx->msm_force_c > 1 ? ctx->msm_force_c : 0);
    if (ctx->msm_chunk) g.chunk = ctx->msm_chunk;
    const G1Affine *bases = points ? points : use_pre ? ctx->pre_table + (start - ctx->pre_lo) : ctx->bases + start;
    const uint64_t max_digits = n * g.n_windows;
    // L batched-affine tree levels in front of the XYZZ chunks (msm.cuh): every bucket's slice of the sorted array is padded
    // to a multiple of 2^L entries, the chunk kernel then sees 1 / 2^L of the entries
    uint32_t L = max_digits >= ctx->msm_affine_min_digits ? ctx->msm_affine_levels : 0;
    if (max_digits + ((uint64_t)g.n_keys << L) >= ((uint64_t)1 << 32)) L = 0;  // offsets are 32-bit
    const uint64_t max_entries = max_digits + (L ? (uint64_t)g.n_keys * (((uint64_t)1 << L) - 1) : 0);
    const uint64_t max_chunks = (max_entries >> L) / g.chunk + 1;
    const uint64_t n_slots = max_chunks + g.n_keys;  // partial (chunk j, bucket b) lives in slot j + b
    const uint32_t n_segs = g.red_windows * g.segs_per_window;
    const uint32_t n_scan_blocks = (g.n_keys + SCAN_BLOCK - 1) / SCAN_BLOCK;
    const uint64_t max_multi = max_chunks / MSM_BIG_SPAN + 1;  // buckets spread over > BIG_SPAN chunks
    bool oom = false;
    auto grab = [&](size_t bytes) -> void * {
        void *p = ctx->pool.alloc(bytes);
        if (!p) oom = true;
        job.scratch.push_back(p);
        return p;
    };
    uint32_t *counts = (uint32_t *)grab((g.n_keys + 1) * 4ull);
    uint32_t *offsets = (uint32_t *)grab((g.n_keys + 1) * 4ull);
    uint32_t *cursor = (uint32_t *)grab((g.n_keys + 1) * 4ull);
    uint32_t *sorted = (uint32_t *)grab(max_entries * 4ull);
    uint32_t *offsets_l = L ? (uint32_t *)grab((g.n_keys + 1) * 4ull) : offsets;  // bucket starts after the tree levels
    // level buffers: outputs of the levels, prefix products, block roots and their inverses.  Only the compute stream touches
    // them and the last of them is consumed by the chunk kernel queued below, so they go back to the pool when this function
    // returns (stream-ordered reuse by the next job) - unless sorts run on their own stream and could be handed the blocks
    Scratch level_tmp(ctx->pool);
    auto grab_level = [&](size_t bytes) -> void * {
        if (ctx->msm_sort_own_stream) return grab(bytes);
        void *p = level_tmp.get<uint8_t>(bytes);
        if (!p) oom = true;
        return p;
    };
    G1Affine *lvl_out[4] = {nullptr, nullptr, nullptr, nullptr};
    Fq *lvl_pre = nullptr, *lvl_root = nullptr, *lvl_inv = nullptr;
    const uint32_t lvl_blocks = L ? blocks_for(max_entries >> 1, AFF_BLOCK_PAIRS) : 0;
    if (L) {
        for (uint32_t l = 0; l < L; l++) lvl_out[l] = (G1Affine *)grab_level((max_entries >> (l + 1)) * sizeof(G1Affine) + 512);
        lvl_pre = (Fq *)grab_level((max_entries >> 1) * sizeof(Fq) + 512);
        lvl_root = (Fq *)grab_level((size_t)lvl_blocks * sizeof(Fq));
        lvl_inv = (Fq *)grab_level((size_t)lvl_blocks * sizeof(Fq));
    }
    G1XYZZ *partials = (G1XYZZ *)grab(n_slots * sizeof(G1XYZZ));
    G1XYZZ *seg_sums = (G1XYZZ *)grab((uint64_t)n_segs * sizeof(G1XYZZ));
    G1XYZZ *win_sums = (G1XYZZ *)grab((uint64_t)g.red_windows * g.slices * sizeof(G1XYZZ));
    uint32_t *block_sums = (uint32_t *)grab((size_t)n_scan_blocks * 4ull);
    uint32_t *multi_keys = (uint32_t *)grab((max_multi + 1) * 4ull);  // [0] = counter, then keys
    job.err = (uint32_t *)grab(4);
    if (oom) return fail(ctx, DP_E_OOM, "msm scratch for %llu points", (unsigned long long)n);
    if (!job.ev_head) DP_CUDA(ctx, cudaEventCreateWithFlags(&job.ev_head, cudaEventDisableTiming));
    if (!job.ev_sorted) DP_CUDA(ctx, cudaEventCreateWithFlags(&job.ev_sorted, cudaEventDisableTiming));
    if (record_breakdown) cudaEventRecord(ctx->ev_msm[0], st);
    if (!ready) {
        if (!job.ev_ready) DP_CUDA(ctx, cudaEventCreateWithFlags(&job.ev_ready, cudaEventDisableTiming));
        DP_CUDA(ctx, cudaEventRecord(job.ev_ready, st));
        ready = job.ev_ready;
    }
    DP_CUDA(ctx, cudaStreamWaitEvent(so, ready, 0));
    cudaMemsetAsync(counts, 0, (g.n_keys + 1) * 4ull, so);
    cudaMemsetAsync(job.err, 0, 4, so);
    cudaMemsetAsync(multi_keys, 0, 4, so);
    DP_LAUNCH(msm_count_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, so, scalars_dev, n, g, counts, job.err);
    if (L) {  // bucket slices padded to multiples of 2^L; the holes keep the filler = infinity
        DP_LAUNCH(msm_pad_counts_kernel, dim3(blocks_for(g.n_keys, 256)), dim3(256), 0, so, counts, g.n_keys, L);
        cudaMemsetAsync(sorted, 0xff, max_entries * 4ull, so);
    }
    DP_LAUNCH(scan_block_sums_kernel, dim3(n_scan_blocks), dim3(SCAN_TPB), 0, so, counts, g.n_keys, block_sums);
    DP_LAUNCH(scan_block_offsets_kernel, dim3(1), dim3(SCAN_TPB), 0, so, block_sums, n_scan_blocks, offsets, g.n_keys);
    DP_LAUNCH(scan_write_kernel, dim3(n_scan_blocks), dim3(SCAN_TPB), 0, so, counts, g.n_keys, block_sums, offsets);
    cudaMemcpyAsync(cursor, offsets, (g.n_keys + 1) * 4ull, cudaMemcpyDeviceToDevice, so);
    DP_LAUNCH(msm_scatter_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, so, scalars_dev, n, g, cursor, sorted);
    if (!L)
        DP_LAUNCH(msm_find_big_kernel, dim3(blocks_for(g.n_keys, 256)), dim3(256), 0, so, offsets, g.n_keys, g.chunk, multi_keys + 1,
                  multi_keys);
    DP_CUDA(ctx, cudaEventRecord(job.ev_sorted, so));
    DP_CUDA(ctx, cudaStreamWaitEvent(st, job.ev_sorted, 0));
    if (record_breakdown) cudaEventRecord(ctx->ev_msm[1], st);
    if (L) {
        AffSrc src{sorted, bases};
        const uint32_t *n_elems = offsets + g.n_keys;  // total entries of the padded array (device side)
        for (uint32_t l = 0; l < L; l++) {
            const uint32_t nb = blocks_for(max_entries >> (l + 1), AFF_BLOCK_PAIRS);
            if (l == 0) {
                DP_LAUNCH(aff_k1_kernel<true>, dim3(nb), dim3(AFF_TPB), 0, st, src, n_elems, l, lvl_pre, lvl_root);
                DP_LAUNCH(aff_k2_kernel, dim3(blocks_for(nb, 32)), dim3(32), 0, st, (const Fq *)lvl_root, lvl_inv, nb);
                DP_LAUNCH(aff_k3_kernel<true>, dim3(nb), dim3(AFF_TPB), 0, st, src, n_elems, l, (const Fq *)lvl_pre, (const Fq *)lvl_inv, lvl_out[l]);
            } else {
                DP_LAUNCH(aff_k1_kernel<false>, dim3(nb), dim3(AFF_TPB), 0, st, src, n_elems, l, lvl_pre, lvl_root);
                DP_LAUNCH(aff_k2_kernel, dim3(blocks_for(nb, 32)), dim3(32), 0, st, (const Fq *)lvl_root, lvl_inv, nb);
                DP_LAUNCH(aff_k3_kernel<false>, dim3(nb), dim3(AFF_TPB), 0, st, src, n_elems, l, (const Fq *)lvl_pre, (const Fq *)lvl_inv, lvl_out[l]);
            }
            src = AffSrc{nullptr, lvl_out[l]};
        }
        DP_LAUNCH(msm_shift_offsets_kernel, dim3(blocks_for(g.n_keys + 1, 256)), dim3(256), 0, st, (const uint32_t *)offsets, g.n_keys, L, offsets_l);
        DP_LAUNCH(msm_find_big_kernel, dim3(blocks_for(g.n_keys, 256)), dim3(256), 0, st, (const uint32_t *)offsets_l, g.n_keys, g.chunk,
                  multi_keys + 1, multi_keys);
        DP_LAUNCH((msm_accumulate_kernel<3, true>), dim3(blocks_for(max_chunks, MSM_TPB)), dim3(MSM_TPB), 0, st, (const uint32_t *)offsets_l, g.n_keys,
                  g.chunk, (const uint32_t *)nullptr, (const G1Affine *)lvl_out[L - 1], partials);
        ctx->launches += 3 * L + 2;
    } else if (ctx->msm_min_blocks == 4)
        DP_LAUNCH(msm_accumulate_kernel<4>, dim3(blocks_for(max_chunks, MSM_TPB)), dim3(MSM_TPB), 0, st, offsets, g.n_keys, g.chunk, sorted,
                  bases, partials);
    else if (ctx->msm_min_blocks == 5)
        DP_LAUNCH(msm_accumulate_kernel<5>, dim3(blocks_for(max_chunks, MSM_TPB)), dim3(MSM_TPB), 0, st, offsets, g.n_keys, g.chunk, sorted,
                  bases, partials);
    else
        DP_LAUNCH(msm_accumulate_kernel<3>, dim3(blocks_for(max_chunks, MSM_TPB)), dim3(MSM_TPB), 0, st, offsets, g.n_keys, g.chunk, sorted,
                  bases, partials);
    const uint64_t collapse_cap = (uint64_t)ctx->n_sms * 8;  // one resident wave of blocks
    DP_LAUNCH(msm_collapse_kernel, dim3(max_multi * 32 < collapse_cap * MSM_TPB ? blocks_for(max_multi * 32, MSM_TPB) : (unsigned)collapse_cap),
              dim3(MSM_TPB), 0, st, multi_keys + 1, multi_keys, (const uint32_t *)offsets_l, g.chunk, partials);
    if (record_breakdown) cudaEventRecord(ctx->ev_msm[2], st);
    DP_CUDA(ctx, cudaEventRecord(job.ev_head, st));
    DP_CUDA(ctx, cudaStreamWaitEvent(tl, job.ev_head, 0));
    DP_LAUNCH(msm_reduce_kernel, dim3(blocks_for(n_segs, MSM_TPB)), dim3(MSM_TPB), 0, tl, partials, (const uint32_t *)offsets_l, g, seg_sums);
    DP_LAUNCH(msm_window_sum_kernel, dim3(g.red_windows * g.slices), dim3(MSM_TPB), 0, tl, seg_sums, g, win_sums);
    DP_LAUNCH(msm_final_kernel, dim3(1), dim3(32), 0, tl, win_sums, g, out_dev);
    if (record_breakdown) cudaEventRecord(ctx->ev_msm[3], tl);
    ctx->launches += 11;
    DP_CUDA(ctx, cudaGetLastError());
    return DP_OK;
}

// wait for every job, collect the error flags, give the scratch back
int msm_finish(dp_ctx *ctx, std::vector<MsmJob> &jobs, bool breakdown) {
    cudaError_t e = cudaStreamSynchronize(ctx->s_sort);  // (only matters when a job failed between its sort and its accumulation)
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->s_tail);
    uint32_t bad = 0;
    for (MsmJob &j : jobs) {
        if (e == cudaSuccess && j.err) {
            uint32_t flag = 0;
            e = cudaMemcpy(&flag, j.err, 4, cudaMemcpyDeviceToHost);
            bad |= flag;
        }
        for (void *p : j.scratch) ctx->pool.release(p);
        j.scratch.clear();
        job_destroy_events(j);
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DP_E_CUDA, "msm kernels: %s", cudaGetErrorString(e));
    if (breakdown)
        for (int k = 0; k < 3; k++) cudaEventElapsedTime(&ctx->msm_ms[k], ctx->ev_msm[k], ctx->ev_msm[k + 1]);
    if (bad) return fail(ctx, DP_E_ARG, "msm: a scalar is not a canonical Fr integer (>= 2^255)");
    return DP_OK;
}

int msm_device(dp_ctx *ctx, uint64_t start, const uint4 *scalars_dev, uint64_t n, G1JacobianOut *out_dev,
               uint32_t *err_host_out, const G1Affine *points = nullptr) {
    (void)err_host_out;
    std::vector<MsmJob> jobs(1);
    int rc = msm_enqueue(ctx, start, scalars_dev, n, out_dev, jobs[0], n != 0, nullptr, points);
    int rc2 = msm_finish(ctx, jobs, rc == DP_OK && n != 0);
    return rc != DP_OK ? rc : rc2;
}

// dp_init's choice between the plain MSM pipeline and batched-affine tree levels in front of it (2; with DP_MSM_TUNE=2 also 1 and 3):
// one MSM over the context's own window-multiple table per candidate (pseudo-random scalars, warm-up + best of two), every
// result compared byte for byte with the plain pipeline's; the fastest candidate that agrees is kept if it is at least
// 2 % faster than the plain pipeline.  Only the geometry of the hot path is tuned (the whole table range); a worker's
// shard of a multi-GPU MSM is its own context and tunes itself.
int msm_tune(dp_ctx *ctx) {
    ctx->tune_ms[0] = ctx->tune_ms[1] = 0.f;
    for (float &v : ctx->tune_all_ms) v = 0.f;
    ctx->tune_equal = -1;
    if (ctx->msm_affine_forced >= 0) {
        ctx->msm_affine_levels = (uint32_t)ctx->msm_affine_forced;
        return DP_OK;
    }
    ctx->msm_affine_levels = 0;
    const uint64_t span = ctx->pre_hi - ctx->pre_lo, digits = span * ctx->pre_nw;
    if (ctx->msm_tune_mode == 0 || !ctx->pre_table || digits < ctx->msm_affine_min_digits) return DP_OK;
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    if (digits * 200ull > free_b / 2) return DP_OK;  // level buffers: ~ 150 B per digit on top of the plain pipeline's 12
    Scratch tmp(ctx->pool);
    constexpr int N_CAND = 4;                         // levels 0 (plain), 1, 2, 3
    uint4 *sc = tmp.get<uint4>(2 * span);
    G1JacobianOut *out = tmp.get<G1JacobianOut>(N_CAND);
    if (!sc || !out) return DP_OK;  // not enough memory to try: stay on the plain pipeline
    DP_LAUNCH(msm_tune_scalars_kernel, dim3(blocks_for(span, 256)), dim3(256), 0, ctx->stream, sc, span, 0x7A11E5ull);
    ctx->launches++;
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    float ms[N_CAND] = {0.f, 0.f, 0.f, 0.f};
    bool ran[N_CAND] = {false, false, false, false};
    for (int lv = 0; lv < N_CAND; lv++) {
        if (ctx->msm_tune_mode < 2 && (lv == 1 || lv == 3)) continue;
        ctx->msm_affine_levels = (uint32_t)lv;
        double best = 1e30;
        int rc = DP_OK;
        for (int rep = 0; rep < 3 && rc == DP_OK; rep++) {
            const auto t0 = std::chrono::steady_clock::now();
            rc = msm_device(ctx, ctx->pre_lo, sc, span, out + lv, nullptr);
            const double t = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            if (rep && t < best) best = t;
        }
        if (rc != DP_OK) {
            ctx->msm_affine_levels = 0;
            if (lv == 0) return rc;
            // a candidate failed where the plain pipeline had just worked: keep the plain pipeline and say so
            // (tune_equal = 0); a sticky CUDA error will surface again at the caller's next call
            cudaGetLastError();
            ctx->tune_equal = 0;
            return DP_OK;
        }
        ms[lv] = (float)best;
        ran[lv] = true;
    }
    ctx->msm_affine_levels = 0;
    G1JacobianOut host[N_CAND];
    DP_CUDA(ctx, cudaMemcpy(host, out, sizeof host, cudaMemcpyDeviceToHost));
    ctx->tune_ms[0] = ms[0];
    ctx->tune_equal = 1;
    int best_lv = 0;
    for (int lv = 1; lv < N_CAND; lv++) {
        if (!ran[lv]) continue;
        if (memcmp(&host[0], &host[lv], sizeof(G1JacobianOut)) != 0) {
            ctx->tune_equal = 0;  // a candidate that disagrees disqualifies the whole experiment
            continue;
        }
        if (best_lv == 0 ? ms[lv] < 0.98f * ms[0] : ms[lv] < ms[best_lv]) best_lv = lv;
        if (ctx->tune_ms[1] == 0.f || ms[lv] < ctx->tune_ms[1]) ctx->tune_ms[1] = ms[lv];  // the best candidate's time, kept or not
    }
    ctx->msm_affine_levels = ctx->tune_equal == 1 ? (uint32_t)best_lv : 0u;
    for (int lv = 0; lv < N_CAND; lv++) ctx->tune_all_ms[lv] = ms[lv];
    return DP_OK;
}

// give back everything a pending MSM holds; the caller has made sure its kernels are done
void release_pending(dp_ctx *ctx, MsmPending *p) {
    for (void *q : p->job.scratch) ctx->pool.release(q);
    job_destroy_events(p->job);
    ctx->pool_io.release(p->scalars);
    ctx->pool.release(p->out);
    if (p->ev_in) cudaEventDestroy(p->ev_in);
    if (p->ev_done) cudaEventDestroy(p->ev_done);
    ctx->msm_slots_used &= ~(1ull << p->slot);
    delete p;
}

// dp_init / dp_destroy: every stream has been synchronised
void drop_pending_msms(dp_ctx *ctx) {
    for (auto &kv : ctx->msm_pending) release_pending(ctx, kv.second);
    ctx->msm_pending.clear();
}

FftTask *find_task(dp_ctx *ctx, uint64_t id) {
    auto it = ctx->tasks.find(id);
    return it == ctx->tasks.end() ? nullptr : &it->second;
}

constexpr uint64_t ARENA_HEADER_BYTES = 1024;  // arrival counter of the device-side barrier, then the receive slots

bool p2p_ready(const dp_ctx *ctx) {
    if (ctx->W <= 1 || !ctx->arena) return false;
    for (uint64_t q = 0; q < ctx->W; q++)
        if (!ctx->peer_arena[q]) return false;
    return true;
}

// Receive slots of the arena.  One slot holds the receive matrix [r][c/W] of the LARGER of the two domains; the arena
// holds as many as fit (every rank creates it with the same size and has the same domains, so every rank computes
// the same geometry), at least two.  Exchange number k uses slot k mod n_slots on every rank - the ranks issue their
// exchanges in the same order, as they would for a collective - so at most n_slots fused exchanges may be between
// their row phase and their column phase per context: one more would overwrite a receive matrix nobody has read
// yet.  The reference dispatcher keeps up to 26 transforms in flight (join_all, dispatcher2.rs:382-414): a worker
// serving it creates an arena of 32 slots (rust/worker_gpu.rs); bench.py's resident path needs two.
// The slot is only reserved here; p2p_commit_slot() consumes the sequence number once the row kernels were queued
// without error, so a failed call leaves every rank's sequence where it was.
struct SlotGeom {
    uint64_t slot_elems, n_slots;
};
SlotGeom p2p_slot_geom(const dp_ctx *ctx) {
    uint64_t need = 0;
    for (int k = 0; k < 2; k++) {
        const uint64_t b = ctx->dom[k].n() / ctx->W;  // r * (c / W) elements
        if (ctx->dom[k].H && b > need) need = b;
    }
    SlotGeom g{need, 0};
    if (need == 0 || !ctx->arena) return g;
    g.n_slots = (ctx->arena_bytes - ARENA_HEADER_BYTES) / (need * sizeof(Fr));
    if (g.n_slots > dp_ctx::P2P_MAX_SLOTS) g.n_slots = dp_ctx::P2P_MAX_SLOTS;
    return g;
}
int p2p_next_slot(dp_ctx *ctx, uint64_t recv_bytes, PeerDst &dst, Fr *&my_slot, uint64_t row_off) {
    const SlotGeom g = p2p_slot_geom(ctx);
    if (g.n_slots < 2 || recv_bytes > g.slot_elems * sizeof(Fr))
        return fail(ctx, DP_E_COMM, "peer arena of %llu B holds %llu receive matrices of %llu B: at least 2 are needed", (unsigned long long)ctx->arena_bytes,
                    (unsigned long long)g.n_slots, (unsigned long long)(g.slot_elems * sizeof(Fr)));
    const uint64_t s = ctx->p2p_seq % g.n_slots;
    if (ctx->p2p_slot_busy[s])
        return fail(ctx, DP_E_STATE, "fused exchange: all %llu receive slots hold transforms whose column phase has not run (that many may sit "
                                     "between fft2_prepare and fft2 per context); finish one with dp_fft2, create a larger arena, or use dp_fft_exchange_begin/_end",
                    (unsigned long long)g.n_slots);
    const uint64_t off = ARENA_HEADER_BYTES / sizeof(Fr) + s * g.slot_elems;
    for (uint64_t q = 0; q < ctx->W; q++) dst.base[q] = ctx->peer_arena[q] + off;
    dst.row_off = row_off;
    my_slot = ctx->arena + off;
    return DP_OK;
}
void p2p_commit_slot(dp_ctx *ctx) {
    ctx->p2p_slot_busy[ctx->p2p_seq % p2p_slot_geom(ctx).n_slots] = true;
    ctx->p2p_seq++;
}
void p2p_release_slot(dp_ctx *ctx, const Fr *slot) {
    if (!slot || !ctx->arena) return;
    const SlotGeom g = p2p_slot_geom(ctx);
    if (!g.slot_elems) return;
    const uint64_t s = (uint64_t)(slot - (ctx->arena + ARENA_HEADER_BYTES / sizeof(Fr))) / g.slot_elems;
    if (s < dp_ctx::P2P_MAX_SLOTS) ctx->p2p_slot_busy[s] = false;
}

// rows handed in short (dp_fft1 with len < c, dp_fft1_rows_short): the first pass reads rd columns of every row;
// whatever lies between a row's own length and rd is zero-filled here (compute stream, after the copy-in), the rest
// of the tail is never touched.  Returns rd.
uint64_t fill_short_rows(dp_ctx *ctx, FftTask &t, const DomainDev &d) {
    const uint64_t c = d.c();
    uint64_t valid = 1;
    bool same = true;
    for (uint64_t i = 0; i < t.n_rows; i++) {
        if (t.row_len[i] > valid) valid = t.row_len[i];
        same = same && t.row_len[i] == t.row_len[0];
    }
    const uint64_t rd = row_read_cols(ctx, d, valid);
    if (same) {
        if (t.n_rows && t.row_len[0] < rd)
            cudaMemset2DAsync(t.rows + t.row_len[0], c * sizeof(Fr), 0, (rd - t.row_len[0]) * sizeof(Fr), t.n_rows, ctx->stream);
    } else {
        for (uint64_t i = 0; i < t.n_rows; i++)
            if (t.row_len[i] < rd) cudaMemsetAsync(t.rows + i * c + t.row_len[i], 0, (rd - t.row_len[i]) * sizeof(Fr), ctx->stream);
    }
    return rd;
}

// one worker: the whole transform of a task as three passes rows -> scratch -> rows -> cols (plan_single_worker3)
int run_single_worker(dp_ctx *ctx, FftTask &t) {
    if (t.exchanged) return fail(ctx, DP_E_STATE, "fft task: the transform of this task was already queued");
    if (t.rows_filled != t.n_rows) return fail(ctx, DP_E_STATE, "fft task: %llu of %llu rows received", (unsigned long long)t.rows_filled, (unsigned long long)t.n_rows);
    const DomainDev &d = ctx->dom[t.is_quot ? 1 : 0];
    const Split3 s3 = single_worker_split(ctx, d);
    Scratch tmp(ctx->pool);  // stream-ordered: handed back when the kernels that use it are already queued
    Fr *w1 = tmp.get<Fr>(d.n());
    if (!t.cols) t.cols = (Fr *)ctx->pool.alloc(t.n_cols * d.r() * sizeof(Fr));
    if (!w1 || !t.cols) return fail(ctx, DP_E_OOM, "single-worker transform buffers");
    cudaStreamWaitEvent(ctx->stream, t.ev_in, 0);
    const uint64_t rd = fill_short_rows(ctx, t, d);
    DP_TRY(plan_single_worker3(ctx, d, s3, t.rows, w1, t.rows, t.cols, t.is_inv, t.is_coset, rd));
    DP_CUDA(ctx, cudaEventRecord(t.ev_c, ctx->stream));
    t.send = t.recv = t.rows;
    t.row_phase_done = t.exchanged = true;
    return DP_OK;
}

int run_row_phase(dp_ctx *ctx, FftTask &t, bool use_p2p = false) {
    if (t.row_phase_done) return DP_OK;
    if (t.rows_filled != t.n_rows) return fail(ctx, DP_E_STATE, "fft task: %llu of %llu rows received", (unsigned long long)t.rows_filled, (unsigned long long)t.n_rows);
    const DomainDev &d = ctx->dom[t.is_quot ? 1 : 0];
    const uint64_t c = d.c();
    Fr *scratch = nullptr;
    if (d.log_c > ctx->max_contig_log_k) {
        scratch = (Fr *)ctx->pool.alloc(t.n_rows * c * sizeof(Fr));
        if (!scratch) return fail(ctx, DP_E_OOM, "row-phase scratch");
    }
    PeerDst peers;
    Fr *slot = nullptr;
    if (use_p2p) {
        // block q of my rows goes straight to rows [me*n_rows, ...) of worker q's receive matrix
        int rc0 = p2p_next_slot(ctx, d.r() * t.n_cols * sizeof(Fr), peers, slot, ctx->me * t.n_rows * t.n_cols);
        if (rc0 != DP_OK) {
            ctx->pool.release(scratch);
            return rc0;
        }
    } else if (ctx->W > 1 && !t.send) {
        t.send = (Fr *)ctx->pool.alloc(t.n_rows * c * sizeof(Fr));
        if (!t.send) {
            ctx->pool.release(scratch);
            return fail(ctx, DP_E_OOM, "exchange send buffer");
        }
    } else if (ctx->W == 1) {
        t.send = t.rows;
    }
    cudaStreamWaitEvent(ctx->stream, t.ev_in, 0);
    const uint64_t rd = fill_short_rows(ctx, t, d);
    int rc = plan_row_phase(ctx, d, t.rows, t.send, scratch, t.n_rows, t.row_start, t.is_inv, t.is_coset, ctx->W,
                            use_p2p ? &peers : nullptr, rd);
    ctx->pool.release(scratch);
    if (rc == DP_OK) {
        t.row_phase_done = true;
        if (use_p2p) {
            t.recv = slot;
            t.p2p = true;
            p2p_commit_slot(ctx);
        }
    }
    return rc;
}

// queue the column phase of a task whose recv matrix is complete; result lands in t.cols
int queue_col_phase(dp_ctx *ctx, FftTask &t) {
    const DomainDev &d = ctx->dom[t.is_quot ? 1 : 0];
    // the two-pass column plan works in place on `recv`: running it twice would transform garbage
    if (t.exchanged) return fail(ctx, DP_E_STATE, "fft task: the column phase of this task was already queued");
    if (!t.cols) {
        t.cols = (Fr *)ctx->pool.alloc(t.n_cols * d.r() * sizeof(Fr));
        if (!t.cols) return fail(ctx, DP_E_OOM, "column buffer");
    }
    DP_TRY(plan_col_phase(ctx, d, t.recv, t.cols, t.n_cols, t.col_start, t.is_inv, t.is_coset));
    DP_CUDA(ctx, cudaEventRecord(t.ev_c, ctx->stream));
    t.exchanged = true;
    return DP_OK;
}

}  // namespace

// =================================================================== C ABI
extern "C" {

const char *dp_version(void) { return "distributed_plonk_b200 0.1 (sm_90a)"; }

const char *dp_last_error(const dp_ctx *ctx) { return ctx ? ctx->err.c_str() : g_err_noctx.c_str(); }

int dp_create(int cuda_device, uint64_t me, uint64_t n_workers, dp_ctx **out) {
    if (!out) return fail(nullptr, DP_E_ARG, "dp_create: out is NULL");
    *out = nullptr;
    if (n_workers == 0 || (n_workers & (n_workers - 1)) || me >= n_workers)
        return fail(nullptr, DP_E_ARG, "dp_create: n_workers must be a power of two and me < n_workers");
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0)
        return fail(nullptr, DP_E_CUDA, "dp_create: no CUDA device (this library has no CPU path)");
    if (cuda_device < 0 || cuda_device >= n_dev) return fail(nullptr, DP_E_ARG, "dp_create: device %d of %d", cuda_device, n_dev);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, cuda_device) != cudaSuccess) return fail(nullptr, DP_E_CUDA, "cudaGetDeviceProperties");
    // the library holds sm_90a code only, which runs on compute capability 9.0 and nothing else
    if (prop.major != 9 || prop.minor != 0)
        return fail(nullptr, DP_E_CUDA, "dp_create: device %d is sm_%d%d, need sm_90 (H100)", cuda_device, prop.major, prop.minor);
    dp_ctx *ctx = new dp_ctx();
    ctx->device = cuda_device;
    ctx->n_sms = (uint32_t)prop.multiProcessorCount;
    if (const char *e = getenv("DP_MSM_CHUNK")) ctx->msm_chunk = (uint32_t)atoi(e) >= 8 ? (uint32_t)atoi(e) : 0;
    if (const char *e = getenv("DP_NTT_BLOCKS")) ctx->ntt_min_blocks = atoi(e) == 2 ? 2 : 3;
    if (const char *e = getenv("DP_NTT_PREFETCH")) ctx->ntt_tw_prefetch = atoi(e) != 0;
    if (const char *e = getenv("DP_NTT_NO_3PASS")) ctx->no_three_pass = atoi(e) != 0;
    if (const char *e = getenv("DP_MSM_BLOCKS")) ctx->msm_min_blocks = atoi(e) >= 3 && atoi(e) <= 5 ? atoi(e) : 3;
    if (const char *e = getenv("DP_QUOT_TABLE")) ctx->quot_table = atoi(e) != 0 ? 1 : 0;
    if (const char *e = getenv("DP_MSM_SORT_STREAM")) ctx->msm_sort_own_stream = atoi(e) != 0;
    if (const char *e = getenv("DP_MSM_AFFINE")) {
        ctx->msm_affine_forced = atoi(e) < 0 ? 0 : atoi(e) > 3 ? 3 : atoi(e);
        ctx->msm_affine_levels = (uint32_t)ctx->msm_affine_forced;
    }
    if (const char *e = getenv("DP_MSM_AFFINE_MIN")) ctx->msm_affine_min_digits = strtoull(e, nullptr, 10);
    if (const char *e = getenv("DP_MSM_TUNE")) ctx->msm_tune_mode = atoi(e) < 0 ? 0 : atoi(e) > 2 ? 2 : atoi(e);
    if (const char *e = getenv("DP_MSM_PRE_C")) {
        char *end = nullptr;
        const long v = strtol(e, &end, 10);
        ctx->msm_pre_c = end != e && *end == '\0' && v >= 0 && v <= 64 ? (int)v : 1000;
        ctx->pre_disabled = ctx->msm_pre_c == 0;
    }
    ctx->me = me;
    ctx->W = n_workers;
    int rc = DP_OK;
    do {
        if (cudaSetDevice(cuda_device) != cudaSuccess) { rc = DP_E_CUDA; break; }
        if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { rc = DP_E_CUDA; break; }
        if (cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking) != cudaSuccess) { rc = DP_E_CUDA; break; }
        if (cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking) != cudaSuccess) { rc = DP_E_CUDA; break; }
        if (cudaStreamCreateWithFlags(&ctx->s_tail, cudaStreamNonBlocking) != cudaSuccess) { rc = DP_E_CUDA; break; }
        if (cudaStreamCreateWithFlags(&ctx->s_sort, cudaStreamNonBlocking) != cudaSuccess) { rc = DP_E_CUDA; break; }
        cudaEventCreate(&ctx->ev0);
        cudaEventCreate(&ctx->ev1);
        for (int k = 0; k < 4; k++) cudaEventCreate(&ctx->ev_msm[k]);
        if (cudaFuncSetAttribute(ntt_tile_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)ntt_pass_smem_bytes(NTT_WTAB_LOG, 0)) != cudaSuccess) { rc = DP_E_CUDA; break; }
        if (cudaFuncSetAttribute(ntt_tile_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)ntt_pass_smem_bytes(NTT_WTAB_LOG, 0)) != cudaSuccess) { rc = DP_E_CUDA; break; }
        const size_t wb = ((size_t)1 << NTT_WTAB_LOG) * sizeof(uint4);
        ctx->wf_lo = (uint4 *)ctx->pool.alloc(wb);
        ctx->wf_hi = (uint4 *)ctx->pool.alloc(wb);
        ctx->wi_lo = (uint4 *)ctx->pool.alloc(wb);
        ctx->wi_hi = (uint4 *)ctx->pool.alloc(wb);
        if (!ctx->wf_lo || !ctx->wf_hi || !ctx->wi_lo || !ctx->wi_hi) { rc = DP_E_OOM; break; }
        const unsigned nb = (1u << NTT_WTAB_LOG) / 256;
        DP_LAUNCH(ntt_gen_level_table_kernel, dim3(nb), dim3(256), 0, ctx->stream, ctx->wf_lo, ctx->wf_hi, 0u);
        DP_LAUNCH(ntt_gen_level_table_kernel, dim3(nb), dim3(256), 0, ctx->stream, ctx->wi_lo, ctx->wi_hi, 1u);
        ctx->launches += 2;
        if (cudaStreamSynchronize(ctx->stream) != cudaSuccess || cudaGetLastError() != cudaSuccess) { rc = DP_E_CUDA; break; }
    } while (0);
    if (rc != DP_OK) {
        fail(nullptr, rc, "dp_create: CUDA initialisation failed on device %d", cuda_device);
        ctx->pool.destroy();
        ctx->pool_io.destroy();
        delete ctx;
        return rc;
    }
    *out = ctx;
    return DP_OK;
}

int dp_destroy(dp_ctx *ctx) {
    if (!ctx) return DP_OK;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->s_in);
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->s_out);
    for (auto &kv : ctx->tasks) {
        if (kv.second.ev_in) cudaEventDestroy(kv.second.ev_in);
        if (kv.second.ev_c) cudaEventDestroy(kv.second.ev_c);
    }
    cudaStreamSynchronize(ctx->s_sort);
    cudaStreamSynchronize(ctx->s_tail);
    drop_pending_msms(ctx);
    if (ctx->msm_pinned) cudaFreeHost(ctx->msm_pinned);
    ctx->pool.destroy();
    ctx->pool_io.destroy();
    for (uint64_t q = 0; q < 8; q++)
        if (ctx->peer_arena[q] && q != ctx->me) cudaIpcCloseMemHandle(ctx->peer_arena[q]);
    if (ctx->arena) cudaFree(ctx->arena);
    if (ctx->s_in) cudaStreamDestroy(ctx->s_in);
    if (ctx->s_out) cudaStreamDestroy(ctx->s_out);
    if (ctx->s_tail) cudaStreamDestroy(ctx->s_tail);
    if (ctx->s_sort) cudaStreamDestroy(ctx->s_sort);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    for (int k = 0; k < 4; k++)
        if (ctx->ev_msm[k]) cudaEventDestroy(ctx->ev_msm[k]);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return DP_OK;
}

static int p2p_check_timeout(dp_ctx *ctx);
int dp_sync(dp_ctx *ctx) {
    if (!ctx) return DP_E_ARG;
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->s_in));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->s_sort));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->s_tail));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->s_out));
    return p2p_check_timeout(ctx);
}

int dp_last_timing(const dp_ctx *ctx, float *kernel_ms, uint64_t *launches) {
    if (!ctx) return DP_E_ARG;
    if (kernel_ms) *kernel_ms = ctx->last_ms;
    if (launches) *launches = ctx->launches - ctx->launches_at_call;
    return DP_OK;
}

uint64_t dp_launch_count(const dp_ctx *ctx) { return ctx ? ctx->launches : 0; }

// g1_decompress_kernel's reason codes (msm.cuh)
static const char *const G1_DECOMPRESS_WHY[] = {"", "x is not a canonical field element", "both flag bits set",
                                                "x^3 + 4 is not a square: no such point", "the point is not in the r-torsion subgroup"};

// format 0: raw ark GroupAffine structs (104 B, utils.rs:27-43) - what the reference's init RPC carries;
// format 1: ark-serialize compressed points (48 B) - what SRS files hold ("next" row 4)
static int init_impl(dp_ctx *ctx, const void *bases, size_t n_bases, uint64_t domain_size, uint64_t quot_domain_size, int format,
                     int check_subgroup) {
    if (!ctx) return DP_E_ARG;
    if (n_bases && !bases) return fail(ctx, DP_E_ARG, "dp_init: bases is NULL");
    if (domain_size == 0 || quot_domain_size == 0) return fail(ctx, DP_E_ARG, "dp_init: domain sizes must be >= 1");
    if (ctx->msm_pre_c > 0 && (ctx->msm_pre_c < 8 || ctx->msm_pre_c > 22))
        return fail(ctx, DP_E_ARG, "dp_init: DP_MSM_PRE_C must be 0 or a table width of 8 to 22");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    // drop previous state (init may be called again, worker.rs:135-141 overwrites)
    cudaStreamSynchronize(ctx->s_in);
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->s_out);
    for (auto &kv : ctx->tasks) free_task(ctx, kv.second);
    ctx->tasks.clear();
    for (bool &b : ctx->p2p_slot_busy) b = false;  // (the slot geometry follows the new domains; every rank re-initialises alike)
    ctx->dev_p2p_slot = nullptr;
    cudaStreamSynchronize(ctx->s_sort);
    cudaStreamSynchronize(ctx->s_tail);
    drop_pending_msms(ctx);
    ctx->pool.release(ctx->bases);
    ctx->pool.release(ctx->pre_table);
    ctx->bases = nullptr;
    ctx->pre_table = nullptr;
    ctx->pre_c = ctx->pre_nw = 0;
    ctx->pre_lo = ctx->pre_hi = 0;
    free_domain(ctx, ctx->dom[0]);
    free_domain(ctx, ctx->dom[1]);
    ctx->pool.release(ctx->quot_inv);
    ctx->quot_inv = nullptr;
    ctx->pool.release(ctx->srs_table);
    ctx->srs_table = nullptr;
    ctx->inited = false;
    ctx->n_bases = n_bases;
    if (n_bases) {
        ctx->bases = (G1Affine *)ctx->pool.alloc(n_bases * sizeof(G1Affine));
        const size_t in_bytes = n_bases * (size_t)(format == 0 ? DP_G1_AFFINE_BYTES : DP_G1_COMPRESSED_BYTES);
        Scratch stage(ctx->pool);
        void *staging = stage.get<uint8_t>(in_bytes);
        if (!ctx->bases || !staging) return fail(ctx, DP_E_OOM, "dp_init: %zu bases", n_bases);
        DP_CUDA(ctx, cudaMemcpyAsync(staging, bases, in_bytes, cudaMemcpyDefault, ctx->stream));  // host or device memory
        if (format == 0) {
            DP_LAUNCH(g1_import_ark_kernel, dim3(blocks_for(n_bases, 256)), dim3(256), 0, ctx->stream,
                      (const uint64_t *)staging, ctx->bases, (uint64_t)n_bases);
        } else {
            unsigned long long *err = stage.get<unsigned long long>(1), verdict = ~0ull;
            if (!err) return fail(ctx, DP_E_OOM, "dp_init_compressed scratch");
            DP_CUDA(ctx, cudaMemcpyAsync(err, &verdict, sizeof verdict, cudaMemcpyHostToDevice, ctx->stream));
            DP_LAUNCH(g1_decompress_kernel, dim3(blocks_for(n_bases, 128)), dim3(128), 0, ctx->stream, (const uint32_t *)staging,
                      ctx->bases, (uint64_t)n_bases, check_subgroup ? 1u : 0u, err);
            DP_CUDA(ctx, cudaMemcpyAsync(&verdict, err, sizeof verdict, cudaMemcpyDeviceToHost, ctx->stream));
            DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            if (verdict != ~0ull) {
                ctx->pool.release(ctx->bases);
                ctx->bases = nullptr;
                ctx->n_bases = 0;
                return fail(ctx, DP_E_ARG, "dp_init_compressed: point %llu rejected: %s", (unsigned long long)((verdict >> 8) - 1),
                            G1_DECOMPRESS_WHY[verdict & 7]);
            }
        }
        ctx->launches++;
        // window multiples for the MSM (skipped for tiny SRS or when memory is short)
        size_t free_b = 0, total_b = 0;
        cudaMemGetInfo(&free_b, &total_b);
        const uint64_t lo = ctx->me * n_bases / ctx->W, hi = (ctx->me + 1) * n_bases / ctx->W, span = hi - lo;
        uint32_t c = span >= (1u << 11) && !ctx->pre_disabled ? msm_pick_pre_c(span, free_b / 4) : 0;
        if (ctx->msm_pre_c > 0) {  // pinned width: exactly this table or an error, never another width
            c = (uint32_t)ctx->msm_pre_c;
            const uint64_t nw = (256 + c - 1) / c;
            if (span < (1u << 11) || nw * span >= (1ull << 31))
                return fail(ctx, DP_E_ARG, "dp_init: DP_MSM_PRE_C=%u does not fit a shard of %llu bases (needs >= 2^11 and %llu windows * bases < 2^31)",
                            c, (unsigned long long)span, (unsigned long long)nw);
        }
        if (c) {
            const uint32_t nw = (256 + c - 1) / c;
            ctx->pre_table = nw <= (uint32_t)MSM_PRE_MAX_WINDOWS ? (G1Affine *)ctx->pool.alloc((size_t)nw * span * sizeof(G1Affine)) : nullptr;
            if (!ctx->pre_table && ctx->msm_pre_c > 0)
                return fail(ctx, DP_E_OOM, "dp_init: DP_MSM_PRE_C=%u: no room for the %.1f GB window table of %llu bases", c,
                            (double)nw * span * sizeof(G1Affine) / 1e9, (unsigned long long)span);
            if (ctx->pre_table) {
                ctx->pre_c = c;
                ctx->pre_nw = nw;
                ctx->pre_lo = lo;
                ctx->pre_hi = hi;
                DP_LAUNCH(msm_precompute_kernel, dim3(blocks_for(span, 128)), dim3(128), 0, ctx->stream, ctx->bases + lo,
                          ctx->pre_table, span, span, c, nw);
                ctx->launches++;
            }
        }
    }
    DP_TRY(build_domain(ctx, ctx->dom[0], domain_size));
    DP_TRY(build_domain(ctx, ctx->dom[1], quot_domain_size));
    DP_TRY(build_slice_tables(ctx, ctx->dom[0], ctx->dom[1]));
    for (int k = 0; k < 2; k++) {
        const DomainDev &d = ctx->dom[k];
        if (d.r() < ctx->W || d.c() < ctx->W)
            return fail(ctx, DP_E_ARG, "dp_init: domain 2^%u too small to split over %llu workers", d.log_n, (unsigned long long)ctx->W);
    }
    DP_TRY(call_end(ctx, true));
    DP_TRY(msm_tune(ctx));
    ctx->inited = true;
    return DP_OK;
}

int dp_init(dp_ctx *ctx, const void *bases, size_t n_bases, uint64_t domain_size, uint64_t quot_domain_size) {
    return init_impl(ctx, bases, n_bases, domain_size, quot_domain_size, 0, 0);
}

int dp_init_compressed(dp_ctx *ctx, const void *bases48, size_t n_bases, uint64_t domain_size, uint64_t quot_domain_size, int check_subgroup) {
    return init_impl(ctx, bases48, n_bases, domain_size, quot_domain_size, 1, check_subgroup);
}

int dp_get_bases(dp_ctx *ctx, uint64_t start, size_t n, void *out104) {
    if (!ctx || (n && !out104)) return fail(ctx, DP_E_ARG, "dp_get_bases: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_get_bases before dp_init");
    if (start > ctx->n_bases || n > ctx->n_bases - start) return fail(ctx, DP_E_ARG, "dp_get_bases: range outside %llu bases", (unsigned long long)ctx->n_bases);
    if (n == 0) return DP_OK;
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    uint64_t *ark = tmp.get<uint64_t>(n * 13);
    if (!ark) return fail(ctx, DP_E_OOM, "dp_get_bases buffer");
    DP_LAUNCH(g1_export_ark_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, ctx->stream, (const G1Affine *)(ctx->bases + start), ark, (uint64_t)n);
    ctx->launches++;
    DP_CUDA(ctx, cudaMemcpyAsync(out104, ark, n * (size_t)DP_G1_AFFINE_BYTES, cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

int dp_msm(dp_ctx *ctx, uint64_t start, uint64_t end, const void *scalars, size_t n_scalars, void *out) {
    if (!ctx || !out) return fail(ctx, DP_E_ARG, "dp_msm: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_msm before dp_init");
    if (start > end || end > ctx->n_bases) return fail(ctx, DP_E_ARG, "dp_msm: range [%llu,%llu) outside %llu bases", (unsigned long long)start, (unsigned long long)end, (unsigned long long)ctx->n_bases);
    if (n_scalars && !scalars) return fail(ctx, DP_E_ARG, "dp_msm: scalars is NULL");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint64_t n = (end - start) < n_scalars ? (end - start) : n_scalars;
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    uint4 *sc = tmp.get<uint4>(2 * n);
    G1JacobianOut *od = tmp.get<G1JacobianOut>(1);
    if (!sc || !od) return fail(ctx, DP_E_OOM, "dp_msm buffers");
    if (n) DP_CUDA(ctx, cudaMemcpyAsync(sc, scalars, n * 32, cudaMemcpyHostToDevice, ctx->stream));
    DP_TRY(msm_device(ctx, start, sc, n, od, nullptr));
    DP_CUDA(ctx, cudaMemcpyAsync(out, od, sizeof(G1JacobianOut), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

int dp_msm_dev(dp_ctx *ctx, uint64_t start, uint64_t end, const void *scalars_dev, size_t n_scalars, void *out_dev) {
    if (!ctx || !out_dev) return fail(ctx, DP_E_ARG, "dp_msm_dev: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_msm_dev before dp_init");
    if (start > end || end > ctx->n_bases) return fail(ctx, DP_E_ARG, "dp_msm_dev: bad range");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint64_t n = (end - start) < n_scalars ? (end - start) : n_scalars;
    call_begin(ctx);
    DP_TRY(msm_device(ctx, start, (const uint4 *)scalars_dev, n, (G1JacobianOut *)out_dev, nullptr));
    return call_end(ctx, true);
}

int dp_msm_dev_batch(dp_ctx *ctx, size_t n_jobs, const uint64_t *starts, const uint64_t *ends, const void *const *scalars_dev,
                     const size_t *n_scalars, void *const *outs_dev) {
    if (!ctx || (n_jobs && (!starts || !ends || !scalars_dev || !n_scalars || !outs_dev))) return fail(ctx, DP_E_ARG, "dp_msm_dev_batch: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_msm_dev_batch before dp_init");
    for (size_t k = 0; k < n_jobs; k++)
        if (starts[k] > ends[k] || ends[k] > ctx->n_bases || !outs_dev[k]) return fail(ctx, DP_E_ARG, "dp_msm_dev_batch: job %zu has a bad range / output", k);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    std::vector<MsmJob> jobs(n_jobs);
    int rc = DP_OK;
    // every job's scalars are complete where the compute stream stands now (the caller's contract for *_dev inputs), and so
    // is every earlier user of the pool blocks the jobs will be handed: one event lets all the sorts run ahead
    cudaEvent_t ev_batch = nullptr;
    if (cudaEventCreateWithFlags(&ev_batch, cudaEventDisableTiming) != cudaSuccess || cudaEventRecord(ev_batch, ctx->stream) != cudaSuccess)
        rc = fail(ctx, DP_E_CUDA, "dp_msm_dev_batch: event");
    for (size_t k = 0; k < n_jobs && rc == DP_OK; k++) {
        const uint64_t n = (ends[k] - starts[k]) < n_scalars[k] ? (ends[k] - starts[k]) : n_scalars[k];
        rc = msm_enqueue(ctx, starts[k], (const uint4 *)scalars_dev[k], n, (G1JacobianOut *)outs_dev[k], jobs[k], false, ev_batch);
    }
    int rc2 = msm_finish(ctx, jobs, false);
    if (ev_batch) cudaEventDestroy(ev_batch);
    if (rc != DP_OK) return rc;
    if (rc2 != DP_OK) return rc2;
    return call_end(ctx, true);
}

int dp_msm_batch(dp_ctx *ctx, size_t n_jobs, const uint64_t *starts, const uint64_t *ends, const void *const *scalars,
                 const size_t *n_scalars, void *const *outs) {
    if (!ctx || (n_jobs && (!starts || !ends || !scalars || !n_scalars || !outs))) return fail(ctx, DP_E_ARG, "dp_msm_batch: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_msm_batch before dp_init");
    for (size_t k = 0; k < n_jobs; k++)
        if (starts[k] > ends[k] || ends[k] > ctx->n_bases || !outs[k] || (n_scalars[k] && !scalars[k]))
            return fail(ctx, DP_E_ARG, "dp_msm_batch: job %zu has a bad range / buffer", k);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    // copy-in of job k+1 runs on s_in under the kernels of job k; tails overlap as in dp_msm_dev_batch
    std::vector<MsmJob> jobs(n_jobs);
    std::vector<uint4 *> sc(n_jobs, nullptr);
    std::vector<cudaEvent_t> ev(n_jobs, nullptr);
    G1JacobianOut *od = (G1JacobianOut *)ctx->pool.alloc((n_jobs ? n_jobs : 1) * sizeof(G1JacobianOut));
    int rc = od ? DP_OK : fail(ctx, DP_E_OOM, "dp_msm_batch outputs");
    for (size_t k = 0; k < n_jobs && rc == DP_OK; k++) {
        const uint64_t n = (ends[k] - starts[k]) < n_scalars[k] ? (ends[k] - starts[k]) : n_scalars[k];
        sc[k] = (uint4 *)ctx->pool_io.alloc((n ? n : 1) * 32);
        if (!sc[k] || cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming) != cudaSuccess) {
            rc = fail(ctx, DP_E_OOM, "dp_msm_batch staging");
            break;
        }
        cudaError_t e = n ? cudaMemcpyAsync(sc[k], scalars[k], n * 32, cudaMemcpyHostToDevice, ctx->s_in) : cudaSuccess;
        if (e == cudaSuccess) e = cudaEventRecord(ev[k], ctx->s_in);
        if (e != cudaSuccess) rc = fail(ctx, DP_E_CUDA, "dp_msm_batch H2D: %s", cudaGetErrorString(e));
    }
    // the sorts wait for their own copy-in (s_in) and for whatever the compute stream held when the batch began (earlier
    // users of recycled scratch); then they run ahead of the accumulations
    cudaEvent_t ev_batch = nullptr;
    if (rc == DP_OK && (cudaEventCreateWithFlags(&ev_batch, cudaEventDisableTiming) != cudaSuccess || cudaEventRecord(ev_batch, ctx->stream) != cudaSuccess))
        rc = fail(ctx, DP_E_CUDA, "dp_msm_batch: event");
    for (size_t k = 0; k < n_jobs && rc == DP_OK; k++) {
        const uint64_t n = (ends[k] - starts[k]) < n_scalars[k] ? (ends[k] - starts[k]) : n_scalars[k];
        cudaStreamWaitEvent(ctx->msm_sort_own_stream ? ctx->s_sort : ctx->stream, ev[k], 0);
        rc = msm_enqueue(ctx, starts[k], sc[k], n, od + k, jobs[k], false, ev_batch);
    }
    int rc2 = msm_finish(ctx, jobs, false);   // drains the sort, compute and tail streams
    if (ev_batch) cudaEventDestroy(ev_batch);
    if (rc == DP_OK) rc = rc2;
    if (rc == DP_OK) {
        std::vector<G1JacobianOut> host(n_jobs);
        cudaError_t e = n_jobs ? cudaMemcpy(host.data(), od, n_jobs * sizeof(G1JacobianOut), cudaMemcpyDeviceToHost) : cudaSuccess;
        if (e != cudaSuccess) rc = fail(ctx, DP_E_CUDA, "dp_msm_batch D2H: %s", cudaGetErrorString(e));
        for (size_t k = 0; k < n_jobs && rc == DP_OK; k++) memcpy(outs[k], &host[k], sizeof(G1JacobianOut));
    }
    cudaStreamSynchronize(ctx->s_in);
    for (size_t k = 0; k < n_jobs; k++) {
        ctx->pool_io.release(sc[k]);
        if (ev[k]) cudaEventDestroy(ev[k]);
    }
    ctx->pool.release(od);
    if (rc != DP_OK) return rc;
    return call_end(ctx, true);
}

// varMsm without blocking the caller: the Rust worker answers the RPC from a Promise (like fft2Prepare,
// worker.rs:293), so that transforms and commitments of concurrent requests share the GPU: the copy-in
// runs on s_in, the kernels queue behind whatever the compute stream holds, the 144-byte result lands in
// pinned host memory.  dp_msm_collect waits for that one job only.
int dp_msm_submit(dp_ctx *ctx, uint64_t id, uint64_t start, uint64_t end, const void *scalars, size_t n_scalars) {
    if (!ctx) return DP_E_ARG;
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_msm_submit before dp_init");
    if (start > end || end > ctx->n_bases) return fail(ctx, DP_E_ARG, "dp_msm_submit: range [%llu,%llu) outside %llu bases", (unsigned long long)start, (unsigned long long)end, (unsigned long long)ctx->n_bases);
    if (n_scalars && !scalars) return fail(ctx, DP_E_ARG, "dp_msm_submit: scalars is NULL");
    if (ctx->msm_pending.count(id)) return fail(ctx, DP_E_STATE, "dp_msm_submit: id %llu is already pending", (unsigned long long)id);
    if (ctx->msm_slots_used == ~0ull) return fail(ctx, DP_E_STATE, "dp_msm_submit: %u jobs pending, collect some first", MSM_SLOTS);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->msm_pinned) DP_CUDA(ctx, cudaMallocHost((void **)&ctx->msm_pinned, (size_t)MSM_SLOTS * MSM_SLOT_BYTES));
    const uint64_t n = (end - start) < n_scalars ? (end - start) : n_scalars;
    MsmPending *p = new MsmPending();
    while (ctx->msm_slots_used & (1ull << p->slot)) p->slot++;
    ctx->msm_slots_used |= 1ull << p->slot;
    uint8_t *pin = ctx->msm_pinned + (size_t)p->slot * MSM_SLOT_BYTES;
    memset(pin, 0, MSM_SLOT_BYTES);
    p->scalars = (uint4 *)ctx->pool_io.alloc((n ? n : 1) * 32);
    p->out = (G1JacobianOut *)ctx->pool.alloc(sizeof(G1JacobianOut));
    int rc = DP_OK;
    cudaError_t e = cudaSuccess;
    if (!p->scalars || !p->out) rc = fail(ctx, DP_E_OOM, "dp_msm_submit buffers");
    if (rc == DP_OK) e = cudaEventCreateWithFlags(&p->ev_in, cudaEventDisableTiming);
    if (rc == DP_OK && e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_done, cudaEventDisableTiming);
    if (rc == DP_OK && e == cudaSuccess && n) e = cudaMemcpyAsync(p->scalars, scalars, n * 32, cudaMemcpyHostToDevice, ctx->s_in);
    if (rc == DP_OK && e == cudaSuccess) e = cudaEventRecord(p->ev_in, ctx->s_in);
    if (rc == DP_OK && e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, p->ev_in, 0);
    if (rc == DP_OK && e == cudaSuccess) rc = msm_enqueue(ctx, start, p->scalars, n, p->out, p->job, false);
    if (rc == DP_OK && e == cudaSuccess && n == 0) {  // the identity was written on the compute stream: order the tail stream after it
        e = cudaEventCreateWithFlags(&p->job.ev_head, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventRecord(p->job.ev_head, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->s_tail, p->job.ev_head, 0);
    }
    if (rc == DP_OK && e == cudaSuccess) e = cudaMemcpyAsync(pin, p->out, sizeof(G1JacobianOut), cudaMemcpyDeviceToHost, ctx->s_tail);
    if (rc == DP_OK && e == cudaSuccess && p->job.err) e = cudaMemcpyAsync(pin + 192, p->job.err, 4, cudaMemcpyDeviceToHost, ctx->s_tail);
    if (rc == DP_OK && e == cudaSuccess) e = cudaEventRecord(p->ev_done, ctx->s_tail);
    if (rc == DP_OK && e != cudaSuccess) rc = fail(ctx, DP_E_CUDA, "dp_msm_submit: %s", cudaGetErrorString(e));
    if (rc != DP_OK) {  // nothing of this job may still be running when its buffers go back
        cudaStreamSynchronize(ctx->s_in);
        cudaStreamSynchronize(ctx->s_sort);
        cudaStreamSynchronize(ctx->stream);
        cudaStreamSynchronize(ctx->s_tail);
        release_pending(ctx, p);
        return rc;
    }
    ctx->msm_pending[id] = p;
    return DP_OK;
}

int dp_msm_collect(dp_ctx *ctx, uint64_t id, void *out) {
    if (!ctx || !out) return fail(ctx, DP_E_ARG, "dp_msm_collect: NULL argument");
    auto it = ctx->msm_pending.find(id);
    if (it == ctx->msm_pending.end()) return fail(ctx, DP_E_STATE, "dp_msm_collect: no pending job %llu", (unsigned long long)id);
    MsmPending *p = it->second;
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaError_t e = cudaEventSynchronize(p->ev_done);
    if (e == cudaSuccess) e = cudaGetLastError();
    const uint8_t *pin = ctx->msm_pinned + (size_t)p->slot * MSM_SLOT_BYTES;
    uint32_t bad = 0;
    memcpy(out, pin, sizeof(G1JacobianOut));
    memcpy(&bad, pin + 192, 4);
    if (e != cudaSuccess) {  // make sure nothing is running before the buffers go back
        cudaStreamSynchronize(ctx->s_sort);
        cudaStreamSynchronize(ctx->stream);
        cudaStreamSynchronize(ctx->s_tail);
    }
    release_pending(ctx, p);
    ctx->msm_pending.erase(it);
    if (e != cudaSuccess) return fail(ctx, DP_E_CUDA, "msm kernels: %s", cudaGetErrorString(e));
    if (bad) return fail(ctx, DP_E_ARG, "msm: a scalar is not a canonical Fr integer (>= 2^255)");
    return DP_OK;
}

static int commit_device(dp_ctx *ctx, const Fr *coeffs_dev, uint64_t n, G1JacobianOut *out_dev) {
    // into_repr + zero-pad to bases.len() (worker.rs:118-120)
    const uint64_t nb = ctx->n_bases;
    if (n > nb) return fail(ctx, DP_E_ARG, "commit: %llu coefficients > %llu bases", (unsigned long long)n, (unsigned long long)nb);
    Scratch tmp(ctx->pool);
    Fr *sc = tmp.get<Fr>(nb);
    if (!sc) return fail(ctx, DP_E_OOM, "commit scalars");
    if (nb) {
        DP_LAUNCH(fr_into_repr_kernel, dim3(blocks_for(nb, 256)), dim3(256), 0, ctx->stream, coeffs_dev, sc, n, nb);
        ctx->launches++;
    }
    return msm_device(ctx, 0, (const uint4 *)sc, nb, out_dev, nullptr);  // synchronises before sc goes back
}

int dp_commit(dp_ctx *ctx, const void *coeffs, size_t n, void *out) {
    if (!ctx || !out) return fail(ctx, DP_E_ARG, "dp_commit: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_commit before dp_init");
    if (n && !coeffs) return fail(ctx, DP_E_ARG, "dp_commit: coeffs is NULL");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    Fr *cd = tmp.get<Fr>(n);
    G1JacobianOut *od = tmp.get<G1JacobianOut>(1);
    if (!cd || !od) return fail(ctx, DP_E_OOM, "dp_commit buffers");
    if (n) DP_CUDA(ctx, cudaMemcpyAsync(cd, coeffs, n * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    DP_TRY(commit_device(ctx, cd, n, od));
    DP_CUDA(ctx, cudaMemcpyAsync(out, od, sizeof(G1JacobianOut), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

int dp_fft_init(dp_ctx *ctx, uint64_t id, const dp_fft_workload *workloads, size_t n_workloads, int is_quot, int is_inv,
                int is_coset) {
    if (!ctx || !workloads) return fail(ctx, DP_E_ARG, "dp_fft_init: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_fft_init before dp_init");
    if (n_workloads != ctx->W) return fail(ctx, DP_E_ARG, "dp_fft_init: %zu workloads for %llu workers", n_workloads, (unsigned long long)ctx->W);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    const DomainDev &d = ctx->dom[is_quot ? 1 : 0];
    const uint64_t r = d.r(), c = d.c(), W = ctx->W;
    for (uint64_t w = 0; w < W; w++) {
        const dp_fft_workload &x = workloads[w];
        if (x.row_start != w * r / W || x.row_end != (w + 1) * r / W || x.col_start != w * c / W || x.col_end != (w + 1) * c / W)
            return fail(ctx, DP_E_ARG, "dp_fft_init: workload %llu is not the equal block split of %llu x %llu", (unsigned long long)w, (unsigned long long)r, (unsigned long long)c);
    }
    if (FftTask *old_task = find_task(ctx, id)) {
        // `fft_tasks.insert(id, ..)` (worker.rs:215) replaces an open task with the same id: drop it, once
        // nothing of it is in flight any more
        cudaStreamSynchronize(ctx->s_in);
        cudaStreamSynchronize(ctx->stream);
        cudaStreamSynchronize(ctx->s_out);
        free_task(ctx, *old_task);
        ctx->tasks.erase(id);
    }
    FftTask t;
    t.is_quot = is_quot != 0;
    t.is_inv = is_inv != 0;
    t.is_coset = is_coset != 0;
    t.wl.assign(workloads, workloads + n_workloads);
    const dp_fft_workload &mine = workloads[ctx->me];
    t.n_rows = mine.row_end - mine.row_start;
    t.n_cols = mine.col_end - mine.col_start;
    t.row_start = mine.row_start;
    t.col_start = mine.col_start;
    t.rows = (Fr *)ctx->pool_io.alloc(t.n_rows * c * sizeof(Fr));
    if (!t.rows) return fail(ctx, DP_E_OOM, "dp_fft_init: rows buffer");
    if (cudaEventCreateWithFlags(&t.ev_in, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&t.ev_c, cudaEventDisableTiming) != cudaSuccess) {
        ctx->pool_io.release(t.rows);
        return fail(ctx, DP_E_CUDA, "dp_fft_init: event creation");
    }
    t.row_len.assign(t.n_rows, 0);
    ctx->tasks.emplace(id, std::move(t));
    return DP_OK;
}

int dp_fft1_rows(dp_ctx *ctx, uint64_t id, uint64_t i_first, uint64_t n_rows, const void *rows) {
    if (!ctx || !rows) return fail(ctx, DP_E_ARG, "dp_fft1: NULL argument");
    FftTask *t = find_task(ctx, id);
    if (!t) return fail(ctx, DP_E_ARG, "dp_fft1: unknown task %llu", (unsigned long long)id);
    if (t->row_phase_done) return fail(ctx, DP_E_STATE, "dp_fft1 after fft2_prepare");
    if (i_first > t->n_rows || n_rows > t->n_rows - i_first) return fail(ctx, DP_E_ARG, "dp_fft1: rows [%llu,%llu) of %llu", (unsigned long long)i_first, (unsigned long long)(i_first + n_rows), (unsigned long long)t->n_rows);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint64_t c = ctx->dom[t->is_quot ? 1 : 0].c();
    DP_CUDA(ctx, cudaMemcpyAsync(t->rows + i_first * c, rows, n_rows * c * sizeof(Fr), cudaMemcpyHostToDevice, ctx->s_in));
    DP_CUDA(ctx, cudaEventRecord(t->ev_in, ctx->s_in));
    for (uint64_t i = i_first; i < i_first + n_rows; i++) {
        if (!t->row_len[i]) t->rows_filled++;
        t->row_len[i] = (uint32_t)c;
    }
    return DP_OK;
}

// n_rows consecutive local rows of row_len <= c leading entries each (compact: n_rows * row_len Fr); the tail of
// every row is the implicit zero padding of Radix2EvaluationDomain::fft_in_place's resize (worker.rs:81-85)
int dp_fft1_rows_short(dp_ctx *ctx, uint64_t id, uint64_t i_first, uint64_t n_rows, const void *rows, size_t row_len) {
    if (!ctx || !rows) return fail(ctx, DP_E_ARG, "dp_fft1_rows_short: NULL argument");
    FftTask *t = find_task(ctx, id);
    if (!t) return fail(ctx, DP_E_ARG, "dp_fft1_rows_short: unknown task %llu", (unsigned long long)id);
    if (t->row_phase_done) return fail(ctx, DP_E_STATE, "dp_fft1 after fft2_prepare");
    if (i_first > t->n_rows || n_rows > t->n_rows - i_first) return fail(ctx, DP_E_ARG, "dp_fft1_rows_short: rows [%llu,%llu) of %llu", (unsigned long long)i_first, (unsigned long long)(i_first + n_rows), (unsigned long long)t->n_rows);
    const uint64_t c = ctx->dom[t->is_quot ? 1 : 0].c();
    if (row_len == 0 || row_len > c) return fail(ctx, DP_E_ARG, "dp_fft1_rows_short: row length %zu outside 1..%llu", row_len, (unsigned long long)c);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    DP_CUDA(ctx, cudaMemcpy2DAsync(t->rows + i_first * c, c * sizeof(Fr), rows, row_len * sizeof(Fr), row_len * sizeof(Fr), n_rows,
                                   cudaMemcpyHostToDevice, ctx->s_in));
    DP_CUDA(ctx, cudaEventRecord(t->ev_in, ctx->s_in));
    for (uint64_t i = i_first; i < i_first + n_rows; i++) {
        if (!t->row_len[i]) t->rows_filled++;
        t->row_len[i] = (uint32_t)row_len;
    }
    return DP_OK;
}

int dp_fft1(dp_ctx *ctx, uint64_t id, uint64_t i, const void *row, size_t len) {
    if (!ctx) return DP_E_ARG;
    FftTask *t = find_task(ctx, id);
    if (!t) return fail(ctx, DP_E_ARG, "dp_fft1: unknown task %llu", (unsigned long long)id);
    const uint64_t c = ctx->dom[t->is_quot ? 1 : 0].c();
    if (len >= c) return dp_fft1_rows(ctx, id, i, 1, row);  // a longer row is cut to c, as the resize does
    // a shorter row is zero-extended: c_domain.fft_in_place resizes v to the domain size (worker.rs:81-85)
    if (len && !row) return fail(ctx, DP_E_ARG, "dp_fft1: NULL argument");
    if (t->row_phase_done) return fail(ctx, DP_E_STATE, "dp_fft1 after fft2_prepare");
    if (i >= t->n_rows) return fail(ctx, DP_E_ARG, "dp_fft1: row %llu of %llu", (unsigned long long)i, (unsigned long long)t->n_rows);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    if (len == 0) {  // an empty row is a row of zeros: one explicit zero, the rest is the implicit tail
        DP_CUDA(ctx, cudaMemsetAsync(t->rows + i * c, 0, sizeof(Fr), ctx->s_in));
        len = 1;
    } else {
        DP_CUDA(ctx, cudaMemcpyAsync(t->rows + i * c, row, len * sizeof(Fr), cudaMemcpyHostToDevice, ctx->s_in));
    }
    DP_CUDA(ctx, cudaEventRecord(t->ev_in, ctx->s_in));
    if (!t->row_len[i]) t->rows_filled++;
    t->row_len[i] = (uint32_t)len;   // the zero tail is filled in (as far as the row phase reads) by run_row_phase
    return DP_OK;
}

static int exchange_begin(dp_ctx *ctx, uint64_t id, void **send_dev, void **recv_dev, uint64_t *block_elems, bool wait);

int dp_fft_exchange_begin(dp_ctx *ctx, uint64_t id, void **send_dev, void **recv_dev, uint64_t *block_elems) {
    return exchange_begin(ctx, id, send_dev, recv_dev, block_elems, true);
}

// Same, but returns without waiting for the row phase: the buffers are complete only for work that is
// enqueued on the context's compute stream (dp_compute_stream), e.g. the ncclSend / ncclRecv group of the
// exchange.  With dp_fft_exchange_end right behind it a whole multi-worker transform is asynchronous.
int dp_fft_exchange_begin_async(dp_ctx *ctx, uint64_t id, void **send_dev, void **recv_dev, uint64_t *block_elems) {
    return exchange_begin(ctx, id, send_dev, recv_dev, block_elems, false);
}

int dp_compute_stream(dp_ctx *ctx, void **stream) {
    if (!ctx || !stream) return fail(ctx, DP_E_ARG, "dp_compute_stream: NULL argument");
    *stream = (void *)ctx->stream;
    return DP_OK;
}

static int exchange_begin(dp_ctx *ctx, uint64_t id, void **send_dev, void **recv_dev, uint64_t *block_elems, bool wait) {
    if (!ctx || !send_dev || !recv_dev || !block_elems) return fail(ctx, DP_E_ARG, "dp_fft_exchange_begin: NULL argument");
    FftTask *t = find_task(ctx, id);
    if (!t) return fail(ctx, DP_E_ARG, "dp_fft_exchange_begin: unknown task %llu", (unsigned long long)id);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    DP_TRY(run_row_phase(ctx, *t));
    if (!t->recv) {
        if (ctx->W == 1) {
            t->recv = t->send;
        } else {
            const uint64_t r = ctx->dom[t->is_quot ? 1 : 0].r();
            t->recv = (Fr *)ctx->pool.alloc(r * t->n_cols * sizeof(Fr));
            if (!t->recv) return fail(ctx, DP_E_OOM, "exchange recv buffer");
        }
    }
    DP_TRY(call_end(ctx, wait));  // buffers must be complete before the caller's collective reads them (or ordered behind them)
    *send_dev = t->send;
    *recv_dev = t->recv;
    *block_elems = t->n_rows * t->n_cols;
    return DP_OK;
}

int dp_fft_exchange_end(dp_ctx *ctx, uint64_t id) {
    if (!ctx) return DP_E_ARG;
    FftTask *t = find_task(ctx, id);
    if (!t) return fail(ctx, DP_E_ARG, "dp_fft_exchange_end: unknown task %llu", (unsigned long long)id);
    if (!t->row_phase_done || !t->recv) return fail(ctx, DP_E_STATE, "dp_fft_exchange_end before dp_fft_exchange_begin");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    return queue_col_phase(ctx, *t);
}

int dp_fft2_prepare(dp_ctx *ctx, uint64_t id) {
    if (!ctx) return DP_E_ARG;
    FftTask *t = find_task(ctx, id);
    if (!t) return fail(ctx, DP_E_ARG, "dp_fft2_prepare: unknown task %llu", (unsigned long long)id);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    if (ctx->W > 1) {
        if (!p2p_ready(ctx))
            return fail(ctx, DP_E_COMM, "dp_fft2_prepare: %llu workers but no peer transport attached; use dp_fft_exchange_begin/_end around an all-to-all", (unsigned long long)ctx->W);
        // fused exchange: the row kernel stores into the owners' arenas over NVLink.  Returning only
        // after the stream drained makes "every worker answered fft2Prepare" (the dispatcher's join,
        // dispatcher2.rs:767-772) the barrier that orders these stores before any fft2.
        call_begin(ctx);
        DP_TRY(run_row_phase(ctx, *t, true));
        return call_end(ctx, true);
    }
    call_begin(ctx);
    if (single_worker_split(ctx, ctx->dom[t->is_quot ? 1 : 0]).ok) {
        DP_TRY(run_single_worker(ctx, *t));
        return call_end(ctx, false);
    }
    DP_TRY(run_row_phase(ctx, *t));
    t->recv = t->send;
    DP_TRY(queue_col_phase(ctx, *t));
    return call_end(ctx, false);
}

int dp_fft2(dp_ctx *ctx, uint64_t id, void *out, size_t out_bytes) {
    if (!ctx || !out) return fail(ctx, DP_E_ARG, "dp_fft2: NULL argument");
    FftTask *t = find_task(ctx, id);
    if (!t) return fail(ctx, DP_E_ARG, "dp_fft2: unknown task %llu", (unsigned long long)id);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    if (t->p2p && t->row_phase_done && !t->cols) DP_TRY(queue_col_phase(ctx, *t));  // peers' stores are complete by now
    if (!t->exchanged || !t->cols) return fail(ctx, DP_E_STATE, "dp_fft2 before fft2_prepare / exchange");
    const uint64_t r = ctx->dom[t->is_quot ? 1 : 0].r();
    const size_t bytes = t->n_cols * r * sizeof(Fr);
    if (out_bytes < bytes) return fail(ctx, DP_E_ARG, "dp_fft2: out buffer %zu < %zu bytes", out_bytes, bytes);
    // the column phase was queued by fft2_prepare; only the copy-out happens here, on its own stream,
    // so the next task's copy-in and compute keep running underneath
    int rc = DP_OK;
    cudaError_t e = cudaStreamWaitEvent(ctx->s_out, t->ev_c, 0);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, t->cols, bytes, cudaMemcpyDeviceToHost, ctx->s_out);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->s_out);
    if (e != cudaSuccess) rc = fail(ctx, DP_E_CUDA, "dp_fft2 D2H: %s", cudaGetErrorString(e));
    free_task(ctx, *t);  // worker.rs:378
    ctx->tasks.erase(id);
    return rc;
}

// rows handed to the dp_fft_dev* entries: how many columns the row phase has to read (0 = all)
static uint64_t dev_rd_cols(const dp_ctx *ctx, const DomainDev &d, int is_quot, int is_inv) {
    const uint64_t v = ctx->dev_valid[is_quot ? 1 : 0];
    return (v && !is_inv) ? row_read_cols(ctx, d, v) : 0;
}

int dp_fft_dev_hint_valid_cols(dp_ctx *ctx, int is_quot, uint64_t valid_cols) {
    if (!ctx) return DP_E_ARG;
    ctx->dev_valid[is_quot ? 1 : 0] = valid_cols;
    return DP_OK;
}

int dp_fft_dev(dp_ctx *ctx, const void *rows_dev, void *cols_dev, int is_quot, int is_inv, int is_coset) {
    if (!ctx || !rows_dev || !cols_dev) return fail(ctx, DP_E_ARG, "dp_fft_dev: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_fft_dev before dp_init");
    if (ctx->W != 1) return fail(ctx, DP_E_COMM, "dp_fft_dev: multi-worker exchange needs the split API");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    const DomainDev &d = ctx->dom[is_quot ? 1 : 0];
    const uint64_t N = d.n();
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    Fr *work = tmp.get<Fr>(N);
    const Split3 s3 = single_worker_split(ctx, d);
    const bool need_scratch = s3.ok || d.log_c > ctx->max_contig_log_k;
    Fr *scratch = need_scratch ? tmp.get<Fr>(N) : nullptr;
    if (!work || (need_scratch && !scratch)) return fail(ctx, DP_E_OOM, "dp_fft_dev buffers");
    if (s3.ok) {
        DP_TRY(plan_single_worker3(ctx, d, s3, (const Fr *)rows_dev, work, scratch, (Fr *)cols_dev, is_inv != 0, is_coset != 0,
                                   dev_rd_cols(ctx, d, is_quot, is_inv)));
        return call_end(ctx, true);  // synchronises before the scratch goes back to the pool
    }
    DP_TRY(plan_row_phase(ctx, d, (const Fr *)rows_dev, work, scratch, d.r(), 0, is_inv != 0, is_coset != 0, 1, nullptr,
                          dev_rd_cols(ctx, d, is_quot, is_inv)));
    DP_TRY(plan_col_phase(ctx, d, work, (Fr *)cols_dev, d.c(), 0, is_inv != 0, is_coset != 0));
    return call_end(ctx, true);  // synchronises before the scratch goes back to the pool
}

int dp_fft_dev_rows(dp_ctx *ctx, const void *rows_dev, int is_quot, int is_inv, int is_coset, void **send_dev,
                    void **recv_dev, uint64_t *block_elems) {
    if (!ctx || !rows_dev || !send_dev || !recv_dev || !block_elems) return fail(ctx, DP_E_ARG, "dp_fft_dev_rows: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_fft_dev_rows before dp_init");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    const DomainDev &d = ctx->dom[is_quot ? 1 : 0];
    const uint64_t W = ctx->W, n_rows = d.r() / W, n_cols = d.c() / W, c = d.c();
    call_begin(ctx);
    ctx->pool.release(ctx->dev_send);
    ctx->pool.release(ctx->dev_recv);
    ctx->dev_send = (Fr *)ctx->pool.alloc(n_rows * c * sizeof(Fr));
    ctx->dev_recv = W > 1 ? (Fr *)ctx->pool.alloc(d.r() * n_cols * sizeof(Fr)) : nullptr;
    const bool need_scratch = d.log_c > ctx->max_contig_log_k;
    Scratch tmp(ctx->pool);
    Fr *scratch = need_scratch ? tmp.get<Fr>(n_rows * c) : nullptr;
    if (!ctx->dev_send || (W > 1 && !ctx->dev_recv) || (need_scratch && !scratch)) return fail(ctx, DP_E_OOM, "dp_fft_dev_rows buffers");
    DP_TRY(plan_row_phase(ctx, d, (const Fr *)rows_dev, ctx->dev_send, scratch, n_rows, ctx->me * n_rows, is_inv != 0, is_coset != 0, W, nullptr,
                          dev_rd_cols(ctx, d, is_quot, is_inv)));
    DP_TRY(call_end(ctx, true));
    ctx->dev_flags = (is_quot ? 4 : 0) | (is_inv ? 2 : 0) | (is_coset ? 1 : 0);
    *send_dev = ctx->dev_send;
    *recv_dev = W > 1 ? ctx->dev_recv : ctx->dev_send;
    *block_elems = n_rows * n_cols;
    return DP_OK;
}

int dp_fft_dev_cols(dp_ctx *ctx, void *cols_dev) {
    if (!ctx || !cols_dev) return fail(ctx, DP_E_ARG, "dp_fft_dev_cols: NULL argument");
    if (ctx->dev_flags < 0) return fail(ctx, DP_E_STATE, "dp_fft_dev_cols before dp_fft_dev_rows");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    const int f = ctx->dev_flags;
    const DomainDev &d = ctx->dom[(f & 4) ? 1 : 0];
    const uint64_t n_cols = d.c() / ctx->W;
    call_begin(ctx);
    Fr *p2p_slot = ctx->dev_p2p_slot;
    Fr *src = p2p_slot ? p2p_slot : (ctx->W > 1 ? ctx->dev_recv : ctx->dev_send);
    ctx->dev_p2p_slot = nullptr;
    ctx->dev_flags = -1;
    int rc = plan_col_phase(ctx, d, src, (Fr *)cols_dev, n_cols, ctx->me * n_cols, (f & 2) != 0, (f & 1) != 0);
    if (rc == DP_OK) rc = call_end(ctx, true);
    p2p_release_slot(ctx, p2p_slot);  // read (or given up): peers may store the next exchange into it
    return rc;
}

static int ntt_device(dp_ctx *ctx, Fr *x, uint32_t log_n, bool is_inv, bool is_coset, uint64_t n_valid = 0) {
    // twiddles: reuse a resident domain table when it is at least as large, else build one.
    // Everything is queued on the compute stream, so handing the scratch back at scope exit is
    // stream-ordered with respect to every later user of the pool.
    const DomainDev *d = nullptr;
    for (int k = 0; k < 2; k++)
        if (ctx->dom[k].H && ctx->dom[k].log_n >= log_n && (!d || ctx->dom[k].log_n < d->log_n)) d = &ctx->dom[k];
    const uint64_t N = (uint64_t)1 << log_n;
    Scratch tmp(ctx->pool);
    const Fr *H = d ? d->H : nullptr;
    uint32_t H_log = d ? d->log_n : log_n;
    const bool multi = log_n > ctx->max_contig_log_k;
    if (!H && multi) {
        Fr *tmpH = tmp.get<Fr>(N / 2);
        if (!tmpH) return fail(ctx, DP_E_OOM, "dp_ntt twiddles");
        DP_TRY(gen_powers(ctx, tmpH, N / 2, fr_domain_gen(log_n), 0, 1, Fr::one()));
        H = tmpH;
    }
    Fr *scratch = multi ? tmp.get<Fr>(N) : nullptr;
    if (multi && !scratch) return fail(ctx, DP_E_OOM, "dp_ntt scratch");
    return plan_whole_ntt(ctx, d, x, scratch, log_n, is_inv, is_coset, H, H_log, is_inv ? 0 : n_valid);
}

int dp_ntt_dev(dp_ctx *ctx, void *data_dev, uint32_t log_n, int is_inv, int is_coset) {
    if (!ctx || !data_dev) return fail(ctx, DP_E_ARG, "dp_ntt_dev: NULL argument");
    if (log_n > 32) return fail(ctx, DP_E_ARG, "dp_ntt_dev: log_n %u", log_n);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    DP_TRY(ntt_device(ctx, (Fr *)data_dev, log_n, is_inv != 0, is_coset != 0));
    return call_end(ctx, true);
}

// in place on a device buffer of 2^log_n Fr whose entries from n_valid on are zero (a resident coefficient vector
// shorter than the domain, e.g. n coefficients evaluated on the 8n-point coset): the forward transform neither reads
// nor multiplies the zero tail.  Asynchronous variant of dp_ntt_dev when `wait` is 0 (dp_sync waits).
int dp_ntt_dev_padded(dp_ctx *ctx, void *data_dev, size_t n_valid, uint32_t log_n, int is_inv, int is_coset, int wait) {
    if (!ctx || !data_dev) return fail(ctx, DP_E_ARG, "dp_ntt_dev_padded: NULL argument");
    if (log_n > 32 || n_valid > ((uint64_t)1 << log_n)) return fail(ctx, DP_E_ARG, "dp_ntt_dev_padded: %zu valid entries, log_n %u", n_valid, log_n);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    DP_TRY(ntt_device(ctx, (Fr *)data_dev, log_n, is_inv != 0, is_coset != 0, n_valid));
    return call_end(ctx, wait != 0);
}

// Slice k of the coset evaluation on the quotient domain: out[i] = p(s_k * omega_n^i), i < n, an n-point transform of the
// gate domain with the coset shift s_k (slice_shift), out of place.  coeffs[0, n_valid) is read, never written.
static int slice_ntt_device(dp_ctx *ctx, const Fr *coeffs, uint64_t n_valid, uint32_t k, Fr *out) {
    const DomainDev &dg = ctx->dom[0];
    const uint32_t L = dg.log_n;
    const uint64_t N = dg.n();
    const bool multi = L > ctx->max_contig_log_k;
    Scratch tmp(ctx->pool);
    Fr *scratch = multi ? tmp.get<Fr>(N) : nullptr;
    if (multi && !scratch) return fail(ctx, DP_E_OOM, "dp_ntt_dev_quot_slice scratch");
    // Fused: the first pass reads coeffs and multiplies by slice k's factor tables as it loads.  Its zero-input cut reads
    // the leading 2^v points of each of its 2^(L - l1) lanes, which is exactly coeffs[0, n_valid) when n_valid is a power
    // of two of at least that many lanes (the prover's n coefficients, and n/8 from 2^(3 + L - l1) on).
    const uint64_t lanes = N >> dg.w_l1;
    const bool exact_cut = n_valid && (n_valid & (n_valid - 1)) == 0 && n_valid >= lanes;
    if (dg.ws_a && whole_tables_fit(ctx, &dg, L) && exact_cut) {
        const CosetTables t{dg.ws_a + k * lanes, dg.ws_b + ((uint64_t)k << dg.w_l1)};
        return plan_whole_ntt(ctx, &dg, out, scratch, L, false, true, dg.H, L, n_valid, coeffs, &t);
    }
    // otherwise (single-pass domains, a split the tables were not built for, other lengths): scale-and-copy into out,
    // then the plain transform in place
    DP_LAUNCH(fr_scale_powers_copy_kernel, dim3(blocks_for(N, 256)), dim3(256), 0, ctx->stream, coeffs, out, n_valid, N,
              slice_shift(ctx->dom[1], k));
    ctx->launches++;
    DP_CUDA(ctx, cudaGetLastError());
    return plan_whole_ntt(ctx, &dg, out, scratch, L, false, false, dg.H, L, n_valid);
}

static bool ranges_overlap(const void *a, uint64_t a_bytes, const void *b, uint64_t b_bytes) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + b_bytes && y < x + a_bytes;
}

int dp_ntt_dev_quot_slice(dp_ctx *ctx, const void *coeffs_dev, size_t n_valid, uint32_t slice, void *out_dev, int wait) {
    if (!ctx || !coeffs_dev || !out_dev) return fail(ctx, DP_E_ARG, "dp_ntt_dev_quot_slice: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_ntt_dev_quot_slice before dp_init");
    const DomainDev &dg = ctx->dom[0], &dq = ctx->dom[1];
    const uint64_t n = dg.n();
    if (dq.log_n < dg.log_n || slice >= (dq.n() >> dg.log_n))
        return fail(ctx, DP_E_ARG, "dp_ntt_dev_quot_slice: slice %u of %llu", slice, (unsigned long long)(dq.log_n < dg.log_n ? 0 : dq.n() >> dg.log_n));
    if (n_valid > n) return fail(ctx, DP_E_ARG, "dp_ntt_dev_quot_slice: %zu coefficients > n = %llu", n_valid, (unsigned long long)n);
    if (ranges_overlap(coeffs_dev, n_valid * sizeof(Fr), out_dev, n * sizeof(Fr)))
        return fail(ctx, DP_E_ARG, "dp_ntt_dev_quot_slice: the output overlaps the coefficients");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    DP_TRY(slice_ntt_device(ctx, (const Fr *)coeffs_dev, n_valid, slice, (Fr *)out_dev));
    return call_end(ctx, wait != 0);
}

int dp_ntt(dp_ctx *ctx, void *data, size_t n, uint32_t log_n, int is_inv, int is_coset) {
    if (!ctx || !data) return fail(ctx, DP_E_ARG, "dp_ntt: NULL argument");
    if (log_n > 32) return fail(ctx, DP_E_ARG, "dp_ntt: log_n %u", log_n);
    const uint64_t N = (uint64_t)1 << log_n;
    if (n > N) return fail(ctx, DP_E_ARG, "dp_ntt: %zu elements > domain 2^%u", n, log_n);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    Fr *x = tmp.get<Fr>(N);
    if (!x) return fail(ctx, DP_E_OOM, "dp_ntt buffer");
    DP_CUDA(ctx, cudaMemcpyAsync(x, data, n * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    if (n < N) DP_CUDA(ctx, cudaMemsetAsync(x + n, 0, (N - n) * sizeof(Fr), ctx->stream));
    DP_TRY(ntt_device(ctx, x, log_n, is_inv != 0, is_coset != 0, n));
    DP_CUDA(ctx, cudaMemcpyAsync(data, x, N * sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

// coeffs += b(X) * (X^n - 1), b = b_0 + b_1 X + ... + b_(k-1) X^(k-1), k <= RND_MAX_TAIL: for each j in turn, b_j comes
// off coefficient j and onto coefficient n + j.  For n < k the two ranges meet, and the order gives the right sum: n == 1,
// k == 2 leaves c_1 + b_0 - b_1 at index 1 (worker.rs:400-401 blinds a wire with k = 2)
struct BlindScalars {
    Fr b[RND_MAX_TAIL];
};
__global__ void poly_blind_kernel(Fr *coeffs, uint64_t n, uint32_t k, BlindScalars s) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    for (uint32_t j = 0; j < k; j++) {
        coeffs[j] = coeffs[j] - s.b[j];
        coeffs[n + j] = coeffs[n + j] + s.b[j];
    }
}

// k secret scalars, uniform over [0, r).  The reference blinds with ThreadRng, a CSPRNG (worker.rs:400, dispatcher2.rs:
// 294-361): the scalars must be unpredictable, so they come from the kernel's entropy pool, as canonical residues < r by
// rejection (r is 255 bits: one try in ~2.2 is rejected).  Any residue < r is a valid Montgomery-form element.
static int draw_secret_fr(dp_ctx *ctx, Fr *out, uint32_t k, const char *who) {
    for (uint32_t j = 0; j < k; j++) {
        Fr v;
        do {
            size_t got = 0;
            while (got < sizeof(Fr)) {
                const ssize_t r = getrandom(reinterpret_cast<uint8_t *>(v.l) + got, sizeof(Fr) - got, 0);
                if (r < 0) return fail(ctx, DP_E_STATE, "%s: getrandom failed; pass the blinders in `blind`", who);
                got += (size_t)r;
            }
            v.l[7] &= 0x7fffffffu;
        } while (!v.canon_is_reduced());
        out[j] = v;
    }
    return DP_OK;
}

int dp_round1(dp_ctx *ctx, const void *evals, size_t n, const void *blind, void *out) {
    if (!ctx || !evals || !out) return fail(ctx, DP_E_ARG, "dp_round1: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_round1 before dp_init");
    const DomainDev &d = ctx->dom[0];
    const uint64_t N = d.n();
    if (n > N) return fail(ctx, DP_E_ARG, "dp_round1: %zu evaluations > domain %llu", n, (unsigned long long)N);
    if (N + 2 > ctx->n_bases) return fail(ctx, DP_E_ARG, "dp_round1: %llu bases cannot commit a degree-%llu polynomial", (unsigned long long)ctx->n_bases, (unsigned long long)(N + 1));
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    ctx->pool.release(ctx->wire);
    ctx->wire = (Fr *)ctx->pool.alloc((N + 2) * sizeof(Fr));
    Scratch tmp(ctx->pool);
    G1JacobianOut *od = tmp.get<G1JacobianOut>(1);
    if (!ctx->wire || !od) return fail(ctx, DP_E_OOM, "dp_round1 buffers");
    ctx->wire_len = N + 2;
    DP_CUDA(ctx, cudaMemcpyAsync(ctx->wire, evals, n * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    DP_CUDA(ctx, cudaMemsetAsync(ctx->wire + n, 0, (N + 2 - n) * sizeof(Fr), ctx->stream));
    DP_TRY(ntt_device(ctx, ctx->wire, d.log_n, true, false));
    BlindScalars b;
    memset((void *)&b, 0, sizeof b);
    if (blind) memcpy(b.b, blind, 2 * sizeof(Fr));
    else DP_TRY(draw_secret_fr(ctx, b.b, 2, "dp_round1"));
    DP_LAUNCH(poly_blind_kernel, dim3(1), dim3(32), 0, ctx->stream, ctx->wire, N, 2u, b);
    ctx->launches++;
    DP_TRY(commit_device(ctx, ctx->wire, N + 2, od));
    DP_CUDA(ctx, cudaMemcpyAsync(out, od, sizeof(G1JacobianOut), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

int dp_poly_blind_dev(dp_ctx *ctx, void *coeffs_dev, size_t n, uint32_t k, const void *blind) {
    if (!ctx || !coeffs_dev) return fail(ctx, DP_E_ARG, "dp_poly_blind_dev: NULL argument");
    if (k > RND_MAX_TAIL) return fail(ctx, DP_E_ARG, "dp_poly_blind_dev: %u blinding scalars, at most %u", k, RND_MAX_TAIL);
    BlindScalars b;
    memset((void *)&b, 0, sizeof b);
    if (blind) {
        memcpy(b.b, blind, k * sizeof(Fr));
        for (uint32_t j = 0; j < k; j++)
            if (!b.b[j].canon_is_reduced()) return fail(ctx, DP_E_ARG, "dp_poly_blind_dev: blinding scalar %u is not below r", j);
    } else {
        DP_TRY(draw_secret_fr(ctx, b.b, k, "dp_poly_blind_dev"));
    }
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    DP_LAUNCH(poly_blind_kernel, dim3(1), dim3(32), 0, ctx->stream, (Fr *)coeffs_dev, (uint64_t)n, k, b);
    ctx->launches++;
    DP_CUDA(ctx, cudaGetLastError());
    const int rc = call_end(ctx, true);
    explicit_bzero((void *)&b, sizeof b);   // drawn scalars never leave the library; the launch copied its parameters
    return rc;
}

// multiplicative scan of n Fr on the compute stream: out[i] = product of the logical elements before
// (exclusive) or up to (inclusive) i, logical order reversed when `reverse`; *total_dev = whole product
static int perm_scan(dp_ctx *ctx, const Fr *x, uint64_t n, bool reverse, bool inclusive, Fr *out, Fr *total_dev) {
    const uint32_t n_blocks = (uint32_t)((n + PERM_BLOCK - 1) / PERM_BLOCK);
    Scratch tmp(ctx->pool);  // stream-ordered: only the compute stream touches it
    Fr *block_tot = tmp.get<Fr>(n_blocks);
    if (!block_tot) return fail(ctx, DP_E_OOM, "perm scan scratch");
    DP_LAUNCH(perm_block_products_kernel, dim3(n_blocks), dim3(PERM_TPB), 0, ctx->stream, x, n, reverse ? 1u : 0u, block_tot);
    DP_LAUNCH(perm_block_offsets_kernel, dim3(1), dim3(PERM_TPB), 0, ctx->stream, block_tot, n_blocks, total_dev);
    DP_LAUNCH(perm_scan_write_kernel, dim3(n_blocks), dim3(PERM_TPB), 0, ctx->stream, x, n, reverse ? 1u : 0u, inclusive ? 1u : 0u,
              (const Fr *)block_tot, out);
    ctx->launches += 3;
    DP_CUDA(ctx, cudaGetLastError());
    return DP_OK;
}

static int perm_product_device(dp_ctx *ctx, const Fr *wires, const Fr *id, const Fr *sigma, uint32_t n_types, uint64_t n,
                               const Fr &beta, const Fr &gamma, Fr *z_dev) {
    Scratch tmp(ctx->pool);
    Fr *a = tmp.get<Fr>(n), *b = tmp.get<Fr>(n), *tot = tmp.get<Fr>(2);
    if (!a || !b || !tot) return fail(ctx, DP_E_OOM, "dp_perm_product scratch");
    DP_LAUNCH(perm_terms_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, ctx->stream, wires, id, sigma, n_types, n, beta, gamma, a, b);
    ctx->launches++;
    DP_TRY(perm_scan(ctx, a, n, false, false, a, tot));        // a <- exclusive prefix products (in place)
    DP_TRY(perm_scan(ctx, b, n, true, true, b, tot + 1));      // b <- inclusive suffix products; tot[1] = T
    DP_LAUNCH(perm_invert_kernel, dim3(1), dim3(32), 0, ctx->stream, tot + 1);
    DP_LAUNCH(perm_finish_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, ctx->stream, (const Fr *)a, (const Fr *)b,
              (const Fr *)(tot + 1), n, z_dev);
    ctx->launches += 2;
    Fr t_inv;
    DP_CUDA(ctx, cudaMemcpyAsync(&t_inv, tot + 1, sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    DP_CUDA(ctx, cudaGetLastError());
    if (t_inv.is_zero()) return fail(ctx, DP_E_ARG, "dp_perm_product: a denominator is zero (the reference's division panics)");
    return DP_OK;
}

int dp_perm_product(dp_ctx *ctx, const void *wires, const void *id_perm, const void *sigma_perm, size_t num_wire_types, size_t n,
                    const void *beta, const void *gamma, void *out) {
    if (!ctx || !wires || !id_perm || !sigma_perm || !beta || !gamma || !out) return fail(ctx, DP_E_ARG, "dp_perm_product: NULL argument");
    if (n == 0 || num_wire_types == 0 || num_wire_types > 16) return fail(ctx, DP_E_ARG, "dp_perm_product: n = %zu, %zu wire types", n, num_wire_types);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    const size_t count = num_wire_types * n, bytes = count * sizeof(Fr);
    Scratch tmp(ctx->pool);
    Fr *w = tmp.get<Fr>(count), *i = tmp.get<Fr>(count), *s = tmp.get<Fr>(count), *z = tmp.get<Fr>(n);
    if (!w || !i || !s || !z) return fail(ctx, DP_E_OOM, "dp_perm_product buffers");
    DP_CUDA(ctx, cudaMemcpyAsync(w, wires, bytes, cudaMemcpyHostToDevice, ctx->stream));
    DP_CUDA(ctx, cudaMemcpyAsync(i, id_perm, bytes, cudaMemcpyHostToDevice, ctx->stream));
    DP_CUDA(ctx, cudaMemcpyAsync(s, sigma_perm, bytes, cudaMemcpyHostToDevice, ctx->stream));
    Fr be, ga;
    memcpy(&be, beta, sizeof be);
    memcpy(&ga, gamma, sizeof ga);
    DP_TRY(perm_product_device(ctx, w, i, s, (uint32_t)num_wire_types, n, be, ga, z));
    DP_CUDA(ctx, cudaMemcpyAsync(out, z, n * sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

int dp_perm_product_dev(dp_ctx *ctx, const void *wires_dev, const void *id_dev, const void *sigma_dev, size_t num_wire_types, size_t n,
                        const void *beta, const void *gamma, void *out_dev) {
    if (!ctx || !wires_dev || !id_dev || !sigma_dev || !beta || !gamma || !out_dev) return fail(ctx, DP_E_ARG, "dp_perm_product_dev: NULL argument");
    if (n == 0 || num_wire_types == 0 || num_wire_types > 16) return fail(ctx, DP_E_ARG, "dp_perm_product_dev: n = %zu, %zu wire types", n, num_wire_types);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Fr be, ga;
    memcpy(&be, beta, sizeof be);
    memcpy(&ga, gamma, sizeof ga);
    DP_TRY(perm_product_device(ctx, (const Fr *)wires_dev, (const Fr *)id_dev, (const Fr *)sigma_dev, (uint32_t)num_wire_types, n, be, ga, (Fr *)out_dev));
    return call_end(ctx, true);
}

// ------------------------------------------------------------------ circuit preprocessing and witness gather (circuit.cuh)
// Sort scratch of dp_wire_permutation_dev, offsets in bytes: key / value buffers (one pair for a single radix pass, two to
// ping-pong between), the digit histograms of every block, their scan's block sums, the id-check flag.
struct WirePermLayout {
    uint32_t passes = 0, n_blocks = 0, hist_n = 0, scan_blocks = 0;
    uint64_t keys[2] = {0, 0}, vals[2] = {0, 0}, hist = 0, bsum = 0, flag = 0, total = 0;
};

static WirePermLayout wire_perm_layout(uint64_t count, uint64_t num_vars) {
    WirePermLayout L;
    uint64_t top = num_vars - 1;                       // largest id; ids are u32
    if (top > 0xffffffffull) top = 0xffffffffull;
    uint32_t bits = 0;
    while (bits < 64 && (top >> bits)) bits++;
    L.passes = (bits + CIRC_RADIX_BITS - 1) / CIRC_RADIX_BITS;
    L.n_blocks = (uint32_t)((count + CIRC_TILE - 1) / CIRC_TILE);
    L.hist_n = CIRC_RADIX * L.n_blocks;
    L.scan_blocks = (L.hist_n + SCAN_BLOCK - 1) / SCAN_BLOCK;
    uint64_t off = 0;
    auto take = [&](uint64_t bytes) {
        const uint64_t at = off;
        off += (bytes + 255) & ~(uint64_t)255;
        return at;
    };
    const uint32_t pairs = L.passes < 2 ? L.passes : 2;
    for (uint32_t p = 0; p < pairs; p++) {
        L.keys[p] = take(count * sizeof(uint32_t));
        L.vals[p] = take(count * sizeof(uint32_t));
    }
    if (L.passes) {
        L.hist = take((uint64_t)L.hist_n * sizeof(uint32_t));
        L.bsum = take((uint64_t)L.scan_blocks * sizeof(uint32_t));
    }
    L.flag = take(sizeof(uint32_t));
    L.total = off;
    return L;
}

// *ok = every ids[i] < bound; flag_dev: one u32 of device scratch.  Waits for the answer.
static int ids_below(dp_ctx *ctx, const uint32_t *ids, uint64_t count, uint64_t bound, uint32_t *flag_dev, bool *ok) {
    DP_CUDA(ctx, cudaMemsetAsync(flag_dev, 0, sizeof(uint32_t), ctx->stream));
    uint64_t grid = blocks_for(count, 256);
    if (grid > (uint64_t)ctx->n_sms * 8) grid = (uint64_t)ctx->n_sms * 8;
    DP_LAUNCH(circ_check_ids_kernel, dim3((unsigned)(grid ? grid : 1)), dim3(256), 0, ctx->stream, ids, count, bound, flag_dev);
    ctx->launches++;
    uint32_t flag = 0;
    DP_CUDA(ctx, cudaMemcpyAsync(&flag, flag_dev, sizeof flag, cudaMemcpyDeviceToHost, ctx->stream));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    DP_CUDA(ctx, cudaGetLastError());
    *ok = flag == 0;
    return DP_OK;
}

// the arguments every circuit entry shares: after dp_init, 1..5 wire types over the gate domain, slots indexable by u32
static int circuit_args(dp_ctx *ctx, size_t num_wire_types, size_t n, const char *who) {
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "%s before dp_init", who);
    if (num_wire_types < 1 || num_wire_types > 5) return fail(ctx, DP_E_ARG, "%s: %zu wire types (1..5)", who, num_wire_types);
    if (n != ctx->dom[0].n()) return fail(ctx, DP_E_ARG, "%s: n = %zu is not the gate domain (%llu)", who, n, (unsigned long long)ctx->dom[0].n());
    if ((uint64_t)num_wire_types * n > 0xffffffffull) return fail(ctx, DP_E_ARG, "%s: %zu slots do not fit 32-bit slot ids", who, num_wire_types * n);
    return DP_OK;
}

int dp_wire_permutation_scratch_bytes(size_t num_wire_types, size_t n, uint64_t num_vars, size_t *bytes) {
    if (!bytes || num_wire_types < 1 || num_wire_types > 5 || n == 0 || num_vars == 0 || (uint64_t)num_wire_types * n > 0xffffffffull)
        return fail(nullptr, DP_E_ARG, "dp_wire_permutation_scratch_bytes: %zu wire types, n = %zu, %llu variables", num_wire_types, n,
                    (unsigned long long)num_vars);
    *bytes = wire_perm_layout((uint64_t)num_wire_types * n, num_vars).total;
    return DP_OK;
}

int dp_wire_permutation_dev(dp_ctx *ctx, const uint32_t *vars_dev, size_t num_wire_types, size_t n, uint64_t num_vars, void *scratch_dev,
                            size_t scratch_bytes, uint32_t *succ_out_dev) {
    const char *who = "dp_wire_permutation_dev";
    if (!ctx) return fail(ctx, DP_E_ARG, "%s: NULL context", who);
    DP_TRY(circuit_args(ctx, num_wire_types, n, who));
    if (!vars_dev || !scratch_dev || !succ_out_dev) return fail(ctx, DP_E_ARG, "%s: NULL argument", who);
    if (num_vars == 0) return fail(ctx, DP_E_ARG, "%s: num_vars = 0", who);
    const uint64_t count = (uint64_t)num_wire_types * n;
    const WirePermLayout L = wire_perm_layout(count, num_vars);
    if (scratch_bytes < L.total) return fail(ctx, DP_E_ARG, "%s: %zu scratch bytes, %llu needed", who, scratch_bytes, (unsigned long long)L.total);
    if (ranges_overlap(vars_dev, count * 4, succ_out_dev, count * 4) || ranges_overlap(vars_dev, count * 4, scratch_dev, L.total) ||
        ranges_overlap(succ_out_dev, count * 4, scratch_dev, L.total))
        return fail(ctx, DP_E_ARG, "%s: the variable map, the scratch and the output overlap", who);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    uint8_t *S = (uint8_t *)scratch_dev;
    bool ok = false;
    DP_TRY(ids_below(ctx, vars_dev, count, num_vars, (uint32_t *)(S + L.flag), &ok));
    if (!ok) return fail(ctx, DP_E_ARG, "%s: a variable id is >= num_vars = %llu", who, (unsigned long long)num_vars);
    const uint32_t *keys = vars_dev, *vals = nullptr;
    uint32_t *hist = (uint32_t *)(S + L.hist), *bsum = (uint32_t *)(S + L.bsum);
    for (uint32_t p = 0; p < L.passes; p++) {
        uint32_t *ko = (uint32_t *)(S + L.keys[p & 1]), *vo = (uint32_t *)(S + L.vals[p & 1]);
        const uint32_t shift = p * CIRC_RADIX_BITS;
        DP_LAUNCH(circ_radix_hist_kernel, dim3(L.n_blocks), dim3(CIRC_TPB), 0, ctx->stream, keys, count, shift, L.n_blocks, hist);
        DP_LAUNCH(scan_block_sums_kernel, dim3(L.scan_blocks), dim3(SCAN_TPB), 0, ctx->stream, (const uint32_t *)hist, L.hist_n, bsum);
        DP_LAUNCH(circ_scan_offsets_kernel, dim3(1), dim3(CIRC_TPB), 0, ctx->stream, bsum, L.scan_blocks);
        DP_LAUNCH(circ_scan_write_kernel, dim3(L.scan_blocks), dim3(SCAN_TPB), 0, ctx->stream, hist, L.hist_n, (const uint32_t *)bsum);
        DP_LAUNCH(circ_radix_scatter_kernel, dim3(L.n_blocks), dim3(CIRC_TPB), 0, ctx->stream, keys, vals, count, shift,
                  (const uint32_t *)hist, L.n_blocks, ko, vo);
        ctx->launches += 5;
        DP_CUDA(ctx, cudaGetLastError());
        keys = ko;
        vals = vo;
    }
    DP_LAUNCH(circ_successor_kernel, dim3(blocks_for(count, 256)), dim3(256), 0, ctx->stream, keys, vals, count, succ_out_dev);
    ctx->launches++;
    DP_CUDA(ctx, cudaGetLastError());
    return call_end(ctx, true);
}

int dp_perm_evals_dev(dp_ctx *ctx, const uint32_t *succ_dev, size_t num_wire_types, size_t n, const void *k, void *id_out_dev,
                      void *sigma_out_dev) {
    const char *who = "dp_perm_evals_dev";
    if (!ctx) return fail(ctx, DP_E_ARG, "%s: NULL context", who);
    DP_TRY(circuit_args(ctx, num_wire_types, n, who));
    if (!k || !id_out_dev || !sigma_out_dev) return fail(ctx, DP_E_ARG, "%s: NULL argument", who);
    const uint64_t count = (uint64_t)num_wire_types * n;
    if (ranges_overlap(id_out_dev, count * 32, sigma_out_dev, count * 32) ||
        (succ_dev && (ranges_overlap(succ_dev, count * 4, id_out_dev, count * 32) || ranges_overlap(succ_dev, count * 4, sigma_out_dev, count * 32))))
        return fail(ctx, DP_E_ARG, "%s: the successor map and the outputs overlap", who);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    if (succ_dev) {
        Scratch tmp(ctx->pool);
        uint32_t *flag = tmp.get<uint32_t>(1);
        if (!flag) return fail(ctx, DP_E_OOM, "%s flag", who);
        bool ok = false;
        DP_TRY(ids_below(ctx, succ_dev, count, count, flag, &ok));
        if (!ok) return fail(ctx, DP_E_ARG, "%s: a successor slot is >= num_wire_types * n = %llu", who, (unsigned long long)count);
    }
    CircK kk;
    memset((void *)&kk, 0, sizeof kk);
    memcpy(kk.k, k, num_wire_types * sizeof(Fr));
    DP_LAUNCH(circ_perm_evals_kernel, dim3(blocks_for(count, 256)), dim3(256), 0, ctx->stream, succ_dev, count, ctx->dom[0].log_n,
              (const Fr *)ctx->dom[0].H, kk, (Fr *)id_out_dev, (Fr *)sigma_out_dev);
    ctx->launches++;
    DP_CUDA(ctx, cudaGetLastError());
    return call_end(ctx, true);
}

int dp_witness_gather_dev(dp_ctx *ctx, const void *witness_dev, uint64_t num_vars, const uint32_t *vars_dev, size_t num_wire_types, size_t n,
                          size_t num_inputs, void *wires_out_dev, void *pub_out_dev) {
    const char *who = "dp_witness_gather_dev";
    if (!ctx) return fail(ctx, DP_E_ARG, "%s: NULL context", who);
    DP_TRY(circuit_args(ctx, num_wire_types, n, who));
    if (!witness_dev || !vars_dev || !wires_out_dev || !pub_out_dev) return fail(ctx, DP_E_ARG, "%s: NULL argument", who);
    if (num_vars == 0) return fail(ctx, DP_E_ARG, "%s: num_vars = 0", who);
    if (num_inputs > n) return fail(ctx, DP_E_ARG, "%s: %zu public inputs > n = %zu", who, num_inputs, n);
    const uint64_t count = (uint64_t)num_wire_types * n;
    const uint64_t wit_bytes = (num_vars < ((uint64_t)1 << 32) ? num_vars : ((uint64_t)1 << 32)) * 32;   // ids are u32
    if (ranges_overlap(wires_out_dev, count * 32, witness_dev, wit_bytes) || ranges_overlap(wires_out_dev, count * 32, vars_dev, count * 4) ||
        ranges_overlap(wires_out_dev, count * 32, pub_out_dev, n * 32) || ranges_overlap(pub_out_dev, n * 32, witness_dev, wit_bytes) ||
        ranges_overlap(pub_out_dev, n * 32, vars_dev, count * 4))
        return fail(ctx, DP_E_ARG, "%s: an output overlaps an input or the other output", who);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    uint32_t *flag = tmp.get<uint32_t>(1);
    if (!flag) return fail(ctx, DP_E_OOM, "%s flag", who);
    bool ok = false;
    DP_TRY(ids_below(ctx, vars_dev, count, num_vars, flag, &ok));
    if (!ok) return fail(ctx, DP_E_ARG, "%s: a variable id is >= num_vars = %llu", who, (unsigned long long)num_vars);
    DP_LAUNCH(circ_gather_kernel, dim3(blocks_for(count, 256)), dim3(256), 0, ctx->stream, (const Fr *)witness_dev, vars_dev, count, (uint64_t)n,
              (uint64_t)(num_wire_types - 1) * n, (uint64_t)num_inputs, (Fr *)wires_out_dev, (Fr *)pub_out_dev);
    ctx->launches++;
    DP_CUDA(ctx, cudaGetLastError());
    return call_end(ctx, true);
}

int dp_commit_dev_batch(dp_ctx *ctx, size_t n_jobs, void *const *coeffs_dev, const size_t *lens, void *outs144) {
    const char *who = "dp_commit_dev_batch";
    if (!ctx || (n_jobs && (!coeffs_dev || !lens || !outs144))) return fail(ctx, DP_E_ARG, "%s: NULL argument", who);
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "%s before dp_init", who);
    for (size_t j = 0; j < n_jobs; j++) {
        if (lens[j] && !coeffs_dev[j]) return fail(ctx, DP_E_ARG, "%s: polynomial %zu is NULL", who, j);
        if (lens[j] > ctx->n_bases) return fail(ctx, DP_E_ARG, "%s: polynomial %zu has %zu coefficients > %llu bases", who, j, lens[j],
                                                (unsigned long long)ctx->n_bases);
    }
    if (n_jobs == 0) return DP_OK;
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    G1JacobianOut *od = tmp.get<G1JacobianOut>(n_jobs);
    if (!od) return fail(ctx, DP_E_OOM, "%s outputs", who);
    // into_repr in place (the MSM takes canonical scalars), one MSM batch, back to Montgomery form: no n-sized scratch per job
    for (size_t j = 0; j < n_jobs; j++)
        if (lens[j]) {
            DP_LAUNCH(fr_into_repr_kernel, dim3(blocks_for(lens[j], 256)), dim3(256), 0, ctx->stream, (const Fr *)coeffs_dev[j],
                      (Fr *)coeffs_dev[j], (uint64_t)lens[j], (uint64_t)lens[j]);
            ctx->launches++;
        }
    std::vector<uint64_t> starts(n_jobs, 0), ends(lens, lens + n_jobs);
    std::vector<void *> outs(n_jobs);
    for (size_t j = 0; j < n_jobs; j++) outs[j] = od + j;
    const int rc = dp_msm_dev_batch(ctx, n_jobs, starts.data(), ends.data(), (const void *const *)coeffs_dev, lens, outs.data());
    for (size_t j = 0; j < n_jobs; j++)
        if (lens[j]) {
            DP_LAUNCH(fr_to_mont_kernel, dim3(blocks_for(lens[j], 256)), dim3(256), 0, ctx->stream, (Fr *)coeffs_dev[j], (uint64_t)lens[j]);
            ctx->launches++;
        }
    DP_CUDA(ctx, cudaGetLastError());
    if (rc != DP_OK) {
        DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return rc;
    }
    DP_CUDA(ctx, cudaMemcpyAsync(outs144, od, n_jobs * sizeof(G1JacobianOut), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

int dp_get_wire(dp_ctx *ctx, void *out, size_t out_bytes, size_t *n_coeffs) {
    if (!ctx) return DP_E_ARG;
    if (!ctx->wire) return fail(ctx, DP_E_STATE, "dp_get_wire before dp_round1");
    if (n_coeffs) *n_coeffs = ctx->wire_len;
    if (!out) return DP_OK;
    if (out_bytes < ctx->wire_len * sizeof(Fr)) return fail(ctx, DP_E_ARG, "dp_get_wire: buffer too small");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    DP_CUDA(ctx, cudaMemcpyAsync(out, ctx->wire, ctx->wire_len * sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return DP_OK;
}

int dp_last_msm_breakdown(const dp_ctx *ctx, float *sort_ms, float *accumulate_ms, float *reduce_ms) {
    if (!ctx) return DP_E_ARG;
    if (sort_ms) *sort_ms = ctx->msm_ms[0];
    if (accumulate_ms) *accumulate_ms = ctx->msm_ms[1];
    if (reduce_ms) *reduce_ms = ctx->msm_ms[2];
    return DP_OK;
}

int dp_msm_tuning(const dp_ctx *ctx, float *plain_ms, float *affine_ms, int *levels, int *equal) {
    if (!ctx) return DP_E_ARG;
    if (plain_ms) *plain_ms = ctx->tune_ms[0];
    if (affine_ms) *affine_ms = ctx->tune_ms[1];
    if (levels) *levels = (int)ctx->msm_affine_levels;
    if (equal) *equal = ctx->tune_equal;
    return DP_OK;
}

int dp_msm_tuning_all(const dp_ctx *ctx, float ms_by_levels[4]) {
    if (!ctx || !ms_by_levels) return DP_E_ARG;
    for (int k = 0; k < 4; k++) ms_by_levels[k] = ctx->tune_all_ms[k];
    return DP_OK;
}

int dp_debug_gen_bases(dp_ctx *ctx, uint64_t seed, size_t n, void *out) {
    if (!ctx || (n && !out)) return fail(ctx, DP_E_ARG, "dp_debug_gen_bases: NULL argument");
    if (n == 0) return DP_OK;
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    uint64_t *dev = (uint64_t *)ctx->pool.alloc(n * (size_t)DP_G1_AFFINE_BYTES);
    if (!dev) return fail(ctx, DP_E_OOM, "dp_debug_gen_bases");
    DP_LAUNCH(g1_gen_bases_kernel, dim3(blocks_for(n, 128)), dim3(128), 0, ctx->stream, dev, (uint64_t)n, seed);
    ctx->launches++;
    cudaError_t e = cudaMemcpyAsync(out, dev, n * (size_t)DP_G1_AFFINE_BYTES, cudaMemcpyDefault, ctx->stream);  // host or device memory
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    ctx->pool.release(dev);
    if (e != cudaSuccess) return fail(ctx, DP_E_CUDA, "dp_debug_gen_bases: %s", cudaGetErrorString(e));
    return DP_OK;
}

// tau^i = A[i mod 2^h] * B[i >> h] for i < n: A[a] = tau^a, B[b] = tau^(2^h b), about sqrt(n) host products each
// (Montgomery form; h >= min_log_a).  Returns h.
static uint32_t srs_power_tables(const Fr &tau, uint64_t n, uint32_t min_log_a, std::vector<Fr> &pow_a, std::vector<Fr> &pow_b) {
    uint32_t log_a = (log2_ceil_u64(n) + 1) / 2;
    if (log_a < min_log_a) log_a = min_log_a;
    const uint64_t n_a = (uint64_t)1 << log_a, n_b = (n + n_a - 1) >> log_a;
    pow_a.assign(n_a, Fr::one());
    pow_b.assign(n_b, Fr::one());
    const Fr t = tau.to_mont();
    for (uint64_t a = 1; a < n_a; a++) pow_a[a] = pow_a[a - 1] * t;
    const Fr step = pow_a[n_a - 1] * t;
    for (uint64_t b = 1; b < n_b; b++) pow_b[b] = pow_b[b - 1] * step;
    return log_a;
}

int dp_srs_powers_of_tau(dp_ctx *ctx, const void *tau32, size_t n, void *out104) {
    if (!ctx) return fail(ctx, DP_E_ARG, "dp_srs_powers_of_tau: ctx is NULL");
    if (n && (!tau32 || !out104)) return fail(ctx, DP_E_ARG, "dp_srs_powers_of_tau: NULL argument");
    if (n == 0) return DP_OK;
    if (n > ((uint64_t)1 << 32)) return fail(ctx, DP_E_ARG, "dp_srs_powers_of_tau: %zu points exceed 2^32", n);
    Fr tau;
    memcpy(tau.l, tau32, sizeof tau.l);
    if (tau.is_zero()) return fail(ctx, DP_E_ARG, "dp_srs_powers_of_tau: tau is zero");
    if (!tau.canon_is_reduced()) return fail(ctx, DP_E_ARG, "dp_srs_powers_of_tau: tau is not a canonical scalar (tau >= r)");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<Fr> pow_a, pow_b;
    const uint32_t log_a = srs_power_tables(tau, n, 0, pow_a, pow_b);
    const uint64_t n_a = pow_a.size(), n_b = pow_b.size();
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    Fr *da = tmp.get<Fr>(n_a), *db = tmp.get<Fr>(n_b);
    const uint64_t chunk = n < SRS_CHUNK ? n : SRS_CHUNK;
    uint64_t *staging = tmp.get<uint64_t>(chunk * 13);
    if (!da || !db || !staging) return fail(ctx, DP_E_OOM, "dp_srs_powers_of_tau buffers");
    DP_CUDA(ctx, cudaMemcpyAsync(da, pow_a.data(), n_a * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    DP_CUDA(ctx, cudaMemcpyAsync(db, pow_b.data(), n_b * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    G1Affine *table = ctx->srs_table;
    const bool build_table = !table;
    std::vector<G1Affine> half_base;
    if (build_table) {
        // P_q = 2^(q c / 2) G, q < 2 * windows: the points whose small multiples build the fixed-base table
        half_base.resize(2 * SRS_WINDOWS);
        G1XYZZ p = G1XYZZ::from_affine(g1_generator());
        for (uint32_t q = 0; q < 2 * SRS_WINDOWS; q++) {
            if (q)
                for (uint32_t k = 0; k < SRS_HALF; k++) p = p.dbl();
            half_base[q] = p.to_affine(true);
        }
        G1Affine *dbase = tmp.get<G1Affine>(2 * SRS_WINDOWS), *mult = tmp.get<G1Affine>(SRS_MULTIPLES);
        table = (G1Affine *)ctx->pool.alloc((size_t)SRS_WINDOWS * SRS_ROW * sizeof(G1Affine));
        if (!dbase || !mult || !table) {
            ctx->pool.release(table);
            return fail(ctx, DP_E_OOM, "dp_srs_powers_of_tau table");
        }
        const cudaError_t e = cudaMemcpyAsync(dbase, half_base.data(), 2 * SRS_WINDOWS * sizeof(G1Affine), cudaMemcpyHostToDevice, ctx->stream);
        if (e != cudaSuccess) {
            ctx->pool.release(table);
            return fail(ctx, DP_E_CUDA, "dp_srs_powers_of_tau: %s", cudaGetErrorString(e));
        }
        DP_LAUNCH(srs_multiples_kernel, dim3(blocks_for(SRS_MULTIPLES, AFF_TPB)), dim3(AFF_TPB), 0, ctx->stream, (const G1Affine *)dbase, mult);
        DP_LAUNCH(srs_table_kernel, dim3(blocks_for(SRS_WINDOWS * SRS_ROW / SRS_TABLE_GROUP, 128)), dim3(128), 0, ctx->stream,
                  (const G1Affine *)mult, table);
        ctx->launches += 2;
    }
    const MsmGeom g = msm_make_geom(SRS_C, true, 0);
    int rc = DP_OK;
    for (uint64_t first = 0; first < n && rc == DP_OK; first += chunk) {
        const uint64_t end = first + chunk < n ? first + chunk : n;
        DP_LAUNCH(srs_powers_kernel, dim3(blocks_for(end - first, AFF_TPB)), dim3(AFF_TPB), 0, ctx->stream, (const Fr *)da,
                  (const Fr *)db, log_a, first, end, g, (const G1Affine *)table, staging);
        ctx->launches++;
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess)
            e = cudaMemcpyAsync((uint8_t *)out104 + first * DP_G1_AFFINE_BYTES, staging, (end - first) * DP_G1_AFFINE_BYTES, cudaMemcpyDefault,
                                ctx->stream);  // host or device memory
        if (e != cudaSuccess) rc = fail(ctx, DP_E_CUDA, "dp_srs_powers_of_tau: %s", cudaGetErrorString(e));
    }
    if (rc == DP_OK) rc = call_end(ctx, true);
    if (build_table) {  // kept for the next call only when its build is known to have completed
        if (rc == DP_OK) {
            ctx->srs_table = table;
        } else {
            cudaStreamSynchronize(ctx->stream);
            ctx->pool.release(table);
        }
    }
    return rc;
}

// ---- verifier: decoding, an MSM over caller-given points, the G2 open key and the multi-pairing (pairing.cuh)
int dp_g1_decompress(dp_ctx *ctx, const void *in48, size_t n, int check_subgroup, void *out104, size_t *bad_index, int *why) {
    if (!ctx) return fail(ctx, DP_E_ARG, "dp_g1_decompress: ctx is NULL");
    if (n && (!in48 || !out104)) return fail(ctx, DP_E_ARG, "dp_g1_decompress: NULL argument");
    if (bad_index) *bad_index = n;
    if (why) *why = 0;
    if (n == 0) return DP_OK;
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    uint32_t *staging = tmp.get<uint32_t>(n * 12);
    G1Affine *pts = tmp.get<G1Affine>(n);
    uint64_t *raw = tmp.get<uint64_t>(n * 13);
    unsigned long long *err = tmp.get<unsigned long long>(1), verdict = ~0ull;
    if (!staging || !pts || !raw || !err) return fail(ctx, DP_E_OOM, "dp_g1_decompress buffers");
    DP_CUDA(ctx, cudaMemcpyAsync(staging, in48, n * (size_t)DP_G1_COMPRESSED_BYTES, cudaMemcpyHostToDevice, ctx->stream));
    DP_CUDA(ctx, cudaMemcpyAsync(err, &verdict, sizeof verdict, cudaMemcpyHostToDevice, ctx->stream));
    DP_LAUNCH(g1_decompress_kernel, dim3(blocks_for(n, 128)), dim3(128), 0, ctx->stream, (const uint32_t *)staging, pts, (uint64_t)n,
              check_subgroup ? 1u : 0u, err);
    DP_LAUNCH(g1_export_ark_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, ctx->stream, (const G1Affine *)pts, raw, (uint64_t)n);
    ctx->launches += 2;
    DP_CUDA(ctx, cudaMemcpyAsync(&verdict, err, sizeof verdict, cudaMemcpyDeviceToHost, ctx->stream));
    DP_TRY(call_end(ctx, true));
    if (verdict != ~0ull) {
        const size_t idx = (size_t)((verdict >> 8) - 1);
        if (bad_index) *bad_index = idx;
        if (why) *why = (int)(verdict & 7);
        return fail(ctx, DP_E_ARG, "dp_g1_decompress: point %zu rejected: %s", idx, G1_DECOMPRESS_WHY[verdict & 7]);
    }
    DP_CUDA(ctx, cudaMemcpy(out104, raw, n * (size_t)DP_G1_AFFINE_BYTES, cudaMemcpyDeviceToHost));
    return DP_OK;
}

int dp_msm_points(dp_ctx *ctx, const void *points104, const void *scalars32, size_t n, void *out144) {
    if (!ctx) return fail(ctx, DP_E_ARG, "dp_msm_points: ctx is NULL");
    if (!out144 || (n && (!points104 || !scalars32))) return fail(ctx, DP_E_ARG, "dp_msm_points: NULL argument");
    if (n >= ((uint64_t)1 << 31)) return fail(ctx, DP_E_ARG, "dp_msm_points: %zu points exceed 2^31", n);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    uint64_t *raw = tmp.get<uint64_t>(n * 13);
    G1Affine *pts = tmp.get<G1Affine>(n);
    uint4 *sc = tmp.get<uint4>(2 * n);
    G1JacobianOut *od = tmp.get<G1JacobianOut>(1);
    if (!raw || !pts || !sc || !od) return fail(ctx, DP_E_OOM, "dp_msm_points buffers for %zu points", n);
    if (n) {
        DP_CUDA(ctx, cudaMemcpyAsync(raw, points104, n * (size_t)DP_G1_AFFINE_BYTES, cudaMemcpyHostToDevice, ctx->stream));
        DP_CUDA(ctx, cudaMemcpyAsync(sc, scalars32, n * 32, cudaMemcpyHostToDevice, ctx->stream));
        DP_LAUNCH(g1_import_ark_kernel, dim3(blocks_for(n, 256)), dim3(256), 0, ctx->stream, (const uint64_t *)raw, pts, (uint64_t)n);
        ctx->launches++;
    }
    DP_TRY(msm_device(ctx, 0, sc, n, od, nullptr, pts));
    DP_CUDA(ctx, cudaMemcpyAsync(out144, od, sizeof(G1JacobianOut), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

int dp_srs_open_key(dp_ctx *ctx, const void *tau32, void *out400) {
    if (!ctx) return fail(ctx, DP_E_ARG, "dp_srs_open_key: ctx is NULL");
    if (!tau32 || !out400) return fail(ctx, DP_E_ARG, "dp_srs_open_key: NULL argument");
    Fr tau;
    memcpy(tau.l, tau32, sizeof tau.l);
    if (tau.is_zero()) return fail(ctx, DP_E_ARG, "dp_srs_open_key: tau is zero");
    if (!tau.canon_is_reduced()) return fail(ctx, DP_E_ARG, "dp_srs_open_key: tau is not a canonical scalar (tau >= r)");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    uint64_t *dev = tmp.get<uint64_t>(2 * 25);
    if (!dev) return fail(ctx, DP_E_OOM, "dp_srs_open_key buffer");
    DP_LAUNCH(g2_open_key_kernel, dim3(1), dim3(32), 0, ctx->stream, tau, dev);
    ctx->launches++;
    DP_CUDA(ctx, cudaMemcpyAsync(out400, dev, 2 * (size_t)DP_G2_AFFINE_BYTES, cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

int dp_multi_pairing(dp_ctx *ctx, const void *g1_104, const void *g2_200, size_t k, void *out576) {
    if (!ctx) return fail(ctx, DP_E_ARG, "dp_multi_pairing: ctx is NULL");
    if (!out576 || (k && (!g1_104 || !g2_200))) return fail(ctx, DP_E_ARG, "dp_multi_pairing: NULL argument");
    if (k > ((size_t)1 << 20)) return fail(ctx, DP_E_ARG, "dp_multi_pairing: %zu pairs exceed 2^20", k);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    uint64_t *p = tmp.get<uint64_t>(k * 13), *q = tmp.get<uint64_t>(k * 25);
    Fq12 *f = tmp.get<Fq12>(k), *out = tmp.get<Fq12>(1);
    unsigned long long *bad = tmp.get<unsigned long long>(1), verdict = ~0ull;
    if (!p || !q || !f || !out || !bad) return fail(ctx, DP_E_OOM, "dp_multi_pairing buffers for %zu pairs", k);
    DP_CUDA(ctx, cudaMemcpyAsync(bad, &verdict, sizeof verdict, cudaMemcpyHostToDevice, ctx->stream));
    if (k) {
        DP_CUDA(ctx, cudaMemcpyAsync(p, g1_104, k * (size_t)DP_G1_AFFINE_BYTES, cudaMemcpyHostToDevice, ctx->stream));
        DP_CUDA(ctx, cudaMemcpyAsync(q, g2_200, k * (size_t)DP_G2_AFFINE_BYTES, cudaMemcpyHostToDevice, ctx->stream));
        DP_LAUNCH(pairing_miller_kernel, dim3(blocks_for(2 * (uint64_t)k, 64)), dim3(64), 0, ctx->stream, (const uint64_t *)p,
                  (const uint64_t *)q, (uint32_t)k, f, bad);
        ctx->launches++;
    }
    DP_LAUNCH(pairing_final_kernel, dim3(1), dim3(32), 0, ctx->stream, (const Fq12 *)f, (uint32_t)k, (const unsigned long long *)bad, out);
    ctx->launches++;
    DP_CUDA(ctx, cudaMemcpyAsync(&verdict, bad, sizeof verdict, cudaMemcpyDeviceToHost, ctx->stream));
    DP_TRY(call_end(ctx, true));
    if (verdict != ~0ull) {
        static const char *const reason[] = {"", "a G1 coordinate is not below p", "the G1 point is not on the curve",
                                             "a G2 coordinate is not below p", "the G2 point is not on the twist",
                                             "the G2 point is not in the r-torsion subgroup"};
        return fail(ctx, DP_E_ARG, "dp_multi_pairing: pair %llu rejected: %s", (unsigned long long)((verdict >> 8) - 1),
                    reason[(verdict & 0xff) < 6 ? verdict & 0xff : 0]);
    }
    DP_CUDA(ctx, cudaMemcpy(out576, out, sizeof(Fq12), cudaMemcpyDeviceToHost));
    return DP_OK;
}

// ---- setup files: the encoders, the G2 decoder and the consistency check of a loaded SRS (DESIGN.md section 3.9)
// n points to 48 compressed bytes each, SRS_CHUNK points at a time: `src_dev` (resident 96-byte bases) or, when it is NULL,
// the raw structs at in104 (host or device memory), staged chunk by chunk
static int g1_compress_chunks(dp_ctx *ctx, const G1Affine *src_dev, const void *in104, size_t n, void *out48, const char *who) {
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    const uint64_t chunk = n < SRS_CHUNK ? n : SRS_CHUNK;
    uint32_t *packed = tmp.get<uint32_t>(chunk * 12);
    uint64_t *raw = src_dev ? nullptr : tmp.get<uint64_t>(chunk * 13);
    if (!packed || (!src_dev && !raw)) return fail(ctx, DP_E_OOM, "%s buffers", who);
    for (uint64_t first = 0; first < n; first += chunk) {
        const uint64_t m = first + chunk < n ? chunk : n - first;
        if (src_dev) {
            DP_LAUNCH(g1_compress_kernel, dim3(blocks_for(m, 256)), dim3(256), 0, ctx->stream, src_dev + first, packed, m);
        } else {
            DP_CUDA(ctx, cudaMemcpyAsync(raw, (const uint8_t *)in104 + first * DP_G1_AFFINE_BYTES, m * DP_G1_AFFINE_BYTES, cudaMemcpyDefault,
                                         ctx->stream));
            DP_LAUNCH(g1_compress_ark_kernel, dim3(blocks_for(m, 256)), dim3(256), 0, ctx->stream, (const uint64_t *)raw, packed, m);
        }
        ctx->launches++;
        DP_CUDA(ctx, cudaMemcpyAsync((uint8_t *)out48 + first * DP_G1_COMPRESSED_BYTES, packed, m * DP_G1_COMPRESSED_BYTES, cudaMemcpyDefault,
                                     ctx->stream));
    }
    return call_end(ctx, true);
}

int dp_g1_compress(dp_ctx *ctx, const void *in104, size_t n, void *out48) {
    if (!ctx) return fail(ctx, DP_E_ARG, "dp_g1_compress: ctx is NULL");
    if (n && (!in104 || !out48)) return fail(ctx, DP_E_ARG, "dp_g1_compress: NULL argument");
    if (n == 0) return DP_OK;
    return g1_compress_chunks(ctx, nullptr, in104, n, out48, "dp_g1_compress");
}

int dp_get_bases_compressed(dp_ctx *ctx, uint64_t start, size_t n, void *out48) {
    if (!ctx || (n && !out48)) return fail(ctx, DP_E_ARG, "dp_get_bases_compressed: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_get_bases_compressed before dp_init");
    if (start > ctx->n_bases || n > ctx->n_bases - start)
        return fail(ctx, DP_E_ARG, "dp_get_bases_compressed: range outside %llu bases", (unsigned long long)ctx->n_bases);
    if (n == 0) return DP_OK;
    return g1_compress_chunks(ctx, ctx->bases + start, nullptr, n, out48, "dp_get_bases_compressed");
}

int dp_g2_compress(dp_ctx *ctx, const void *in200, size_t n, void *out96) {
    if (!ctx) return fail(ctx, DP_E_ARG, "dp_g2_compress: ctx is NULL");
    if (n && (!in200 || !out96)) return fail(ctx, DP_E_ARG, "dp_g2_compress: NULL argument");
    if (n > ((size_t)1 << 20)) return fail(ctx, DP_E_ARG, "dp_g2_compress: %zu points exceed 2^20", n);
    if (n == 0) return DP_OK;
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    uint64_t *raw = tmp.get<uint64_t>(n * 25);
    uint32_t *packed = tmp.get<uint32_t>(n * 24);
    if (!raw || !packed) return fail(ctx, DP_E_OOM, "dp_g2_compress buffers");
    DP_CUDA(ctx, cudaMemcpyAsync(raw, in200, n * (size_t)DP_G2_AFFINE_BYTES, cudaMemcpyDefault, ctx->stream));
    DP_LAUNCH(g2_compress_kernel, dim3(blocks_for(n, 32)), dim3(32), 0, ctx->stream, (const uint64_t *)raw, packed, (uint64_t)n);
    ctx->launches++;
    DP_CUDA(ctx, cudaMemcpyAsync(out96, packed, n * (size_t)DP_G2_COMPRESSED_BYTES, cudaMemcpyDefault, ctx->stream));
    return call_end(ctx, true);
}

int dp_g2_decompress(dp_ctx *ctx, const void *in96, size_t n, int check_subgroup, void *out200, size_t *bad_index, int *why) {
    if (!ctx) return fail(ctx, DP_E_ARG, "dp_g2_decompress: ctx is NULL");
    if (n && (!in96 || !out200)) return fail(ctx, DP_E_ARG, "dp_g2_decompress: NULL argument");
    if (n > ((size_t)1 << 20)) return fail(ctx, DP_E_ARG, "dp_g2_decompress: %zu points exceed 2^20", n);
    if (bad_index) *bad_index = n;
    if (why) *why = 0;
    if (n == 0) return DP_OK;
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    uint32_t *packed = tmp.get<uint32_t>(n * 24);
    uint64_t *raw = tmp.get<uint64_t>(n * 25);
    unsigned long long *err = tmp.get<unsigned long long>(1), verdict = ~0ull;
    if (!packed || !raw || !err) return fail(ctx, DP_E_OOM, "dp_g2_decompress buffers");
    DP_CUDA(ctx, cudaMemcpyAsync(packed, in96, n * (size_t)DP_G2_COMPRESSED_BYTES, cudaMemcpyDefault, ctx->stream));
    DP_CUDA(ctx, cudaMemcpyAsync(err, &verdict, sizeof verdict, cudaMemcpyHostToDevice, ctx->stream));
    DP_LAUNCH(g2_decompress_kernel, dim3(blocks_for(n, 32)), dim3(32), 0, ctx->stream, (const uint32_t *)packed, raw, (uint64_t)n,
              check_subgroup ? 1u : 0u, err);
    ctx->launches++;
    DP_CUDA(ctx, cudaMemcpyAsync(&verdict, err, sizeof verdict, cudaMemcpyDeviceToHost, ctx->stream));
    DP_TRY(call_end(ctx, true));
    if (verdict != ~0ull) {
        const size_t idx = (size_t)((verdict >> 8) - 1);
        if (bad_index) *bad_index = idx;
        if (why) *why = (int)(verdict & 7);
        static const char *const reason[] = {"", "a coordinate is not a canonical field element", "both flag bits set",
                                             "x^3 + 4 (u + 1) is not a square: no such point", "the point is not in the r-torsion subgroup"};
        return fail(ctx, DP_E_ARG, "dp_g2_decompress: point %zu rejected: %s", idx, reason[verdict & 7]);
    }
    DP_CUDA(ctx, cudaMemcpy(out200, raw, n * (size_t)DP_G2_AFFINE_BYTES, cudaMemcpyDefault));
    return DP_OK;
}

int dp_srs_check(dp_ctx *ctx, const void *g2_400, const void *seed32, int *ok) {
    if (!ctx) return fail(ctx, DP_E_ARG, "dp_srs_check: ctx is NULL");
    if (!g2_400 || !ok) return fail(ctx, DP_E_ARG, "dp_srs_check: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_srs_check before dp_init");
    const uint64_t n = ctx->n_bases;
    if (n == 0) return fail(ctx, DP_E_STATE, "dp_srs_check: the context holds no bases");
    *ok = 0;
    ChaChaKey key;
    if (seed32) {
        memcpy(key.w, seed32, sizeof key.w);
    } else {
        size_t got = 0;
        while (got < sizeof key.w) {
            const ssize_t r = getrandom(reinterpret_cast<uint8_t *>(key.w) + got, sizeof key.w - got, 0);
            if (r < 0) return fail(ctx, DP_E_STATE, "dp_srs_check: getrandom failed; pass a seed");
            got += (size_t)r;
        }
    }
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    using clock = std::chrono::steady_clock;
    auto ms_since = [](clock::time_point t0) { return std::chrono::duration<float, std::milli>(clock::now() - t0).count(); };
    for (float &v : ctx->srs_check_ms) v = 0.f;
    ctx->srs_check_ab[0] = ctx->srs_check_ab[1] = G1JacobianOut::from_affine(G1Affine::inf());
    G1Affine first;
    DP_CUDA(ctx, cudaMemcpy(&first, ctx->bases, sizeof first, cudaMemcpyDeviceToHost));
    const G1Affine gen = g1_generator();
    if (!(first.x == gen.x) || !(first.y == gen.y)) return DP_OK;  // P_0 is not the generator
    if (n == 1) {
        *ok = 1;
        return DP_OK;
    }
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    uint4 *sa = tmp.get<uint4>(2 * n), *sb = tmp.get<uint4>(2 * n);
    G1JacobianOut *od = tmp.get<G1JacobianOut>(2);
    if (!sa || !sb || !od) return fail(ctx, DP_E_OOM, "dp_srs_check: scalars for %llu bases", (unsigned long long)n);
    clock::time_point t0 = clock::now();
    DP_LAUNCH(srs_check_scalars_kernel, dim3(blocks_for((n + 2) / 4, 128)), dim3(128), 0, ctx->stream, key, n, sa, sb);
    ctx->launches++;
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->srs_check_ms[0] = ms_since(t0);
    // both over the whole SRS from base 0, the range the window-multiple table of dp_init covers
    t0 = clock::now();
    DP_TRY(msm_device(ctx, 0, sa, n, od, nullptr));
    DP_TRY(msm_device(ctx, 0, sb, n, od + 1, nullptr));
    DP_CUDA(ctx, cudaMemcpyAsync(ctx->srs_check_ab, od, 2 * sizeof(G1JacobianOut), cudaMemcpyDeviceToHost, ctx->stream));
    DP_TRY(call_end(ctx, true));
    ctx->srs_check_ms[1] = ms_since(t0);
    // e(A, beta h) * e(-B, h) == 1  <=>  sum rho_i (tau P_i - P_(i+1)) == 0
    t0 = clock::now();
    uint8_t g1[2 * DP_G1_AFFINE_BYTES] = {};  // raw structs: the limbs of a Montgomery Fq are its 48 little-endian bytes
    for (int k = 0; k < 2; k++) {
        const G1JacobianOut &j = ctx->srs_check_ab[k];
        const bool inf = j.z.is_zero();
        const Fq x = inf ? Fq::zero() : j.x, y = inf ? Fq::one() : k == 0 ? j.y : j.y.neg();
        memcpy(g1 + DP_G1_AFFINE_BYTES * k, x.l, 48);
        memcpy(g1 + DP_G1_AFFINE_BYTES * k + 48, y.l, 48);
        g1[DP_G1_AFFINE_BYTES * k + 96] = inf ? 1 : 0;
    }
    uint8_t pair[2 * DP_G2_AFFINE_BYTES];
    memcpy(pair, (const uint8_t *)g2_400 + DP_G2_AFFINE_BYTES, DP_G2_AFFINE_BYTES);  // beta h pairs with A
    memcpy(pair + DP_G2_AFFINE_BYTES, g2_400, DP_G2_AFFINE_BYTES);                   // h with -B
    uint8_t e[DP_FQ12_BYTES], one[DP_FQ12_BYTES] = {};  // 1 in Fq12: the first of the 12 coefficients is 1
    const Fq fq_one = Fq::one();
    memcpy(one, fq_one.l, 48);
    DP_TRY(dp_multi_pairing(ctx, g1, pair, 2, e));
    ctx->srs_check_ms[2] = ms_since(t0);
    *ok = memcmp(e, one, sizeof e) == 0 ? 1 : 0;
    return DP_OK;
}

// ---- ceremony: one contribution Q_i = s^i P_i over the resident bases, and s h, s beta h (DESIGN.md section 3.10)
static int srs_update(dp_ctx *ctx, const void *s32, const void *g2_400, void *out48, void *out400, bool glv, const char *who) {
    if (!ctx) return fail(ctx, DP_E_ARG, "%s: ctx is NULL", who);
    if (!g2_400 || !out48 || !out400) return fail(ctx, DP_E_ARG, "%s: NULL argument", who);
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "%s before dp_init", who);
    const uint64_t n = ctx->n_bases;
    if (n == 0) return fail(ctx, DP_E_STATE, "%s: the context holds no bases", who);
    // the secret and everything derived from it on the host: wiped on every return
    Fr s = Fr::zero();
    std::vector<Fr> pow_a, pow_b;
    struct HostWipe {
        Fr &s;
        std::vector<Fr> &a, &b;
        ~HostWipe() {
            explicit_bzero((void *)&s, sizeof s);
            if (!a.empty()) explicit_bzero((void *)a.data(), a.size() * sizeof(Fr));
            if (!b.empty()) explicit_bzero((void *)b.data(), b.size() * sizeof(Fr));
        }
    } host_wipe{s, pow_a, pow_b};
    if (s32) {
        memcpy(s.l, s32, sizeof s.l);
        if (s.is_zero()) return fail(ctx, DP_E_ARG, "%s: s is zero", who);
        if (!s.canon_is_reduced()) return fail(ctx, DP_E_ARG, "%s: s is not a canonical scalar (s >= r)", who);
    } else {
        while (s.is_zero() || !s.canon_is_reduced()) {  // uniform in 1 .. r - 1: r > 2^254, so 255 random bits hit it often
            size_t got = 0;
            while (got < sizeof s.l) {
                const ssize_t r = getrandom(reinterpret_cast<uint8_t *>(s.l) + got, sizeof s.l - got, 0);
                if (r < 0) return fail(ctx, DP_E_STATE, "%s: getrandom failed; pass s", who);
                got += (size_t)r;
            }
            s.l[7] &= 0x7fffffffu;
        }
    }
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint32_t log_a = srs_power_tables(s, n, 1, pow_a, pow_b);  // h >= 1: pow_a[1] = s for the G2 kernel
    const uint64_t n_a = pow_a.size(), n_b = pow_b.size();
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    Fr *da = tmp.get<Fr>(n_a), *db = tmp.get<Fr>(n_b);
    const uint64_t chunk = n < SRS_CHUNK ? n : SRS_CHUNK;
    uint32_t *staging = tmp.get<uint32_t>(chunk * 12);
    uint64_t *g2_in = tmp.get<uint64_t>(2 * 25), *g2_out = tmp.get<uint64_t>(2 * 25);
    unsigned long long *bad = tmp.get<unsigned long long>(1), verdict = ~0ull;
    // the pool hands its blocks out again (DESIGN.md section 3.5): the power tables are zeroed, in stream order, before
    // Scratch returns them, on every path
    struct DeviceWipe {
        dp_ctx *ctx;
        Fr *a, *b;
        uint64_t n_a, n_b;
        ~DeviceWipe() {
            if (a) cudaMemsetAsync(a, 0, n_a * sizeof(Fr), ctx->stream);
            if (b) cudaMemsetAsync(b, 0, n_b * sizeof(Fr), ctx->stream);
            cudaStreamSynchronize(ctx->stream);
        }
    } device_wipe{ctx, da, db, n_a, n_b};
    if (!da || !db || !staging || !g2_in || !g2_out || !bad) return fail(ctx, DP_E_OOM, "%s buffers", who);
    DP_CUDA(ctx, cudaMemcpyAsync(da, pow_a.data(), n_a * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    DP_CUDA(ctx, cudaMemcpyAsync(db, pow_b.data(), n_b * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    DP_CUDA(ctx, cudaMemcpyAsync(g2_in, g2_400, 2 * (size_t)DP_G2_AFFINE_BYTES, cudaMemcpyDefault, ctx->stream));
    DP_CUDA(ctx, cudaMemcpyAsync(bad, &verdict, sizeof verdict, cudaMemcpyHostToDevice, ctx->stream));
    DP_LAUNCH(srs_update_g2_kernel, dim3(1), dim3(32), 0, ctx->stream, (const Fr *)da, (const uint64_t *)g2_in, g2_out, bad);
    ctx->launches++;
    DP_CUDA(ctx, cudaMemcpyAsync(&verdict, bad, sizeof verdict, cudaMemcpyDeviceToHost, ctx->stream));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // a rejected G2 point is refused before the bulk work
    if (verdict != ~0ull) {
        static const char *const reason[] = {"", "", "", "a coordinate is not below p", "the point is not on the twist",
                                             "the point is not in the r-torsion subgroup"};
        return fail(ctx, DP_E_ARG, "%s: %s rejected: %s", who, (verdict >> 8) == 1 ? "h" : "beta h", reason[(verdict & 0xff) < 6 ? verdict & 0xff : 0]);
    }
    const Fq beta = glv_beta();
    for (uint64_t first = 0; first < n; first += chunk) {
        const uint64_t end = first + chunk < n ? first + chunk : n;
        if (glv)
            DP_LAUNCH(srs_update_kernel<true>, dim3(blocks_for(end - first, AFF_TPB)), dim3(AFF_TPB), 0, ctx->stream, (const G1Affine *)ctx->bases,
                      (const Fr *)da, (const Fr *)db, log_a, first, end, beta, staging);
        else
            DP_LAUNCH(srs_update_kernel<false>, dim3(blocks_for(end - first, AFF_TPB)), dim3(AFF_TPB), 0, ctx->stream, (const G1Affine *)ctx->bases,
                      (const Fr *)da, (const Fr *)db, log_a, first, end, beta, staging);
        ctx->launches++;
        DP_CUDA(ctx, cudaGetLastError());
        DP_CUDA(ctx, cudaMemcpyAsync((uint8_t *)out48 + first * DP_G1_COMPRESSED_BYTES, staging, (end - first) * DP_G1_COMPRESSED_BYTES,
                                     cudaMemcpyDefault, ctx->stream));  // host or device memory
    }
    DP_CUDA(ctx, cudaMemcpyAsync(out400, g2_out, 2 * (size_t)DP_G2_AFFINE_BYTES, cudaMemcpyDefault, ctx->stream));
    return call_end(ctx, true);
}

int dp_srs_update(dp_ctx *ctx, const void *s32, const void *g2_400, void *out48, void *out400) {
    return srs_update(ctx, s32, g2_400, out48, out400, true, "dp_srs_update");
}

int dp_debug_srs_update_plain(dp_ctx *ctx, const void *s32, const void *g2_400, void *out48, void *out400) {
    return srs_update(ctx, s32, g2_400, out48, out400, false, "dp_debug_srs_update_plain");
}

int dp_last_srs_check(const dp_ctx *ctx, float *scalars_ms, float *msm_ms, float *pairing_ms, void *ab288) {
    if (!ctx) return DP_E_ARG;
    if (scalars_ms) *scalars_ms = ctx->srs_check_ms[0];
    if (msm_ms) *msm_ms = ctx->srs_check_ms[1];
    if (pairing_ms) *pairing_ms = ctx->srs_check_ms[2];
    if (ab288) memcpy(ab288, ctx->srs_check_ab, sizeof ctx->srs_check_ab);
    return DP_OK;
}

int dp_debug_set_limits(dp_ctx *ctx, uint32_t max_contig_log_k, uint32_t max_strided_log_k, int msm_window_bits) {
    if (!ctx) return DP_E_ARG;
    if (max_contig_log_k < 1 || max_contig_log_k > NTT_WTAB_LOG || max_strided_log_k < 1 || max_strided_log_k > NTT_MAX_STRIDED_LOG_K ||
        msm_window_bits < 0 || msm_window_bits > 20)
        return fail(ctx, DP_E_ARG, "dp_debug_set_limits: out of range");
    ctx->max_contig_log_k = max_contig_log_k;
    ctx->max_strided_log_k = max_strided_log_k;
    ctx->msm_force_c = msm_window_bits;
    return DP_OK;
}

int dp_debug_set_three_pass(dp_ctx *ctx, uint32_t min_log_n) {
    if (!ctx) return DP_E_ARG;
    ctx->no_three_pass = min_log_n == 0;
    ctx->three_pass_min_log = min_log_n ? min_log_n : 20;
    return DP_OK;
}

int dp_peer_arena_create(dp_ctx *ctx, uint64_t arena_bytes, void *handle_out) {
    if (!ctx || !handle_out) return fail(ctx, DP_E_ARG, "dp_peer_arena_create: NULL argument");
    if (ctx->arena) return fail(ctx, DP_E_STATE, "dp_peer_arena_create: arena already exists");
    if (arena_bytes < 2 * sizeof(Fr)) return fail(ctx, DP_E_ARG, "dp_peer_arena_create: arena too small");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    arena_bytes = ((arena_bytes + 1023) & ~(uint64_t)1023) + ARENA_HEADER_BYTES;
    void *p = nullptr;
    // a dedicated cudaMalloc (not the pool): IPC handles cover whole allocations
    if (cudaMalloc(&p, arena_bytes) != cudaSuccess) return fail(ctx, DP_E_OOM, "peer arena of %llu bytes", (unsigned long long)arena_bytes);
    cudaMemset(p, 0, ARENA_HEADER_BYTES);
    cudaIpcMemHandle_t h;
    static_assert(sizeof(cudaIpcMemHandle_t) == DP_IPC_HANDLE_BYTES, "IPC handle size");
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        return fail(ctx, DP_E_CUDA, "cudaIpcGetMemHandle: %s", cudaGetErrorString(e));
    }
    memcpy(handle_out, &h, sizeof h);
    ctx->arena = (Fr *)p;
    ctx->arena_bytes = arena_bytes;
    ctx->peer_arena[ctx->me] = ctx->arena;
    return DP_OK;
}

int dp_peer_attach(dp_ctx *ctx, uint64_t peer, const void *handle) {
    if (!ctx || !handle) return fail(ctx, DP_E_ARG, "dp_peer_attach: NULL argument");
    if (peer >= ctx->W || peer >= 8) return fail(ctx, DP_E_ARG, "dp_peer_attach: peer %llu of %llu", (unsigned long long)peer, (unsigned long long)ctx->W);
    if (!ctx->arena) return fail(ctx, DP_E_STATE, "dp_peer_attach before dp_peer_arena_create");
    if (peer == ctx->me) return DP_OK;
    if (ctx->peer_arena[peer]) return fail(ctx, DP_E_STATE, "dp_peer_attach: peer %llu already attached", (unsigned long long)peer);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof h);
    void *p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return fail(ctx, DP_E_COMM, "cudaIpcOpenMemHandle(peer %llu): %s", (unsigned long long)peer, cudaGetErrorString(e));
    ctx->peer_arena[peer] = (Fr *)p;
    return DP_OK;
}

int dp_peer_ready(const dp_ctx *ctx) { return ctx && p2p_ready(ctx) ? 1 : 0; }

int dp_fft_dev_rows_p2p(dp_ctx *ctx, const void *rows_dev, int is_quot, int is_inv, int is_coset) {
    if (!ctx || !rows_dev) return fail(ctx, DP_E_ARG, "dp_fft_dev_rows_p2p: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_fft_dev_rows_p2p before dp_init");
    if (!p2p_ready(ctx)) return fail(ctx, DP_E_COMM, "dp_fft_dev_rows_p2p: peers not attached");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    const DomainDev &d = ctx->dom[is_quot ? 1 : 0];
    const uint64_t W = ctx->W, n_rows = d.r() / W, n_cols = d.c() / W, c = d.c();
    call_begin(ctx);
    PeerDst peers;
    Fr *slot = nullptr;
    DP_TRY(p2p_next_slot(ctx, d.r() * n_cols * sizeof(Fr), peers, slot, ctx->me * n_rows * n_cols));
    const bool need_scratch = d.log_c > ctx->max_contig_log_k;
    Scratch tmp(ctx->pool);
    Fr *scratch = need_scratch ? tmp.get<Fr>(n_rows * c) : nullptr;
    if (need_scratch && !scratch) return fail(ctx, DP_E_OOM, "dp_fft_dev_rows_p2p scratch");
    if (ctx->dev_p2p_slot) return fail(ctx, DP_E_STATE, "dp_fft_dev_rows_p2p: the previous transform still waits for dp_fft_dev_cols");
    DP_TRY(plan_row_phase(ctx, d, (const Fr *)rows_dev, nullptr, scratch, n_rows, ctx->me * n_rows, is_inv != 0, is_coset != 0, W, &peers,
                          dev_rd_cols(ctx, d, is_quot, is_inv)));
    p2p_commit_slot(ctx);
    ctx->dev_p2p_slot = slot;
    DP_TRY(call_end(ctx, true));
    ctx->pool.release(ctx->dev_send);
    ctx->pool.release(ctx->dev_recv);
    ctx->dev_send = nullptr;
    ctx->dev_recv = nullptr;
    ctx->dev_p2p_slot = slot;
    ctx->dev_flags = (is_quot ? 4 : 0) | (is_inv ? 2 : 0) | (is_coset ? 1 : 0);
    return DP_OK;
}

static int fft_dev_p2p(dp_ctx *ctx, const void *rows_dev, void *cols_dev, int is_quot, int is_inv, int is_coset, bool wait);

// rows -> peer memory -> device-side barrier -> columns, all queued on the compute stream
int dp_fft_dev_p2p(dp_ctx *ctx, const void *rows_dev, void *cols_dev, int is_quot, int is_inv, int is_coset) {
    return fft_dev_p2p(ctx, rows_dev, cols_dev, is_quot, is_inv, is_coset, true);
}
// The same without waiting: the whole transform (and any number of following ones) stays queued on the
// compute stream; dp_sync() waits and reports a barrier time-out.  Two receive slots are enough for an
// unbounded stream of transforms: rank A stores transform k+2 into the slot of transform k only after its
// own column phase k+1, which waited at barrier k+1 for every rank B to finish its row phase k+1, which B's
// stream runs after B's column phase k - the last reader of that slot.
int dp_fft_dev_p2p_async(dp_ctx *ctx, const void *rows_dev, void *cols_dev, int is_quot, int is_inv, int is_coset) {
    return fft_dev_p2p(ctx, rows_dev, cols_dev, is_quot, is_inv, is_coset, false);
}

static int p2p_check_timeout(dp_ctx *ctx) {
    if (!ctx->arena || !ctx->bar_seq) return DP_OK;
    uint32_t timed_out = 0;  // word 1 of the arena header, set by p2p_barrier_kernel when a peer never arrived
    DP_CUDA(ctx, cudaMemcpy(&timed_out, reinterpret_cast<uint32_t *>(ctx->arena) + 1, 4, cudaMemcpyDeviceToHost));
    if (timed_out) return fail(ctx, DP_E_COMM, "fused exchange: a peer did not reach the device-side barrier within 20 s");
    return DP_OK;
}

static int fft_dev_p2p(dp_ctx *ctx, const void *rows_dev, void *cols_dev, int is_quot, int is_inv, int is_coset, bool wait) {
    if (!ctx || !rows_dev || !cols_dev) return fail(ctx, DP_E_ARG, "dp_fft_dev_p2p: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_fft_dev_p2p before dp_init");
    if (!p2p_ready(ctx)) return fail(ctx, DP_E_COMM, "dp_fft_dev_p2p: peers not attached");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    const DomainDev &d = ctx->dom[is_quot ? 1 : 0];
    const uint64_t W = ctx->W, n_rows = d.r() / W, n_cols = d.c() / W, c = d.c();
    call_begin(ctx);
    PeerDst peers;
    Fr *slot = nullptr;
    DP_TRY(p2p_next_slot(ctx, d.r() * n_cols * sizeof(Fr), peers, slot, ctx->me * n_rows * n_cols));
    Scratch tmp(ctx->pool);
    const bool need_scratch = d.log_c > ctx->max_contig_log_k;
    Fr *scratch = need_scratch ? tmp.get<Fr>(n_rows * c) : nullptr;
    if (need_scratch && !scratch) return fail(ctx, DP_E_OOM, "dp_fft_dev_p2p scratch");
    DP_TRY(plan_row_phase(ctx, d, (const Fr *)rows_dev, nullptr, scratch, n_rows, ctx->me * n_rows, is_inv != 0, is_coset != 0, W, &peers,
                          dev_rd_cols(ctx, d, is_quot, is_inv)));
    p2p_commit_slot(ctx);
    struct SlotGuard {  // the slot is free again once this call returns: the column kernels read it before the stream drains
        dp_ctx *c;
        Fr *s;
        ~SlotGuard() { p2p_release_slot(c, s); }
    } slot_guard{ctx, slot};
    PeerCounters pc;
    for (uint64_t q = 0; q < 8; q++) pc.c[q] = q < W ? reinterpret_cast<uint32_t *>(ctx->peer_arena[q]) : nullptr;
    ctx->bar_seq++;
    DP_LAUNCH(p2p_barrier_kernel, dim3(1), dim3(32), 0, ctx->stream, pc, (uint32_t)W, (uint32_t)ctx->me, (uint32_t)(W * ctx->bar_seq));
    ctx->launches++;
    DP_TRY(plan_col_phase(ctx, d, slot, (Fr *)cols_dev, n_cols, ctx->me * n_cols, is_inv != 0, is_coset != 0));
    DP_TRY(call_end(ctx, wait));
    return wait ? p2p_check_timeout(ctx) : DP_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ rounds 3-5 ("next" row 1)
namespace {

// z^(2^j), j < RND_POW_TABLE, computed on the host and uploaded (80 squarings)
int upload_pow_table(dp_ctx *ctx, const Fr &z, Fr *pw_dev) {
    Fr host[RND_POW_TABLE];
    host[0] = z;
    for (int j = 1; j < RND_POW_TABLE; j++) host[j] = host[j - 1].sqr();
    DP_CUDA(ctx, cudaMemcpyAsync(pw_dev, host, sizeof host, cudaMemcpyHostToDevice, ctx->stream));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // `host` is a stack buffer
    return DP_OK;
}

// *out_dev = sum_k in[k] * (z^(2^e))^k
int poly_fold_device(dp_ctx *ctx, const Fr *in, uint64_t n, const Fr *pw, uint32_t e, Fr *out_dev) {
    Scratch tmp(ctx->pool);
    while (true) {
        const uint64_t nb = (n + RND_CHUNK - 1) / RND_CHUNK;
        Fr *dst = nb == 1 ? out_dev : tmp.get<Fr>(nb);
        if (!dst) return fail(ctx, DP_E_OOM, "poly fold scratch");
        DP_LAUNCH(poly_fold_kernel, dim3((unsigned)nb), dim3(RND_TPB), 0, ctx->stream, in, n, pw, e, dst);
        ctx->launches++;
        if (nb == 1) break;
        in = dst;
        n = nb;
        e += RND_LOG_CHUNK;
    }
    DP_CUDA(ctx, cudaGetLastError());
    return DP_OK;
}

// E_j = sum_{k >= j} in[k] * y^(k-j), y = z^(2^e); stored at out[j - shift]; E_0 -> *rem when shift = 1
int poly_suffix_device(dp_ctx *ctx, const Fr *in, uint64_t n, const Fr *pw, uint32_t e, Fr *out, uint32_t shift, Fr *rem) {
    const uint64_t nb = (n + RND_CHUNK - 1) / RND_CHUNK;
    Scratch tmp(ctx->pool);
    Fr *carry = nullptr;
    if (nb > 1) {
        Fr *tot = tmp.get<Fr>(nb);
        carry = tmp.get<Fr>(nb);
        if (!tot || !carry) return fail(ctx, DP_E_OOM, "poly suffix scratch");
        DP_LAUNCH(poly_fold_kernel, dim3((unsigned)nb), dim3(RND_TPB), 0, ctx->stream, in, n, pw, e, tot);
        ctx->launches++;
        DP_TRY(poly_suffix_device(ctx, tot, nb, pw, e + RND_LOG_CHUNK, carry, 0, nullptr));
    }
    DP_LAUNCH(poly_suffix_kernel, dim3((unsigned)nb), dim3(RND_TPB), 0, ctx->stream, in, n, pw, e, (const Fr *)carry, nb, out, shift, rem);
    ctx->launches++;
    DP_CUDA(ctx, cudaGetLastError());
    return DP_OK;
}

// slice < 0: the whole quotient coset (25 arrays of m points); else slice k of it (25 arrays of n points, DESIGN.md 3.4):
// points g * omega_m^(k + (m/n) i), written to out_dev[k + (m/n) i]
// tails (checked by quotient_tails_check, not all empty): the wires and z have more than n coefficients, the arrays hold the
// evaluations of their first n (QuotientTailArgs)
// scale (accumulating form, QuotientAcc): out_dev[pt] += scale * quotient(pt) instead of out_dev[pt] = quotient(pt)
int quotient_device(dp_ctx *ctx, const dp_quotient_args &a, const Fr *const *arrays /* 25 device arrays */, Fr *out_dev,
                    int slice = -1, const dp_quotient_tails *tails = nullptr, const Fr *scale = nullptr) {
    const DomainDev &dq = ctx->dom[1], &dg = ctx->dom[0];
    const uint64_t m = dq.n(), n = dg.n();
    if (m < n || m / n > RND_MAX_RATIO) return fail(ctx, DP_E_ARG, "quotient domain / gate domain = %llu, supported: 1..%d", (unsigned long long)(m / n), RND_MAX_RATIO);
    QuotientArgs q;
    for (int i = 0; i < 13; i++) q.sel[i] = arrays[i];
    for (int i = 0; i < 5; i++) q.sig[i] = arrays[13 + i];
    for (int i = 0; i < 5; i++) q.w[i] = arrays[18 + i];
    q.z = arrays[23];
    q.pi = arrays[24];
    Fr k[5];
    memcpy(k, a.k, sizeof k);
    memcpy(&q.alpha, a.alpha, sizeof(Fr));
    memcpy(&q.beta, a.beta, sizeof(Fr));
    memcpy(&q.gamma, a.gamma, sizeof(Fr));
    for (int i = 0; i < 5; i++) q.k_beta[i] = k[i] * q.beta;
    q.alpha_sq_div_n = q.alpha.sqr() * dg.n_inv;           // dispatcher2.rs:363
    q.gen = fr_from_u64(7);
    q.ratio = (uint32_t)(m / n);
    // 1 / Z_H(x_i), x_i = g omega_m^i, i < m/n: x_i^n = g^n (omega_m^n)^i   (dispatcher2.rs:372-379)
    const Fr gn = q.gen.pow(n), wn = fr_domain_gen(dq.log_n).pow(n);
    Fr cur = gn, xn[RND_MAX_RATIO];
    for (uint32_t i = 0; i < q.ratio; i++) {
        const Fr zh = cur - Fr::one();
        if (zh.is_zero()) return fail(ctx, DP_E_ARG, "Z_H vanishes on the quotient coset (domains %llu / %llu)", (unsigned long long)n, (unsigned long long)m);
        q.zh_inv[i] = zh.inverse();
        xn[i] = cur;
        cur = cur * wn;
    }
    for (uint32_t i = q.ratio; i < RND_MAX_RATIO; i++) q.zh_inv[i] = Fr::zero();
    if (slice >= (int)q.ratio) return fail(ctx, DP_E_ARG, "quotient slice %d of %u", slice, q.ratio);
    if (scale) {   // scale * (zh_inv (gate + alpha perm) + alpha^2/n (z - 1)/(x - 1)): both products take the scale
        for (uint32_t i = 0; i < q.ratio; i++) q.zh_inv[i] = q.zh_inv[i] * *scale;
        q.alpha_sq_div_n = q.alpha_sq_div_n * *scale;
    }
    q.H = dq.H;
    q.m = m;
    q.log_m = dq.log_n;
    q.out = out_dev;
    const QuotPts pts = slice < 0 ? QuotPts{m, 0, 1} : QuotPts{n, (uint32_t)slice, q.ratio};
    q.pts = pts.pts;
    q.first = pts.first;
    q.step = pts.step;
    q.z_next = slice < 0 ? q.ratio : 1;   // z(omega x): omega_n = omega_m^ratio, one step within a slice
    // all blocks' 1 / prod(x_i - 1) up front, one thread per block, instead of one serial inversion inside each block
    const unsigned n_blocks = blocks_for(pts.pts, QUO_TPB), m_blocks = blocks_for(m, QUO_TPB);
    Scratch tmp(ctx->pool);
    // the 1/(x_i - 1) are the same for every proof on this domain: keep them when the table fits
    bool want_table = ctx->quot_table == 1;
    if (ctx->quot_table < 0) {
        size_t free_b = 0, total_b = 0;
        cudaMemGetInfo(&free_b, &total_b);
        want_table = (ctx->quot_inv && ctx->quot_inv_log == dq.log_n) || m * sizeof(Fr) <= free_b / 8;
    }
    if (want_table && !(ctx->quot_inv && ctx->quot_inv_log == dq.log_n)) {
        ctx->pool.release(ctx->quot_inv);
        ctx->quot_inv = (Fr *)ctx->pool.alloc(m * sizeof(Fr));
        if (ctx->quot_inv) {   // (over the whole coset, whichever points this call covers)
            Fr *prod = tmp.get<Fr>(m_blocks);
            if (!prod) return fail(ctx, DP_E_OOM, "quotient scratch");
            DP_LAUNCH(quotient_xm1_products_kernel, dim3(m_blocks), dim3(QUO_TPB), 0, ctx->stream, q.gen, q.H, q.log_m, QuotPts{m, 0, 1}, prod);
            DP_LAUNCH(fr_invert_kernel, dim3(blocks_for(m_blocks, 128)), dim3(128), 0, ctx->stream, prod, (uint64_t)m_blocks);
            DP_LAUNCH(quotient_inv_table_kernel, dim3(m_blocks), dim3(QUO_TPB), 0, ctx->stream, q.gen, q.H, q.log_m, m, (const Fr *)prod,
                      ctx->quot_inv);
            ctx->launches += 3;
            ctx->quot_inv_log = dq.log_n;
        } else if (ctx->quot_table == 1) {
            return fail(ctx, DP_E_OOM, "quotient: table of 1/(x - 1) over 2^%u points", dq.log_n);
        }
    }
    q.prod_inv = nullptr;
    q.inv_xm1 = nullptr;
    // the same launches with either argument type: QuotientArgs, or QuotientTailArgs for blinded wires and z
    auto launch = [&](auto &args) -> int {
        using Args = std::decay_t<decltype(args)>;
        if (want_table && ctx->quot_inv) {
            args.inv_xm1 = ctx->quot_inv;
            const auto kernel = quotient_kernel<true, Args>;
            DP_LAUNCH(kernel, dim3(n_blocks), dim3(QUO_TPB), 0, ctx->stream, args);
            ctx->launches += 1;
        } else {
            Fr *prod = tmp.get<Fr>(n_blocks);
            if (!prod) return fail(ctx, DP_E_OOM, "quotient scratch");
            DP_LAUNCH(quotient_xm1_products_kernel, dim3(n_blocks), dim3(QUO_TPB), 0, ctx->stream, q.gen, q.H, q.log_m, pts, prod);
            DP_LAUNCH(fr_invert_kernel, dim3(blocks_for(n_blocks, 128)), dim3(128), 0, ctx->stream, prod, (uint64_t)n_blocks);
            args.prod_inv = prod;
            const auto kernel = quotient_kernel<false, Args>;
            DP_LAUNCH(kernel, dim3(n_blocks), dim3(QUO_TPB), 0, ctx->stream, args);
            ctx->launches += 3;
        }
        DP_CUDA(ctx, cudaGetLastError());
        return DP_OK;
    };
    if (!tails) {
        if (!scale) return launch(q);
        QuotientAcc<QuotientArgs> qa;
        static_cast<QuotientArgs &>(qa) = q;
        return launch(qa);
    }
    QuotientTailArgs qt;
    static_cast<QuotientArgs &>(qt) = q;
    for (int j = 0; j < 5; j++) {
        qt.w_tail[j] = (const Fr *)tails->wires[j];
        qt.w_tail_len[j] = (uint32_t)tails->wire_len[j];
    }
    qt.z_tail = (const Fr *)tails->perm;
    qt.z_tail_len = (uint32_t)tails->perm_len;
    for (uint32_t i = 0; i < RND_MAX_RATIO; i++) qt.xn[i] = i < q.ratio ? xn[i] : Fr::zero();
    qt.omega_n = fr_domain_gen(dg.log_n);
    if (!scale) return launch(qt);
    QuotientAcc<QuotientTailArgs> qta;
    static_cast<QuotientTailArgs &>(qta) = qt;
    return launch(qta);
}

const void *const *quotient_ptrs(const dp_quotient_args &a, const void *flat[25]) {
    for (int i = 0; i < 13; i++) flat[i] = a.selectors[i];
    for (int i = 0; i < 5; i++) flat[13 + i] = a.sigmas[i];
    for (int i = 0; i < 5; i++) flat[18 + i] = a.wires[i];
    flat[23] = a.perm;
    flat[24] = a.pub_input;
    return flat;
}

// DP_E_ARG for a tail longer than RND_MAX_TAIL, a NULL tail of nonzero length, or one that overlaps the m-entry output.
// *any = some tail is not empty.
int quotient_tails_check(dp_ctx *ctx, const dp_quotient_tails *t, const void *out, bool *any, const char *who) {
    if (!t) return fail(ctx, DP_E_ARG, "%s: NULL tails", who);
    const uint64_t m = ctx->dom[1].n();
    *any = false;
    for (int j = 0; j < 6; j++) {
        const void *p = j < 5 ? t->wires[j] : t->perm;
        const size_t len = j < 5 ? t->wire_len[j] : t->perm_len;
        if (len > RND_MAX_TAIL) return fail(ctx, DP_E_ARG, "%s: tail %d has %zu coefficients, at most %u", who, j, len, RND_MAX_TAIL);
        if (!len) continue;
        if (!p) return fail(ctx, DP_E_ARG, "%s: tail %d is NULL", who, j);
        if (ranges_overlap(p, len * sizeof(Fr), out, m * sizeof(Fr))) return fail(ctx, DP_E_ARG, "%s: the output overlaps tail %d", who, j);
        *any = true;
    }
    return DP_OK;
}

int quotient_check(dp_ctx *ctx, const dp_quotient_args *a, const void *out, const char *who) {
    if (!ctx || !a || !out) return fail(ctx, DP_E_ARG, "%s: NULL argument", who);
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "%s before dp_init", who);
    const void *flat[25];
    quotient_ptrs(*a, flat);
    for (int i = 0; i < 25; i++)
        if (!flat[i]) return fail(ctx, DP_E_ARG, "%s: polynomial %d is NULL", who, i);
    if (!a->k || !a->alpha || !a->beta || !a->gamma) return fail(ctx, DP_E_ARG, "%s: NULL challenge", who);
    return DP_OK;
}

}  // namespace

extern "C" {

int dp_quotient_evals(dp_ctx *ctx, const dp_quotient_args *a, void *out) {
    DP_TRY(quotient_check(ctx, a, out, "dp_quotient_evals"));
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    const uint64_t m = ctx->dom[1].n();
    const void *flat[25];
    quotient_ptrs(*a, flat);
    Scratch tmp(ctx->pool);
    const Fr *dev[25];
    for (int i = 0; i < 25; i++) {
        Fr *d = tmp.get<Fr>(m);
        if (!d) return fail(ctx, DP_E_OOM, "dp_quotient_evals: 26 x %llu B of device memory", (unsigned long long)(m * sizeof(Fr)));
        DP_CUDA(ctx, cudaMemcpyAsync(d, flat[i], m * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
        dev[i] = d;
    }
    Fr *o = tmp.get<Fr>(m);
    if (!o) return fail(ctx, DP_E_OOM, "dp_quotient_evals output");
    DP_TRY(quotient_device(ctx, *a, dev, o));
    DP_CUDA(ctx, cudaMemcpyAsync(out, o, m * sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

int dp_quotient_evals_dev(dp_ctx *ctx, const dp_quotient_args *a, void *out_dev) {
    DP_TRY(quotient_check(ctx, a, out_dev, "dp_quotient_evals_dev"));
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    const void *flat[25];
    quotient_ptrs(*a, flat);
    DP_TRY(quotient_device(ctx, *a, reinterpret_cast<const Fr *const *>(flat), (Fr *)out_dev));
    return call_end(ctx, true);
}

int dp_quotient_evals_tail_dev(dp_ctx *ctx, const dp_quotient_args *a, const dp_quotient_tails *tails, void *out_dev) {
    DP_TRY(quotient_check(ctx, a, out_dev, "dp_quotient_evals_tail_dev"));
    bool any = false;
    DP_TRY(quotient_tails_check(ctx, tails, out_dev, &any, "dp_quotient_evals_tail_dev"));
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    const void *flat[25];
    quotient_ptrs(*a, flat);
    DP_TRY(quotient_device(ctx, *a, reinterpret_cast<const Fr *const *>(flat), (Fr *)out_dev, -1, any ? tails : nullptr));
    return call_end(ctx, true);
}

static int quotient_slice_any(dp_ctx *ctx, const dp_quotient_args *slice_arrays, const dp_quotient_tails *tails, uint32_t slice,
                              void *out_dev, const char *who) {
    DP_TRY(quotient_check(ctx, slice_arrays, out_dev, who));
    bool any = false;
    if (tails) DP_TRY(quotient_tails_check(ctx, tails, out_dev, &any, who));
    const DomainDev &dg = ctx->dom[0], &dq = ctx->dom[1];
    const uint64_t n = dg.n(), m = dq.n();
    if (m < n || slice >= m / n) return fail(ctx, DP_E_ARG, "%s: slice %u of %llu", who, slice, (unsigned long long)(m < n ? 0 : m / n));
    const void *flat[25];
    quotient_ptrs(*slice_arrays, flat);
    for (int i = 0; i < 25; i++)
        if (ranges_overlap(flat[i], n * sizeof(Fr), out_dev, m * sizeof(Fr)))
            return fail(ctx, DP_E_ARG, "%s: the output overlaps input %d", who, i);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    DP_TRY(quotient_device(ctx, *slice_arrays, reinterpret_cast<const Fr *const *>(flat), (Fr *)out_dev, (int)slice, any ? tails : nullptr));
    return call_end(ctx, true);
}

int dp_quotient_evals_slice_dev(dp_ctx *ctx, const dp_quotient_args *slice_arrays, uint32_t slice, void *out_dev) {
    return quotient_slice_any(ctx, slice_arrays, nullptr, slice, out_dev, "dp_quotient_evals_slice_dev");
}

int dp_quotient_evals_slice_tail_dev(dp_ctx *ctx, const dp_quotient_args *slice_arrays, const dp_quotient_tails *tails, uint32_t slice,
                                     void *out_dev) {
    if (!tails) return fail(ctx, DP_E_ARG, "dp_quotient_evals_slice_tail_dev: NULL tails");
    return quotient_slice_any(ctx, slice_arrays, tails, slice, out_dev, "dp_quotient_evals_slice_tail_dev");
}

// the accumulating entries: slice < 0 = the whole coset (25 arrays of m points), else one slice (25 arrays of n points)
static int quotient_acc_any(dp_ctx *ctx, const dp_quotient_args *arrays, const dp_quotient_tails *tails, int slice, const void *scale32,
                            void *out_dev, const char *who) {
    DP_TRY(quotient_check(ctx, arrays, out_dev, who));
    if (!scale32) return fail(ctx, DP_E_ARG, "%s: NULL scale", who);
    Fr scale;
    memcpy(&scale, scale32, sizeof scale);
    if (!scale.canon_is_reduced()) return fail(ctx, DP_E_ARG, "%s: the scale is not below r", who);
    bool any = false;
    if (tails) DP_TRY(quotient_tails_check(ctx, tails, out_dev, &any, who));
    const DomainDev &dg = ctx->dom[0], &dq = ctx->dom[1];
    const uint64_t n = dg.n(), m = dq.n();
    if (slice >= 0 && (m < n || (uint64_t)slice >= m / n))
        return fail(ctx, DP_E_ARG, "%s: slice %d of %llu", who, slice, (unsigned long long)(m < n ? 0 : m / n));
    const uint64_t in_len = slice < 0 ? m : n;
    const void *flat[25];
    quotient_ptrs(*arrays, flat);
    for (int i = 0; i < 25; i++)   // the output is read as well as written: no input may share its memory
        if (ranges_overlap(flat[i], in_len * sizeof(Fr), out_dev, m * sizeof(Fr)))
            return fail(ctx, DP_E_ARG, "%s: the output overlaps input %d", who, i);
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    DP_TRY(quotient_device(ctx, *arrays, reinterpret_cast<const Fr *const *>(flat), (Fr *)out_dev, slice, any ? tails : nullptr, &scale));
    return call_end(ctx, true);
}

int dp_quotient_evals_acc_dev(dp_ctx *ctx, const dp_quotient_args *dev_arrays, const dp_quotient_tails *tails, const void *scale32,
                              void *out_dev) {
    return quotient_acc_any(ctx, dev_arrays, tails, -1, scale32, out_dev, "dp_quotient_evals_acc_dev");
}

int dp_quotient_evals_slice_acc_dev(dp_ctx *ctx, const dp_quotient_args *slice_arrays, const dp_quotient_tails *tails, uint32_t slice,
                                    const void *scale32, void *out_dev) {
    if (slice > (uint32_t)RND_MAX_RATIO) return fail(ctx, DP_E_ARG, "dp_quotient_evals_slice_acc_dev: slice %u", slice);
    return quotient_acc_any(ctx, slice_arrays, tails, (int)slice, scale32, out_dev, "dp_quotient_evals_slice_acc_dev");
}

static int poly_eval_any(dp_ctx *ctx, const void *coeffs, size_t n, const void *point, void *out32, bool on_device, const char *who) {
    if (!ctx || !point || !out32 || (n && !coeffs)) return fail(ctx, DP_E_ARG, "%s: NULL argument", who);
    if (n == 0) {  // the zero polynomial
        memset(out32, 0, sizeof(Fr));
        return DP_OK;
    }
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    Fr *pw = tmp.get<Fr>(RND_POW_TABLE), *res = tmp.get<Fr>(1);
    const Fr *src = (const Fr *)coeffs;
    if (!on_device) {
        Fr *c = tmp.get<Fr>(n);
        if (!c) return fail(ctx, DP_E_OOM, "%s buffers", who);
        DP_CUDA(ctx, cudaMemcpyAsync(c, coeffs, n * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
        src = c;
    }
    if (!pw || !res) return fail(ctx, DP_E_OOM, "%s buffers", who);
    Fr z;
    memcpy(&z, point, sizeof z);
    DP_TRY(upload_pow_table(ctx, z, pw));
    DP_TRY(poly_fold_device(ctx, src, n, pw, 0, res));
    DP_CUDA(ctx, cudaMemcpyAsync(out32, res, sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}
int dp_poly_eval(dp_ctx *ctx, const void *coeffs, size_t n, const void *point, void *out32) {
    return poly_eval_any(ctx, coeffs, n, point, out32, false, "dp_poly_eval");
}
int dp_poly_eval_dev(dp_ctx *ctx, const void *coeffs_dev, size_t n, const void *point, void *out32) {
    return poly_eval_any(ctx, coeffs_dev, n, point, out32, true, "dp_poly_eval_dev");
}

static int poly_div_any(dp_ctx *ctx, const void *coeffs, size_t n, const void *point, void *out, void *rem32, bool on_device, const char *who) {
    if (!ctx || !point || (n && !coeffs) || (n > 1 && !out)) return fail(ctx, DP_E_ARG, "%s: NULL argument", who);
    if (n == 0) {
        if (rem32) memset(rem32, 0, sizeof(Fr));
        return DP_OK;
    }
    if (on_device && n > 1) {
        // blocks of poly_suffix_kernel read coefficients that other blocks' quotient stores may already have
        // replaced: the quotient cannot be written over (or into) the dividend
        const uintptr_t a0 = (uintptr_t)coeffs, a1 = a0 + n * sizeof(Fr), b0 = (uintptr_t)out, b1 = b0 + (n - 1) * sizeof(Fr);
        if (a0 < b1 && b0 < a1) return fail(ctx, DP_E_ARG, "%s: out_dev overlaps coeffs_dev (in-place division is not supported)", who);
    }
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    Fr *pw = tmp.get<Fr>(RND_POW_TABLE), *rem = tmp.get<Fr>(1);
    if (!pw || !rem) return fail(ctx, DP_E_OOM, "%s buffers", who);
    const Fr *src = (const Fr *)coeffs;
    Fr *dst = (Fr *)out;
    if (!on_device) {
        Fr *c = tmp.get<Fr>(n), *q = tmp.get<Fr>(n);
        if (!c || !q) return fail(ctx, DP_E_OOM, "%s buffers", who);
        DP_CUDA(ctx, cudaMemcpyAsync(c, coeffs, n * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
        src = c;
        dst = q;
    }
    Fr z;
    memcpy(&z, point, sizeof z);
    DP_TRY(upload_pow_table(ctx, z, pw));
    DP_TRY(poly_suffix_device(ctx, src, n, pw, 0, dst, 1, rem));
    if (!on_device && n > 1) DP_CUDA(ctx, cudaMemcpyAsync(out, dst, (n - 1) * sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
    if (rem32) DP_CUDA(ctx, cudaMemcpyAsync(rem32, rem, sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}
int dp_poly_div_linear(dp_ctx *ctx, const void *coeffs, size_t n, const void *point, void *out, void *rem32) {
    return poly_div_any(ctx, coeffs, n, point, out, rem32, false, "dp_poly_div_linear");
}
int dp_poly_div_linear_dev(dp_ctx *ctx, const void *coeffs_dev, size_t n, const void *point, void *out_dev, void *rem32) {
    return poly_div_any(ctx, coeffs_dev, n, point, out_dev, rem32, true, "dp_poly_div_linear_dev");
}

static int poly_lincomb_any(dp_ctx *ctx, const void *const *polys, const size_t *lens, const void *coeffs, size_t k, void *out, size_t out_len,
                            bool on_device, const char *who) {
    if (!ctx || !polys || !lens || !coeffs || (out_len && !out)) return fail(ctx, DP_E_ARG, "%s: NULL argument", who);
    if (k == 0 || k > RND_MAX_POLYS) return fail(ctx, DP_E_ARG, "%s: %zu polynomials (1..%d)", who, k, RND_MAX_POLYS);
    if (out_len == 0) return DP_OK;
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    LincombArgs a;
    memset(&a, 0, sizeof a);
    a.k = (uint32_t)k;
    a.out_len = out_len;
    memcpy(a.coeff, coeffs, k * sizeof(Fr));
    for (size_t i = 0; i < k; i++) {
        a.len[i] = lens[i] < out_len ? lens[i] : out_len;
        if (a.len[i] && !polys[i]) return fail(ctx, DP_E_ARG, "%s: polynomial %zu is NULL", who, i);
        if (on_device || a.len[i] == 0) {
            a.poly[i] = (const Fr *)polys[i];
        } else {
            Fr *d = tmp.get<Fr>(a.len[i]);
            if (!d) return fail(ctx, DP_E_OOM, "%s buffers", who);
            DP_CUDA(ctx, cudaMemcpyAsync(d, polys[i], a.len[i] * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
            a.poly[i] = d;
        }
    }
    Fr *dst = on_device ? (Fr *)out : tmp.get<Fr>(out_len);
    if (!dst) return fail(ctx, DP_E_OOM, "%s buffers", who);
    a.out = dst;
    DP_LAUNCH(poly_lincomb_kernel, dim3(blocks_for(out_len, 256)), dim3(256), 0, ctx->stream, a);
    ctx->launches++;
    DP_CUDA(ctx, cudaGetLastError());
    if (!on_device) DP_CUDA(ctx, cudaMemcpyAsync(out, dst, out_len * sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}
int dp_poly_lincomb(dp_ctx *ctx, const void *const *polys, const size_t *lens, const void *coeffs, size_t k, void *out, size_t out_len) {
    return poly_lincomb_any(ctx, polys, lens, coeffs, k, out, out_len, false, "dp_poly_lincomb");
}
int dp_poly_lincomb_dev(dp_ctx *ctx, const void *const *polys_dev, const size_t *lens, const void *coeffs, size_t k, void *out_dev, size_t out_len) {
    return poly_lincomb_any(ctx, polys_dev, lens, coeffs, k, out_dev, out_len, true, "dp_poly_lincomb_dev");
}

// ------------------------------------------------------------------ worker-resident polynomials
// What `state.wire` is in the reference (worker.rs:58,400-405), generalised: named device buffers
// that the *_dev entries of rounds 2-5, dp_ntt_dev and dp_commit_dev work on, so that a polynomial
// crosses PCIe once (or never).  All copies and kernels touching them run on the compute stream.
int dp_poly_put(dp_ctx *ctx, uint64_t poly_id, const void *coeffs, size_t n, size_t capacity) {
    if (!ctx || (n && !coeffs)) return fail(ctx, DP_E_ARG, "dp_poly_put: NULL argument");
    if (capacity < n) capacity = n;
    if (capacity == 0) return fail(ctx, DP_E_ARG, "dp_poly_put: empty polynomial");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    dp_ctx::Poly &p = ctx->polys[poly_id];
    if (p.cap != capacity) {  // (re)allocate; stream-ordered pool: earlier kernels on the old buffer are ordered before its reuse
        ctx->pool.release(p.dev);
        p.dev = (Fr *)ctx->pool.alloc(capacity * sizeof(Fr));
        p.cap = p.dev ? capacity : 0;
        if (!p.dev) {
            ctx->polys.erase(poly_id);
            return fail(ctx, DP_E_OOM, "dp_poly_put: %zu coefficients", capacity);
        }
    }
    if (n) DP_CUDA(ctx, cudaMemcpyAsync(p.dev, coeffs, n * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    if (capacity > n) DP_CUDA(ctx, cudaMemsetAsync(p.dev + n, 0, (capacity - n) * sizeof(Fr), ctx->stream));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // `coeffs` is the caller's again
    return DP_OK;
}

int dp_poly_ptr(dp_ctx *ctx, uint64_t poly_id, void **dev, size_t *capacity) {
    if (!ctx) return DP_E_ARG;
    auto it = ctx->polys.find(poly_id);
    if (it == ctx->polys.end()) return fail(ctx, DP_E_ARG, "dp_poly_ptr: unknown polynomial %llu", (unsigned long long)poly_id);
    if (dev) *dev = it->second.dev;
    if (capacity) *capacity = it->second.cap;
    return DP_OK;
}

int dp_poly_get(dp_ctx *ctx, uint64_t poly_id, size_t offset, size_t n, void *out) {
    if (!ctx || (n && !out)) return fail(ctx, DP_E_ARG, "dp_poly_get: NULL argument");
    auto it = ctx->polys.find(poly_id);
    if (it == ctx->polys.end()) return fail(ctx, DP_E_ARG, "dp_poly_get: unknown polynomial %llu", (unsigned long long)poly_id);
    if (offset > it->second.cap || n > it->second.cap - offset) return fail(ctx, DP_E_ARG, "dp_poly_get: [%zu, +%zu) outside %zu coefficients", offset, n, it->second.cap);
    if (n == 0) return DP_OK;
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    DP_CUDA(ctx, cudaMemcpyAsync(out, it->second.dev + offset, n * sizeof(Fr), cudaMemcpyDeviceToHost, ctx->stream));
    DP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return DP_OK;
}

int dp_poly_free(dp_ctx *ctx, uint64_t poly_id) {
    if (!ctx) return DP_E_ARG;
    auto it = ctx->polys.find(poly_id);
    if (it == ctx->polys.end()) return fail(ctx, DP_E_ARG, "dp_poly_free: unknown polynomial %llu", (unsigned long long)poly_id);
    ctx->pool.release(it->second.dev);
    ctx->polys.erase(it);
    return DP_OK;
}

// commit_polynomial (worker.rs:117-123) of coefficients that already live on the device
int dp_commit_dev(dp_ctx *ctx, const void *coeffs_dev, size_t n, void *out144) {
    if (!ctx || !out144 || (n && !coeffs_dev)) return fail(ctx, DP_E_ARG, "dp_commit_dev: NULL argument");
    if (!ctx->inited) return fail(ctx, DP_E_STATE, "dp_commit_dev before dp_init");
    DP_CUDA(ctx, cudaSetDevice(ctx->device));
    call_begin(ctx);
    Scratch tmp(ctx->pool);
    G1JacobianOut *od = tmp.get<G1JacobianOut>(1);
    if (!od) return fail(ctx, DP_E_OOM, "dp_commit_dev buffers");
    DP_TRY(commit_device(ctx, (const Fr *)coeffs_dev, n, od));
    DP_CUDA(ctx, cudaMemcpyAsync(out144, od, sizeof(G1JacobianOut), cudaMemcpyDeviceToHost, ctx->stream));
    return call_end(ctx, true);
}

}  // extern "C"
