// Batched-affine tree level, second attempt (DESIGN.md section 7): serial prefix products per thread instead of a
// product tree over single pairs.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -o tools/microbench6 tools/microbench6.cu
//   ./tools/microbench6 [log2 pairs, default 24]
// tools/microbench4.cu (round 2) measured one level of P_k + Q_k with a 256-leaf product tree over 2 pairs per thread:
// 1.69x SLOWER than the XYZZ mixed addition, because the tree levels run with mostly idle warps (36 warp-products per
// 512 pairs = 2.25 lane-products per pair on top of the 6 useful ones) and sit behind 16 block barriers.  Here a thread
// chains KP pairs (Montgomery's trick inside the thread: 1 product per pair on the way up, 2 on the way down), so the
// tree over the 128 thread totals costs 36*32/(128*KP) = 9/KP lane-products per pair:
//   K1  d = x2 - x1, prefix products -> global (48 B per pair), thread totals -> block tree -> root[b]   (1 + 3/KP)
//   K2  root[b] <- 1/root[b]: Fermat (inverse) or binary Euclid per lane (inverse_vartime), both timed
//   K3  thread total again (1 product), tree up + down (9/KP), then per pair 2 + 3 products             (5 + 10/KP)
// = 6.4 products per addition at KP = 16 against 10 for the XYZZ mixed addition.  Operands: (a) gathered at random from
// a 384 MiB table, as the first level gathers window multiples; (b) contiguous pairs (in[2q], in[2q+1]), as the later
// levels read the previous level's output.  Prints the times next to the XYZZ mixed addition on the same operands and
// checks every result against it.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include "../distributed_plonk_b200/csrc/g1.cuh"
using namespace dp;

constexpr int TPB = 128;

#define CK(x)                                                                      \
    do {                                                                           \
        cudaError_t e_ = (x);                                                      \
        if (e_ != cudaSuccess) {                                                   \
            printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); \
            exit(1);                                                               \
        }                                                                          \
    } while (0)

__device__ inline G1Affine ld_affine(const G1Affine *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    G1Affine r;
    uint32_t *w = reinterpret_cast<uint32_t *>(&r);
#pragma unroll
    for (int k = 0; k < 6; k++) {
        const uint4 v = q[k];
        w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
    }
    return r;
}
__device__ inline Fq ld_fq(const Fq *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    Fq r;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const uint4 v = q[k];
        r.l[4 * k] = v.x; r.l[4 * k + 1] = v.y; r.l[4 * k + 2] = v.z; r.l[4 * k + 3] = v.w;
    }
    return r;
}
__device__ inline void st_fq(Fq *p, const Fq &v) {
    uint4 *q = reinterpret_cast<uint4 *>(p);
#pragma unroll
    for (int k = 0; k < 3; k++) q[k] = make_uint4(v.l[4 * k], v.l[4 * k + 1], v.l[4 * k + 2], v.l[4 * k + 3]);
}
__device__ inline void st_affine(G1Affine *p, const G1Affine &v) {
    st_fq(&p->x, v.x);
    st_fq(&p->y, v.y);
}

// table[i] = (i + 1) * G, distinct points
__global__ void gen_table(G1Affine *table, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t gx[12] = {0xfd530c16u, 0x5cb38790u, 0x9976fff5u, 0x7817fc67u, 0x143ba1c1u, 0x154f95c7u,
                             0xf3d0e747u, 0xf0ae6acdu, 0x21dbf440u, 0xedce6eccu, 0x9e0bfb75u, 0x12017741u};
    const uint32_t gy[12] = {0x0ce72271u, 0xbaac93d5u, 0x7918fd8eu, 0x8c22631au, 0x570725ceu, 0xdd595f13u,
                             0x50405194u, 0x51ac5829u, 0xad0059c0u, 0x0e1c8c3fu, 0x5008a26au, 0x0bbc3efcu};
    G1Affine g;
    for (int k = 0; k < 12; k++) {
        g.x.l[k] = gx[k];
        g.y.l[k] = gy[k];
    }
    G1XYZZ acc = G1XYZZ::inf();
    const uint32_t s = i + 1;
    for (int b = 31; b >= 0; b--) {
        acc = acc.dbl();
        if ((s >> b) & 1) acc = acc.add_mixed(g);
    }
    table[i] = acc.to_affine();
}

// operand indices of pair k: GATHER = pseudo-random distinct table entries, else the contiguous pair (2k, 2k+1) mod table
template <bool GATHER>
__device__ inline void operands(uint64_t k, uint32_t table_n, uint32_t &ip, uint32_t &iq) {
    if (GATHER) {
        uint64_t z = (k + 1) * 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z ^= z >> 27;
        ip = (uint32_t)(z % table_n);
        iq = (uint32_t)((ip + 1 + (z >> 32) % (table_n - 1)) % table_n);
    } else {
        ip = (uint32_t)((2 * k) % table_n);
        iq = ip + 1;
    }
}

// product of the 128 thread totals: tree[1]; leaves at tree[TPB + t]
__device__ inline void tree_up(Fq *tree, const Fq &mine) {
    const uint32_t t = threadIdx.x;
    tree[TPB + t] = mine;
    __syncthreads();
    for (uint32_t s = TPB >> 1; s >= 1; s >>= 1) {
        if (t < s) tree[s + t] = tree[2 * (s + t)] * tree[2 * (s + t) + 1];
        __syncthreads();
    }
}

template <int KP, bool GATHER>
__global__ void __launch_bounds__(TPB) k1_prefix(const G1Affine *table, uint32_t table_n, uint64_t m, Fq *pre, Fq *root) {
    __shared__ Fq tree[2 * TPB];
    const uint32_t t = threadIdx.x;
    Fq run = Fq::one();
    for (int j = 0; j < KP; j++) {
        const uint64_t k = ((uint64_t)blockIdx.x * KP + j) * TPB + t;
        if (k < m) {
            uint32_t ip, iq;
            operands<GATHER>(k, table_n, ip, iq);
            st_fq(pre + k, run);  // product of this thread's earlier denominators
            run = run * (ld_fq(&table[iq].x) - ld_fq(&table[ip].x));
        }
    }
    tree_up(tree, run);
    if (t == 0) st_fq(root + blockIdx.x, tree[1]);
}

__global__ void k2_invert_fermat(const Fq *root, Fq *inv, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) inv[i] = root[i].inverse();
}
__global__ void k2_invert_euclid(const Fq *root, Fq *inv, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) inv[i] = root[i].inverse_vartime();
}

template <int KP, bool GATHER>
__global__ void __launch_bounds__(TPB) k3_finish(const G1Affine *table, uint32_t table_n, uint64_t m, const Fq *pre, const Fq *root_inv,
                                                 G1Affine *out) {
    __shared__ Fq tree[2 * TPB];
    const uint32_t t = threadIdx.x;
    // this thread's total again: prefix of its last pair times that pair's denominator
    int last = -1;
    for (int j = KP - 1; j >= 0 && last < 0; j--)
        if (((uint64_t)blockIdx.x * KP + j) * TPB + t < m) last = j;
    Fq total = Fq::one();
    if (last >= 0) {
        const uint64_t k = ((uint64_t)blockIdx.x * KP + last) * TPB + t;
        uint32_t ip, iq;
        operands<GATHER>(k, table_n, ip, iq);
        total = ld_fq(pre + k) * (ld_fq(&table[iq].x) - ld_fq(&table[ip].x));
    }
    tree_up(tree, total);
    if (t == 0) tree[1] = ld_fq(root_inv + blockIdx.x);
    __syncthreads();
    for (uint32_t s = 1; s < TPB; s <<= 1) {
        if (t < s) {
            const uint32_t node = s + t;
            const Fq iv = tree[node], l = tree[2 * node], r = tree[2 * node + 1];
            tree[2 * node] = iv * r;
            tree[2 * node + 1] = iv * l;
        }
        __syncthreads();
    }
    Fq inv_run = tree[TPB + t];  // 1 / (product of this thread's denominators)
    for (int j = last; j >= 0; j--) {
        const uint64_t k = ((uint64_t)blockIdx.x * KP + j) * TPB + t;
        uint32_t ip, iq;
        operands<GATHER>(k, table_n, ip, iq);
        const G1Affine a = ld_affine(table + ip), b = ld_affine(table + iq);
        const Fq d = b.x - a.x;
        const Fq inv_d = inv_run * ld_fq(pre + k);
        inv_run = inv_run * d;
        const Fq lambda = (b.y - a.y) * inv_d;
        G1Affine r;
        r.x = lambda.sqr() - a.x - b.x;
        r.y = lambda * (a.x - r.x) - a.y;
        st_affine(out + k, r);
    }
}

template <bool GATHER>
__global__ void __launch_bounds__(TPB) k_xyzz(const G1Affine *table, uint32_t table_n, uint64_t m, G1XYZZ *out) {
    const uint64_t k = (uint64_t)blockIdx.x * TPB + threadIdx.x;
    if (k >= m) return;
    uint32_t ip, iq;
    operands<GATHER>(k, table_n, ip, iq);
    out[k] = G1XYZZ::from_affine(ld_affine(table + ip)).add_mixed(ld_affine(table + iq));
}

__global__ void k_compare(const G1Affine *a, const G1XYZZ *b, uint64_t m, uint32_t *bad) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= m) return;
    const G1Affine r = b[k].to_affine();
    if (r.x != a[k].x || r.y != a[k].y) atomicAdd(bad, 1u);
}

struct Bufs {
    G1Affine *table, *out;
    G1XYZZ *out_x;
    Fq *pre, *root, *inv;
    uint32_t *bad;
    uint32_t table_n;
    uint64_t m;
    cudaEvent_t e0, e1;
};

template <class F>
static float timed(Bufs &B, F launch, int reps = 3) {
    float sum = 0;
    for (int rep = 0; rep <= reps; rep++) {  // first repetition = warm-up
        float t;
        cudaEventRecord(B.e0);
        launch();
        cudaEventRecord(B.e1);
        CK(cudaEventSynchronize(B.e1));
        cudaEventElapsedTime(&t, B.e0, B.e1);
        if (rep) sum += t / reps;
    }
    CK(cudaGetLastError());
    return sum;
}

template <int KP, bool GATHER>
static void run(Bufs &B, float ms_xyzz) {
    const uint64_t m = B.m;
    const uint32_t n_blocks = (uint32_t)((m + (uint64_t)TPB * KP - 1) / ((uint64_t)TPB * KP));
    const float t1 = timed(B, [&] { k1_prefix<KP, GATHER><<<n_blocks, TPB>>>(B.table, B.table_n, m, B.pre, B.root); });
    const float t2f = timed(B, [&] { k2_invert_fermat<<<(n_blocks + 127) / 128, 128>>>(B.root, B.inv, n_blocks); });
    const float t2e = timed(B, [&] { k2_invert_euclid<<<(n_blocks + 31) / 32, 32>>>(B.root, B.inv, n_blocks); });
    const float t3 = timed(B, [&] { k3_finish<KP, GATHER><<<n_blocks, TPB>>>(B.table, B.table_n, m, B.pre, B.inv, B.out); });
    CK(cudaMemset(B.bad, 0, 4));
    k_compare<<<(unsigned)((m + 255) / 256), 256>>>(B.out, B.out_x, m, B.bad);
    uint32_t h_bad = 0;
    CK(cudaMemcpy(&h_bad, B.bad, 4, cudaMemcpyDeviceToHost));
    const float k2 = t2f < t2e ? t2f : t2e, total = t1 + k2 + t3;
    printf("%s KP=%2d (%u roots): K1 %.3f + K2 %.3f (Fermat %.3f / Euclid per lane %.3f) + K3 %.3f = %.3f ms -> %.2f G additions/s, "
           "ratio to XYZZ %.2f, mismatches %u\n",
           GATHER ? "gathered  " : "contiguous", KP, n_blocks, t1, k2, t2f, t2e, t3, total, m / (total * 1e-3) / 1e9, total / ms_xyzz, h_bad);
    fflush(stdout);
}

template <bool GATHER>
static void suite(Bufs &B) {
    const uint64_t m = B.m;
    const float ms_x = timed(B, [&] { k_xyzz<GATHER><<<(unsigned)((m + TPB - 1) / TPB), TPB>>>(B.table, B.table_n, m, B.out_x); });
    printf("%s XYZZ mixed addition (one kernel, 10 products): %.3f ms -> %.2f G additions/s\n", GATHER ? "gathered  " : "contiguous", ms_x,
           m / (ms_x * 1e-3) / 1e9);
    run<4, GATHER>(B, ms_x);
    run<8, GATHER>(B, ms_x);
    run<16, GATHER>(B, ms_x);
}

int main(int argc, char **argv) {
    const int log_m = argc > 1 ? atoi(argv[1]) : 24;
    Bufs B;
    B.m = 1ull << log_m;
    B.table_n = 1u << 22;  // 384 MiB of points: well beyond L2, like the real window-multiple table
    const uint64_t m = B.m;
    CK(cudaMalloc(&B.table, (size_t)B.table_n * sizeof(G1Affine)));
    CK(cudaMalloc(&B.out, m * sizeof(G1Affine)));
    CK(cudaMalloc(&B.out_x, m * sizeof(G1XYZZ)));
    CK(cudaMalloc(&B.pre, m * sizeof(Fq)));
    CK(cudaMalloc(&B.root, (m / (TPB * 4) + 1) * sizeof(Fq)));
    CK(cudaMalloc(&B.inv, (m / (TPB * 4) + 1) * sizeof(Fq)));
    CK(cudaMalloc(&B.bad, 4));
    gen_table<<<(B.table_n + 127) / 128, 128>>>(B.table, B.table_n);
    CK(cudaDeviceSynchronize());
    cudaEventCreate(&B.e0);
    cudaEventCreate(&B.e1);
    printf("additions per level: 2^%d, %d threads per block, KP pairs per thread\n", log_m, TPB);
    suite<true>(B);
    suite<false>(B);
    return 0;
}
