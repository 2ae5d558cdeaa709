// Feasibility microbenchmark for batched-affine bucket accumulation (DESIGN.md §7, planned for round 2).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -o tools/microbench4 tools/microbench4.cu
//   ./tools/microbench4 [log2 pairs, default 24]
//
// One tree level of a batched-affine reduction = M independent affine additions P_k + Q_k sharing field
// inversions.  An inversion (x^(p-2): ~570 multiplications, strictly serial) inside a block would idle the
// block for ~80 us, so a level is three kernels, the shape the quotient kernel already uses for 1/(x-1):
//   K1  d_k = x(Q_k) - x(P_k), product tree per block -> root[b]                      (1 mul / addition)
//   K2  root[b] <- 1 / root[b], one thread per block                                  (~570 mul / 1024 additions)
//   K3  rebuild the tree, push the inverse down, lambda = (y2 - y1)/d, x3, y3          (1 + 2 + 3 mul / addition)
// = ~7.6 Fq multiplications per addition against 10 for the XYZZ mixed addition msm_accumulate uses today
// (2.81 G additions/s measured), at the price of two passes over the operands and an output array.
// Operands are gathered at random from a table (as the bucket method gathers bases), results are written
// contiguously.  Prints additions/s for the three-kernel level and for the XYZZ mixed addition on the same
// operands, and checks the two against each other.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include "../distributed_plonk_b200/csrc/g1.cuh"
using namespace dp;

constexpr int TPB = 256;
constexpr int PAIRS = 2;  // additions per thread and level (x1, d and the prefix product of each stay in registers)

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

// table[i] = (i + 1) * G, distinct points
__global__ void gen_table(G1Affine *table, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    // generator, Montgomery form (same constants as msm.cuh:g1_generator)
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

// pseudo-random operand indices; P and Q never equal (so no doubling / cancellation in this benchmark)
__device__ inline void operands(uint64_t k, uint32_t table_n, uint32_t &ip, uint32_t &iq) {
    uint64_t z = (k + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27;
    ip = (uint32_t)(z % table_n);
    iq = (uint32_t)((ip + 1 + (z >> 32) % (table_n - 1)) % table_n);
}

__global__ void __launch_bounds__(TPB) k1_denominators(const G1Affine *table, uint32_t table_n, uint64_t m, Fq *root) {
    __shared__ Fq sh[TPB];
    const uint32_t t = threadIdx.x;
    Fq prod = Fq::one();
    for (int j = 0; j < PAIRS; j++) {
        const uint64_t k = ((uint64_t)blockIdx.x * PAIRS + j) * TPB + t;
        if (k < m) {
            uint32_t ip, iq;
            operands(k, table_n, ip, iq);
            prod = prod * (table[iq].x - table[ip].x);
        }
    }
    sh[t] = prod;
    __syncthreads();
    for (uint32_t s = TPB >> 1; s >= 1; s >>= 1) {
        if (t < s) sh[t] = sh[t] * sh[t + s];
        __syncthreads();
    }
    if (t == 0) root[blockIdx.x] = sh[0];
}

__global__ void k2_invert(Fq *root, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) root[i] = root[i].inverse();
}

__global__ void __launch_bounds__(TPB) k3_finish(const G1Affine *table, uint32_t table_n, uint64_t m, const Fq *root_inv, G1Affine *out) {
    __shared__ Fq tree[2 * TPB];
    const uint32_t t = threadIdx.x;
    Fq x1[PAIRS], d[PAIRS], pre[PAIRS];  // x(P), denominators and the thread's exclusive prefix products
    Fq prod = Fq::one();
    for (int j = 0; j < PAIRS; j++) {
        const uint64_t k = ((uint64_t)blockIdx.x * PAIRS + j) * TPB + t;
        d[j] = Fq::one();
        x1[j] = Fq::zero();
        if (k < m) {
            uint32_t ip, iq;
            operands(k, table_n, ip, iq);
            x1[j] = table[ip].x;
            d[j] = table[iq].x - x1[j];
        }
        pre[j] = prod;
        prod = prod * d[j];
    }
    tree[TPB + t] = prod;
    __syncthreads();
    for (uint32_t s = TPB >> 1; s >= 1; s >>= 1) {
        if (t < s) tree[s + t] = tree[2 * (s + t)] * tree[2 * (s + t) + 1];
        __syncthreads();
    }
    if (t == 0) tree[1] = root_inv[blockIdx.x];
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
    Fq inv_suffix = tree[TPB + t];  // 1 / (d_0 ... d_{PAIRS-1}) of this thread
    for (int j = PAIRS - 1; j >= 0; j--) {
        const uint64_t k = ((uint64_t)blockIdx.x * PAIRS + j) * TPB + t;
        const Fq inv_d = inv_suffix * pre[j];
        inv_suffix = inv_suffix * d[j];
        if (k < m) {  // the y coordinates are fetched only now (second touch of the operands: L2 / DRAM)
            uint32_t ip, iq;
            operands(k, table_n, ip, iq);
            const Fq y1 = table[ip].y;
            const Fq lambda = (table[iq].y - y1) * inv_d;
            G1Affine r;
            r.x = lambda.sqr() - x1[j].dbl() - d[j];  // lambda^2 - x1 - x2, x2 = x1 + d
            r.y = lambda * (x1[j] - r.x) - y1;
            out[k] = r;
        }
    }
}

// the same additions with the formula msm_accumulate uses (result left in XYZZ, as the buckets are)
__global__ void __launch_bounds__(TPB) k_xyzz(const G1Affine *table, uint32_t table_n, uint64_t m, G1XYZZ *out) {
    const uint64_t k = (uint64_t)blockIdx.x * TPB + threadIdx.x;
    if (k >= m) return;
    uint32_t ip, iq;
    operands(k, table_n, ip, iq);
    out[k] = G1XYZZ::from_affine(ld_affine(table + ip)).add_mixed(ld_affine(table + iq));
}

__global__ void k_compare(const G1Affine *a, const G1XYZZ *b, uint64_t m, uint32_t *bad) {
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= m) return;
    const G1Affine r = b[k].to_affine();
    if (r.x != a[k].x || r.y != a[k].y) atomicAdd(bad, 1u);
}

int main(int argc, char **argv) {
    const int log_m = argc > 1 ? atoi(argv[1]) : 24;
    const uint64_t m = 1ull << log_m;
    const uint32_t table_n = 1u << 22;  // 384 MiB of points: well beyond L2, like the real window-multiple table
    G1Affine *table, *out;
    G1XYZZ *out_x;
    Fq *root;
    uint32_t *bad;
    const uint32_t n_blocks = (uint32_t)((m + TPB * PAIRS - 1) / (TPB * PAIRS));
    CK(cudaMalloc(&table, (size_t)table_n * sizeof(G1Affine)));
    CK(cudaMalloc(&out, m * sizeof(G1Affine)));
    CK(cudaMalloc(&out_x, m * sizeof(G1XYZZ)));
    CK(cudaMalloc(&root, (size_t)n_blocks * sizeof(Fq)));
    CK(cudaMalloc(&bad, 4));
    CK(cudaMemset(bad, 0, 4));
    gen_table<<<(table_n + 127) / 128, 128>>>(table, table_n);
    CK(cudaDeviceSynchronize());
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    float ms[4] = {0, 0, 0, 0}, ms_x = 0;
    for (int rep = 0; rep < 4; rep++) {  // first repetition = warm-up
        float t;
        cudaEventRecord(e0);
        k1_denominators<<<n_blocks, TPB>>>(table, table_n, m, root);
        cudaEventRecord(e1);
        CK(cudaEventSynchronize(e1));
        cudaEventElapsedTime(&t, e0, e1);
        if (rep) ms[0] += t / 3;
        cudaEventRecord(e0);
        k2_invert<<<(n_blocks + 127) / 128, 128>>>(root, n_blocks);
        cudaEventRecord(e1);
        CK(cudaEventSynchronize(e1));
        cudaEventElapsedTime(&t, e0, e1);
        if (rep) ms[1] += t / 3;
        cudaEventRecord(e0);
        k3_finish<<<n_blocks, TPB>>>(table, table_n, m, root, out);
        cudaEventRecord(e1);
        CK(cudaEventSynchronize(e1));
        cudaEventElapsedTime(&t, e0, e1);
        if (rep) ms[2] += t / 3;
        cudaEventRecord(e0);
        k_xyzz<<<(unsigned)((m + TPB - 1) / TPB), TPB>>>(table, table_n, m, out_x);
        cudaEventRecord(e1);
        CK(cudaEventSynchronize(e1));
        cudaEventElapsedTime(&t, e0, e1);
        if (rep) ms_x += t / 3;
    }
    k_compare<<<(unsigned)((m + 255) / 256), 256>>>(out, out_x, m, bad);
    uint32_t h_bad = 0;
    CK(cudaMemcpy(&h_bad, bad, 4, cudaMemcpyDeviceToHost));
    const float total = ms[0] + ms[1] + ms[2];
    printf("additions: 2^%d, %u per block, mismatches vs XYZZ: %u\n", log_m, TPB * PAIRS, h_bad);
    printf("batched affine level: K1 %.3f ms + K2 %.3f ms + K3 %.3f ms = %.3f ms -> %.2f G additions/s\n", ms[0], ms[1], ms[2], total,
           m / (total * 1e-3) / 1e9);
    printf("XYZZ mixed addition (one kernel, same gathers): %.3f ms -> %.2f G additions/s\n", ms_x, m / (ms_x * 1e-3) / 1e9);
    printf("ratio batched-affine / XYZZ time: %.2f (a level pays off when well below 1)\n", total / ms_x);
    return h_bad ? 1 : 0;
}
