// Pipe-throughput microbenchmarks on the real part (exploratory; numbers quoted in DESIGN.md).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/microbench tools/microbench.cu
#include <cstdio>
#include <cuda_runtime.h>
#include "../distributed_plonk_b200/csrc/g1.cuh"
using namespace dp;

template <int MODE>
__global__ void mb_imad(uint32_t *out, int iters, uint32_t seed) {
    uint32_t a = threadIdx.x * 2654435761u + seed, b = a ^ 0x9e3779b9u;
    uint64_t acc[8];
#pragma unroll
    for (int k = 0; k < 8; k++) acc[k] = a + k;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int k = 0; k < 8; k++) {
            if (MODE == 0) {  // IMAD.WIDE.U32 : 64-bit acc += a*b
                asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[k]) : "r"(a), "r"(b));
            } else if (MODE == 1) {  // IMAD (lo)
                uint32_t lo = (uint32_t)acc[k];
                asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(lo) : "r"(a), "r"(b));
                acc[k] = lo;
            } else if (MODE == 2) {  // IMAD.HI
                uint32_t lo = (uint32_t)acc[k];
                asm volatile("mad.hi.u32 %0, %1, %2, %0;" : "+r"(lo) : "r"(a), "r"(b));
                acc[k] = lo;
            } else {  // IADD3 chain
                uint32_t lo = (uint32_t)acc[k];
                asm volatile("add.u32 %0, %0, %1;" : "+r"(lo) : "r"(a));
                acc[k] = lo;
            }
        }
    }
    uint64_t s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s += acc[k];
    out[blockIdx.x * blockDim.x + threadIdx.x] = (uint32_t)s ^ (uint32_t)(s >> 32);
}

template <class F>
__global__ void mb_field_mul(F *out, int iters) {
    F x = F::one(), y = F::r2();
    x.l[0] += threadIdx.x;
    F u = y, v = x;
    for (int it = 0; it < iters; it++) {
        x = x * y;
        u = u * v;
        y = y * x;
        v = v * u;
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = x + y + u + v;
}

template <class F>
__global__ void mb_field_addsub(F *out, int iters) {
    F x = F::one(), y = F::r2();
    x.l[0] += threadIdx.x;
    for (int it = 0; it < iters; it++) {
        x = x + y;
        y = y - x;
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = x + y;
}

__global__ void mb_madd(G1XYZZ *out, int iters) {
    G1Affine g;
    g.x = Fq::r2();
    g.y = Fq::one();
    g.x.l[0] += threadIdx.x;
    G1XYZZ acc = G1XYZZ::from_affine(g);
    acc.x.l[1] ^= 5;
    for (int it = 0; it < iters; it++) {
        acc = acc.add_mixed(g);
        g.x = g.x + acc.zz;
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <class K, class... A>
float time_kernel(K k, dim3 grid, dim3 block, A... args) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    k<<<grid, block>>>(args...);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    k<<<grid, block>>>(args...);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    return ms;
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount;
    int clk_khz = 0;
    cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    printf("%s, %d SMs, max clock %.0f MHz\n", p.name, sms, clk_khz / 1e3);
    void *buf;
    cudaMalloc(&buf, (size_t)sms * 8 * 256 * sizeof(G1XYZZ));
    const char *names[4] = {"IMAD.WIDE.U32 (mad.wide)", "IMAD lo (mad.lo)", "IMAD.HI (mad.hi)", "IADD (add.u32)"};
    for (int occ_blocks = 2; occ_blocks <= 8; occ_blocks *= 2) {
        dim3 grid(sms * occ_blocks), block(256);
        int iters = 4096;
        float ms[4];
        ms[0] = time_kernel(mb_imad<0>, grid, block, (uint32_t *)buf, iters, 1u);
        ms[1] = time_kernel(mb_imad<1>, grid, block, (uint32_t *)buf, iters, 1u);
        ms[2] = time_kernel(mb_imad<2>, grid, block, (uint32_t *)buf, iters, 1u);
        ms[3] = time_kernel(mb_imad<3>, grid, block, (uint32_t *)buf, iters, 1u);
        for (int m = 0; m < 4; m++) {
            double ops = (double)grid.x * 256 * iters * 8;
            printf("blocks/SM=%d %-26s %.3f ms  %.2f Tlane-op/s  (%.1f lane-ops/clk/SM at max clock)\n", occ_blocks, names[m], ms[m],
                   ops / ms[m] / 1e9, ops / (ms[m] * 1e-3) / sms / (clk_khz * 1e3));
        }
    }
    for (int tpb = 128; tpb <= 256; tpb *= 2)
        for (int occ_blocks = 1; occ_blocks <= 4; occ_blocks *= 2) {
            dim3 grid(sms * occ_blocks), block(tpb);
            int iters = 512;
            float a = time_kernel(mb_field_mul<Fr>, grid, block, (Fr *)buf, iters);
            float b = time_kernel(mb_field_mul<Fq>, grid, block, (Fq *)buf, iters);
            float c = time_kernel(mb_madd, grid, block, (G1XYZZ *)buf, iters / 4);
            float d = time_kernel(mb_field_addsub<Fq>, grid, block, (Fq *)buf, iters * 8);
            double n = (double)grid.x * tpb;
            printf("tpb=%d blocks/SM=%d  Fr mul %.2f G/s | Fq mul %.2f G/s | XYZZ mixed add %.3f G/s | Fq add+sub pair %.2f G/s\n", tpb,
                   occ_blocks, n * iters * 4 / a / 1e6, n * iters * 4 / b / 1e6, n * (iters / 4) / c / 1e6, n * iters * 8 / d / 1e6);
        }
    return 0;
}
