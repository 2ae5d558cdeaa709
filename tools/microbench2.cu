// Carry-chain throughput: is IMAD.WIDE.U32.X (carry-in/out) slower than plain IMAD.WIDE.U32 ?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/microbench2 tools/microbench2.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <stdint.h>

// MODE 0: 4 independent carry chains of 6 fused mad.lo.cc/madc.hi.cc pairs (IMAD.WIDE.U32.X)
// MODE 1: the same 24 products as plain mad.wide.u32 into 64-bit accumulators (no carries)
// MODE 2: 4 carry chains of 12 add.cc/addc.cc (IADD3.X)
// MODE 3: 24 plain mad.wide + 48 IADD3(.X) carry adds (products on the FMA pipe, carries on ALU)
template <int MODE>
__global__ void mb(uint32_t *out, int iters) {
    uint32_t a[6], acc[4][12];
    uint64_t wacc[4][6];
    uint32_t b = threadIdx.x * 2654435761u + 12345u;
    for (int k = 0; k < 6; k++) a[k] = b * (k + 3) + k;
    for (int c = 0; c < 4; c++)
        for (int k = 0; k < 12; k++) acc[c][k] = b ^ (c * 131 + k);
    for (int c = 0; c < 4; c++)
        for (int k = 0; k < 6; k++) wacc[c][k] = b ^ (c * 17 + k);
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int c = 0; c < 4; c++) {
            uint32_t bb = b + c;
            if (MODE == 0) {
                asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(acc[c][0]), "+r"(acc[c][1]) : "r"(a[0]), "r"(bb));
#pragma unroll
                for (int k = 1; k < 6; k++)
                    asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(acc[c][2 * k]), "+r"(acc[c][2 * k + 1]) : "r"(a[k]), "r"(bb));
            } else if (MODE == 1) {
#pragma unroll
                for (int k = 0; k < 6; k++) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(wacc[c][k]) : "r"(a[k]), "r"(bb));
            } else if (MODE == 2) {
                asm volatile("add.cc.u32 %0, %0, %1;" : "+r"(acc[c][0]) : "r"(a[0]));
#pragma unroll
                for (int k = 1; k < 12; k++) asm volatile("addc.cc.u32 %0, %0, %1;" : "+r"(acc[c][k]) : "r"(a[k % 6]));
            } else {
                uint64_t p[6];
#pragma unroll
                for (int k = 0; k < 6; k++) asm volatile("mul.wide.u32 %0, %1, %2;" : "=l"(p[k]) : "r"(a[k]), "r"(bb));
                asm volatile("add.cc.u32 %0, %0, %1;" : "+r"(acc[c][0]) : "r"((uint32_t)p[0]));
                asm volatile("addc.cc.u32 %0, %0, %1;" : "+r"(acc[c][1]) : "r"((uint32_t)(p[0] >> 32)));
#pragma unroll
                for (int k = 1; k < 6; k++) {
                    asm volatile("addc.cc.u32 %0, %0, %1;" : "+r"(acc[c][2 * k]) : "r"((uint32_t)p[k]));
                    asm volatile("addc.cc.u32 %0, %0, %1;" : "+r"(acc[c][2 * k + 1]) : "r"((uint32_t)(p[k] >> 32)));
                }
            }
        }
        b = b * 3 + acc[0][11] + (uint32_t)wacc[0][5];
    }
    uint32_t s = 0;
    for (int c = 0; c < 4; c++)
        for (int k = 0; k < 12; k++) s ^= acc[c][k] ^ (uint32_t)(wacc[c][k % 6] >> 7);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <class K>
float run(K k, int blocks, uint32_t *buf, int iters) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    k<<<blocks, 256>>>(buf, iters);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    k<<<blocks, 256>>>(buf, iters);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    return ms;
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount, khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    uint32_t *buf;
    cudaMalloc(&buf, (size_t)sms * 8 * 256 * 4);
    const char *names[4] = {"IMAD.WIDE.U32.X chains (24 MAC)", "IMAD.WIDE.U32 no carry (24 MAC)", "IADD3.X chains (48 adds)",
                            "mul.wide + ALU carry adds (24 MAC)"};
    for (int occ = 1; occ <= 4; occ *= 2) {
        int blocks = sms * occ, iters = 2048;
        float ms[4] = {run(mb<0>, blocks, buf, iters), run(mb<1>, blocks, buf, iters), run(mb<2>, blocks, buf, iters), run(mb<3>, blocks, buf, iters)};
        for (int m = 0; m < 4; m++) {
            double units = (double)blocks * 256 * iters * (m == 2 ? 48 : 24);
            printf("blocks/SM=%d %-36s %.3f ms  %.1f lane-units/clk/SM\n", occ, names[m], ms[m], units / (ms[m] * 1e-3) / sms / (khz * 1e3));
        }
    }
    return 0;
}
