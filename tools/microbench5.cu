// FP64-pipe field multiplication (tools/experiments/dfield.cuh) against the 32-bit carry-chain product.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -o tools/microbench5 tools/microbench5.cu
// Prints: raw DFMA rate; the hi/lo split mix (2 DFMA + DADD + 64-bit integer adds); Fr / Fq Montgomery
// products per second on the FP64 pipe, on the integer pipe, and with both kinds of warps resident
// together (do the pipes overlap?); a bit-for-bit check of the FP64 product against field.cuh.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include "../distributed_plonk_b200/csrc/field.cuh"
#include "experiments/dfield.cuh"
using namespace dp;
using namespace dpd;

__global__ void mb_dfma(double *out, int iters) {
    double a[8], x = 1.0 + threadIdx.x * 1e-9, y = 1.0 - 1e-9;
    for (int k = 0; k < 8; k++) a[k] = k;
    for (int it = 0; it < iters; it++)
#pragma unroll
        for (int k = 0; k < 8; k++) a[k] = fma(a[k], x, y);
    double s = 0;
    for (int k = 0; k < 8; k++) s += a[k];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// the split of 8 independent limb products per iteration, accumulated as integers
__global__ void mb_split(uint64_t *out, int iters) {
    double x[8], y = 4503599627370495.0 - threadIdx.x;
    uint64_t ah = 0, al = 0;
    for (int k = 0; k < 8; k++) x[k] = 1234567890123.0 + k * 77 + threadIdx.x;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const double hi = __fma_rz(x[k], y, DF_C1);
            const double lo = __fma_rz(x[k], y, DF_C2 - hi);
            ah += d2b(hi);
            al += d2b(lo);
        }
        y = b2d((al & MASK52) | EXP_LO) - 0x1p52;  // data dependence between iterations
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = ah + al;
}

template <class P>
__device__ __forceinline__ void dmul(double *x, const double *y) {
    uint64_t o[P::L];
    mont_mul_dfma<P>(x, y, o);
#pragma unroll
    for (int i = 0; i < P::L; i++) x[i] = u52_to_double(o[i]);
}

template <class P>
__device__ __forceinline__ void dfield_chain(double *out, int iters) {
    constexpr int L = P::L;
    double x[L], y[L], u[L], v[L];
    for (int i = 0; i < L; i++) {
        x[i] = (double)((P::mod(i) >> 1) + threadIdx.x);
        y[i] = (double)((P::mod(i) >> 2) + 3 * i);
        u[i] = y[i];
        v[i] = x[i];
    }
    for (int it = 0; it < iters; it++) {
        dmul<P>(x, y);
        dmul<P>(u, v);
        dmul<P>(y, x);
        dmul<P>(v, u);
    }
    double s = 0;
    for (int i = 0; i < L; i++) s += x[i] + y[i] + u[i] + v[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <class F>
__device__ __forceinline__ void ifield_chain(F *out, int iters) {
    F x = F::one(), y = F::r2();
    x.l[0] += threadIdx.x;
    F u = y, v = x;
    for (int it = 0; it < iters; it++) {
        x = F::mul_inline(x, y);
        u = F::mul_inline(u, v);
        y = F::mul_inline(y, x);
        v = F::mul_inline(v, u);
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = x + y + u + v;
}

template <class P>
__global__ void __launch_bounds__(256) mb_dfield(double *out, int iters) { dfield_chain<P>(out, iters); }
template <class F>
__global__ void __launch_bounds__(256) mb_ifield(F *out, int iters) { ifield_chain<F>(out, iters); }
// warps alternate between the two pipes: even warps integer, odd warps FP64 (same number of products each)
template <class P, class F>
__global__ void __launch_bounds__(256) mb_both(void *out, int iters_i, int iters_d) {
    if ((threadIdx.x >> 5) & 1)
        dfield_chain<P>((double *)out, iters_d);
    else
        ifield_chain<F>((F *)out + (size_t)gridDim.x * blockDim.x, iters_i);
}

// bit-for-bit: 16 * dfma(a, b) == a * b (field.cuh) for Montgomery words a, b
__global__ void check_fr(const Fr *a, const Fr *b, int n, int *bad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t la[5], lb[5], lo[5];
    double da[5], db[5];
    fr_words_to_limbs(a[i].l, la);
    fr_words_to_limbs(b[i].l, lb);
    for (int k = 0; k < 5; k++) {
        da[k] = u52_to_double(la[k]);
        db[k] = u52_to_double(lb[k]);
    }
    mont_mul_dfma<FrDParams>(da, db, lo);
    Fr z;
    fr_limbs_to_words(lo, z.l);
    Fr::final_sub(z.l);
    for (int k = 0; k < 4; k++) z = z.dbl();
    if (z != a[i] * b[i]) atomicAdd(bad, 1);
}
__global__ void gen_fr(Fr *x, int n, uint32_t seed) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr v = Fr::one();
    v.l[0] += i * 2654435761u + seed;
    v.l[3] ^= i * 40503u;
    Fr w = v * v;
    x[i] = w * v + w;
}

template <class K, class... A>
float tk(K k, int blocks, int tpb, A... args) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    k<<<blocks, tpb>>>(args...);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    k<<<blocks, tpb>>>(args...);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) printf("CUDA error: %s\n", cudaGetErrorString(e));
    return ms;
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount, clk_khz = 0;
    cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    printf("%s, %d SMs, max clock %.0f MHz\n", p.name, sms, clk_khz / 1e3);
    void *buf;
    cudaMalloc(&buf, (size_t)sms * 8 * 256 * 128);
    {   // correctness first
        const int n = 1 << 16;
        Fr *a, *b;
        int *bad, hbad = -1;
        cudaMalloc(&a, n * sizeof(Fr));
        cudaMalloc(&b, n * sizeof(Fr));
        cudaMalloc(&bad, 4);
        cudaMemset(bad, 0, 4);
        gen_fr<<<n / 256, 256>>>(a, n, 1u);
        gen_fr<<<n / 256, 256>>>(b, n, 7777u);
        check_fr<<<n / 256, 256>>>(a, b, n, bad);
        cudaMemcpy(&hbad, bad, 4, cudaMemcpyDeviceToHost);
        printf("FP64 Fr product vs field.cuh on %d random pairs: %d mismatches (%s)\n", n, hbad, cudaGetErrorString(cudaGetLastError()));
    }
    for (int occ = 1; occ <= 4; occ *= 2) {
        const int blocks = sms * occ, tpb = 256, iters = 2048;
        const double lanes = (double)blocks * tpb;
        float a = tk(mb_dfma, blocks, tpb, (double *)buf, iters);
        float b = tk(mb_split, blocks, tpb, (uint64_t *)buf, iters);
        printf("blocks/SM=%d  DFMA %.1f lane-op/clk/SM | split mix (2 DFMA + DADD + 2 add64 per product) %.1f products/clk/SM\n", occ,
               lanes * iters * 8 / (a * 1e-3) / sms / (clk_khz * 1e3), lanes * iters * 8 / (b * 1e-3) / sms / (clk_khz * 1e3));
    }
    for (int occ = 1; occ <= 4; occ *= 2) {
        const int blocks = sms * occ, tpb = 256, iters = 256;
        const double n = (double)blocks * tpb * iters * 4;
        float a = tk(mb_ifield<Fr>, blocks, tpb, (Fr *)buf, iters);
        float b = tk(mb_dfield<FrDParams>, blocks, tpb, (double *)buf, iters);
        float c = tk(mb_ifield<Fq>, blocks, tpb, (Fq *)buf, iters);
        float d = tk(mb_dfield<FqDParams>, blocks, tpb, (double *)buf, iters);
        // both pipes: integer warps get iters_i, FP64 warps iters_d; total products = half the threads each
        float e = tk(mb_both<FrDParams, Fr>, blocks, tpb, buf, iters, iters);
        float f = tk(mb_both<FrDParams, Fr>, blocks, tpb, buf, iters, iters * 3 / 2);
        float g = tk(mb_both<FqDParams, Fq>, blocks, tpb, buf, iters, iters);
        printf("blocks/SM=%d  Fr mul: int %.1f G/s, fp64 %.1f G/s, mixed warps 1:1 %.1f G/s, 1:1.5 %.1f G/s | Fq mul: int %.1f G/s, fp64 %.1f G/s, mixed 1:1 %.1f G/s\n",
               occ, n / a / 1e6, n / b / 1e6, n / e / 1e6, n * 1.25 / f / 1e6, n / c / 1e6, n / d / 1e6, n / g / 1e6);
    }
    return 0;
}
