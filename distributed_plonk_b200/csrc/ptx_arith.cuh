// 32-bit carry-chain primitives.
//
// On the device every primitive is ONE PTX instruction that reads and/or writes the PTX
// condition-code register (add.cc / addc / mad.lo.cc / madc.hi.cc ...).  ptxas keeps the CC
// dependency between consecutive `asm volatile` statements, fuses mad.lo/mad.hi pairs into
// IMAD.WIDE.U32 and turns the chains into IADD3.X / IMAD.WIDE.U32.X on sm_90a.
//
// On the host (g++ or nvcc's host pass) the same functions are emulated with an explicit
// carry flag, so the multi-precision algorithms in field.cuh / g1.cuh can be unit-tested
// bit-for-bit on a machine without a GPU (tests/emul).  The host path is NOT a product path:
// the library never computes field arithmetic on the CPU for its results.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define DP_HD __host__ __device__ __forceinline__
#define DP_D __device__ __forceinline__
#else
#define DP_HD inline
#define DP_D inline
#endif

namespace dp {
namespace ptx {

#if defined(__CUDA_ARCH__)

DP_HD uint32_t add_cc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
DP_HD uint32_t addc_cc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
DP_HD uint32_t addc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
DP_HD uint32_t sub_cc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
DP_HD uint32_t subc_cc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
DP_HD uint32_t subc(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
DP_HD uint32_t mul_lo(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
DP_HD uint32_t mul_hi(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
DP_HD uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
DP_HD uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
DP_HD uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("mad.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
DP_HD uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
DP_HD uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}

// ---- fused lo/hi pairs: one asm statement per 32x32->64 multiply-accumulate so that ptxas
// emits a single IMAD.WIDE.U32(.X) for it (verified with cuobjdump -sass on sm_90a).
// {hi:lo} = a*b
DP_HD void mul_wide(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    asm("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
// {hi:lo} += a*b, carry-out -> CC
DP_HD void mad_wide_cc(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
                 : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
// {hi:lo} += a*b + CC, carry-out -> CC
DP_HD void madc_wide_cc(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;"
                 : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
// {hi:lo} = a*b + {chi:clo} + CC, carry-out -> CC
DP_HD void madc_wide_cc(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;"
                 : "=r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
}
// {hi:lo} = a*b + CC   (cannot overflow: hi(a*b) <= 2^32-2)
DP_HD void madc_wide_last(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, 0; madc.hi.u32 %1, %2, %3, 0;"
                 : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}

#else  // ---------------------------------------------------------------- host emulation

inline uint32_t &cc_flag() {
    static thread_local uint32_t cc = 0;
    return cc;
}
inline uint32_t emul_add(uint32_t a, uint32_t b, uint32_t cin, bool set) {
    uint64_t s = (uint64_t)a + b + cin;
    if (set) cc_flag() = (uint32_t)(s >> 32);
    return (uint32_t)s;
}
inline uint32_t emul_sub(uint32_t a, uint32_t b, uint32_t bin, bool set) {
    // PTX: CC.CF after sub.cc is the BORROW (1 = borrow out), consumed as borrow-in by subc.
    uint64_t d = (uint64_t)a - b - bin;
    if (set) cc_flag() = (uint32_t)((d >> 32) & 1);
    return (uint32_t)d;
}
inline uint32_t add_cc(uint32_t a, uint32_t b) { return emul_add(a, b, 0, true); }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { return emul_add(a, b, cc_flag(), true); }
inline uint32_t addc(uint32_t a, uint32_t b) { return emul_add(a, b, cc_flag(), false); }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { return emul_sub(a, b, 0, true); }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { return emul_sub(a, b, cc_flag(), true); }
inline uint32_t subc(uint32_t a, uint32_t b) { return emul_sub(a, b, cc_flag(), false); }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return (uint32_t)((uint64_t)a * b); }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return emul_add(mul_lo(a, b), c, 0, true); }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return emul_add(mul_lo(a, b), c, cc_flag(), true); }
inline uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return emul_add(mul_hi(a, b), c, 0, true); }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return emul_add(mul_hi(a, b), c, cc_flag(), true); }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return emul_add(mul_hi(a, b), c, cc_flag(), false); }

inline void mul_wide(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    lo = mul_lo(a, b);
    hi = mul_hi(a, b);
}
inline void mad_wide_cc(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    lo = mad_lo_cc(a, b, lo);
    hi = madc_hi_cc(a, b, hi);
}
inline void madc_wide_cc(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    lo = madc_lo_cc(a, b, lo);
    hi = madc_hi_cc(a, b, hi);
}
inline void madc_wide_cc(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
    lo = madc_lo_cc(a, b, clo);
    hi = madc_hi_cc(a, b, chi);
}
inline void madc_wide_last(uint32_t &lo, uint32_t &hi, uint32_t a, uint32_t b) {
    lo = madc_lo_cc(a, b, 0u);
    hi = madc_hi(a, b, 0u);
}

#endif

}  // namespace ptx
}  // namespace dp
