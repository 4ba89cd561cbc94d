// wn_math.cuh -- device math of the WaveNet kernels.
//
// "Portable" functions: exp / tanh / sigmoid built only from IEEE-754 double +,*,/,fma,rint and one
// double->float rounding, so that the fp32 kernel is bit-reproducible against a CPU evaluation of the
// same formulas (DESIGN.md §4).  They stand in for the libm expf/tanhf the reference CPU model calls
// (nv_wavenet_reference.cpp:36-40) and are correctly rounded except in ~1e-9 of cases.
//
// "Fast" functions: MUFU-based approximations for the fp16 tensor-core path (replaces the
// --use_fast_math expf/tanhf of nv_wavenet_util.cuh:78-86).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace wn {

__device__ __forceinline__ double exp_core(double x)
{
    // -150 <= x <= 100
    const double LOG2E = 0x1.71547652b82fep+0;
    const double LN2_HI = 0x1.62e42fee00000p-1;
    const double LN2_LO = 0x1.a39ef35793c76p-33;
    double kd = rint(x * LOG2E);
    double r = fma(-kd, LN2_HI, x);
    r = fma(-kd, LN2_LO, r);
    // degree-13 Taylor polynomial of exp(r), Estrin evaluation (same association as the CPU checker)
    double a0 = fma(1.0, r, 1.0);                                           // c0 + c1 r
    double a1 = fma(0x1.5555555555555p-3, r, 0.5);                           // c2 + c3 r
    double a2 = fma(0x1.1111111111111p-7, r, 0x1.5555555555555p-5);          // c4 + c5 r
    double a3 = fma(0x1.a01a01a01a01ap-13, r, 0x1.6c16c16c16c17p-10);        // c6 + c7 r
    double a4 = fma(0x1.71de3a556c734p-19, r, 0x1.a01a01a01a01ap-16);        // c8 + c9 r
    double a5 = fma(0x1.ae64567f544e4p-26, r, 0x1.27e4fb7789f5cp-22);        // c10 + c11 r
    double a6 = fma(0x1.6124613a86d09p-33, r, 0x1.1eed8eff8d898p-29);        // c12 + c13 r
    double r2 = r * r;
    double b0 = fma(a1, r2, a0);
    double b1 = fma(a3, r2, a2);
    double b2 = fma(a5, r2, a4);
    double r4 = r2 * r2;
    double d0 = fma(b1, r4, b0);
    double d1 = fma(a6, r4, b2);
    double r8 = r4 * r4;
    double p = fma(d1, r8, d0);
    long long k = (long long)kd;
    double scale = __longlong_as_double((k + 1023) << 52);
    return p * scale;
}

__device__ __forceinline__ float expf_portable(float x)
{
    if (x != x) return x;
    if (x < -150.0f) return 0.0f;
    if (x > 100.0f) return __int_as_float(0x7f800000);
    return __double2float_rn(exp_core((double)x));
}

__device__ __forceinline__ float tanhf_portable(float x)
{
    if (x != x) return x;
    double xd = (double)x;
    double ax = fabs(xd);
    double t;
    if (ax < 0x1p-12) {
        double x2 = ax * ax;
        t = fma(-(x2 * ax), 0x1.5555555555555p-2, ax);
    } else if (ax >= 20.0) {
        t = 1.0;
    } else {
        double e = exp_core(2.0 * ax);
        t = __ddiv_rn(e - 1.0, e + 1.0);
    }
    return __double2float_rn(xd < 0.0 ? -t : t);
}

// 1.f / (1.f + exp(-f)) in float, as nv_wavenet_reference.cpp:36
__device__ __forceinline__ float sigmoidf_portable(float x)
{
    float e = expf_portable(-x);
    float den = __fadd_rn(1.0f, e);
    return __fdiv_rn(1.0f, den);
}

// ---- fast approximations (fp16 path) ----
__device__ __forceinline__ float tanhf_fast(float x)
{
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float sigmoidf_fast(float x)
{
    // sigmoid(x) = 0.5 * tanh(0.5 x) + 0.5 : one MUFU instead of ex2 + rcp
    return fmaf(0.5f, tanhf_fast(0.5f * x), 0.5f);
}
// two fp16 tanh for one MUFU issue slot
__device__ __forceinline__ __half2 tanh_h2(__half2 x)
{
    uint32_t y, xi = *reinterpret_cast<const uint32_t*>(&x);
    asm("tanh.approx.f16x2 %0, %1;" : "=r"(y) : "r"(xi));
    return *reinterpret_cast<const __half2*>(&y);
}
__device__ __forceinline__ float exp2f_fast(float x)
{
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// two floats <-> one 32-bit word of two fp16 (round to nearest even)
__device__ __forceinline__ uint32_t pack_h2(float a, float b)
{
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_h2(uint32_t v) { return __half22float2(*reinterpret_cast<__half2*>(&v)); }

}  // namespace wn
