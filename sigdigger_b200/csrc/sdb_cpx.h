// sdb_cpx.h -- complex binary32 arithmetic for the FFT and chain kernels (sm_90a).
//
// One explicit round-to-nearest intrinsic per component, so the compiler can neither contract nor reorder a
// rounding: the parity with oracle/fft_spec.c rests on these exact expressions.
#pragma once
#include <cuda_runtime.h>

static __device__ __forceinline__ float2 sdb_add2(float2 a, float2 b)
{
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
static __device__ __forceinline__ float2 sdb_sub2(float2 a, float2 b)
{
  return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y));
}
static __device__ __forceinline__ float2 sdb_mul2(float2 a, float2 b)
{
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
static __device__ __forceinline__ float2 sdb_fma2(float2 a, float2 b, float2 c)
{
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

static __device__ __forceinline__ float2 cadd(float2 a, float2 b) { return sdb_add2(a, b); }
static __device__ __forceinline__ float2 csub(float2 a, float2 b) { return sdb_sub2(a, b); }
static __device__ __forceinline__ float2 mul_mi(float2 a) { return make_float2(a.y, -a.x); }   // a * (-i)
static __device__ __forceinline__ float2 mul_pi(float2 a) { return make_float2(-a.y, a.x); }   // a * (+i)

// SPEC F.1 twiddle product: re = fma(a.re, b.re, -(a.im b.im)), im = fma(a.re, b.im, a.im b.re).
static __device__ __forceinline__ float2 cmulf(float2 a, float2 b)
{
  return make_float2(__fmaf_rn(a.x, b.x, -__fmul_rn(a.y, b.y)), __fmaf_rn(a.x, b.y, __fmul_rn(a.y, b.x)));
}
// a * conj(b), same rounding pattern with b.im negated: re = fma(a.re, b.re, a.im b.im),
// im = fma(a.re, -b.im, a.im b.re)
static __device__ __forceinline__ float2 cmulf_conj(float2 a, float2 b)
{
  return make_float2(__fmaf_rn(a.x, b.x, __fmul_rn(a.y, b.y)), __fmaf_rn(a.x, -b.y, __fmul_rn(a.y, b.x)));
}

// forward 4-point DFT in place: (a, b, c, d) <- DFT4, b = d0 - i t and d = d0 + i t with t = b - d
// (one rounded add or subtract per lane, as in oracle/fft_spec.c)
static __device__ __forceinline__ void fft4(float2 &a, float2 &b, float2 &c, float2 &d)
{
  const float2 s0 = cadd(a, c), d0 = csub(a, c), s1 = cadd(b, d), t = csub(b, d);
  a = cadd(s0, s1); c = csub(s0, s1);
  b = make_float2(__fadd_rn(d0.x, t.y), __fsub_rn(d0.y, t.x));
  d = make_float2(__fsub_rn(d0.x, t.y), __fadd_rn(d0.y, t.x));
}
// inverse 4-point DFT (kernel exp(+i...)): b = d0 + i t, d = d0 - i t
static __device__ __forceinline__ void ifft4(float2 &a, float2 &b, float2 &c, float2 &d)
{
  const float2 s0 = cadd(a, c), d0 = csub(a, c), s1 = cadd(b, d), t = csub(b, d);
  a = cadd(s0, s1); c = csub(s0, s1);
  b = make_float2(__fsub_rn(d0.x, t.y), __fadd_rn(d0.y, t.x));
  d = make_float2(__fadd_rn(d0.x, t.y), __fsub_rn(d0.y, t.x));
}
