// sdb_fft_block.h -- the transform building blocks of SPEC F.1 / F.2 shared by the kernels that run them
// (fft_kernels.cu, fac_kernels.cu): the twiddle product and the shared-memory Stockham transform.
#pragma once
#include <cuda_runtime.h>
#include "sdb_cpx.h"

// SPEC F.1 twiddle product: one rounded product + one fused multiply-add per component
static __device__ __forceinline__ float2 cmul(float2 a, float2 b)
{
  return make_float2(__fmaf_rn(a.x, b.x, -(a.y * b.y)), __fmaf_rn(a.x, b.y, a.y * b.x));
}
static __device__ __forceinline__ float2 ldtw(const float2 *__restrict__ tw, int i)
{
  return __ldg(tw + i);
}

// ---------------------------------------------------------------------------------------------
// In-place shared-memory FFT of M = 2^logM points.  `nthr` threads (lane = 0..nthr-1) cooperate,
// nthr * BPT >= M / 4.  Every thread of the CTA must call this with the same M (CTA-wide barriers).
// DIR = -1 forward, +1 inverse (unnormalised).
// ---------------------------------------------------------------------------------------------
template <int DIR, int BPT>
static __device__ __forceinline__ void block_fft_inplace(float2 *s, const int M, const int logM,
                                                         const int lane, const int nthr,
                                                         const float2 *__restrict__ tw)
{
  const int q = M >> 2;
  int logNs = 0;
  for (; logNs + 2 <= logM; logNs += 2) {
    const int Ns = 1 << logNs;
    float2 v[BPT][4];
#pragma unroll
    for (int b = 0; b < BPT; ++b) {
      const int j = lane + b * nthr;
      if (j < q) {
#pragma unroll
        for (int t = 0; t < 4; ++t) v[b][t] = s[j + t * q];
      }
    }
    __syncthreads();
#pragma unroll
    for (int b = 0; b < BPT; ++b) {
      const int j = lane + b * nthr;
      if (j < q) {
        const int k = j & (Ns - 1);
        // complex arithmetic of sdb_cpx.h: the same IEEE operations per component as the scalar statement of
        // SPEC F.1 / F.2, so the results are bit-identical
        if (logNs > 0) {
          const int step = M >> (logNs + 2);
          float2 w1 = ldtw(tw, k * step), w2 = ldtw(tw, 2 * k * step), w3 = ldtw(tw, 3 * k * step);
          if (DIR > 0) { w1.y = -w1.y; w2.y = -w2.y; w3.y = -w3.y; }
          v[b][1] = cmulf(v[b][1], w1);
          v[b][2] = cmulf(v[b][2], w2);
          v[b][3] = cmulf(v[b][3], w3);
        }
        const float2 a = cadd(v[b][0], v[b][2]);
        const float2 bb = csub(v[b][0], v[b][2]);
        const float2 c = cadd(v[b][1], v[b][3]);
        const float2 dd = csub(v[b][1], v[b][3]);
        // forward: d = -i * dd ; inverse: d = +i * dd
        const float2 d = DIR < 0 ? make_float2(dd.y, -dd.x) : make_float2(-dd.y, dd.x);
        const int j0 = ((j - k) << 2) + k;
        s[j0]          = cadd(a, c);
        s[j0 + Ns]     = cadd(bb, d);
        s[j0 + 2 * Ns] = csub(a, c);
        s[j0 + 3 * Ns] = csub(bb, d);
      }
    }
    __syncthreads();
  }
  if (logNs < logM) {  // one radix-2 stage with Ns = M/2: in place, butterfly j touches s[j], s[j+h]
    const int h = M >> 1;
#pragma unroll
    for (int b = 0; b < 2 * BPT; ++b) {
      const int j = lane + b * nthr;
      if (j < h) {
        float2 w = ldtw(tw, j);
        if (DIR > 0) w.y = -w.y;
        const float2 a = s[j], t = cmulf(s[j + h], w);
        s[j]     = cadd(a, t);
        s[j + h] = csub(a, t);
      }
    }
    __syncthreads();
  }
}

