// sdb_snr_step.h -- one step of the SNR estimator of the inspector's decision-space histogram
// (Misc/SNREstimator.cpp:30-169; SPEC Y.7), shared by the stand-alone estimator (k_snr_feed, tasks_kernels.cu) and the
// engine's SNR meter (k_snr, snr_kernels.cu).  One 256-thread CTA per histogram.  The model (a comb of 2^bps
// Gaussians) is built bin-parallel -- every bin's sum over the intervals keeps the reference's order --; the two
// order-dependent reductions (the maximum is order-free, the gradient sum is not) are done by thread 0 in bin order.
// expf(t) = 10^(t log10 e) of SPEC M.  Included by units compiled with -fmad=false.
#pragma once
#include "sdb_math.h"

struct SdbSnrState { float sigma, alpha, delta; unsigned intervals; };

// h[length] counts in; g, H, Ht, T [length] work arrays (H is the normalised model afterwards, Ht the normalised
// histogram).  Thread 0 writes out->delta and out->sigma.  With st.intervals == 0 only Ht is computed.
static __device__ __forceinline__ void sdb_snr_step(const unsigned *__restrict__ h, unsigned length, const SdbSnrState st,
                                                    float *__restrict__ g, float *__restrict__ H,
                                                    float *__restrict__ Ht, float *__restrict__ T,
                                                    SdbSnrState *__restrict__ out)
{
  __shared__ unsigned s_max;
  __shared__ float s_fmax;
  const float hx = 1.f / length;
  if (threadIdx.x == 0) { s_max = 0; s_fmax = 0.f; }
  __syncthreads();
  unsigned m = 0;
  for (unsigned i = threadIdx.x; i < length; i += blockDim.x) m = max(m, h[i]);
  atomicMax(&s_max, m);
  __syncthreads();
  const unsigned hmax = s_max == 0 ? 1u : s_max;
  for (unsigned i = threadIdx.x; i < length; i += blockDim.x) Ht[i] = (float) h[i] / hmax;
  if (st.intervals == 0) return;
  const float sigma2 = st.sigma * st.sigma;
  for (unsigned i = threadIdx.x; i < length; i += blockDim.x) {
    float x = i * hx;
    if (x >= .5f) x -= 1.f;
    g[i] = d_exp10f((-x * x / sigma2) * 0.4342944819032518f);
  }
  __syncthreads();
  const float intlen = 1.f / st.intervals, start = .5f * intlen;
  float lmax = 0.f;
  for (unsigned i = threadIdx.x; i < length; i += blockDim.x) {
    float v = 0.f;
    for (unsigned j = 0; j < st.intervals; ++j) {
      const float skip = start + j * intlen;
      const float t = 1.f - (skip - floorf(skip));
      const unsigned skipint = (unsigned) floorf(length * skip);
      const unsigned i1 = (length + i - skipint) % length;
      const unsigned i2 = (length + i1 - 1) % length;
      v += t * g[i1];
      v += (1 - t) * g[i2];
    }
    H[i] = v;
    lmax = fmaxf(lmax, v);
  }
  // non-negative floats order like their bit patterns
  atomicMax(reinterpret_cast<unsigned *>(&s_fmax), __float_as_uint(lmax));
  __syncthreads();
  const float fmx = s_fmax;
  const float sigmainv = 1.f / st.sigma, sigma3inv = sigmainv * sigmainv * sigmainv;
  for (unsigned i = threadIdx.x; i < length; i += blockDim.x) {
    float hv = H[i];
    if (fmx > 0.f) { hv /= fmx; H[i] = hv; }
    float x = i * hx;
    if (x >= .5f) x -= 1.f;
    float tm = 0;
    for (unsigned j = 0; j < st.intervals; ++j) {
      const float skip = start + j * intlen;
      tm += (x - skip) * (x - skip);
    }
    T[i] = tm * ((hv - Ht[i]) / sigma3inv);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float delta = 0;
    for (unsigned i = 0; i < length; ++i) delta += T[i];
    delta = delta / length;
    out->delta = delta;
    out->sigma = st.sigma + -st.alpha * delta;
  }
}
