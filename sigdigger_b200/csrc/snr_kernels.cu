// snr_kernels.cu -- the generic inspector's SNR meter (InspectorUI::feed, Default/GenericInspector/InspectorUI.cpp:
// 807-833; oracle/SPEC_SN.md) over the engine's device-side symbols: per (channel, stream) the feed's soft symbols
// are binned into the decision-space histogram (SN.1) and one SPEC Y.7 step fits the comb model to it (SN.2).
// Compiled with -fmad=false: float expressions round exactly as written.
#include "sdb_internal.h"
#include "sdb_math.h"
#include "sdb_snr_step.h"

// One 256-thread CTA per (channel, stream): grid (n_streams, n_chans).  Dynamic shared memory: the counts and the
// four float work arrays of Y.7, 5 L words.
__global__ void __launch_bounds__(256) k_snr(const SdbSnrChan *__restrict__ chans, int n_channels,
                                             const float2 *__restrict__ soft, const uint32_t *__restrict__ counts,
                                             size_t sym_cap, uint32_t *__restrict__ hist, float *__restrict__ model,
                                             sdb_snr_status *__restrict__ status)
{
  const SdbSnrChan ch = chans[blockIdx.y];
  const unsigned s = blockIdx.x, L = ch.L;
  const size_t row = (size_t) s * n_channels + ch.k;
  sdb_snr_status *__restrict__ st = status + ch.chain0 + s;
  const unsigned n = counts[row];
  if (n == 0) {                                     // SN.2: no symbols, no counts and no step
    if (threadIdx.x == 0) st->stepped = 0;
    return;
  }
  extern __shared__ unsigned s_snr[];
  unsigned *h = s_snr;
  float *g = reinterpret_cast<float *>(h + L), *H = g + L, *Ht = H + L, *T = Ht + L;
  __shared__ SdbSnrState s_out;
  __shared__ unsigned long long s_sum;
  for (unsigned i = threadIdx.x; i < L; i += blockDim.x) h[i] = 0;
  if (threadIdx.x == 0) s_sum = 0;
  __syncthreads();
  // SN.1: shared-memory counts are exact whatever the order
  const float2 *__restrict__ x = soft + row * sym_cap;
  const float fL = (float) L;
  for (unsigned i = threadIdx.x; i < n; i += blockDim.x) {
    const float2 v2 = x[i];
    const float v = ch.mode == 0 ? d_atan2f(v2.y, v2.x) : d_cabsf(v2.x, v2.y);
    const float b = floorf((v - ch.dmin) / ch.dh * fL);
    if (ch.mode == 0) {
      if (b == b) atomicAdd(&h[b < fL ? (unsigned) b : L - 1], 1u);     // v >= min: b >= 0
    } else if (b < fL) {
      atomicAdd(&h[(unsigned) b], 1u);                                  // |x| >= 0: b >= 0
    }
  }
  __syncthreads();
  // SN.2: add into the stream's histogram; every bin halves once one reaches 2^31 (the sum stays below 2^32)
  uint32_t *__restrict__ gh = hist + ch.hist_off + (size_t) s * L;
  int big = 0;
  for (unsigned i = threadIdx.x; i < L; i += blockDim.x) {
    const unsigned v = gh[i] + h[i];
    h[i] = v;
    big |= v >= 0x80000000u;
  }
  const int halve = __syncthreads_or(big);
  unsigned long long sum = 0;
  for (unsigned i = threadIdx.x; i < L; i += blockDim.x) {
    unsigned v = h[i];
    if (halve) { v >>= 1; h[i] = v; }
    gh[i] = v;
    sum += v;
  }
  atomicAdd(&s_sum, sum);
  SdbSnrState in;
  in.sigma = st->sigma; in.alpha = ch.alpha; in.delta = 0.f; in.intervals = ch.K;
  sdb_snr_step(h, L, in, g, H, Ht, T, &s_out);
  __syncthreads();
  float *__restrict__ gm = model + ch.hist_off + (size_t) s * L;
  for (unsigned i = threadIdx.x; i < L; i += blockDim.x) gm[i] = H[i];
  if (threadIdx.x == 0) {
    sdb_snr_status o;
    o.counted = s_sum; o.steps = st->steps + 1; o.stepped = 1;
    o.sigma = s_out.sigma; o.snr = 1.f / (ch.K * s_out.sigma); o.delta = s_out.delta;
    *st = o;
  }
}

cudaError_t sdb_launch_snr(const SdbLaunchCtx &c, const SdbSnrArgs &a)
{
  if (a.n_chans <= 0) return cudaSuccess;
  const size_t smem = (size_t) 5 * a.max_L * sizeof(uint32_t);
  k_snr<<<dim3((unsigned) a.n_streams, (unsigned) a.n_chans), 256, smem, c.stream>>>(
      a.chans, a.n_channels, a.soft, a.counts, a.sym_cap, a.hist, a.model, a.status);
  if (c.launch_counter) ++*c.launch_counter;
  return cudaGetLastError();
}
