// tasks_kernels.cu -- the GUI's offline TimeWindow tasks whose arithmetic is fully present in the reference
// (SPEC.md section Y), over a batch of captured buffers:
//   delayed conjugate product    Tasks/DelayedConjTask.cpp:58-100
//   histogram feeder             Tasks/HistogramFeeder.cpp:35-87
//   manual (box-car) sampler     Tasks/WaveSampler.cpp:28-46, 96-175
//   zero-crossing sampler        Tasks/WaveSampler.cpp:222-292
//   carrier detector             Tasks/CarrierDetector.cpp:49-147
//   decider                      Default/GenericInspector/InspectorUI.cpp:836-846 (SPEC D)
// The reference runs them as sequential loops on one buffer.  Here every loop iteration that carries no state
// is one thread; where the reference carries state (the sampler's `prev`, the zero-crossing run lengths)
// the state a thread needs is recomputed from the inputs or passed through a one-byte-per-sample event map.
// The Tasks/ primitives (carrier translator, quadrature demodulator, Costas, PLL, AGC, low-pass filter) and the SNR
// estimator of the inspector's histogram live here too, with the host side of every task behind the C-ABI.
// Compiled with -fmad=false: float and double expressions round exactly as written.
#include "sdb_internal.h"
#include "sdb_math.h"
#include "sdb_chain_steps.h"
#include "sdb_snr_step.h"
#include "host_design.h"
#include <string.h>
#include <vector>

#define TASK_BLOCK 4096  // SIGDIGGER_WAVESAMPLER_FEEDER_BLOCK_LENGTH (include/WaveSampler.h:28)

__global__ void k_task_delayed_conj(const float2 *__restrict__ src, float2 *__restrict__ dst, size_t n, size_t batch,
                                    size_t delay)
{
  const size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (i >= n * batch) return;
  const size_t p = i % n;
  if (p < delay) { dst[i] = make_float2(0.0f, 0.0f); return; }
  const float2 x = src[i], prev = src[i - delay];
  const float kinv = (float) (1.0 / ((double) d_cabsf(prev.x, prev.y) + 1e-3));
  const float tr = kinv * x.x, ti = kinv * x.y;
  dst[i] = make_float2(tr * prev.x + ti * prev.y, ti * prev.x - tr * prev.y);
}

// space: 0 amplitude, 1 phase, 2 frequency (n - 1 values per buffer)
__global__ void k_task_hist(const float2 *__restrict__ src, float *__restrict__ out, size_t n, size_t batch, int space)
{
  const size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (i >= n * batch) return;
  const float2 x = src[i];
  if (space == 0) { out[i] = d_cabsf(x.x, x.y); return; }
  if (space == 1) { out[i] = d_atan2f(x.y, x.x); return; }
  const size_t b = i / n, p = i - b * n;
  if (p == 0) return;
  const float2 pv = src[i - 1];
  out[b * (n - 1) + p - 1] = d_atan2f(x.y * pv.x - x.x * pv.y, x.x * pv.x + x.y * pv.y);
}

struct SymGeom { long long i0, i1; float t0, t1; };

static __device__ __forceinline__ SymGeom sym_geom(long long p, double samp_offset, double delta, double sync)
{
  SymGeom g;
  const double start = ((double) p - samp_offset) * delta + sync;
  const double end = start + delta;
  g.i0 = (long long) floor(start);
  g.i1 = (long long) ceil(end);
  g.t0 = (float) (1 - (start - (double) g.i0));
  g.t1 = (float) (1 - ((double) g.i1 - end));
  return g;
}

static __device__ __forceinline__ float2 sym_tap(const float2 *__restrict__ x, long long n, const SymGeom &g,
                                                 long long i)
{
  if (i < 0 || i >= n) return make_float2(0.0f, 0.0f);
  const float2 v = x[i];
  if (i == g.i0) return make_float2(g.t0 * v.x, g.t0 * v.y);
  if (i == g.i1) return make_float2(g.t1 * v.x, g.t1 * v.y);
  return v;
}

// one thread per (buffer, symbol); `prev` at the start of a symbol is the last tap of the previous one
__global__ void k_task_sample_manual(const float2 *__restrict__ src, size_t n, size_t batch, int space, double sync,
                                     double delta, double samp_offset, float delta_inv, long long count,
                                     float2 *__restrict__ out)
{
  const size_t t = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (t >= (size_t) count * batch) return;
  const size_t b = t / (size_t) count;
  const long long p = (long long) (t - b * (size_t) count);
  const float2 *__restrict__ x = src + b * n;
  float2 prev = make_float2(0.0f, 0.0f);
  if (p > 0) {
    const SymGeom q = sym_geom(p - 1, samp_offset, delta, sync);
    if (q.i1 >= q.i0) prev = sym_tap(x, (long long) n, q, q.i1);
  }
  const SymGeom g = sym_geom(p, samp_offset, delta, sync);
  float ar = 0.0f, ai = 0.0f;
  for (long long i = g.i0; i <= g.i1; ++i) {
    const float2 v = sym_tap(x, (long long) n, g, i);
    if (space == 0) {
      ar += v.x * v.x + v.y * v.y;
      ai += v.y * v.x - v.x * v.y;
    } else {
      ar += v.x * prev.x + v.y * prev.y;
      ai += v.y * prev.x - v.x * prev.y;
    }
    prev = v;
  }
  out[t] = space == 0 ? make_float2(sqrtf(delta_inv * ar), 0.0f) : make_float2(delta_inv * ar, delta_inv * ai);
}

// Zero-crossing sampler, pass 1: one thread per (buffer, 4096-sample work() block).  Every block starts from
// prevVar = -1 and prev = 0 (the reference never stores them back), so blocks are independent here; what
// couples them (lastZc, the per-block cap) is handled by pass 2.  ev[p]: 0 none, 1 crossing with var <= 0,
// 2 crossing with var > 0.
__global__ void k_task_zc_events(const float2 *__restrict__ src, size_t n, size_t batch, size_t blocks, int space,
                                 int amplitude, float thres, float2 zca, unsigned char *__restrict__ ev,
                                 size_t ev_pitch)
{
  const size_t t = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (t >= blocks * batch) return;
  const size_t b = t / blocks, k = t - b * blocks;
  const float2 *__restrict__ x = src + b * n;
  unsigned char *__restrict__ e = ev + b * ev_pitch;
  const size_t p0 = k * TASK_BLOCK;
  const size_t p1 = p0 + TASK_BLOCK < n ? p0 + TASK_BLOCK : n;
  const bool last = p1 >= n;
  float2 prev = make_float2(0.0f, 0.0f);
  float var = 0.0f, prev_var = -1.0f;
  for (size_t p = p0; p < p1; ++p) {
    const float2 d = x[p];
    if (space == 0) {
      var = amplitude ? d.x * d.x + d.y * d.y : d.x * zca.x - d.y * zca.y;
      var -= thres;
    } else if (space == 1) {
      var = d_atan2f(d.x * zca.y + d.y * zca.x, d.x * zca.x - d.y * zca.y);
    } else {
      const float ir = -d.y, ii = d.x;
      var = d_atan2f(ii * prev.x - ir * prev.y, ir * prev.x + ii * prev.y);
      prev = d;
    }
    unsigned char c = 0;
    if (((var > 0 || var < 0) || last) && (var * prev_var < 0 || last)) {
      c = var > 0 ? 2 : 1;
      prev_var = var;
    }
    e[p] = c;
  }
}

// pass 2: one thread per buffer walks the event map (8 samples per load when nothing happened)
__global__ void k_task_zc_emit(const unsigned char *__restrict__ ev, size_t ev_pitch, size_t n, size_t batch,
                               float bnor, unsigned char *__restrict__ sym, unsigned *__restrict__ counts, size_t cap)
{
  const size_t b = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const unsigned char *__restrict__ e = ev + b * ev_pitch;
  unsigned char *__restrict__ o = sym + b * cap;
  size_t total = 0;
  long long last_zc = 0;
  for (size_t p0 = 0; p0 < n; p0 += TASK_BLOCK) {
    const size_t p1 = p0 + TASK_BLOCK < n ? p0 + TASK_BLOCK : n;
    long long i = 0;
    size_t p = p0;
    while (p < p1) {
      if ((p & 7) == 0 && p + 8 <= p1 && *reinterpret_cast<const unsigned long long *>(e + p) == 0ull) { p += 8; continue; }
      const unsigned char c = e[p];
      if (c) {
        const long long samples = (long long) p - last_zc;
        long long symbols = (long long) round((double) ((float) samples * bnor));
        while (symbols-- > 0 && i < TASK_BLOCK) {
          if (total < cap) o[total] = c == 2;
          ++total; ++i;
        }
        last_zc = (long long) p;
      }
      ++p;
    }
  }
  counts[b] = (unsigned) total;
}

// carrier detector, step 1: window (length n) and zero-pad to the transform size
__global__ void k_task_carrier_prep(const float2 *__restrict__ src, const float *__restrict__ w, size_t n, size_t alloc,
                                    size_t batch, float2 *__restrict__ dst)
{
  const size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (i >= alloc * batch) return;
  const size_t b = i / alloc, k = i - b * alloc;
  float2 v = make_float2(0.0f, 0.0f);
  if (k < n) { const float2 x = src[b * n + k]; const float wk = w[k]; v = make_float2(x.x * wk, x.y * wk); }
  dst[i] = v;
}

// step 3 (step 2 is the engine's PSD): strongest bin outside the notch (first one on ties), then the
// power-weighted circular centroid around it, accumulated in bin order by one thread
__global__ void __launch_bounds__(256) k_task_carrier_find(const float *__restrict__ psd, int alloc, int bins, int delta,
                                                           int skip, float *__restrict__ peak)
{
  __shared__ float sv[256];
  __shared__ int si[256];
  const float *__restrict__ P = psd + (size_t) blockIdx.x * alloc;
  float bv = 0.0f; int bi = 0;
  for (int i = skip + threadIdx.x; i < alloc - skip; i += 256) {
    const float v = P[i];
    if (v > bv) { bv = v; bi = i; }
  }
  sv[threadIdx.x] = bv; si[threadIdx.x] = bi;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      const float ov = sv[threadIdx.x + s]; const int oi = si[threadIdx.x + s];
      if (ov > sv[threadIdx.x] || (ov == sv[threadIdx.x] && ov > 0.0f && oi < si[threadIdx.x])) {
        sv[threadIdx.x] = ov; si[threadIdx.x] = oi;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  const int start = si[0] - delta;
  float ar = 0.0f, ai = 0.0f;
  for (int i = 0; i < bins; ++i) {
    int j = i + start;
    if (j < 0) j += alloc;
    j %= alloc;
    const float nfreq = 2.f * (float) j / (float) alloc;
    float s, c;
    d_sincosf(3.14159265358979323846f * nfreq, &s, &c);
    const float pw = P[j];
    ar += pw * c;
    ai += pw * s;
  }
  peak[blockIdx.x] = d_atan2f(ai, ar);
}

// SPEC D decider over a flat array: mode 0 argument, 1 modulus
__global__ void k_task_decide(const float2 *__restrict__ x, unsigned char *__restrict__ sym, size_t n, int mode,
                              float dmin, float dh, int intervals)
{
  const size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float2 v2 = x[i];
  const float v = mode == 0 ? d_atan2f(v2.y, v2.x) : d_cabsf(v2.x, v2.y);
  const float s = floorf((v - dmin) / dh * (float) intervals);
  int k = (int) s;
  if (!(s >= 0.0f)) k = 0;
  if (k > intervals - 1) k = intervals - 1;
  sym[i] = (unsigned char) k;
}

// SNR estimator of the inspector's decision-space histogram (SPEC Y.7; the step is sdb_snr_step.h): one CTA per
// estimator
__global__ void __launch_bounds__(256) k_snr_feed(const unsigned *__restrict__ history, unsigned length,
                                                  SdbSnrState *__restrict__ states, float *__restrict__ gaussian,
                                                  float *__restrict__ hi, float *__restrict__ htilde,
                                                  float *__restrict__ term)
{
  const unsigned b = blockIdx.x;
  const unsigned *__restrict__ h = history + (size_t) b * length;
  float *__restrict__ g = gaussian + (size_t) b * length, *__restrict__ H = hi + (size_t) b * length;
  float *__restrict__ Ht = htilde + (size_t) b * length, *__restrict__ T = term + (size_t) b * length;
  sdb_snr_step(h, length, states[b], g, H, Ht, T, states + b);
}

static cudaError_t sdb_launch_snr_feed(cudaStream_t s, const unsigned *history, unsigned length, unsigned n,
                                       SdbSnrState *states, float *gaussian, float *hi, float *htilde, float *term)
{
  if (n == 0 || length == 0) return cudaSuccess;
  k_snr_feed<<<n, 256, 0, s>>>(history, length, states, gaussian, hi, htilde, term);
  return cudaGetLastError();
}

static inline unsigned grid_for(size_t total, unsigned threads) { return (unsigned) ((total + threads - 1) / threads); }

static cudaError_t sdb_launch_task_delayed_conj(cudaStream_t s, const float2 *src, float2 *dst, size_t n, size_t batch,
                                                size_t delay)
{
  k_task_delayed_conj<<<grid_for(n * batch, 256), 256, 0, s>>>(src, dst, n, batch, delay);
  return cudaGetLastError();
}

static cudaError_t sdb_launch_task_hist(cudaStream_t s, const float2 *src, float *out, size_t n, size_t batch, int space)
{
  k_task_hist<<<grid_for(n * batch, 256), 256, 0, s>>>(src, out, n, batch, space);
  return cudaGetLastError();
}

static cudaError_t sdb_launch_task_sample_manual(cudaStream_t s, const float2 *src, size_t n, size_t batch, int space,
                                                 double sync, double delta, double samp_offset, float delta_inv,
                                                 long long count, float2 *out)
{
  if (count <= 0) return cudaSuccess;
  k_task_sample_manual<<<grid_for((size_t) count * batch, 128), 128, 0, s>>>(src, n, batch, space, sync, delta,
                                                                            samp_offset, delta_inv, count, out);
  return cudaGetLastError();
}

static cudaError_t sdb_launch_task_zero_crossing(cudaStream_t s, const float2 *src, size_t n, size_t batch, int space,
                                                 int amplitude, float thres, float2 zca, float bnor, unsigned char *ev,
                                                 size_t ev_pitch, unsigned char *sym, unsigned *counts, size_t cap)
{
  const size_t blocks = (n + TASK_BLOCK - 1) / TASK_BLOCK;
  k_task_zc_events<<<grid_for(blocks * batch, 64), 64, 0, s>>>(src, n, batch, blocks, space, amplitude, thres, zca,
                                                               ev, ev_pitch);
  k_task_zc_emit<<<grid_for(batch, 32), 32, 0, s>>>(ev, ev_pitch, n, batch, bnor, sym, counts, cap);
  return cudaGetLastError();
}

static cudaError_t sdb_launch_task_carrier_prep(cudaStream_t s, const float2 *src, const float *w, size_t n, size_t alloc,
                                                size_t batch, float2 *dst)
{
  k_task_carrier_prep<<<grid_for(alloc * batch, 256), 256, 0, s>>>(src, w, n, alloc, batch, dst);
  return cudaGetLastError();
}

static cudaError_t sdb_launch_task_carrier_find(cudaStream_t s, const float *psd, size_t alloc, size_t batch, int bins,
                                                int delta, int skip, float *peak)
{
  k_task_carrier_find<<<(unsigned) batch, 256, 0, s>>>(psd, (int) alloc, bins, delta, skip, peak);
  return cudaGetLastError();
}

static cudaError_t sdb_launch_task_decide(cudaStream_t s, const float2 *x, unsigned char *sym, size_t n, int mode, float dmin,
                                          float dh, int intervals)
{
  k_task_decide<<<grid_for(n, 256), 256, 0, s>>>(x, sym, n, mode, dmin, dh, intervals);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// DC removal of the source worker (suscan_analyzer_set_dc_remove, Suscan/Analyzer.cpp:229-236; SPEC R).  Block-wise
// single pole: every sample of block k has the estimate c_k subtracted (one binary32 subtraction per component),
// then c_{k+1} = c_k + alpha (m_k - c_k) with m_k the mean of the RAW block.  The mean is a fixed two-level sum in
// binary64 (runs of 256 samples in index order, then the run sums in index order), so it is reproducible bit for bit
// (oracle/tasks.c sdo_dc_remove).  Output: complex float32 (native formats are converted in the same load).
// ------------------------------------------------------------------------------------------------
#define DC_RUN 256
__global__ void k_dc_partial(const void *__restrict__ x, int fmt, size_t stream_stride, size_t n, size_t runs,
                             double2 *__restrict__ part)
{
  const size_t r = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  const int s = blockIdx.y;
  if (r >= runs) return;
  const char *xs = reinterpret_cast<const char *>(x) + (size_t) s * stream_stride * sdb_fmt_bytes(fmt);
  const size_t i0 = r * DC_RUN, i1 = i0 + DC_RUN < n ? i0 + DC_RUN : n;
  double ar = 0.0, ai = 0.0;
  for (size_t i = i0; i < i1; ++i) { const float2 v = sdb_ld_iq(xs, (long) i, fmt); ar += (double) v.x; ai += (double) v.y; }
  part[(size_t) s * runs + r] = make_double2(ar, ai);
}
// state[s] = {c.re, c.im}; cur[s] receives the estimate this block is corrected with
__global__ void k_dc_finish(const double2 *__restrict__ part, size_t runs, size_t n, float alpha, float2 *__restrict__ state,
                            float2 *__restrict__ cur, int n_streams)
{
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_streams) return;
  double ar = 0.0, ai = 0.0;
  for (size_t r = 0; r < runs; ++r) { const double2 p = part[(size_t) s * runs + r]; ar += p.x; ai += p.y; }
  const float mr = (float) (ar / (double) n), mi = (float) (ai / (double) n);
  const float2 c = state[s];
  cur[s] = c;
  state[s] = make_float2(c.x + alpha * (mr - c.x), c.y + alpha * (mi - c.y));
}
__global__ void k_dc_apply(const void *__restrict__ x, int fmt, size_t stream_stride, size_t n,
                           const float2 *__restrict__ cur, float2 *__restrict__ out)
{
  const size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  const int s = blockIdx.y;
  if (i >= n) return;
  const char *xs = reinterpret_cast<const char *>(x) + (size_t) s * stream_stride * sdb_fmt_bytes(fmt);
  const float2 v = sdb_ld_iq(xs, (long) i, fmt), c = cur[s];
  out[(size_t) s * n + i] = make_float2(v.x - c.x, v.y - c.y);
}
cudaError_t sdb_launch_dc_remove(cudaStream_t st, const void *x, int fmt, size_t stream_stride, size_t n, int n_streams,
                                 float alpha, float2 *state, float2 *cur, double2 *part, float2 *out)
{
  const size_t runs = (n + DC_RUN - 1) / DC_RUN;
  dim3 g1((unsigned) ((runs + 127) / 128), n_streams);
  k_dc_partial<<<g1, 128, 0, st>>>(x, fmt, stream_stride, n, runs, part);
  k_dc_finish<<<(n_streams + 63) / 64, 64, 0, st>>>(part, runs, n, alpha, state, cur, n_streams);
  dim3 g2((unsigned) ((n + 255) / 256), n_streams);
  k_dc_apply<<<g2, 256, 0, st>>>(x, fmt, stream_stride, n, cur, out);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// packed symbol read-out.  The inspector kernel leaves chain c's symbols at [c][0 .. counts[c]) of a [chains][cap]
// array (cap = channel samples per feed, the only static bound: the Gardner loop's baud is free in [0, 1]).  Copying
// the array wholesale moves cap / symbols-per-feed times more bytes over PCIe than there are symbols (cfg3: 3.1 x).
// k_sym_offsets lays the chains out back to back (each start rounded up to 16 symbols, so that every row of the
// copy starts on a 128-byte line of `soft` and a 16-byte word of `hard`); k_sym_pack then WRITES the packed rows
// straight into the destination -- pinned host memory mapped into the device's address space, or device memory --
// with 16-byte stores.  No size has to be known on the host before the copy, so the read stays asynchronous.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_sym_offsets(const uint32_t *__restrict__ counts, size_t chains,
                                                      unsigned long long *__restrict__ offsets)
{
  __shared__ unsigned long long warp_tot[32];
  __shared__ unsigned long long carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (size_t base = 0; base < chains; base += 1024) {
    const size_t c = base + threadIdx.x;
    const unsigned long long v = c < chains ? (unsigned long long) ((counts[c] + 15u) & ~15u) : 0ull;
    unsigned long long x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) warp_tot[warp] = x;
    __syncthreads();
    if (warp == 0) {
      unsigned long long t = warp_tot[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, t, d);
        if (lane >= d) t += y;
      }
      warp_tot[lane] = t;                                 // inclusive totals of the warps
    }
    __syncthreads();
    const unsigned long long before = carry + (warp ? warp_tot[warp - 1] : 0ull) + (x - v);
    if (c < chains) offsets[c] = before;
    __syncthreads();
    if (threadIdx.x == 1023) carry = before + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) offsets[chains] = carry;
}

__global__ void __launch_bounds__(128) k_sym_pack(const uint32_t *__restrict__ counts,
                                                  const unsigned long long *__restrict__ offsets, size_t chains,
                                                  const float2 *__restrict__ soft, const unsigned char *__restrict__ hard,
                                                  size_t cap, float4 *__restrict__ out_soft, uint4 *__restrict__ out_hard,
                                                  unsigned long long cap_total)
{
  for (size_t c = blockIdx.x; c < chains; c += gridDim.x) {
    const uint32_t cnt = counts[c];
    const unsigned long long off = offsets[c];            // multiple of 16
    const uint32_t padded = (cnt + 15u) & ~15u;
    if (off + padded > cap_total) continue;               // does not fit: the caller sees it from offsets[chains]
    if (out_soft) {
      const float2 *__restrict__ src = soft + c * cap;
      float4 *__restrict__ dst = out_soft + off / 2;
      for (uint32_t i = threadIdx.x; i < padded / 2; i += blockDim.x) {
        const uint32_t a = 2 * i, b = 2 * i + 1;
        const float2 u = a < cnt ? src[a] : make_float2(0.0f, 0.0f), v = b < cnt ? src[b] : make_float2(0.0f, 0.0f);
        dst[i] = make_float4(u.x, u.y, v.x, v.y);
      }
    }
    if (out_hard) {
      const unsigned char *__restrict__ src = hard + c * cap;
      uint4 *__restrict__ dst = out_hard + off / 16;
      for (uint32_t i = threadIdx.x; i < padded / 16; i += blockDim.x) {
        uint32_t w[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          uint32_t x = 0;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const uint32_t idx = 16 * i + 4 * k + j;
            x |= (idx < cnt ? (uint32_t) src[idx] : 0u) << (8 * j);
          }
          w[k] = x;
        }
        dst[i] = make_uint4(w[0], w[1], w[2], w[3]);
      }
    }
  }
}

cudaError_t sdb_launch_sym_pack(cudaStream_t stream, const uint32_t *counts, unsigned long long *offsets, size_t chains,
                                const float2 *soft, const unsigned char *hard, size_t cap, void *out_soft,
                                void *out_hard, unsigned long long cap_total, uint64_t *launch_counter)
{
  if (chains == 0) return cudaSuccess;
  k_sym_offsets<<<1, 1024, 0, stream>>>(counts, chains, offsets);
  const unsigned grid = (unsigned) (chains < 132 * 16 ? chains : 132 * 16);   // 16 CTAs on each of an H100's 132 SMs
  k_sym_pack<<<grid, 128, 0, stream>>>(counts, offsets, chains, soft, hard, cap, (float4 *) out_soft, (uint4 *) out_hard,
                                       cap_total);
  if (launch_counter) *launch_counter += 2;
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Tasks/ primitives: one thread per buffer of the batch, the recurrences of the inspector chains with the loop state
// in registers
// ---------------------------------------------------------------------------------------------
__global__ void k_task_xlate(const float2 *__restrict__ src, float2 *__restrict__ dst, size_t n, size_t batch,
                             float omega, float phi0)
{
  size_t b = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (b >= batch) return;
  float phi = phi0;
  const float2 *x = src + b * n;
  float2 *y = dst + b * n;
  for (size_t i = 0; i < n; ++i) {
    float2 ph = ncqo_read(phi, omega);
    float2 v = x[i];
    y[i] = make_float2(v.x * ph.x - v.y * ph.y, v.x * ph.y + v.y * ph.x);
  }
}

// quadrature demod has no loop-carried state beyond x[p-1]: fully parallel over samples
__global__ void k_task_quad(const float2 *__restrict__ src, float2 *__restrict__ dst, size_t n, size_t batch)
{
  size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (i >= n * batch) return;
  size_t p = i % n;
  if (p == 0) { dst[i] = make_float2(0.0f, 0.0f); return; }
  float2 x = src[i], pv = src[i - 1];
  float dr = x.x * pv.x + x.y * pv.y;
  float di = x.y * pv.x - x.x * pv.y;
  dst[i] = make_float2(0.0f, 0.318309886183790671538f * d_atan2f(di, dr));
}

struct CostasKS { CostasK k; CostasS s; };   // a Costas loop's coefficients and state

// mode 0 Costas (st: one CostasKS per buffer), 1 PLL (st: one {alpha, beta, phi, omega} per buffer).  The loop state
// is read at the start and written back at the end, so that a Tasks/ work() block continues where the previous one
// stopped (the bulk twins of su_costas_feed / su_pll_track).
__global__ void k_task_loop(const float2 *__restrict__ src, float2 *__restrict__ dst, size_t n, size_t batch, int mode,
                            void *__restrict__ st)
{
  size_t b = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const float2 *x = src + b * n;
  float2 *y = dst + b * n;
  if (mode == 0) {
    CostasKS *q = (CostasKS *) st + b;
    const CostasK ck = q->k;
    CostasS cs = q->s;
    for (size_t i = 0; i < n; ++i) y[i] = costas_step(ck, cs, x[i]);
    q->s = cs;
  } else {
    float4 *q = (float4 *) st + b;
    const float a = q->x, be = q->y;
    float phi = q->z, omega = q->w;
    for (size_t i = 0; i < n; ++i) y[i] = pll_step(a, be, phi, omega, x[i]);
    q->z = phi; q->w = omega;
  }
}

// AGC from its zero start state.  pool: per buffer the delay line (2 dl_size floats) then the magnitude history
// (mh_size), interleaved by 32 buffers ([slot][lane]).
__global__ void k_task_agc(const float2 *__restrict__ src, float2 *__restrict__ dst, size_t n, size_t batch, AgcK ak,
                           float *pool)
{
  size_t b = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const float2 *x = src + b * n;
  float2 *y = dst + b * n;
  AgcS as;
  as.fast = as.slow = as.peak = -160.0f; as.hang_n = as.dl_ptr = as.mh_ptr = 0;
  float *dl = pool + (b / 32) * 32 * (2 * ak.dl_size + ak.mh_size) + (b % 32), *mh = dl + (size_t) 2 * ak.dl_size * 32;
  for (unsigned i = 0; i < 2 * ak.dl_size; ++i) dl[i * 32] = 0.0f;
  for (unsigned i = 0; i < ak.mh_size; ++i) mh[i * 32] = -160.0f;
  for (size_t i = 0; i < n; ++i) y[i] = agc_step(ak, as, dl, mh, x[i]);
}

// ---------------------------------------------------------------------------------------------
// host side of the tasks: host buffers in and out
// ---------------------------------------------------------------------------------------------
// the task's input on the device (batch buffers of n samples), and an output buffer of the same size when y is given
static int task_in(DevBuf<float2> &x, DevBuf<float2> *y, const sdb_complex *src, size_t n, size_t batch)
{
  if (!src || n == 0 || batch == 0) return fail("invalid task buffer");
  if (sdb_device_count() <= 0) return fail("no CUDA device: sigdigger_b200 has no CPU fallback");
  CK(x.alloc(n * batch));
  if (y) CK(y->alloc(n * batch));
  CK(cudaMemcpy(x, src, n * batch * sizeof(float2), cudaMemcpyHostToDevice));
  return 0;
}

// the first `count` elements of a task's output, once the launches before have finished
template <typename T> static int task_out(void *dst, const DevBuf<T> &d, size_t count)
{
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(dst, d, count * sizeof(T), cudaMemcpyDeviceToHost));
  return 0;
}

// k_task_loop over the input x (task_in) into y, then y to dst; st: batch loop states of st_bytes each, updated in place
static int task_loop(const DevBuf<float2> &x, const DevBuf<float2> &y, sdb_complex *dst, size_t n, size_t batch,
                     int mode, void *st, size_t st_bytes)
{
  DevBuf<unsigned char> d_st;
  CK(d_st.alloc(batch * st_bytes));
  CK(cudaMemcpy(d_st, st, batch * st_bytes, cudaMemcpyHostToDevice));
  k_task_loop<<<(unsigned) ((batch + 31) / 32), 32>>>(x, y, n, batch, mode, d_st);
  CK(cudaGetLastError());
  if (task_out(dst, y, n * batch)) return -1;
  CK(cudaMemcpy(st, d_st, batch * st_bytes, cudaMemcpyDeviceToHost));
  return 0;
}

// the same with every buffer starting from the loop state s0
template <typename S> static int task_loop_from(const DevBuf<float2> &x, const DevBuf<float2> &y, sdb_complex *dst,
                                                size_t n, size_t batch, int mode, const S &s0)
{
  std::vector<S> st;
  try { st.assign(batch, s0); } catch (const std::bad_alloc &) { return fail("out of host memory"); }
  return task_loop(x, y, dst, n, batch, mode, st.data(), sizeof(S));
}

extern "C" int sdb_task_carrier_xlate(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch,
                                      float rel_freq, float phase)
{
  DevBuf<float2> x, y;
  if (task_in(x, &y, src, n, batch)) return -1;
  // su_ncqo_init(-relFreq); su_ncqo_set_phase(-phase)   (Tasks/CarrierXlator.cpp:36-37)
  float omega = 3.14159265358979323846f * (-rel_freq);
  float phi = -phase;
  phi = phi - 6.28318530717958647692f * floorf(phi / 6.28318530717958647692f);
  if (phi >= 6.28318530717958647692f) phi = 0.0f;
  k_task_xlate<<<(unsigned) ((batch + 31) / 32), 32>>>(x, y, n, batch, omega, phi);
  CK(cudaGetLastError());
  return task_out(dst, y, n * batch);
}

extern "C" int sdb_task_quad_demod(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch)
{
  DevBuf<float2> x, y;
  if (task_in(x, &y, src, n, batch)) return -1;
  k_task_quad<<<(unsigned) ((n * batch + 255) / 256), 256>>>(x, y, n, batch);
  CK(cudaGetLastError());
  return task_out(dst, y, n * batch);
}

extern "C" int sdb_task_costas(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch, int kind,
                               float tau, float loop_bw)
{
  if (kind < 1 || kind > 3) return fail("invalid Costas kind");
  DevBuf<float2> x, y;
  if (task_in(x, &y, src, n, batch)) return -1;
  // su_costas_init(&costas, kind, 0, 1/tau, 3, loopbw)   (Tasks/CostasRecoveryTask.cpp:36-41), from the zero state
  CostasKS c;
  memset(&c, 0, sizeof(c));
  c.k.kind = kind;
  c.k.a = 3.14159265358979323846f * loop_bw;
  c.k.b = 0.5f * c.k.a * c.k.a;
  if (!sdbh::butter_lp(2, 1.0f / tau, c.k.af_b, c.k.af_a)) return fail("invalid arm bandwidth");
  c.k.af_n = 3;
  return task_loop_from(x, y, dst, n, batch, 0, c);
}

extern "C" int sdb_task_pll(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch, float bw)
{
  DevBuf<float2> x, y;
  if (task_in(x, &y, src, n, batch)) return -1;
  float fc = 3.14159265358979323846f * bw;
  float dinv = 1.0f / (1.0f + 2.0f * 0.707f * fc + fc * fc);
  return task_loop_from(x, y, dst, n, batch, 1,
                        make_float4(4.0f * fc * fc * dinv, 4.0f * 0.707f * fc * dinv, 0.0f, 0.0f));
}

extern "C" int sdb_task_agc(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch, float tau)
{
  DevBuf<float2> x, y;
  DevBuf<float> pool;
  if (task_in(x, &y, src, n, batch)) return -1;
  // AGCTask sets only the five time constants; delay line / history keep the defaults (20)
  // (Tasks/AGCTask.cpp:43-47 and the comment in SURVEY.md 8a row a6)
  const sdbh::AgcDesign d = sdbh::agc_from_tau(tau, 2.0f);
  const AgcK k = { d.knee, d.gain_slope - 1.0f, d.fixed_gain, d.far_, d.faf, d.sar, d.saf, d.hang_max, 20, 20 };
  CK(pool.alloc(((batch + 31) / 32) * 32 * (2 * k.dl_size + k.mh_size)));
  k_task_agc<<<(unsigned) ((batch + 31) / 32), 32>>>(x, y, n, batch, k, pool);
  CK(cudaGetLastError());
  return task_out(dst, y, n * batch);
}

// ---- bulk twins of the per-sample sigutils calls: one buffer, continuing from (and returning) the caller's loop state
static int task_state(const sdb_complex *src, sdb_complex *dst, size_t n, int mode, void *st, size_t st_bytes)
{
  if (!src || !dst || !st) return fail("null argument");
  if (sdb_device_count() <= 0) return fail("no CUDA device: sigdigger_b200 has no CPU fallback");
  if (n == 0) return 0;
  DevBuf<float2> x, y;
  if (task_in(x, &y, src, n, 1)) return -1;
  return task_loop(x, y, dst, n, 1, mode, st, st_bytes);
}
extern "C" int sdb_task_costas_state(const sdb_complex *src, sdb_complex *dst, size_t n, const void *k, size_t k_bytes,
                                     void *s, size_t s_bytes)
{
  if (k_bytes != sizeof(CostasK) || s_bytes != sizeof(CostasS)) return fail("costas state size mismatch");
  CostasKS st;
  memcpy(&st.k, k, k_bytes); memcpy(&st.s, s, s_bytes);
  if (task_state(src, dst, n, 0, &st, sizeof(st))) return -1;
  memcpy(s, &st.s, s_bytes);
  return 0;
}
extern "C" int sdb_task_pll_state(const sdb_complex *src, sdb_complex *dst, size_t n, float alpha, float beta,
                                  float state[2])
{
  float4 st = make_float4(alpha, beta, state[0], state[1]);
  if (task_state(src, dst, n, 1, &st, sizeof(st))) return -1;
  state[0] = st.z; state[1] = st.w;
  return 0;
}

// ---- TimeWindow tasks that are fully specified in-repo (SPEC Y)
extern "C" int sdb_task_delayed_conj(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch, size_t delay)
{
  if (delay == 0) return fail("Delay is zero samples");   // DelayedConjTask.cpp:36-37
  if (!dst) return fail("null argument");
  DevBuf<float2> x, y;
  if (task_in(x, &y, src, n, batch)) return -1;
  CK(sdb_launch_task_delayed_conj(0, x, y, n, batch, delay));
  return task_out(dst, y, n * batch);
}

extern "C" long sdb_task_histogram_feed(const sdb_complex *src, float *out, size_t n, size_t batch, int space)
{
  if (!out) return fail("null argument");
  if (space < SDB_SPACE_AMPLITUDE || space > SDB_SPACE_FREQUENCY) return fail("unknown decision space");
  DevBuf<float2> x;
  DevBuf<float> o;
  if (task_in(x, nullptr, src, n, batch)) return -1;
  const size_t count = space == SDB_SPACE_FREQUENCY ? n - 1 : n;
  if (count == 0) return 0;
  CK(o.alloc(count * batch));
  CK(sdb_launch_task_hist(0, x, o, n, batch, space));
  if (task_out(out, o, count * batch)) return -1;
  return (long) count;
}

extern "C" long sdb_task_sample_manual(const sdb_complex *src, size_t n, size_t batch, int space, size_t symbol_sync,
                                       double symbol_count, sdb_complex *out)
{
  if (!out) return fail("null argument");
  if (space < SDB_SPACE_AMPLITUDE || space > SDB_SPACE_FREQUENCY) return fail("unknown decision space");
  if (!(symbol_count >= 1.0) || symbol_count > (double) n) return fail("symbol_count must be in [1, n]");
  DevBuf<float2> x, o;
  if (task_in(x, nullptr, src, n, batch)) return -1;
  // WaveSampler.cpp:44-45: delta = length / symbolCount; sampOffset = symbolSync / delta
  const double delta = (double) n / symbol_count;
  const double samp_offset = (double) symbol_sync / delta;
  const float delta_inv = 1.f / (float) delta;
  const long long count = (long long) symbol_count;
  CK(o.alloc((size_t) count * batch));
  CK(sdb_launch_task_sample_manual(0, x, n, batch, space, (double) symbol_sync, delta, samp_offset, delta_inv, count,
                                   o));
  if (task_out(out, o, (size_t) count * batch)) return -1;
  return (long) count;
}

extern "C" int sdb_task_sample_zero_crossing(const sdb_complex *src, size_t n, size_t batch, int space, int amplitude,
                                             float threshold_re, float threshold_im, float zc_angle_re,
                                             float zc_angle_im, float bnor, uint8_t *sym, uint32_t *counts, size_t cap)
{
  if (!sym || !counts || cap == 0) return fail("null argument");
  if (space < SDB_SPACE_AMPLITUDE || space > SDB_SPACE_FREQUENCY) return fail("unknown decision space");
  if (!(bnor > 0.0f)) return fail("bnor must be positive");
  if (bnor > 1.0f) bnor = 1.0f;                            // WaveSampler.cpp:50-51
  DevBuf<float2> x;
  DevBuf<unsigned char> ev, o;
  DevBuf<unsigned> c;
  if (task_in(x, nullptr, src, n, batch)) return -1;
  const size_t pitch = (n + 15) & ~(size_t) 15;
  CK(ev.alloc(pitch * batch));
  CK(o.alloc(cap * batch));
  CK(c.alloc(batch));
  CK(cudaMemset(o, 0, cap * batch));
  // WaveSampler.cpp:236-241
  const float thres = amplitude ? threshold_re * threshold_re + threshold_im * threshold_im
                                : threshold_re * zc_angle_re - threshold_im * zc_angle_im;
  CK(sdb_launch_task_zero_crossing(0, x, n, batch, space, amplitude ? 1 : 0, thres,
                                   make_float2(zc_angle_re, zc_angle_im), bnor, ev, pitch, o, c, cap));
  if (task_out(sym, o, cap * batch)) return -1;
  CK(cudaMemcpy(counts, c, batch * sizeof(unsigned), cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int sdb_task_carrier_detect(const sdb_complex *src, size_t n, size_t batch, double avg_rel_bw,
                                       double dc_notch_rel_bw, float *peak)
{
  if (!peak) return fail("null argument");
  if (n > ((size_t) 1 << 20)) return fail("carrier detector: at most 2^20 samples");
  if (!(avg_rel_bw >= 0.0 && avg_rel_bw <= 1.0)) return fail("avg_rel_bw must be in [0, 1]");
  if (!(dc_notch_rel_bw >= 0.0)) dc_notch_rel_bw = 0.0;   // qBound(0., x, 1.), CarrierDetector.cpp:35
  if (dc_notch_rel_bw > 1.0) dc_notch_rel_bw = 1.0;
  DevBuf<float2> x, buf;
  DevBuf<float> w, pk;
  if (task_in(x, nullptr, src, n, batch)) return -1;
  size_t alloc = 64;                                        // SPEC Y.5: transform size >= 64
  while (alloc < n) alloc <<= 1;
  std::vector<float> win;
  sdbh::window_fill(win, (unsigned) n, SDB_WINDOW_BLACKMANN_HARRIS);
  CK(w.alloc(n));
  CK(cudaMemcpy(w, win.data(), n * sizeof(float), cudaMemcpyHostToDevice));
  CK(buf.alloc(alloc * batch));
  CK(pk.alloc(batch));
  CK(sdb_launch_task_carrier_prep(0, x, w, n, alloc, batch, buf));
  CK(cudaDeviceSynchronize());
  // the transform is the engine's own PSD (rectangular window: the taps are already applied)
  sdb_engine_params prm; memset(&prm, 0, sizeof(prm));
  prm.n_streams = (uint32_t) batch; prm.psd_size = (uint32_t) alloc; prm.psd_window = SDB_WINDOW_NONE;
  prm.max_feed = (uint32_t) alloc;
  sdb_engine_t *e = sdb_engine_new(&prm, 1.0);
  if (!e) return -1;
  int rc = sdb_engine_commit(e);
  if (!rc) rc = sdb_engine_feed_device(e, (const sdb_complex *) buf.get(), alloc, alloc);
  if (!rc) rc = sdb_engine_sync(e);
  if (!rc) {
    const int bins = (int) ((double) alloc * avg_rel_bw) + 1;
    const int skip = (int) (.5 * dc_notch_rel_bw * (double) alloc);
    cudaError_t ce = sdb_launch_task_carrier_find(0, sdb_engine_psd_device(e), alloc, batch, bins, (bins - 1) / 2, skip,
                                                  pk);
    if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
    if (ce == cudaSuccess) ce = cudaMemcpy(peak, pk, batch * sizeof(float), cudaMemcpyDeviceToHost);
    if (ce != cudaSuccess) { g_err = std::string("carrier detector: ") + cudaGetErrorString(ce); rc = -1; }
  }
  sdb_engine_destroy(e);
  return rc;
}

extern "C" int sdb_task_decide(const sdb_complex *soft, uint8_t *sym, size_t n, int mode, unsigned bps, float min,
                               float max)
{
  if (!sym) return fail("null argument");
  if (mode < 0 || mode > 1 || bps < 1 || bps > 8 || !(max > min)) return fail("invalid decider");
  DevBuf<float2> x;
  DevBuf<unsigned char> o;
  if (task_in(x, nullptr, soft, n, 1)) return -1;
  CK(o.alloc(n));
  CK(sdb_launch_task_decide(0, x, o, n, mode, min, max - min, 1 << bps));
  return task_out(sym, o, n);
}

extern "C" int sdb_task_lpf(const sdb_complex *src, sdb_complex *dst, size_t n, size_t batch, float bw)
{
  // LPFTask: specttuner with the default 4096-sample window, one channel at f0 = 0 with
  // guard = 2 pi / bw (no decimation), input flushed with zeros until n outputs exist
  // (Tasks/LPFTask.cpp:52-69,104-107).
  if (!src || !dst || n == 0 || batch == 0) return fail("invalid task buffer");
  const unsigned W = 4096;   // sigutils_specttuner_params_INITIALIZER default window (SURVEY.md A.2)
  sdb_engine_params p; memset(&p, 0, sizeof(p));
  size_t padded = ((n + W / 2 + W / 2 - 1) / (W / 2)) * (W / 2);   // + half-window latency, rounded up
  p.n_streams = (uint32_t) batch; p.psd_size = 0; p.st_window_size = W; p.max_feed = (uint32_t) padded; p.device = 0;
  int dev = 0; cudaGetDevice(&dev); p.device = dev;
  sdb_engine_t *e = sdb_engine_new(&p, 1.0);
  if (!e) return -1;
  sdb_channel_params cp; cp.f0 = 0.0f; cp.bw = 3.14159265358979323846f * bw; cp.guard = 6.28318530717958647692f / cp.bw;
  cp.precise = 0;
  int rc = -1;
  std::vector<float2> in(batch * padded, make_float2(0.f, 0.f)), out(padded);
  for (size_t b = 0; b < batch; ++b) memcpy(&in[b * padded], src + b * n, n * sizeof(float2));
  do {
    int h = sdb_engine_open_channel(e, &cp, nullptr);
    if (h < 0) break;
    if (sdb_engine_commit(e)) break;
    if (sdb_engine_feed_host(e, reinterpret_cast<const sdb_complex *>(in.data()), padded, padded)) break;
    bool ok = true;
    for (size_t b = 0; b < batch && ok; ++b) {
      long got = sdb_engine_read_channel(e, (uint32_t) b, h, reinterpret_cast<sdb_complex *>(out.data()), padded);
      if (got < (long) n) { g_err = "lpf produced too few samples"; ok = false; break; }
      memcpy(dst + b * n, out.data(), n * sizeof(float2));
    }
    if (ok) rc = 0;
  } while (0);
  sdb_engine_destroy(e);
  return rc;
}

// ---- SNR estimator on the inspectors' decision-space histograms (Misc/SNREstimator.cpp; SPEC Y.7)
struct sdb_snr_estimator {
  int device = 0; unsigned n = 0, length = 0;
  std::vector<SdbSnrState> st; std::vector<unsigned> bps;
  bool dirty = true;                       // host copy of the states newer than the device copy
  DevBuf<unsigned> d_hist; DevBuf<SdbSnrState> d_states; DevBuf<float> d_work;   // gaussian | hi | htilde | term
};

extern "C" sdb_snr_estimator_t *sdb_snr_estimator_new(uint32_t n_estimators, uint32_t length, int device)
{
  if (sdb_device_count() <= 0) { g_err = "no CUDA device: sigdigger_b200 has no CPU fallback"; return nullptr; }
  if (n_estimators == 0 || length == 0) { g_err = "snr estimator: empty geometry"; return nullptr; }
  CKP(cudaSetDevice(device));
  sdb_snr_estimator *e = new sdb_snr_estimator();
  e->device = device; e->n = n_estimators; e->length = length;
  e->st.assign(n_estimators, SdbSnrState{ 1.f / 8.f, 1.f, 0.f, 0u });   // SNR_ESTIMATOR_DEFAULT_SIGMA / _ALPHA
  e->bps.assign(n_estimators, 0u);
  const size_t tot = (size_t) n_estimators * length;
  if (e->d_hist.alloc(tot) != cudaSuccess || e->d_states.alloc(n_estimators) != cudaSuccess ||
      e->d_work.alloc(4 * tot) != cudaSuccess) {
    g_err = "out of device memory"; delete e; return nullptr;
  }
  cudaMemset(e->d_work, 0, 4 * tot * sizeof(float));
  return e;
}

extern "C" void sdb_snr_estimator_destroy(sdb_snr_estimator_t *e)
{
  if (!e) return;
  cudaSetDevice(e->device);
  delete e;
}

static int snr_pull(sdb_snr_estimator *e)
{
  if (e->dirty) return 0;
  CK(cudaSetDevice(e->device));
  CK(cudaMemcpy(e->st.data(), e->d_states, e->n * sizeof(SdbSnrState), cudaMemcpyDeviceToHost));
  return 0;
}

// setBps (SNREstimator.cpp:122-131): a change of bps restarts sigma
extern "C" int sdb_snr_estimator_set_bps(sdb_snr_estimator_t *e, uint32_t index, uint32_t bps)
{
  if (!e || index >= e->n) return fail("wrong estimator index");
  if (bps > 8) return fail("bps out of range");
  if (snr_pull(e)) return -1;
  if (e->bps[index] != bps) {                  // as the reference: setBps(0) on a fresh estimator leaves it idle
    e->bps[index] = bps; e->st[index].sigma = 1.f / 8.f; e->st[index].intervals = 1u << bps;
  }
  e->dirty = true;
  return 0;
}

extern "C" int sdb_snr_estimator_set_alpha(sdb_snr_estimator_t *e, uint32_t index, float alpha)
{
  if (!e || index >= e->n) return fail("wrong estimator index");
  if (snr_pull(e)) return -1;
  e->st[index].alpha = alpha; e->dirty = true;
  return 0;
}

extern "C" int sdb_snr_estimator_set_sigma(sdb_snr_estimator_t *e, uint32_t index, float sigma)
{
  if (!e || index >= e->n) return fail("wrong estimator index");
  if (snr_pull(e)) return -1;
  e->st[index].sigma = sigma; e->dirty = true;
  return 0;
}

// feed (SNREstimator.cpp:133-158) for every estimator: histories [n][length] counts, host memory
extern "C" int sdb_snr_estimator_feed(sdb_snr_estimator_t *e, const uint32_t *histories)
{
  if (!e || !histories) return fail("null argument");
  CK(cudaSetDevice(e->device));
  const size_t tot = (size_t) e->n * e->length;
  if (e->dirty) {
    CK(cudaMemcpy(e->d_states, e->st.data(), e->n * sizeof(SdbSnrState), cudaMemcpyHostToDevice));
    e->dirty = false;
  }
  CK(cudaMemcpy(e->d_hist, histories, tot * sizeof(unsigned), cudaMemcpyHostToDevice));
  CK(sdb_launch_snr_feed(0, e->d_hist, e->length, e->n, e->d_states, e->d_work, e->d_work + tot, e->d_work + 2 * tot,
                         e->d_work + 3 * tot));
  CK(cudaDeviceSynchronize());
  return 0;
}

// getSigma / getSNR (include/SNREstimator.h:74-84) and getModel (:61-65); any pointer may be NULL
extern "C" int sdb_snr_estimator_read(sdb_snr_estimator_t *e, float *sigma, float *snr, float *model)
{
  if (!e) return fail("null argument");
  if (snr_pull(e)) return -1;
  for (unsigned i = 0; i < e->n; ++i) {
    if (sigma) sigma[i] = e->st[i].sigma;
    if (snr) snr[i] = 1.f / (e->st[i].intervals * e->st[i].sigma);
  }
  if (model) {
    const size_t tot = (size_t) e->n * e->length;
    CK(cudaSetDevice(e->device));
    CK(cudaMemcpy(model, e->d_work + tot, tot * sizeof(float), cudaMemcpyDeviceToHost));
  }
  return 0;
}
