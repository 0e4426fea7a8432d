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
// Compiled with -fmad=false: float and double expressions round exactly as written.
#include "sdb_internal.h"
#include "sdb_math.h"

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

// SNR estimator of the inspector's decision-space histogram (Misc/SNREstimator.cpp:30-169; SPEC Y.7): one CTA per
// estimator.  The model (a comb of 2^bps Gaussians) is built bin-parallel -- every bin's sum over the intervals keeps
// the reference's order --; the two order-dependent reductions (the maximum is order-free, the gradient sum is not)
// are done by thread 0 in bin order.  expf(t) = 10^(t log10 e) of SPEC M.
struct SdbSnrState { float sigma, alpha, delta; unsigned intervals; };

__global__ void __launch_bounds__(256) k_snr_feed(const unsigned *__restrict__ history, unsigned length,
                                                  SdbSnrState *__restrict__ states, float *__restrict__ gaussian,
                                                  float *__restrict__ hi, float *__restrict__ htilde,
                                                  float *__restrict__ term)
{
  const unsigned b = blockIdx.x;
  const unsigned *__restrict__ h = history + (size_t) b * length;
  float *__restrict__ g = gaussian + (size_t) b * length, *__restrict__ H = hi + (size_t) b * length;
  float *__restrict__ Ht = htilde + (size_t) b * length, *__restrict__ T = term + (size_t) b * length;
  __shared__ unsigned s_max;
  __shared__ float s_fmax;
  const SdbSnrState st = states[b];
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
    states[b].delta = delta;
    states[b].sigma = st.sigma + -st.alpha * delta;
  }
}

cudaError_t sdb_launch_snr_feed(cudaStream_t s, const unsigned *history, unsigned length, unsigned n, void *states,
                                float *gaussian, float *hi, float *htilde, float *term)
{
  if (n == 0 || length == 0) return cudaSuccess;
  k_snr_feed<<<n, 256, 0, s>>>(history, length, (SdbSnrState *) states, gaussian, hi, htilde, term);
  return cudaGetLastError();
}

static inline unsigned grid_for(size_t total, unsigned threads) { return (unsigned) ((total + threads - 1) / threads); }

cudaError_t sdb_launch_task_delayed_conj(cudaStream_t s, const float2 *src, float2 *dst, size_t n, size_t batch,
                                         size_t delay)
{
  k_task_delayed_conj<<<grid_for(n * batch, 256), 256, 0, s>>>(src, dst, n, batch, delay);
  return cudaGetLastError();
}

cudaError_t sdb_launch_task_hist(cudaStream_t s, const float2 *src, float *out, size_t n, size_t batch, int space)
{
  k_task_hist<<<grid_for(n * batch, 256), 256, 0, s>>>(src, out, n, batch, space);
  return cudaGetLastError();
}

cudaError_t sdb_launch_task_sample_manual(cudaStream_t s, const float2 *src, size_t n, size_t batch, int space,
                                          double sync, double delta, double samp_offset, float delta_inv,
                                          long long count, float2 *out)
{
  if (count <= 0) return cudaSuccess;
  k_task_sample_manual<<<grid_for((size_t) count * batch, 128), 128, 0, s>>>(src, n, batch, space, sync, delta,
                                                                            samp_offset, delta_inv, count, out);
  return cudaGetLastError();
}

cudaError_t sdb_launch_task_zero_crossing(cudaStream_t s, const float2 *src, size_t n, size_t batch, int space,
                                          int amplitude, float thres, float2 zca, float bnor, unsigned char *ev,
                                          size_t ev_pitch, unsigned char *sym, unsigned *counts, size_t cap)
{
  const size_t blocks = (n + TASK_BLOCK - 1) / TASK_BLOCK;
  k_task_zc_events<<<grid_for(blocks * batch, 64), 64, 0, s>>>(src, n, batch, blocks, space, amplitude, thres, zca,
                                                               ev, ev_pitch);
  k_task_zc_emit<<<grid_for(batch, 32), 32, 0, s>>>(ev, ev_pitch, n, batch, bnor, sym, counts, cap);
  return cudaGetLastError();
}

cudaError_t sdb_launch_task_carrier_prep(cudaStream_t s, const float2 *src, const float *w, size_t n, size_t alloc,
                                         size_t batch, float2 *dst)
{
  k_task_carrier_prep<<<grid_for(alloc * batch, 256), 256, 0, s>>>(src, w, n, alloc, batch, dst);
  return cudaGetLastError();
}

cudaError_t sdb_launch_task_carrier_find(cudaStream_t s, const float *psd, size_t alloc, size_t batch, int bins,
                                         int delta, int skip, float *peak)
{
  k_task_carrier_find<<<(unsigned) batch, 256, 0, s>>>(psd, (int) alloc, bins, delta, skip, peak);
  return cudaGetLastError();
}

cudaError_t sdb_launch_task_decide(cudaStream_t s, const float2 *x, unsigned char *sym, size_t n, int mode, float dmin,
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
