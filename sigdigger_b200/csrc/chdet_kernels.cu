// chdet_kernels.cu -- channel detector on the main PSD (SPEC.md section K, SURVEY.md 8(f) rank 3).
//
// Replaces what su_channel_detector contributes to the analyzer loop: detector_params.{alpha, gamma, snr}
// (Suscan/AnalyzerParams.cpp:27-66) in, lists of struct sigutils_channel {fc, f_lo, f_hi, bw, snr, S0, N0}
// (Suscan/Messages/ChannelMessage.cpp:25-70, include/Suscan/Channel.h:26-32) out, once per feed
// (channel_update_int).  The upstream algorithm is not in the reference; SPEC K is this project's definition and
// is order-independent on purpose (exact order statistic instead of a mean, maxima instead of sums), so this
// parallel implementation is bit-identical to oracle/chdetect.c.
//
//   k_chdet_avg : one thread per (bin, stream): exponential average over the feed's frames, in frame order.
//   k_chdet_find: one 1024-thread CTA per stream: exact (N/4)-th smallest averaged bin by a 4-pass radix select on
//                 the float bit patterns (shared-memory histogram), noise-floor update, threshold, run detection
//                 with block scans (ordered start / end events in shared memory), width filter + ordered
//                 compaction, per-channel maximum by one warp per channel.
#include "sdb_internal.h"
#include "../../include/sigdigger_b200.h"
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>

#define CHDET_MAXRAW 8192      // raw runs examined per update (SPEC K.4)
#define CHDET_CAP    256       // channels reported per stream

struct SdbDetectedDev { unsigned bin_lo, bin_hi; float s0, n0, snr; };

__global__ void k_chdet_avg(float *__restrict__ avg, const float *__restrict__ psd, int N, int frames,
                            size_t stream_stride, float alpha, int primed)
{
  const int k = blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y;
  if (k >= N) return;
  const float *__restrict__ p = psd + (size_t) s * stream_stride + k;
  float a = avg[(size_t) s * N + k];
  int f = 0;
  if (!primed) { a = p[0]; f = 1; }
  for (; f < frames; ++f) a = a + alpha * (p[(size_t) f * N] - a);
  avg[(size_t) s * N + k] = a;
}

// exclusive scan of one int per thread over a 1024-thread CTA; *total = sum.  s_w: 32 ints of scratch.
static __device__ int block_excl_scan(int v, int *total, int *s_w)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_w[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = s_w[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += t;
    }
    s_w[lane] = w;
  }
  __syncthreads();
  const int off = warp ? s_w[warp - 1] : 0;
  *total = s_w[31];
  __syncthreads();
  return off + incl - v;
}

struct ChdetK {
  const float *avg; float *n0; int *n0_primed;
  int N; float gamma, snr; int min_bins;
  SdbDetectedDev *out; unsigned *count, *total;
};

__global__ void __launch_bounds__(1024) k_chdet_find(const ChdetK p)
{
  extern __shared__ int s_ev[];                 // starts[CHDET_MAXRAW], ends[CHDET_MAXRAW]
  int *starts = s_ev, *ends = s_ev + CHDET_MAXRAW;
  __shared__ unsigned hist[256];
  __shared__ unsigned s_bucket, s_rank;
  __shared__ int s_w[32];
  __shared__ float s_n0;
  const int tid = threadIdx.x, st = blockIdx.x, N = p.N, half = N >> 1;
  const float *__restrict__ avg = p.avg + (size_t) st * N;

  // ---- K.2: exact (N/4)-th smallest value (non-negative floats order like their bit patterns)
  unsigned prefix = 0, mask = 0, rank = (unsigned) N / 4;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < N; i += 1024) {
      const unsigned u = __float_as_uint(avg[i]);
      if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      unsigned cum = 0, b = 0;
      for (; b < 255; ++b) { if (cum + hist[b] > rank) break; cum += hist[b]; }
      s_bucket = b; s_rank = rank - cum;
    }
    __syncthreads();
    prefix |= s_bucket << shift; mask |= 0xffu << shift; rank = s_rank;
    __syncthreads();
  }
  if (tid == 0) {
    const float inst = __uint_as_float(prefix);
    float n0 = p.n0[st];
    n0 = p.n0_primed[st] ? n0 + p.gamma * (inst - n0) : inst;
    p.n0[st] = n0; p.n0_primed[st] = 1;
    s_n0 = n0;
  }
  __syncthreads();
  const float n0 = s_n0, thr = n0 * p.snr;

  // ---- K.3: start / end events of the runs above the threshold, ascending frequency j = (k + N/2) mod N
  const int L = (N + 1023) / 1024;
  const int i0 = min(tid * L, N), i1 = min(i0 + L, N);
  int ns = 0, ne = 0;
  {
    bool prev = i0 > 0 && i0 < N && avg[(i0 - 1 + half) & (N - 1)] > thr;
    for (int i = i0; i < i1; ++i) {
      const bool cur = avg[(i + half) & (N - 1)] > thr;
      ns += cur && !prev; ne += !cur && prev;
      prev = cur;
    }
    if (i1 == N && i0 < N && prev) ++ne;       // a run that reaches the top edge ends at N
  }
  int tot_s, tot_e;
  int os = block_excl_scan(ns, &tot_s, s_w);
  int oe = block_excl_scan(ne, &tot_e, s_w);
  {
    bool prev = i0 > 0 && i0 < N && avg[(i0 - 1 + half) & (N - 1)] > thr;
    for (int i = i0; i < i1; ++i) {
      const bool cur = avg[(i + half) & (N - 1)] > thr;
      if (cur && !prev) { if (os < CHDET_MAXRAW) starts[os] = i; ++os; }
      if (!cur && prev) { if (oe < CHDET_MAXRAW) ends[oe] = i; ++oe; }
      prev = cur;
    }
    if (i1 == N && i0 < N && prev) { if (oe < CHDET_MAXRAW) ends[oe] = N; ++oe; }
  }
  __syncthreads();
  const int R = min(tot_s, CHDET_MAXRAW);

  // ---- K.4: width filter + ordered compaction
  SdbDetectedDev *__restrict__ out = p.out + (size_t) st * CHDET_CAP;
  int running = 0;
  for (int base = 0; base < R; base += 1024) {
    const int r = base + tid;
    const int keep = r < R && ends[r] - starts[r] >= p.min_bins;
    int tile;
    const int pos = running + block_excl_scan(keep, &tile, s_w);
    if (keep && pos < CHDET_CAP) { out[pos].bin_lo = (unsigned) starts[r]; out[pos].bin_hi = (unsigned) ends[r]; }
    running += tile;
  }
  __syncthreads();
  const int nch = min(running, CHDET_CAP);
  if (tid == 0) { p.count[st] = (unsigned) nch; p.total[st] = (unsigned) running; }
  // ---- peak level of every reported channel: one warp per channel
  for (int c = tid >> 5; c < nch; c += 32) {
    const int a = (int) out[c].bin_lo, b = (int) out[c].bin_hi;
    float m = 0.0f;
    for (int i = a + (tid & 31); i < b; i += 32) m = fmaxf(m, avg[(i + half) & (N - 1)]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) { out[c].s0 = m; out[c].n0 = n0; out[c].snr = m / n0; }
  }
}

// ---- fused detector for 2048 <= N <= 65536 (the sizes the analyzer and the panoramic sweep run): one 1024-thread
// ---- CTA per stream keeps the stream's averaged spectrum in REGISTERS (N / 1024 <= 64 values per thread, element
// ---- k = r * 1024 + tid) from the exponential average (K.1, same expression and frame order as k_chdet_avg) through
// ---- the four radix-select passes (K.2); the threshold test leaves a bit map in frequency order in shared memory
// ---- (warp votes; ascending frequency j = k xor N/2), and the run events of K.3 are read off that map word by word.
// ---- One read of the PSD frames, one read + one write of the average.
// ---- Same values as k_chdet_avg + k_chdet_find bit for bit (exact order statistic, ordered events).
#define CHDET_RMAX 64
#define CHDET_RREG 32                           // values per thread kept in registers; the rest in shared memory
#define CHDET_FUSED_SMEM ((CHDET_RMAX - CHDET_RREG) * 1024 * (int) sizeof(float))     // >= 2 * CHDET_MAXRAW ints
struct ChdetFusedK {
  ChdetK k; float *avg_rw; const float *psd; int frames; size_t stream_stride; float alpha; int primed;
};

__global__ void __launch_bounds__(1024) k_chdet_fused(const ChdetFusedK q)
{
  // dynamic shared memory: first the values r >= CHDET_RREG ([r - RREG][1024]), then -- once the bit map exists and
  // the values are dead -- the run events starts[CHDET_MAXRAW], ends[CHDET_MAXRAW]
  extern __shared__ int s_ev[];
  float *vs = reinterpret_cast<float *>(s_ev);
  int *starts = s_ev, *ends = s_ev + CHDET_MAXRAW;
  __shared__ unsigned hist[256];
  __shared__ unsigned bits[CHDET_RMAX * 32];    // N / 32 words, frequency order
  __shared__ unsigned s_bucket, s_rank;
  __shared__ int s_w[32];
  __shared__ float s_n0;
  const ChdetK &p = q.k;
  const int tid = threadIdx.x, lane = tid & 31, st = blockIdx.x, N = p.N, half = N >> 1;
  const int R = N >> 10;                        // values per thread (2 ... 64)
  float *avg = q.avg_rw + (size_t) st * N;

  // ---- K.1: exponential average over the feed's frames, in frame order
  float v[CHDET_RREG];
  const float *__restrict__ ps = q.psd + (size_t) st * q.stream_stride + tid;
  // (loads of all rows first, then the frames in order, then the stores: many requests in flight per thread)
  const int f0 = q.primed ? 0 : 1;
  if (R > CHDET_RREG) {                           // N = 65536: the upper half of the rows lives in shared memory
    float u[CHDET_RMAX - CHDET_RREG];
#pragma unroll
    for (int r = 0; r < CHDET_RMAX - CHDET_RREG; ++r)
      u[r] = q.primed ? avg[(r + CHDET_RREG) * 1024 + tid] : __ldg(ps + (r + CHDET_RREG) * 1024);
    for (int f = f0; f < q.frames; ++f) {
      const float *__restrict__ x = ps + (size_t) f * N + CHDET_RREG * 1024;
#pragma unroll
      for (int r = 0; r < CHDET_RMAX - CHDET_RREG; ++r) u[r] = u[r] + q.alpha * (__ldg(x + r * 1024) - u[r]);
    }
#pragma unroll
    for (int r = 0; r < CHDET_RMAX - CHDET_RREG; ++r) {
      avg[(r + CHDET_RREG) * 1024 + tid] = u[r];
      vs[r * 1024 + tid] = u[r];
    }
  }
#pragma unroll
  for (int r = 0; r < CHDET_RREG; ++r) if (r < R) v[r] = q.primed ? avg[r * 1024 + tid] : __ldg(ps + r * 1024);
  for (int f = f0; f < q.frames; ++f) {
    const float *__restrict__ x = ps + (size_t) f * N;
#pragma unroll
    for (int r = 0; r < CHDET_RREG; ++r) if (r < R) v[r] = v[r] + q.alpha * (__ldg(x + r * 1024) - v[r]);
  }
#pragma unroll
  for (int r = 0; r < CHDET_RREG; ++r) if (r < R) avg[r * 1024 + tid] = v[r];
  // ---- K.2: exact (N/4)-th smallest value (non-negative floats order like their bit patterns)
  unsigned prefix = 0, mask = 0, rank = (unsigned) N / 4;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    // histogram update (R is CTA-uniform: whole warps vote).  A noise floor shares its top byte, so in the first
    // pass nearly every warp is uniform: one add of 32 instead of a 32-way same-address conflict.
    auto count = [&](float x) {
      const unsigned u = __float_as_uint(x);
      const bool in = (u & mask) == prefix;
      const unsigned b = in ? (u >> shift) & 255u : 256u;
      int uniform;
      __match_all_sync(0xffffffffu, b, &uniform);
      if (uniform) { if (in && lane == 0) atomicAdd(&hist[b], 32u); }
      else if (in) atomicAdd(&hist[b], 1u);
    };
#pragma unroll
    for (int r = 0; r < CHDET_RREG; ++r) if (r < R) count(v[r]);
#pragma unroll 8
    for (int r = CHDET_RREG; r < R; ++r) count(vs[(r - CHDET_RREG) * 1024 + tid]);
    __syncthreads();
    if (tid < 32) {
      // bucket b = first with cum(b) + hist[b] > rank: lane l owns buckets 8 l ... 8 l + 7
      unsigned h8[8], sum = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) { h8[i] = hist[lane * 8 + i]; sum += h8[i]; }
      unsigned incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const unsigned t2 = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t2; }
      const unsigned before = incl - sum;
      const unsigned hit = __ballot_sync(0xffffffffu, incl > rank);      // lanes whose range reaches past the rank
      const int owner = hit ? __ffs(hit) - 1 : 31;
      if (lane == owner) {
        unsigned cum = before, b = 0;
        for (; b < 7; ++b) { if (cum + h8[b] > rank) break; cum += h8[b]; }
        // (the serial walk stopped at bucket 255 at the latest without testing it; so does this one)
        s_bucket = (unsigned) lane * 8u + b; s_rank = rank - cum;
      }
    }
    __syncthreads();
    prefix |= s_bucket << shift; mask |= 0xffu << shift; rank = s_rank;
    __syncthreads();
  }
  if (tid == 0) {
    const float inst = __uint_as_float(prefix);
    float n0 = p.n0[st];
    n0 = p.n0_primed[st] ? n0 + p.gamma * (inst - n0) : inst;
    p.n0[st] = n0; p.n0_primed[st] = 1;
    s_n0 = n0;
  }
  __syncthreads();
  const float n0 = s_n0, thr = n0 * p.snr;

  // ---- K.3: threshold bit map in ascending frequency, then the run events word by word
  auto vote = [&](int r, float x) {
    const unsigned m = __ballot_sync(0xffffffffu, x > thr);
    if (lane == 0) bits[((r * 1024 + (tid & ~31)) ^ half) >> 5] = m;
  };
#pragma unroll
  for (int r = 0; r < CHDET_RREG; ++r) if (r < R) vote(r, v[r]);
#pragma unroll 8
  for (int r = CHDET_RREG; r < R; ++r) vote(r, vs[(r - CHDET_RREG) * 1024 + tid]);
  __syncthreads();
  const int W = N >> 5;                         // words
  const int wpt = (W + 1023) / 1024;            // words per thread (1 or 2)
  const int w0 = min(tid * wpt, W), w1 = min(w0 + wpt, W);
  int ns = 0, ne = 0;
  for (int w = w0; w < w1; ++w) {
    const unsigned m = bits[w], prev = (m << 1) | (w > 0 ? bits[w - 1] >> 31 : 0u);
    ns += __popc(m & ~prev); ne += __popc(~m & prev);
    if (w == W - 1 && (m >> 31)) ++ne;          // a run that reaches the top edge ends at N
  }
  int tot_s, tot_e;
  int os = block_excl_scan(ns, &tot_s, s_w);
  int oe = block_excl_scan(ne, &tot_e, s_w);
  for (int w = w0; w < w1; ++w) {
    const unsigned m = bits[w], prev = (m << 1) | (w > 0 ? bits[w - 1] >> 31 : 0u);
    unsigned sb = m & ~prev, eb = ~m & prev;
    while (sb) { const int b = __ffs(sb) - 1; sb &= sb - 1; if (os < CHDET_MAXRAW) starts[os] = w * 32 + b; ++os; }
    while (eb) { const int b = __ffs(eb) - 1; eb &= eb - 1; if (oe < CHDET_MAXRAW) ends[oe] = w * 32 + b; ++oe; }
    if (w == W - 1 && (m >> 31)) { if (oe < CHDET_MAXRAW) ends[oe] = N; ++oe; }
  }
  __syncthreads();
  const int Rr = min(tot_s, CHDET_MAXRAW);

  // ---- K.4: width filter + ordered compaction
  SdbDetectedDev *__restrict__ out = p.out + (size_t) st * CHDET_CAP;
  int running = 0;
  for (int base = 0; base < Rr; base += 1024) {
    const int r = base + tid;
    const int keep = r < Rr && ends[r] - starts[r] >= p.min_bins;
    int tile;
    const int pos = running + block_excl_scan(keep, &tile, s_w);
    if (keep && pos < CHDET_CAP) { out[pos].bin_lo = (unsigned) starts[r]; out[pos].bin_hi = (unsigned) ends[r]; }
    running += tile;
  }
  __syncthreads();
  const int nch = min(running, CHDET_CAP);
  if (tid == 0) { p.count[st] = (unsigned) nch; p.total[st] = (unsigned) running; }
  // ---- peak level of every reported channel: one warp per channel (the average was written above by this CTA)
  for (int c = tid >> 5; c < nch; c += 32) {
    const int a = (int) out[c].bin_lo, b = (int) out[c].bin_hi;
    float m = 0.0f;
    for (int i = a + lane; i < b; i += 32) m = fmaxf(m, avg[(i + half) & (N - 1)]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) { out[c].s0 = m; out[c].n0 = n0; out[c].snr = m / n0; }
  }
}

// ---------------------------------------------------------------------------------------------
// host object + C-ABI
// ---------------------------------------------------------------------------------------------
struct sdb_chdet {
  int device = 0; unsigned N = 0, S = 0, min_bins = 1;
  float alpha = 0, gamma = 0, snr = 0;
  DevBuf<float> d_avg, d_n0; DevBuf<int> d_n0_primed;
  DevBuf<SdbDetectedDev> d_out; DevBuf<unsigned> d_count, d_total;
  bool primed = false;
};

extern "C" void sdb_chdet_destroy(sdb_chdet_t *d)
{
  if (!d) return;
  cudaSetDevice(d->device);
  delete d;
}

extern "C" sdb_chdet_t *sdb_chdet_new(int device, uint32_t n_bins, uint32_t n_streams, float alpha, float gamma,
                                      float snr, uint32_t min_bins)
{
  if (sdb_device_count() <= 0) return nullptr;                        // no CPU fallback
  if (n_bins < 16 || (n_bins & (n_bins - 1)) || n_bins > (1u << 20) || n_streams < 1) return nullptr;
  if (!(snr > 0.0f) || !(alpha >= 0.0f && alpha <= 1.0f) || !(gamma >= 0.0f && gamma <= 1.0f)) return nullptr;
  if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  sdb_chdet *d = new sdb_chdet();
  d->device = device; d->N = n_bins; d->S = n_streams; d->alpha = alpha; d->gamma = gamma; d->snr = snr;
  d->min_bins = min_bins < 1 ? 1 : min_bins;
  const size_t S = n_streams;
  bool ok = d->d_avg.alloc(S * n_bins) == cudaSuccess && d->d_n0.alloc(S) == cudaSuccess &&
            d->d_n0_primed.alloc(S) == cudaSuccess && d->d_out.alloc(S * CHDET_CAP) == cudaSuccess &&
            d->d_count.alloc(S) == cudaSuccess && d->d_total.alloc(S) == cudaSuccess;
  if (ok) {
    cudaMemset(d->d_avg, 0, S * n_bins * sizeof(float));
    cudaMemset(d->d_n0, 0, S * sizeof(float));
    cudaMemset(d->d_n0_primed, 0, S * sizeof(int));
    cudaMemset(d->d_count, 0, S * sizeof(unsigned));
    cudaMemset(d->d_total, 0, S * sizeof(unsigned));
    static std::atomic<unsigned long long> attr_done{ 0 };   // one bit per device: function attributes are per context
    if (sdb_first_on_device(attr_done)) {
      cudaFuncSetAttribute(k_chdet_find, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * CHDET_MAXRAW * (int) sizeof(int));
      cudaFuncSetAttribute(k_chdet_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, CHDET_FUSED_SMEM);
    }
  }
  if (!ok || cudaGetLastError() != cudaSuccess) { sdb_chdet_destroy(d); return nullptr; }
  return d;
}

cudaError_t sdb_chdet_feed_stream(sdb_chdet *d, const float *psd_dev, uint32_t frames, size_t stream_stride,
                                  cudaStream_t stream, uint64_t *launch_counter)
{
  if (frames == 0) return cudaSuccess;
  ChdetK p;
  p.avg = d->d_avg; p.n0 = d->d_n0; p.n0_primed = d->d_n0_primed; p.N = (int) d->N; p.gamma = d->gamma; p.snr = d->snr;
  p.min_bins = (int) d->min_bins; p.out = d->d_out; p.count = d->d_count; p.total = d->d_total;
  static const bool split = getenv("SDB_CHDET_SPLIT") != nullptr;     // the two-kernel path, for A/B runs
  if (d->N >= 2048 && d->N <= 1024 * CHDET_RMAX && !split) {
    ChdetFusedK q;
    q.k = p; q.avg_rw = d->d_avg; q.psd = psd_dev; q.frames = (int) frames; q.stream_stride = stream_stride;
    q.alpha = d->alpha; q.primed = d->primed ? 1 : 0;
    k_chdet_fused<<<d->S, 1024, CHDET_FUSED_SMEM, stream>>>(q);
    if (launch_counter) *launch_counter += 1;
  } else {
    dim3 grid((d->N + 255) / 256, d->S);
    k_chdet_avg<<<grid, 256, 0, stream>>>(d->d_avg, psd_dev, (int) d->N, (int) frames, stream_stride, d->alpha,
                                          d->primed ? 1 : 0);
    k_chdet_find<<<d->S, 1024, 2 * CHDET_MAXRAW * sizeof(int), stream>>>(p);
    if (launch_counter) *launch_counter += 2;
  }
  d->primed = true;
  return cudaGetLastError();
}

extern "C" int sdb_chdet_feed_device(sdb_chdet_t *d, const float *psd_dev, uint32_t frames, size_t stream_stride)
{
  if (!d || !psd_dev) return -1;
  if (cudaSetDevice(d->device) != cudaSuccess) return -1;
  if (sdb_chdet_feed_stream(d, psd_dev, frames, stream_stride, nullptr, nullptr) != cudaSuccess) return -1;
  return cudaStreamSynchronize(nullptr) == cudaSuccess ? 0 : -1;
}

// every stream's list in three copies instead of three per stream (the panoramic sweep reads 128...1024 hops):
// centers[S] host, out[S][cap], counts[S] (clamped to cap)
extern "C" int sdb_chdet_read_all(sdb_chdet_t *d, double samp_rate, const double *centers, sdb_detected_channel *out,
                                  size_t cap, uint32_t *counts)
{
  if (!d || !centers || !out || !counts) return -1;
  if (cudaSetDevice(d->device) != cudaSuccess) return -1;
  const size_t S = d->S;
  std::vector<unsigned> cnt(S);
  std::vector<SdbDetectedDev> h(S * CHDET_CAP);
  if (cudaMemcpy(cnt.data(), d->d_count, S * sizeof(unsigned), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  if (cudaMemcpy(h.data(), d->d_out, h.size() * sizeof(SdbDetectedDev), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  const double df = samp_rate / (double) d->N, half = (double) (d->N / 2);
  for (size_t s = 0; s < S; ++s) {
    const size_t n = cnt[s] < cap ? cnt[s] : cap;
    counts[s] = (uint32_t) n;
    for (size_t i = 0; i < n; ++i) {
      const SdbDetectedDev &q = h[s * CHDET_CAP + i];
      sdb_detected_channel &c = out[s * cap + i];
      c.bin_lo = q.bin_lo; c.bin_hi = q.bin_hi;
      c.f_lo = centers[s] + ((double) q.bin_lo - half) * df;
      c.f_hi = centers[s] + ((double) q.bin_hi - half) * df;
      c.fc = 0.5 * (c.f_lo + c.f_hi); c.bw = c.f_hi - c.f_lo;
      c.S0 = q.s0; c.N0 = q.n0; c.snr = q.snr;
    }
  }
  return 0;
}

// Device-side twin of sdb_chdet_read_all for callers that keep the lists on the GPU (the panoramic sweep packs them
// into its NCCL send block): the same binary64 expressions, one block per stream, stream-ordered, no host copy.
__global__ void k_chdet_pack(const SdbDetectedDev *__restrict__ det, const unsigned *__restrict__ count, unsigned N,
                             double samp_rate, const double *__restrict__ centers, sdb_detected_channel *__restrict__ out,
                             unsigned cap, int *__restrict__ counts_out)
{
  const unsigned s = blockIdx.x;
  const unsigned c = count[s], n = c < cap ? c : cap;
  if (threadIdx.x == 0) counts_out[s] = (int) n;
  const double df = samp_rate / (double) N, half = (double) (N / 2), center = centers[s];
  for (unsigned i = threadIdx.x; i < n; i += blockDim.x) {
    const SdbDetectedDev q = det[(size_t) s * CHDET_CAP + i];
    sdb_detected_channel o;
    o.bin_lo = q.bin_lo; o.bin_hi = q.bin_hi;
    o.f_lo = center + ((double) q.bin_lo - half) * df;
    o.f_hi = center + ((double) q.bin_hi - half) * df;
    o.fc = 0.5 * (o.f_lo + o.f_hi); o.bw = o.f_hi - o.f_lo;
    o.S0 = q.s0; o.N0 = q.n0; o.snr = q.snr;
    out[(size_t) s * cap + i] = o;
  }
}

cudaError_t sdb_chdet_pack_device(sdb_chdet_t *d, double samp_rate, const double *centers_dev, sdb_detected_channel *out_dev,
                                  size_t cap, int *counts_dev, cudaStream_t stream)
{
  if (!d || !centers_dev || !out_dev || !counts_dev) return cudaErrorInvalidValue;
  k_chdet_pack<<<d->S, 64, 0, stream>>>(d->d_out, d->d_count, d->N, samp_rate, centers_dev, out_dev, (unsigned) cap,
                                        counts_dev);
  return cudaGetLastError();
}

extern "C" long sdb_chdet_read(sdb_chdet_t *d, uint32_t stream, double samp_rate, double center_freq,
                               sdb_detected_channel *out, size_t cap, uint32_t *total)
{
  if (!d || stream >= d->S || (!out && cap)) return -1;
  if (cudaSetDevice(d->device) != cudaSuccess) return -1;
  unsigned cnt = 0, tot = 0;
  if (cudaMemcpy(&cnt, d->d_count + stream, sizeof(cnt), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  if (cudaMemcpy(&tot, d->d_total + stream, sizeof(tot), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  if (total) *total = tot;
  std::vector<SdbDetectedDev> h(cnt);
  if (cnt && cudaMemcpy(h.data(), d->d_out + (size_t) stream * CHDET_CAP, cnt * sizeof(SdbDetectedDev),
                        cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  const size_t n = cnt < cap ? cnt : cap;
  const double df = samp_rate / (double) d->N, half = (double) (d->N / 2);
  for (size_t i = 0; i < n; ++i) {
    sdb_detected_channel &c = out[i];
    c.bin_lo = h[i].bin_lo; c.bin_hi = h[i].bin_hi;
    c.f_lo = center_freq + ((double) h[i].bin_lo - half) * df;       // bin edges: bin j spans [j, j+1) df
    c.f_hi = center_freq + ((double) h[i].bin_hi - half) * df;
    c.fc = 0.5 * (c.f_lo + c.f_hi); c.bw = c.f_hi - c.f_lo;
    c.S0 = h[i].s0; c.N0 = h[i].n0; c.snr = h[i].snr;
  }
  return (long) n;
}

// ---------------------------------------------------------------------------------------------
// channel tracking across detector updates (oracle/SPEC_KT.md)
// ---------------------------------------------------------------------------------------------
// k_chtrack: one warp per stream, right after the detector on the same CUDA stream, over the detector's device list
// (d_out / d_count).  The table of the previous update (ascending (a, id), so that index order is the KT.3 tie-break
// order) is read from one parity and the new table written to the other.  Lane l keeps the ranges of tracks l + 32 j
// in registers; each detection, in ascending frequency, takes the warp maximum of (overlap << 8 | 255 - index) over
// the tracks not yet matched.  Survivors and new tracks are then gathered in shared memory and placed by their rank
// in (a, id).
struct SdbTrackDev { unsigned a, b; float s0, snr; unsigned id, age, present, misses; };
struct SdbTrackHdr { unsigned count, issued; float n0; unsigned pad; unsigned long long dropped; };   // ids 1 ... issued

struct ChtrackK {
  const SdbDetectedDev *det; const unsigned *count; const float *n0;
  const SdbTrackDev *tr_in; const SdbTrackHdr *hd_in;
  SdbTrackDev *tr_out; SdbTrackHdr *hd_out;
  float beta; unsigned hold;
};

__global__ void __launch_bounds__(32) k_chtrack(const ChtrackK p)
{
  __shared__ unsigned s_da[CHDET_CAP], s_db[CHDET_CAP];
  __shared__ float s_ds[CHDET_CAP];
  __shared__ short s_dm[CHDET_CAP];             // detection -> matched track, -1: none
  __shared__ short s_tm[CHDET_CAP];             // matched track -> its detection
  __shared__ SdbTrackDev s_new[CHDET_CAP];      // the new table before ordering
  const int lane = threadIdx.x, st = blockIdx.x;
  const SdbTrackHdr h = p.hd_in[st];
  const unsigned nt = h.count, nd = p.count[st];
  const SdbDetectedDev *__restrict__ det = p.det + (size_t) st * CHDET_CAP;
  const SdbTrackDev *__restrict__ in = p.tr_in + (size_t) st * CHDET_CAP;
  for (unsigned d = lane; d < nd; d += 32) { s_da[d] = det[d].bin_lo; s_db[d] = det[d].bin_hi; s_ds[d] = det[d].s0; }
  unsigned ta[CHDET_CAP / 32], tb[CHDET_CAP / 32], matched = 0;
#pragma unroll
  for (int j = 0; j < CHDET_CAP / 32; ++j) {
    const unsigned t = lane + 32 * j;
    ta[j] = t < nt ? in[t].a : 0u; tb[j] = t < nt ? in[t].b : 0u;   // (an empty slot never overlaps)
  }
  __syncwarp();
  // ---- KT.3: detections in ascending frequency; the largest overlap, then the smaller index (= smaller (a, id))
  for (unsigned d = 0; d < nd; ++d) {
    const int ad = (int) s_da[d], bd = (int) s_db[d];
    unsigned best = 0;
#pragma unroll
    for (int j = 0; j < CHDET_CAP / 32; ++j) {
      const int ov = min(bd, (int) tb[j]) - max(ad, (int) ta[j]);
      if (!((matched >> j) & 1u) && ov > 0)
        best = max(best, ((unsigned) ov << 8) | (255u - (unsigned) (lane + 32 * j)));
    }
    best = __reduce_max_sync(0xffffffffu, best);
    const int t = best ? 255 - (int) (best & 255u) : -1;
    if (t >= 0 && (t & 31) == lane) { matched |= 1u << (t >> 5); s_tm[t] = (short) d; }
    if (lane == 0) s_dm[d] = (short) t;
  }
  __syncwarp();
  // ---- KT.4 / KT.5: matched tracks take the detection, unmatched ones age and leave after `hold` misses
  unsigned live = 0;
  const unsigned lt = (1u << lane) - 1u;
#pragma unroll
  for (int j = 0; j < CHDET_CAP / 32; ++j) {
    const unsigned t = lane + 32 * j;
    SdbTrackDev r;
    bool keep = false;
    if (t < nt) {
      r = in[t];
      r.age += 1;
      if ((matched >> j) & 1u) {
        const int d = s_tm[t];
        r.a = s_da[d]; r.b = s_db[d];
        r.s0 = __fadd_rn(r.s0, __fmul_rn(p.beta, __fsub_rn(s_ds[d], r.s0)));
        r.present += 1; r.misses = 0;
        keep = true;
      } else {
        r.misses += 1;
        keep = r.misses <= p.hold;
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (keep) s_new[live + __popc(m & lt)] = r;
    live += __popc(m);
  }
  // ---- KT.6: unmatched detections open tracks in ascending frequency while fewer than 256 are live
  unsigned unm = 0, issued = h.issued;
  for (unsigned d0 = 0; d0 < nd; d0 += 32) {
    const unsigned d = d0 + lane;
    const bool u = d < nd && s_dm[d] < 0;
    const unsigned m = __ballot_sync(0xffffffffu, u);
    const unsigned k = unm + __popc(m & lt);              // rank among the unmatched detections
    if (u && live + k < CHDET_CAP) {
      SdbTrackDev r;
      r.a = s_da[d]; r.b = s_db[d]; r.s0 = s_ds[d]; r.snr = 0.0f;
      r.id = issued + k + 1; r.age = 1; r.present = 1; r.misses = 0;
      s_new[live + k] = r;
    }
    unm += __popc(m);
  }
  const unsigned ins = min(unm, CHDET_CAP - live), n = live + ins;
  __syncwarp();
  // ---- KT.7: ascending (a, id) by rank (ids are unique), snr against the detector's current floor
  const float n0 = p.n0[st];
  SdbTrackDev *__restrict__ out = p.tr_out + (size_t) st * CHDET_CAP;
  for (unsigned i = lane; i < n; i += 32) {
    SdbTrackDev r = s_new[i];
    const unsigned long long ki = ((unsigned long long) r.a << 32) | r.id;
    unsigned rank = 0;
    for (unsigned q = 0; q < n; ++q)
      rank += (((unsigned long long) s_new[q].a << 32) | s_new[q].id) < ki;
    r.snr = r.s0 / n0;
    out[rank] = r;
  }
  if (lane == 0) {
    SdbTrackHdr o;
    o.count = n; o.issued = issued + ins; o.n0 = n0; o.pad = 0; o.dropped = h.dropped + (unm - ins);
    p.hd_out[st] = o;
  }
}

// host object of the tracker: the two tables and headers by update parity; `cur` holds the latest
struct sdb_chtrack {
  int device = 0; unsigned N = 0, S = 0, hold = 0, cur = 0;
  float beta = 1.0f;
  DevBuf<SdbTrackDev> tr[2]; DevBuf<SdbTrackHdr> hd[2];
};

void sdb_chtrack_destroy(sdb_chtrack *t)
{
  if (!t) return;
  cudaSetDevice(t->device);
  delete t;
}

sdb_chtrack *sdb_chtrack_new(int device, uint32_t n_bins, uint32_t n_streams, float beta, uint32_t hold)
{
  if (!(beta > 0.0f && beta <= 1.0f) || hold > SDB_CHTRACK_HOLD_MAX || n_streams < 1) return nullptr;
  if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  sdb_chtrack *t = new sdb_chtrack();
  t->device = device; t->N = n_bins; t->S = n_streams; t->beta = beta; t->hold = hold;
  const size_t S = n_streams;
  bool ok = true;
  for (int i = 0; i < 2 && ok; ++i)
    ok = t->tr[i].alloc(S * CHDET_CAP) == cudaSuccess && t->hd[i].alloc(S) == cudaSuccess &&
         cudaMemset(t->hd[i], 0, S * sizeof(SdbTrackHdr)) == cudaSuccess;   // no track, no id issued, nothing dropped
  if (!ok || cudaDeviceSynchronize() != cudaSuccess) { cudaGetLastError(); sdb_chtrack_destroy(t); return nullptr; }
  return t;
}

// KT.1: one update per detector update, i.e. per feed with frames, after sdb_chdet_feed_stream on the same stream
cudaError_t sdb_chtrack_feed_stream(sdb_chtrack *t, const sdb_chdet *d, uint32_t frames, cudaStream_t stream,
                                    uint64_t *launch_counter)
{
  if (frames == 0) return cudaSuccess;
  ChtrackK p;
  p.det = d->d_out; p.count = d->d_count; p.n0 = d->d_n0;
  p.tr_in = t->tr[t->cur]; p.hd_in = t->hd[t->cur];
  p.tr_out = t->tr[t->cur ^ 1u]; p.hd_out = t->hd[t->cur ^ 1u];
  p.beta = t->beta; p.hold = t->hold;
  k_chtrack<<<t->S, 32, 0, stream>>>(p);
  if (launch_counter) *launch_counter += 1;
  t->cur ^= 1u;
  return cudaGetLastError();
}

static void track_to_host(const SdbTrackDev &q, float n0, double center, double df, double half, sdb_tracked_channel &c)
{
  c.bin_lo = q.a; c.bin_hi = q.b;
  c.f_lo = center + ((double) q.a - half) * df;        // K.4 frequencies over the track's range
  c.f_hi = center + ((double) q.b - half) * df;
  c.fc = 0.5 * (c.f_lo + c.f_hi); c.bw = c.f_hi - c.f_lo;
  c.S0 = q.s0; c.N0 = n0; c.snr = q.snr;
  c.id = q.id; c.age = q.age; c.present = q.present; c.misses = q.misses;
}

// the tracks of one stream after the latest update; *total = live tracks, *dropped = detections not tracked so far
long sdb_chtrack_read(sdb_chtrack *t, uint32_t stream, double samp_rate, double center_freq, sdb_tracked_channel *out,
                      size_t cap, uint32_t *total, uint64_t *dropped)
{
  if (!t || stream >= t->S || (!out && cap)) return -1;
  if (cudaSetDevice(t->device) != cudaSuccess) return -1;
  SdbTrackHdr h;
  if (cudaMemcpy(&h, t->hd[t->cur] + stream, sizeof(h), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  const size_t n = h.count < cap ? h.count : cap;
  std::vector<SdbTrackDev> q(n);
  if (n && cudaMemcpy(q.data(), t->tr[t->cur] + (size_t) stream * CHDET_CAP, n * sizeof(SdbTrackDev),
                      cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  const double df = samp_rate / (double) t->N, half = (double) (t->N / 2);
  for (size_t i = 0; i < n; ++i) track_to_host(q[i], h.n0, center_freq, df, half, out[i]);
  if (total) *total = h.count;
  if (dropped) *dropped = h.dropped;
  return (long) n;
}

// every stream in two copies: centers[S] host, out[S][cap], counts[S] (clamped to cap), dropped[S] (may be NULL)
int sdb_chtrack_read_all(sdb_chtrack *t, double samp_rate, const double *centers, sdb_tracked_channel *out, size_t cap,
                         uint32_t *counts, uint64_t *dropped)
{
  if (!t || !centers || !out || !counts) return -1;
  if (cudaSetDevice(t->device) != cudaSuccess) return -1;
  const size_t S = t->S;
  std::vector<SdbTrackHdr> h(S);
  std::vector<SdbTrackDev> q(S * CHDET_CAP);
  if (cudaMemcpy(h.data(), t->hd[t->cur], S * sizeof(SdbTrackHdr), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  if (cudaMemcpy(q.data(), t->tr[t->cur], q.size() * sizeof(SdbTrackDev), cudaMemcpyDeviceToHost) != cudaSuccess)
    return -1;
  const double df = samp_rate / (double) t->N, half = (double) (t->N / 2);
  for (size_t s = 0; s < S; ++s) {
    const size_t n = h[s].count < cap ? h[s].count : cap;
    counts[s] = (uint32_t) n;
    if (dropped) dropped[s] = h[s].dropped;
    for (size_t i = 0; i < n; ++i) track_to_host(q[s * CHDET_CAP + i], h[s].n0, centers[s], df, half, out[s * cap + i]);
  }
  return 0;
}
