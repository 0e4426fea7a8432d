// sview_kernels.cu -- panoramic-scanner PSD stitcher (SpectrumView) on the GPU.
//
// Reference arithmetic (fully present in the reference, so followed value by value):
//   SpectrumView::feedLinearMode     Panoramic/Scanner.cpp:118-185
//   SpectrumView::feedHistogramMode  Panoramic/Scanner.cpp:187-237
//   SpectrumView::interpolate        Panoramic/Scanner.cpp:56-116   (count > 5 -> reset to 1, gap filling)
//   constants                        include/Scanner.h:26-32
//
// The reference feeds one hop at a time and calls interpolate() after each.  The per-bin state
// (psdAccum, psdCount) only depends on that bin's own contributions in hop order, so the work splits in:
//   project    : per hop, the box average of the source bins that fall in each destination bin (the
//                O(psd_size) part; hops are independent -> shards over GPUs);
//   accumulate : per destination bin, apply the contributions in hop order with the forgetting rule;
//   fill       : the final gap interpolation.
// Between project and accumulate the (tiny) contribution lists are what crosses NVLink (NCCL gather).
// Compiled with -fmad=false; double arithmetic for frequencies / positions exactly as in the C++.
#include "sdb_internal.h"
#include "sdb_math.h"

struct SviewGeom {
  double freq_min, freq_range, fft_bandwidth;
  float  rel_bw;
  unsigned spectrum_size;
};

// one CTA per hop; thread t handles destination bins j0 + t, j0 + t + blockDim, ...
__global__ void k_sview_project(SviewGeom g, const float *__restrict__ psd, size_t psd_size,
                                const double *__restrict__ centers, int n_hops, int adjust_sides,
                                int *__restrict__ j0_out, int *__restrict__ nb_out,
                                float *__restrict__ va, float *__restrict__ vc, int max_bins)
{
  const int h = blockIdx.x;
  if (h >= n_hops) return;
  const double center = centers[h];
  const double fmin = center - g.fft_bandwidth / 2, fmax = center + g.fft_bandwidth / 2;
  const float *__restrict__ src = psd + (size_t) h * psd_size;
  float *__restrict__ oa = va + (size_t) h * max_bins, *__restrict__ oc = vc + (size_t) h * max_bins;
  const double fft_count_rel = (fmax - fmin) / g.freq_range;

  if (fft_count_rel * g.spectrum_size >= 2) {
    // ---- linear mode (Scanner.cpp:118-185)
    const double inp_bw = fmax - fmin;
    const int skip = adjust_sides ? (int) (.5f * (1 - g.rel_bw) * psd_size) : 0;
    const double freq_skip = (double) skip / psd_size * inp_bw;
    const double bw = inp_bw - 2 * freq_skip;
    const double fft_count = g.freq_range / bw;
    const double bins = g.spectrum_size / fft_count;
    const double src_bin_w = inp_bw / psd_size;
    const double dst_bin_w = g.freq_range / g.spectrum_size;
    const double delta = dst_bin_w / src_bin_w;
    double pos = (freq_skip + fmin - g.freq_min) / g.freq_range;
    pos *= g.spectrum_size;
    const int j0 = pos > 0 ? (int) pos : 0;
    const int k = pos + bins < g.spectrum_size ? (int) (pos + bins) : (int) g.spectrum_size;
    int nb = k - j0;
    if (nb < 0) nb = 0;
    if (nb > max_bins) nb = max_bins;
    if (threadIdx.x == 0) { j0_out[h] = j0; nb_out[h] = nb; }
    for (int t = threadIdx.x; t < nb; t += blockDim.x) {
      const int j = j0 + t;
      const double freq_j = g.freq_min + dst_bin_w * j;
      const double src_bin = (freq_j - fmin) / src_bin_w;
      int start_bin = (int) src_bin;
      int end_bin = (int) (src_bin + delta);
      start_bin = start_bin < 0 ? 0 : (start_bin > (int) psd_size - 1 ? (int) psd_size - 1 : start_bin);
      end_bin = end_bin < start_bin + 1 ? start_bin + 1 : (end_bin > (int) psd_size ? (int) psd_size : end_bin);
      float acc = 0, cnt = 0;
      for (int i = start_bin; i < end_bin; ++i) { acc += src[i]; cnt += 1; }
      oa[t] = acc / cnt;      // cnt > 0 always (end_bin > start_bin)
      oc[t] = 1.0f;
    }
  } else {
    // ---- histogram mode (Scanner.cpp:187-237): the hop is narrower than two destination bins
    double rel_bw = (fmax - fmin) / g.freq_range;
    double f_start = (fmin - g.freq_min) / g.freq_range;
    double f_end = (fmax - g.freq_min) / g.freq_range;
    f_start *= g.spectrum_size; f_end *= g.spectrum_size; rel_bw *= g.spectrum_size;
    if (threadIdx.x == 0) {
      unsigned j = f_start < 0 ? 0u : (unsigned) f_start;
      if (j > g.spectrum_size - 1) j = g.spectrum_size - 1;
      const float inv = (float) (1. / psd_size);
      float accum = 0;
      for (size_t i = 0; i < psd_size; ++i) accum += src[i];
      accum *= inv;
      j0_out[h] = (int) j;
      if (floor(f_start) != floor(f_end)) {
        const float t = (float) ((f_start - floor(f_start)) / rel_bw);
        oc[0] = 1 - t; oa[0] = (1 - t) * accum;
        if (j + 1 < g.spectrum_size) { oc[1] = t; oa[1] = t * accum; nb_out[h] = 2; }
        else nb_out[h] = 1;
      } else {
        oc[0] = 1; oa[0] = accum; nb_out[h] = 1;
      }
    }
  }
}

// ---- linear mode, tiled: the same values as k_sview_project, for the sweep's stream-ordered path.
// k_sview_project gives every destination bin one thread that walks its `delta` source bins (512 on cfg5): the lanes
// of a warp read 2 KB apart, 32 cache lines per request -- 0.19 ms per 1024-hop sweep, L1 tag bound.  Here a warp
// owns 32 destination bins and moves their segments through a 32 x 33 shared-memory tile, 32 source bins per segment
// at a time: row after row is read coalesced (lane = source bin), the tile is summed column-wise (lane = destination
// bin, banks (lane + k) mod 32), so every bin still adds its source bins one by one in ascending order.
// LIN: `psd` holds the engine's linear, natural-order PSD and the PSDMessage conversion (fftshift + 10 log10(x + 1e-8),
// the expression of k_psd_shift_db) happens in the load: the separate dB pass and its buffer disappear, and only the
// kept (1 - 2 skip / size) part of each hop is ever converted.  hop_stride: floats between consecutive hops.
template <bool LIN>
__global__ void k_sview_project_tiled(SviewGeom g, const float *__restrict__ psd, size_t psd_size, size_t hop_stride,
                                      const double *__restrict__ centers, int n_hops, int adjust_sides,
                                      int *__restrict__ j0_out, int *__restrict__ nb_out,
                                      float *__restrict__ va, float *__restrict__ vc, int max_bins)
{
  extern __shared__ float s_tile[];               // [warps][32][33]
  const int h = blockIdx.x;
  if (h >= n_hops) return;
  const int lane = (int) (threadIdx.x & 31u), w = (int) (threadIdx.x >> 5);
  float (*tile)[33] = reinterpret_cast<float (*)[33]>(s_tile + (size_t) w * 32 * 33);
  const double center = centers[h];
  const double fmin = center - g.fft_bandwidth / 2, fmax = center + g.fft_bandwidth / 2;
  const float *__restrict__ src = psd + (size_t) h * hop_stride;
  float *__restrict__ oa = va + (size_t) h * max_bins, *__restrict__ oc = vc + (size_t) h * max_bins;
  // ---- geometry exactly as k_sview_project's linear branch (Scanner.cpp:118-185)
  const double inp_bw = fmax - fmin;
  const int skip = adjust_sides ? (int) (.5f * (1 - g.rel_bw) * psd_size) : 0;
  const double freq_skip = (double) skip / psd_size * inp_bw;
  const double bw = inp_bw - 2 * freq_skip;
  const double fft_count = g.freq_range / bw;
  const double bins = g.spectrum_size / fft_count;
  const double src_bin_w = inp_bw / psd_size;
  const double dst_bin_w = g.freq_range / g.spectrum_size;
  const double delta = dst_bin_w / src_bin_w;
  double pos = (freq_skip + fmin - g.freq_min) / g.freq_range;
  pos *= g.spectrum_size;
  const int j0 = pos > 0 ? (int) pos : 0;
  const int k = pos + bins < g.spectrum_size ? (int) (pos + bins) : (int) g.spectrum_size;
  int nb = k - j0;
  if (nb < 0) nb = 0;
  if (nb > max_bins) nb = max_bins;
  if (threadIdx.x == 0) { j0_out[h] = j0; nb_out[h] = nb; }
  const int t = w * 32 + lane;
  int start_bin = 0, end_bin = 0;
  if (t < nb) {
    const int j = j0 + t;
    const double freq_j = g.freq_min + dst_bin_w * j;
    const double src_bin = (freq_j - fmin) / src_bin_w;
    start_bin = (int) src_bin;
    end_bin = (int) (src_bin + delta);
    start_bin = start_bin < 0 ? 0 : (start_bin > (int) psd_size - 1 ? (int) psd_size - 1 : start_bin);
    end_bin = end_bin < start_bin + 1 ? start_bin + 1 : (end_bin > (int) psd_size ? (int) psd_size : end_bin);
  }
  const int len = end_bin - start_bin;
  int maxlen = len;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) maxlen = max(maxlen, __shfl_xor_sync(0xffffffffu, maxlen, o));
  if (w * 32 >= nb) return;                       // whole warp beyond the hop's bins (maxlen == 0)
  const unsigned half = (unsigned) (psd_size >> 1), msk = (unsigned) psd_size - 1u;
  float acc = 0, cnt = 0;
  const int nrows = nb - w * 32 < 32 ? nb - w * 32 : 32;       // destination bins of this warp
  for (int c0 = 0; c0 < maxlen; c0 += 32) {
    // eight rows at a time: the eight loads go out before the first conversion (one row per iteration left one
    // request in flight per warp and the kernel ran at DRAM latency)
#pragma unroll
    for (int rg = 0; rg < 32; rg += 8) {
      if (rg < nrows) {
        float xr[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int rs = __shfl_sync(0xffffffffu, start_bin, rg + u), re = __shfl_sync(0xffffffffu, end_bin, rg + u);
          const int i = rs + c0 + lane;
          xr[u] = i < re ? (LIN ? __ldg(src + (((unsigned) i + half) & msk)) : __ldg(src + i)) : -1.0f;
          if (!LIN && !(i < re)) xr[u] = 0.0f;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          // LIN: a PSD value is non-negative, -1 marks "past the segment" (never summed)
          tile[rg + u][lane] = LIN ? (xr[u] >= 0.0f ? 10.0f * d_log10f(xr[u] + 1e-8f) : 0.0f) : xr[u];
        }
      }
    }
    __syncwarp();
    const int n_here = len - c0 < 32 ? len - c0 : 32;
    for (int q = 0; q < n_here; ++q) { acc += tile[lane][q]; cnt += 1; }
    __syncwarp();
  }
  if (t < nb) {
    oa[t] = acc / cnt;      // cnt > 0 always (end_bin > start_bin)
    oc[t] = 1.0f;
  }
}

// linear mode for every hop <=> the hop covers at least two destination bins (Scanner.cpp:254-262)
static cudaError_t sdb_launch_sview_project_tiled(cudaStream_t s, double freq_min, double freq_range, double fft_bandwidth,
                                                  float rel_bw, unsigned spectrum_size, const float *psd, size_t psd_size,
                                                  size_t hop_stride, int psd_is_linear, const double *centers_dev, int n_hops,
                                                  int adjust_sides, int *j0, int *nb, float *va, float *vc, int max_bins)
{
  SviewGeom g{ freq_min, freq_range, fft_bandwidth, rel_bw, spectrum_size };
  if (n_hops <= 0) return cudaSuccess;
  const int warps = (max_bins + 31) / 32;
  const size_t smem = (size_t) warps * 32 * 33 * sizeof(float);
  if (warps > 32 || smem > 48 * 1024) return cudaErrorInvalidConfiguration;
  if (psd_is_linear)
    k_sview_project_tiled<true><<<n_hops, warps * 32, smem, s>>>(g, psd, psd_size, hop_stride, centers_dev, n_hops,
                                                                adjust_sides, j0, nb, va, vc, max_bins);
  else
    k_sview_project_tiled<false><<<n_hops, warps * 32, smem, s>>>(g, psd, psd_size, hop_stride, centers_dev, n_hops,
                                                                 adjust_sides, j0, nb, va, vc, max_bins);
  return cudaGetLastError();
}

// SpectrumView::feed(SpectrumView const &) (Scanner.cpp:276-286), the zoom path of Scanner::setViewRange: the other
// view's accumulators, weighted by its counts, over its own frequency range, sides untouched.  One contribution
// list of pitch spectrum_size (a view can cover every destination bin); k_sview_accumulate applies it like a hop.
// Grid-stride over the destination bins; the histogram branch (source narrower than two destination bins) is one
// thread, as in k_sview_project.
__global__ void k_sview_project_view(SviewGeom g, const float *__restrict__ src_acc, const float *__restrict__ src_cnt,
                                     unsigned src_size, double fmin, double fmax, int *__restrict__ j0_out,
                                     int *__restrict__ nb_out, float *__restrict__ oa, float *__restrict__ oc)
{
  const double fft_count_rel = (fmax - fmin) / g.freq_range;
  const bool lead = blockIdx.x == 0 && threadIdx.x == 0;
  if (fft_count_rel * g.spectrum_size >= 2) {
    // ---- linear mode (Scanner.cpp:118-185) with adjustSides = false: skip = 0, freqSkip = 0
    const double inp_bw = fmax - fmin;
    const double freq_skip = (double) 0 / src_size * inp_bw;
    const double bw = inp_bw - 2 * freq_skip;
    const double fft_count = g.freq_range / bw;
    const double bins = g.spectrum_size / fft_count;
    const double src_bin_w = inp_bw / src_size;
    const double dst_bin_w = g.freq_range / g.spectrum_size;
    const double delta = dst_bin_w / src_bin_w;
    double pos = (freq_skip + fmin - g.freq_min) / g.freq_range;
    pos *= g.spectrum_size;
    const int j0 = pos > 0 ? (int) pos : 0;
    const int k = pos + bins < g.spectrum_size ? (int) (pos + bins) : (int) g.spectrum_size;
    int nb = k - j0;
    if (nb < 0) nb = 0;
    if (lead) { *j0_out = j0; *nb_out = nb; }
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < nb; t += gridDim.x * blockDim.x) {
      const int j = j0 + t;
      const double freq_j = g.freq_min + dst_bin_w * j;
      const double src_bin = (freq_j - fmin) / src_bin_w;
      int start_bin = (int) src_bin;
      int end_bin = (int) (src_bin + delta);
      start_bin = start_bin < 0 ? 0 : (start_bin > (int) src_size - 1 ? (int) src_size - 1 : start_bin);
      end_bin = end_bin < start_bin + 1 ? start_bin + 1 : (end_bin > (int) src_size ? (int) src_size : end_bin);
      float acc = 0, cnt = 0;
      for (int i = start_bin; i < end_bin; ++i) { acc += src_acc[i]; cnt += src_cnt[i]; }
      // `if (psdCount > 0)`: an empty source range contributes nothing (0 / 0 are no-ops in k_sview_accumulate)
      oa[t] = cnt > 0 ? acc / cnt : 0.0f;
      oc[t] = cnt > 0 ? 1.0f : 0.0f;
    }
  } else if (lead) {
    // ---- histogram mode (Scanner.cpp:187-237); the counts are not used there
    double rel_bw = (fmax - fmin) / g.freq_range;
    double f_start = (fmin - g.freq_min) / g.freq_range;
    double f_end = (fmax - g.freq_min) / g.freq_range;
    f_start *= g.spectrum_size; f_end *= g.spectrum_size; rel_bw *= g.spectrum_size;
    unsigned j = f_start < 0 ? 0u : (unsigned) f_start;
    if (j > g.spectrum_size - 1) j = g.spectrum_size - 1;
    const float inv = (float) (1. / src_size);
    float accum = 0;
    for (unsigned i = 0; i < src_size; ++i) accum += src_acc[i];
    accum *= inv;
    *j0_out = (int) j;
    if (floor(f_start) != floor(f_end)) {
      const float t = (float) ((f_start - floor(f_start)) / rel_bw);
      oc[0] = 1 - t; oa[0] = (1 - t) * accum;
      if (j + 1 < g.spectrum_size) { oc[1] = t; oa[1] = t * accum; *nb_out = 2; }
      else *nb_out = 1;
    } else {
      oc[0] = 1; oa[0] = accum; *nb_out = 1;
    }
  }
}

static cudaError_t sdb_launch_sview_project_view(cudaStream_t s, double freq_min, double freq_range, unsigned spectrum_size,
                                                 const float *src_acc, const float *src_cnt, unsigned src_size, double fmin,
                                                 double fmax, int *j0, int *nb, float *va, float *vc)
{
  SviewGeom g{ freq_min, freq_range, 0.0, 0.0f, spectrum_size };
  k_sview_project_view<<<(spectrum_size + 255) / 256, 256, 0, s>>>(g, src_acc, src_cnt, src_size, fmin, fmax, j0, nb,
                                                                  va, vc);
  return cudaGetLastError();
}

// one thread per destination bin: contributions in hop order + the count > 5 forgetting rule that
// interpolate() applies after every feed (Scanner.cpp:77-81).
// A hop touches the bins [j0, j0 + nb) (and, through the left-neighbour test, bin j0 + nb): the warp reads 32 hop
// headers at a time, votes on which of them reach its 32 bins and walks only those, in hop order.  The per-feed
// block below is idempotent while (a, c, cl) do not change -- p = a / c is recomputed to the same value, and after a
// reset c = 1, a = p -- so skipping the hops that do not reach a bin leaves every value as the hop-by-hop loop had it
// (round 2's first version walked all hops per bin: 0.9 ms per 1024-hop sweep); hop 0 is always evaluated.
__global__ void k_sview_accumulate(unsigned spectrum_size, const int *__restrict__ j0, const int *__restrict__ nb,
                                   const float *__restrict__ va, const float *__restrict__ vc, int n_hops,
                                   int max_bins, float *__restrict__ psd, float *__restrict__ accum,
                                   float *__restrict__ count, const float *__restrict__ count_before)
{
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = j < spectrum_size;
  const int lane = (int) (threadIdx.x & 31u);
  const int wj = (int) j - lane;                       // first bin of this warp
  float a = 0, c = 0, p = 0, cl = 1.0f;
  if (live) {
    a = accum[j]; c = count[j]; p = psd[j];
    // left neighbour's count (only its emptiness matters), from the snapshot taken before this launch: thread j-1
    // rewrites count[j-1] at the end of the kernel, possibly before this thread starts
    cl = j > 0 ? count_before[j - 1] : 1.0f;
  }
  for (int h0 = 0; h0 < n_hops; h0 += 32) {
    int hj = 0, hn = 0;
    if (h0 + lane < n_hops) { hj = j0[h0 + lane]; hn = nb[h0 + lane]; }
    unsigned m = __ballot_sync(0xffffffffu, hn > 0 && hj <= wj + 31 && hj + hn >= wj);
    if (h0 == 0) m |= 1u;
    while (m) {
      const int b = __ffs(m) - 1;
      m &= m - 1;
      const int h = h0 + b;
      const int t = (int) j - __shfl_sync(0xffffffffu, hj, b), n = __shfl_sync(0xffffffffu, hn, b);
      if (t >= 0 && t < n) {
        a += va[(size_t) h * max_bins + t];
        c += vc[(size_t) h * max_bins + t];
      }
      if (t - 1 >= 0 && t - 1 < n) cl += vc[(size_t) h * max_bins + t - 1];
      // interpolate() runs after every feed: a non-empty bin gets psd = accum / count; the count > 5
      // forgetting rule is applied only when the bin does not close a gap (Scanner.cpp:70-90: the branch
      // that ends a run of empty bins computes `right` without the reset).
      if (c > .5f) {
        p = a / c;
        const bool closes_gap = j > 0 && cl <= .5f;
        if (!closes_gap && c > 5.0f) { c = 1.0f; a = p * 1.0f; }
      }
    }
  }
  if (live) { accum[j] = a; count[j] = c; psd[j] = p; }
}

// final gap filling: exactly interpolate()'s treatment of runs of empty bins (Scanner.cpp:56-116).  A gap's fill
// values depend only on the non-empty bins on either side of it (which the fill never touches), so gaps are
// independent: every thread owns the gaps that START in its 64-bin segment, walks each to its end and fills it.
// (Round 1 walked the whole array with one thread: 6.8 ms per sweep for 65536 bins.)
#define SVIEW_SEG 64
__global__ void k_sview_fill(unsigned spectrum_size, float *__restrict__ psd, const float *__restrict__ count)
{
  const unsigned seg = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned i0 = seg * SVIEW_SEG;
  if (i0 >= spectrum_size) return;
  const unsigned i1 = i0 + SVIEW_SEG < spectrum_size ? i0 + SVIEW_SEG : spectrum_size;
  for (unsigned i = i0; i < i1; ++i) {
    if (!(count[i] <= .5f)) continue;
    if (i > 0 && count[i - 1] <= .5f) continue;           // not the first bin of its gap
    const unsigned zero_pos = i;
    const bool first = i == 0;
    const float left = first ? -200.0f : psd[i - 1];
    unsigned e = i;
    while (e < spectrum_size && count[e] <= .5f) ++e;     // e = first non-empty bin after the gap (or the end)
    const unsigned cnt = e - zero_pos;
    if (e == spectrum_size) {
      for (unsigned j = 0; j < cnt; ++j) psd[j + zero_pos] = left;
    } else {
      const float right = psd[e];
      if (first) {
        for (unsigned j = 0; j < cnt; ++j) psd[j + zero_pos] = right;
      } else {
        for (unsigned j = 0; j < cnt; ++j) {
          const float t = (float) (j + .5f) / cnt;
          psd[j + zero_pos] = (1 - t) * left + t * right;
        }
      }
    }
  }
}

static cudaError_t sdb_launch_sview_project(cudaStream_t s, double freq_min, double freq_range, double fft_bandwidth,
                                            float rel_bw, unsigned spectrum_size, const float *psd, size_t psd_size,
                                            const double *centers_dev, int n_hops, int adjust_sides, int *j0, int *nb,
                                            float *va, float *vc, int max_bins)
{
  SviewGeom g{ freq_min, freq_range, fft_bandwidth, rel_bw, spectrum_size };
  if (n_hops <= 0) return cudaSuccess;
  k_sview_project<<<n_hops, 256, 0, s>>>(g, psd, psd_size, centers_dev, n_hops, adjust_sides, j0, nb, va, vc, max_bins);
  return cudaGetLastError();
}

static cudaError_t sdb_launch_sview_accumulate(cudaStream_t s, unsigned spectrum_size, const int *j0, const int *nb,
                                               const float *va, const float *vc, int n_hops, int max_bins, float *psd,
                                               float *accum, float *count, float *count_snapshot)
{
  if (n_hops > 0) {
    cudaError_t e = cudaMemcpyAsync(count_snapshot, count, (size_t) spectrum_size * sizeof(float),
                                    cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) return e;
    k_sview_accumulate<<<(spectrum_size + 255) / 256, 256, 0, s>>>(spectrum_size, j0, nb, va, vc, n_hops, max_bins,
                                                                   psd, accum, count, count_snapshot);
  }
  k_sview_fill<<<((spectrum_size + SVIEW_SEG - 1) / SVIEW_SEG + 127) / 128, 128, 0, s>>>(spectrum_size, psd, count);
  return cudaGetLastError();
}

// PSDMessage post-processing as its own pass (Suscan/Messages/PSDMessage.cpp:32-38: fftshift + 10 log10),
// for engines that keep the linear PSD because the channel detector reads it.  Same expression as the
// fused epilogue of the PSD kernels (SDB_FLAG_PSD_SHIFT_DB), so the results are bit-identical to it.
__global__ void k_psd_shift_db(const float *__restrict__ lin, float *__restrict__ db, size_t total, unsigned n)
{
  const unsigned half = n >> 1;
  for (size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x; i < total; i += (size_t) gridDim.x * blockDim.x) {
    const size_t f = i / n;
    const unsigned k = (unsigned) (i - f * n);
    db[f * n + ((k + half) & (n - 1))] = 10.0f * d_log10f(__ldg(lin + i) + 1e-8f);
  }
}

// Spectrum averager of the GUI (Misc/Averager.cpp:25-50, fed per PSD message at UIMediator/SpectrumMediator.cpp:128):
// last += alpha * (x - last) per bin, frame after frame; the first frame (or alpha >= 1) is copied.
// One thread per (stream, bin); the frames of a feed are applied in order.
__global__ void k_psd_average(const float *__restrict__ psd, size_t stream_stride, unsigned frames, unsigned n,
                              size_t n_streams, float alpha, int primed, float *__restrict__ last)
{
  const size_t t = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (t >= n_streams * n) return;
  const size_t s = t / n;
  const unsigned k = (unsigned) (t - s * n);
  const float *__restrict__ x = psd + s * stream_stride + k;
  float v = last[t];
  for (unsigned f = 0; f < frames; ++f) {
    const float xv = __ldg(x + (size_t) f * n);
    if (!primed || alpha >= 1.0f) v = xv;
    else v += alpha * (xv - v);
    primed = 1;
  }
  last[t] = v;
}

static cudaError_t sdb_launch_psd_average(cudaStream_t s, const float *psd, size_t stream_stride, unsigned frames, unsigned n,
                                          size_t n_streams, float alpha, int primed, float *last)
{
  if (frames == 0 || n_streams * n == 0) return cudaSuccess;
  k_psd_average<<<(unsigned) ((n_streams * n + 255) / 256), 256, 0, s>>>(psd, stream_stride, frames, n, n_streams,
                                                                        alpha, primed, last);
  return cudaGetLastError();
}

// Frame-averaged main PSD (SPEC A, oracle/SPEC_A.md): per (stream, bin), the frames of the feed are added in order to
// the carried partial sum (plain binary32 adds, this unit is built without contraction); every A-th frame of the
// running count finishes a group, whose mean acc / A is one IEEE division.  psd is [S][frames][n], out [S][means][n]
// (fft-shifted and in dB with shift_db, the expression of k_psd_shift_db), carry [S][n].  `carried` frames of the
// current group precede this feed.  Threads of a warp own consecutive bins, so every load and store is coalesced; the
// frame loop issues UNROLL independent loads before the in-order adds.
#define SDB_MEAN_UNROLL 8
__global__ void __launch_bounds__(256) k_psd_group_mean(const float *__restrict__ psd, unsigned frames, unsigned n,
                                                         size_t n_streams, unsigned A, unsigned carried, unsigned means,
                                                         int shift_db, float *__restrict__ carry,
                                                         float *__restrict__ out)
{
  const size_t t = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (t >= n_streams * n) return;
  const size_t s = t / n;
  const unsigned k = (unsigned) (t - s * n);
  const float *__restrict__ x = psd + s * (size_t) frames * n + k;
  float *__restrict__ o = out + s * (size_t) means * n + (shift_db ? ((k + (n >> 1)) & (n - 1)) : k);
  const float fa = (float) A;
  // the carry is only read when a group is open and only written when one stays open: feeds that end on a group
  // boundary move no carry bytes
  float acc = carried ? carry[t] : 0.0f;
  unsigned cnt = carried;
  for (unsigned f0 = 0; f0 < frames; f0 += SDB_MEAN_UNROLL) {
    float v[SDB_MEAN_UNROLL];
#pragma unroll
    for (int u = 0; u < SDB_MEAN_UNROLL; ++u) v[u] = f0 + u < frames ? __ldg(x + (size_t) (f0 + u) * n) : 0.0f;
#pragma unroll
    for (int u = 0; u < SDB_MEAN_UNROLL; ++u) {
      if (f0 + u < frames) {
        acc = __fadd_rn(acc, v[u]);
        if (++cnt == A) {
          const float m = __fdiv_rn(acc, fa);
          *o = shift_db ? 10.0f * d_log10f(m + 1e-8f) : m;
          o += n; acc = 0.0f; cnt = 0;
        }
      }
    }
  }
  if (cnt) carry[t] = acc;
}

cudaError_t sdb_launch_psd_group_mean(const SdbLaunchCtx &c, const float *psd, unsigned frames, unsigned n,
                                      size_t n_streams, unsigned A, unsigned carried, unsigned means, int shift_db,
                                      float *carry, float *out)
{
  if (frames == 0 || n_streams * n == 0) return cudaSuccess;
  k_psd_group_mean<<<(unsigned) ((n_streams * n + 255) / 256), 256, 0, c.stream>>>(psd, frames, n, n_streams, A, carried,
                                                                                   means, shift_db, carry, out);
  if (c.launch_counter) ++*c.launch_counter;
  return cudaGetLastError();
}

// Peak detectors of the main PSD (SPEC PK, oracle/SPEC_PK.md): per (stream, bin), the frames of the feed update the
// carried group maximum and minimum with fmaxf / fminf (maxNum / minNum: a NaN operand is ignored); every P-th frame of
// the running count finishes a group, written to both outputs (fft-shifted and in dB with shift_db, the expression of
// k_psd_shift_db, after the extreme is taken).  An empty group holds NaN, which the group's first frame replaces
// (fmaxf(NaN, x) = x): that is PK.2's "the first frame starts the value" without a branch.  psd is [S][frames][n],
// outputs [S][groups][n], carries [S][n]; `carried` frames of the current group precede this feed.
// Each thread owns 4 consecutive bins (n is a power of two >= 16, so a float4 never straddles a stream or the fft-shift
// seam, and every row is 16-byte aligned): loads and stores are 16-byte and coalesced across the warp, and the frame
// loop issues UNROLL independent loads before the compares.  4 bins a thread moved more bytes per second than 1 on an
// H100 (DESIGN.md, kernel table).
#define SDB_PEAK_UNROLL 8
static __device__ __forceinline__ float4 peak_fmax4(float4 a, float4 b)
{
  return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w));
}
static __device__ __forceinline__ float4 peak_fmin4(float4 a, float4 b)
{
  return make_float4(fminf(a.x, b.x), fminf(a.y, b.y), fminf(a.z, b.z), fminf(a.w, b.w));
}
static __device__ __forceinline__ float4 peak_out4(float4 a, int shift_db)
{
  if (!shift_db) return a;
  return make_float4(10.0f * d_log10f(a.x + 1e-8f), 10.0f * d_log10f(a.y + 1e-8f), 10.0f * d_log10f(a.z + 1e-8f),
                     10.0f * d_log10f(a.w + 1e-8f));
}

static __global__ void __launch_bounds__(256) k_psd_group_peak(const float4 *__restrict__ psd, unsigned frames,
                                                                unsigned n4, size_t n_streams, unsigned P,
                                                                unsigned carried, unsigned groups, int shift_db,
                                                                float4 *__restrict__ carry_max,
                                                                float4 *__restrict__ carry_min,
                                                                float4 *__restrict__ out_max,
                                                                float4 *__restrict__ out_min)
{
  const size_t t = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (t >= n_streams * n4) return;
  const size_t s = t / n4;
  const unsigned k4 = (unsigned) (t - s * n4);
  const float4 *__restrict__ x = psd + s * (size_t) frames * n4 + k4;
  size_t o = s * (size_t) groups * n4 + (shift_db ? ((k4 + (n4 >> 1)) & (n4 - 1)) : k4);
  const float q = __int_as_float(0x7fffffff);
  const float4 empty = make_float4(q, q, q, q);
  // as in k_psd_group_mean, the carries move only while a group stays open across a feed boundary
  float4 mx = carried ? carry_max[t] : empty, mn = carried ? carry_min[t] : empty;
  unsigned cnt = carried;
  for (unsigned f0 = 0; f0 < frames; f0 += SDB_PEAK_UNROLL) {
    float4 v[SDB_PEAK_UNROLL];
#pragma unroll
    for (int u = 0; u < SDB_PEAK_UNROLL; ++u) v[u] = f0 + u < frames ? __ldg(x + (size_t) (f0 + u) * n4) : empty;
#pragma unroll
    for (int u = 0; u < SDB_PEAK_UNROLL; ++u) {
      if (f0 + u < frames) {
        mx = peak_fmax4(mx, v[u]); mn = peak_fmin4(mn, v[u]);
        if (++cnt == P) {
          out_max[o] = peak_out4(mx, shift_db); out_min[o] = peak_out4(mn, shift_db);
          o += n4; mx = mn = empty; cnt = 0;
        }
      }
    }
  }
  if (cnt) { carry_max[t] = mx; carry_min[t] = mn; }
}

cudaError_t sdb_launch_psd_group_peak(const SdbLaunchCtx &c, const float *psd, unsigned frames, unsigned n,
                                      size_t n_streams, unsigned P, unsigned carried, unsigned groups, int shift_db,
                                      float *carry_max, float *carry_min, float *out_max, float *out_min)
{
  if (frames == 0 || n_streams * n == 0) return cudaSuccess;
  const size_t threads = n_streams * (n / 4);
  k_psd_group_peak<<<(unsigned) ((threads + 255) / 256), 256, 0, c.stream>>>(
      reinterpret_cast<const float4 *>(psd), frames, n / 4, n_streams, P, carried, groups, shift_db,
      reinterpret_cast<float4 *>(carry_max), reinterpret_cast<float4 *>(carry_min), reinterpret_cast<float4 *>(out_max),
      reinterpret_cast<float4 *>(out_min));
  if (c.launch_counter) ++*c.launch_counter;
  return cudaGetLastError();
}

static cudaError_t sdb_launch_psd_shift_db(cudaStream_t s, const float *lin, float *db, size_t n_frames, unsigned n)
{
  const size_t total = n_frames * n;
  if (total == 0) return cudaSuccess;
  size_t blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;        // 16 CTAs on each of an H100's 132 SMs, grid-stride beyond
  k_psd_shift_db<<<(unsigned) blocks, 256, 0, s>>>(lin, db, total, n);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// SpectrumView (Panoramic/Scanner.cpp:36-293): panoramic stitcher
// ---------------------------------------------------------------------------------------------

struct sdb_sview {
  int device = 0;
  double freq_min = 0, freq_max = 0, freq_range = 0, fft_bandwidth = 0;
  float rel_bw = 0.5f;                     // include/Scanner.h:70
  unsigned spectrum_size = 65536;          // SIGDIGGER_SCANNER_SPECTRUM_SIZE
  int max_bins = 0;
  DevBuf<float> d_psd, d_accum, d_count, d_count_snap;
  // contribution lists of the last sdb_sview_project: j0 / nb [hops], va / vc [hops][max_bins]
  DevBuf<double> d_centers; DevBuf<int> d_j0, d_nb; DevBuf<float> d_va, d_vc;
};

extern "C" sdb_sview_t *sdb_sview_new(int device)
{
  if (sdb_device_count() <= 0) { g_err = "no CUDA device: sigdigger_b200 has no CPU fallback"; return nullptr; }
  CKP(cudaSetDevice(device));
  sdb_sview *v = new sdb_sview();
  v->device = device;
  const size_t n = 65536 * sizeof(float);
  if (v->d_psd.alloc(65536) != cudaSuccess || v->d_accum.alloc(65536) != cudaSuccess ||
      v->d_count.alloc(65536) != cudaSuccess || v->d_count_snap.alloc(65536) != cudaSuccess) {
    g_err = "out of device memory"; delete v; return nullptr;
  }
  cudaMemset(v->d_psd, 0, n); cudaMemset(v->d_accum, 0, n); cudaMemset(v->d_count, 0, n);
  return v;
}

extern "C" void sdb_sview_destroy(sdb_sview_t *v)
{
  if (!v) return;
  cudaSetDevice(v->device);
  delete v;
}

extern "C" int sdb_sview_reset(sdb_sview_t *v)
{
  if (!v) return fail("null view");
  CK(cudaSetDevice(v->device));
  const size_t n = 65536 * sizeof(float);          // SpectrumView::reset, Scanner.cpp:287-293
  CK(cudaMemset(v->d_psd, 0, n)); CK(cudaMemset(v->d_accum, 0, n)); CK(cudaMemset(v->d_count, 0, n));
  return 0;
}

int sdb_sview_reset_async(sdb_sview_t *v, cudaStream_t st)     // the same, ordered on the caller's stream
{
  if (!v) return fail("null view");
  const size_t n = 65536 * sizeof(float);
  CK(cudaMemsetAsync(v->d_psd, 0, n, st)); CK(cudaMemsetAsync(v->d_accum, 0, n, st));
  CK(cudaMemsetAsync(v->d_count, 0, n, st));
  return 0;
}

extern "C" int sdb_sview_set_range(sdb_sview_t *v, double fmin, double fmax, double fft_bandwidth, float rel_bw)
{
  if (!v) return fail("null view");
  if (!(fmax > fmin) || !(fft_bandwidth > 0)) return fail("invalid frequency range");
  v->freq_min = fmin; v->freq_max = fmax; v->freq_range = fmax - fmin;   // setRange, Scanner.cpp:41-54
  unsigned n = (unsigned) (v->freq_range / 1000.0), sz = 1;               // SIGDIGGER_SCANNER_FREQ_RESOLUTION
  while (sz < n) sz <<= 1;
  if (sz > 65536) sz = 65536;
  v->spectrum_size = sz;
  v->fft_bandwidth = fft_bandwidth; v->rel_bw = rel_bw;
  // a hop contributes at most sz * (fft_bandwidth - 2 skip) / freq_range + 1 bins, and every projection uses THIS
  // fft_bandwidth (the kernels take the geometry from the view, not from the call): the `nb > max_bins` clamp in the
  // projection kernels is a guard that cannot bind
  double mb = (double) sz * fft_bandwidth / v->freq_range + 4.0;
  v->max_bins = mb > (double) sz ? (int) sz : (int) mb;
  if (v->max_bins < 2) v->max_bins = 2;
  v->d_centers.release();   // the contribution lists depend on max_bins: sdb_sview_project reallocates them
  return sdb_sview_reset(v);
}

extern "C" uint32_t sdb_sview_size(const sdb_sview_t *v) { return v ? v->spectrum_size : 0; }
extern "C" uint32_t sdb_sview_max_bins(const sdb_sview_t *v) { return v ? (uint32_t) v->max_bins : 0; }

extern "C" int sdb_sview_project(sdb_sview_t *v, const float *psd_dev, size_t psd_size, const double *centers,
                                 size_t n_hops, int adjust_sides)
{
  if (!v || !psd_dev || !centers) return fail("null argument");
  if (v->max_bins <= 0) return fail("set_range first");
  CK(cudaSetDevice(v->device));
  if (n_hops > v->d_centers.size()) {
    // d_centers is released first and allocated last: its size is 0 until every list has been allocated
    v->d_centers.release();
    CK(v->d_j0.alloc(n_hops)); CK(v->d_nb.alloc(n_hops));
    CK(v->d_va.alloc(n_hops * (size_t) v->max_bins)); CK(v->d_vc.alloc(n_hops * (size_t) v->max_bins));
    CK(v->d_centers.alloc(n_hops));
  }
  CK(cudaMemcpy(v->d_centers, centers, n_hops * sizeof(double), cudaMemcpyHostToDevice));
  CK(cudaMemset(v->d_va, 0, n_hops * (size_t) v->max_bins * sizeof(float)));
  CK(cudaMemset(v->d_vc, 0, n_hops * (size_t) v->max_bins * sizeof(float)));
  CK(sdb_launch_sview_project(0, v->freq_min, v->freq_range, v->fft_bandwidth, v->rel_bw, v->spectrum_size, psd_dev,
                              psd_size, v->d_centers, (int) n_hops, adjust_sides, v->d_j0, v->d_nb, v->d_va, v->d_vc,
                              v->max_bins));
  return 0;
}

// ---- stream-ordered variants for the panoramic sweep (sdb_internal.h)
int sdb_sview_project_async(sdb_sview_t *v, cudaStream_t st, const float *psd_dev, size_t psd_size, size_t hop_stride,
                            int psd_is_linear, const double *centers_dev, size_t n_hops, int adjust_sides, int32_t *j0,
                            int32_t *nb, float *va, float *vc)
{
  if (!v || !psd_dev || !centers_dev || !j0 || !nb || !va || !vc) return fail("null argument");
  if (v->max_bins <= 0) return fail("set_range first");
  const bool linear_mode = v->fft_bandwidth / v->freq_range * v->spectrum_size >= 2.001;  // every hop, with margin
                                                                                              // for the kernel's own test
  if (linear_mode && v->max_bins <= 384) {
    CK(sdb_launch_sview_project_tiled(st, v->freq_min, v->freq_range, v->fft_bandwidth, v->rel_bw, v->spectrum_size,
                                      psd_dev, psd_size, hop_stride, psd_is_linear, centers_dev, (int) n_hops,
                                      adjust_sides, j0, nb, va, vc, v->max_bins));
    return 0;
  }
  if (psd_is_linear || hop_stride != psd_size) return 1;
  CK(sdb_launch_sview_project(st, v->freq_min, v->freq_range, v->fft_bandwidth, v->rel_bw, v->spectrum_size, psd_dev,
                              psd_size, centers_dev, (int) n_hops, adjust_sides, j0, nb, va, vc, v->max_bins));
  return 0;
}

int sdb_sview_accumulate_async(sdb_sview_t *v, cudaStream_t st, const int32_t *j0, const int32_t *nb, const float *va,
                               const float *vc, size_t n_hops)
{
  if (!v) return fail("null view");
  CK(sdb_launch_sview_accumulate(st, v->spectrum_size, j0, nb, va, vc, (int) n_hops, v->max_bins, v->d_psd, v->d_accum,
                                 v->d_count, v->d_count_snap));
  return 0;
}

int sdb_psd_shift_db_async(cudaStream_t st, const float *lin_dev, float *db_dev, size_t n_frames, uint32_t psd_size)
{
  if (!lin_dev || !db_dev || lin_dev == db_dev) return fail("invalid argument");
  CK(sdb_launch_psd_shift_db(st, lin_dev, db_dev, n_frames, psd_size));
  return 0;
}


extern "C" int sdb_psd_shift_db_device(const float *lin_dev, float *db_dev, size_t n_frames, uint32_t psd_size)
{
  if (!lin_dev || !db_dev) return fail("null argument");
  if (lin_dev == db_dev) return fail("in-place conversion is not supported (the halves swap)");
  if (psd_size < 2 || (psd_size & (psd_size - 1))) return fail("psd_size must be a power of two");
  CK(sdb_launch_psd_shift_db(0, lin_dev, db_dev, n_frames, psd_size));
  return 0;
}

// ---- SpectrumView::feed(SpectrumView const &) (Panoramic/Scanner.cpp:276-286; used by the zoom path of
// ---- Scanner::setViewRange, :471-479): project the other view's accumulators / counts, then the same accumulate
// ---- + interpolate pass a hop gets.

extern "C" int sdb_sview_feed_view(sdb_sview_t *v, const sdb_sview_t *detail)
{
  if (!v || !detail) return fail("null view");
  if (v == detail) return fail("a view cannot be fed into itself");
  if (v->max_bins <= 0 || detail->max_bins <= 0) return fail("set_range first");
  if (v->device != detail->device) return fail("both views must live on the same device");
  CK(cudaSetDevice(v->device));
  DevBuf<int> j0, nb; DevBuf<float> va, vc;
  const size_t row = 65536 * sizeof(float);
  cudaError_t e = j0.alloc(1);
  if (e == cudaSuccess) e = nb.alloc(1);
  if (e == cudaSuccess) e = va.alloc(65536);
  if (e == cudaSuccess) e = vc.alloc(65536);
  if (e == cudaSuccess) e = cudaMemset(j0, 0, sizeof(int));
  if (e == cudaSuccess) e = cudaMemset(nb, 0, sizeof(int));
  if (e == cudaSuccess) e = cudaMemset(va, 0, row);
  if (e == cudaSuccess) e = cudaMemset(vc, 0, row);
  if (e == cudaSuccess)
    e = sdb_launch_sview_project_view(0, v->freq_min, v->freq_range, v->spectrum_size, detail->d_accum, detail->d_count,
                                      detail->spectrum_size, detail->freq_min, detail->freq_max, j0, nb, va, vc);
  if (e == cudaSuccess)
    e = sdb_launch_sview_accumulate(0, v->spectrum_size, j0, nb, va, vc, 1, 65536, v->d_psd, v->d_accum, v->d_count,
                                    v->d_count_snap);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(std::string("sdb_sview_feed_view: ") + cudaGetErrorString(e));
  return 0;
}

// ---- spectrum averager (Misc/Averager.cpp:25-60)
struct sdb_averager {
  int device = 0; unsigned n = 0; size_t n_streams = 0; float alpha = 1.0f; bool primed = false;
  DevBuf<float> d_last;
};

extern "C" sdb_averager_t *sdb_averager_new(uint32_t psd_size, uint32_t n_streams, float alpha, int device)
{
  if (sdb_device_count() <= 0) { g_err = "no CUDA device: sigdigger_b200 has no CPU fallback"; return nullptr; }
  if (psd_size == 0 || n_streams == 0) { g_err = "averager: empty geometry"; return nullptr; }
  CKP(cudaSetDevice(device));
  sdb_averager *a = new sdb_averager();
  a->device = device; a->n = psd_size; a->n_streams = n_streams; a->alpha = alpha;
  if (a->d_last.alloc((size_t) psd_size * n_streams) != cudaSuccess) {
    g_err = "out of device memory"; delete a; return nullptr;
  }
  cudaMemset(a->d_last, 0, (size_t) psd_size * n_streams * sizeof(float));
  return a;
}

extern "C" void sdb_averager_destroy(sdb_averager_t *a)
{
  if (!a) return;
  cudaSetDevice(a->device);
  delete a;
}

extern "C" int sdb_averager_set_alpha(sdb_averager_t *a, float alpha)
{
  if (!a) return fail("null averager");
  a->alpha = alpha;
  return 0;
}

extern "C" int sdb_averager_reset(sdb_averager_t *a)
{
  if (!a) return fail("null averager");
  a->primed = false;
  return 0;
}

extern "C" int sdb_averager_feed_device(sdb_averager_t *a, const float *psd_dev, size_t frames, size_t stream_stride)
{
  if (!a || !psd_dev) return fail("null argument");
  if (frames == 0) return 0;
  if (stream_stride < frames * a->n && a->n_streams > 1) return fail("stream stride smaller than the frames");
  CK(cudaSetDevice(a->device));
  CK(sdb_launch_psd_average(0, psd_dev, stream_stride, (unsigned) frames, a->n, a->n_streams, a->alpha,
                            a->primed ? 1 : 0, a->d_last));
  a->primed = true;
  return 0;
}

extern "C" const float *sdb_averager_device(const sdb_averager_t *a) { return a ? a->d_last.get() : nullptr; }

extern "C" int sdb_averager_read(sdb_averager_t *a, float *dst, size_t cap)
{
  if (!a || !dst) return fail("null argument");
  const size_t tot = (size_t) a->n * a->n_streams;
  if (cap < tot) return fail("destination too small");
  CK(cudaSetDevice(a->device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(dst, a->d_last, tot * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int sdb_sview_contrib(sdb_sview_t *v, int32_t **j0, int32_t **nb, float **va, float **vc)
{
  if (!v) return fail("null view");
  if (j0) *j0 = v->d_j0;
  if (nb) *nb = v->d_nb;
  if (va) *va = v->d_va;
  if (vc) *vc = v->d_vc;
  return 0;
}

// copy the last projection's contribution lists into caller-owned DEVICE buffers (the send buffers of the
// NCCL gather): j0/nb [n_hops] int32, va/vc [n_hops][max_bins] float32
extern "C" int sdb_sview_contrib_copy(sdb_sview_t *v, int32_t *j0, int32_t *nb, float *va, float *vc, size_t n_hops)
{
  if (!v || !j0 || !nb || !va || !vc) return fail("null argument");
  if (n_hops > v->d_centers.size()) return fail("more hops than the last projection held");
  CK(cudaSetDevice(v->device));
  const size_t row = (size_t) v->max_bins * sizeof(float);
  CK(cudaMemcpy(j0, v->d_j0, n_hops * sizeof(int), cudaMemcpyDeviceToDevice));
  CK(cudaMemcpy(nb, v->d_nb, n_hops * sizeof(int), cudaMemcpyDeviceToDevice));
  CK(cudaMemcpy(va, v->d_va, n_hops * row, cudaMemcpyDeviceToDevice));
  CK(cudaMemcpy(vc, v->d_vc, n_hops * row, cudaMemcpyDeviceToDevice));
  return 0;
}

extern "C" int sdb_sview_accumulate(sdb_sview_t *v, const int32_t *j0, const int32_t *nb, const float *va,
                                    const float *vc, size_t n_hops)
{
  if (!v) return fail("null view");
  CK(cudaSetDevice(v->device));
  CK(sdb_launch_sview_accumulate(0, v->spectrum_size, j0, nb, va, vc, (int) n_hops, v->max_bins, v->d_psd, v->d_accum,
                                 v->d_count, v->d_count_snap));
  return 0;
}

extern "C" int sdb_sview_read(sdb_sview_t *v, float *psd, float *accum, float *count, size_t cap)
{
  if (!v) return fail("null view");
  if (cap < v->spectrum_size) return fail("destination too small");
  CK(cudaSetDevice(v->device));
  CK(cudaDeviceSynchronize());
  const size_t n = v->spectrum_size * sizeof(float);
  if (psd) CK(cudaMemcpy(psd, v->d_psd, n, cudaMemcpyDeviceToHost));
  if (accum) CK(cudaMemcpy(accum, v->d_accum, n, cudaMemcpyDeviceToHost));
  if (count) CK(cudaMemcpy(count, v->d_count, n, cudaMemcpyDeviceToHost));
  return 0;
}
