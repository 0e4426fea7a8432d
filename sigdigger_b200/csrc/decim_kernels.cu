// decim_kernels.cu -- source decimation (SPEC L, oracle/SPEC_L.md): the FIR decimator behind the source config's `average`
// (Suscan/Source.cpp:195-201, 419-425), batched over streams, and its stand-alone host object sdb_decimator.
//
// y[k] = sum_{i=0}^{16D} h_i x[kD - i] with h = brick-wall LP (SPEC I.3) of 16 D + 1 taps at fc = 1/D; one accumulator
// per component from 0, ascending i, one FFMA per term (SPEC I.1's order), so the result is bit-identical to
// oracle/decimate.c.  Each feed reads a virtual stream: the 16 D float32 samples carried from the previous feed,
// followed by the new input in its native format (converted in the staging load, sdb_iq.h).
#include "sdb_internal.h"
#include "host_design.h"
#include <algorithm>
#include <vector>

constexpr int kT = 128;       // threads per CTA
constexpr int kB = 4;         // consecutive outputs per thread: one staged sample feeds all four accumulators
constexpr int kC = 32;        // steps (input samples per thread) staged per chunk
constexpr int kRow = kC + 1;  // padded run: lane t reads run t at a stride of 33 float2, no bank conflicts

// Thread t of CTA c owns outputs k_t .. k_t + 3, k_t = 512 c + 4 t.  At step s (0 <= s < 19 D + 1) it reads the
// virtual sample v(k_t + 3) - s, where v(k) = 16 D + t0 + kD is the newest sample of output k, and accumulator b
// (output k_t + b) takes it with tap i = s - (3 - b) D when 0 <= i <= 16 D.  So every accumulator takes its taps in
// ascending i, and one shared-memory load of a sample serves four outputs.  The CTA stages, per chunk of 32 steps,
// each thread's 32 samples as one padded run; the taps sit in shared memory for the whole CTA.
template <bool kFull>
static __device__ __forceinline__ void decim_steps(const float2 *__restrict__ run, const float *__restrict__ h, int s0, int C,
                                            int D, int n_taps, float2 (&acc)[kB])
{
#pragma unroll 4
  for (int c = 0; c < C; ++c) {
    const int s = s0 + c;
    const float2 xv = run[c];
#pragma unroll
    for (int b = 0; b < kB; ++b) {
      const int i = s - (kB - 1 - b) * D;
      if (kFull || (i >= 0 && i < n_taps)) {
        const float hv = h[i];
        acc[b].x = __fmaf_rn(hv, xv.x, acc[b].x);
        acc[b].y = __fmaf_rn(hv, xv.y, acc[b].y);
      }
    }
  }
}

__global__ void __launch_bounds__(kT) k_decimate(const void *__restrict__ x, int fmt, size_t x_stride, long m,
                                                 const float2 *__restrict__ carry, int D, int t0, int n_out,
                                                 const float *__restrict__ taps, float2 *__restrict__ y,
                                                 size_t y_stride)
{
  extern __shared__ float4 smem_f4[];
  const int n_taps = 16 * D + 1, L = 16 * D;
  float *h = reinterpret_cast<float *>(smem_f4);
  float2 *st = reinterpret_cast<float2 *>(h + ((n_taps + 3) & ~3));
  const int sid = blockIdx.y;
  const float2 *cs = carry + (size_t) sid * L;
  const long xbase = (long) sid * (long) x_stride;
  for (int i = threadIdx.x; i < n_taps; i += kT) h[i] = taps[i];

  const int k_blk = blockIdx.x * (kT * kB);
  const long vtop = (long) L + t0 + (long) (k_blk + kB - 1) * D;   // newest sample of thread 0's last output
  const long vend = (long) L + m;
  const int s_tot = n_taps + (kB - 1) * D;
  float2 acc[kB];
#pragma unroll
  for (int b = 0; b < kB; ++b) acc[b] = make_float2(0.0f, 0.0f);
  const float2 *run = st + threadIdx.x * kRow;

  for (int s0 = 0; s0 < s_tot; s0 += kC) {
    const int C = min(kC, s_tot - s0);
    __syncthreads();                                   // the previous chunk has been consumed
    // warp w stages runs w, w + 4, ...: lane p loads step s0 + p of the run (descending addresses, coalesced)
    for (int e = threadIdx.x; e < kT * kC; e += kT) {
      const int t = e / kC, p = e % kC;
      const long v = vtop + (long) t * kB * D - s0 - p;
      float2 val = make_float2(0.0f, 0.0f);
      if (p < C && v < vend) val = v < L ? cs[v] : sdb_ld_iq(x, xbase + (v - L), fmt);
      st[t * kRow + p] = val;
    }
    __syncthreads();
    // every accumulator is active over the whole chunk when its first and last steps are inside [0, 16 D]
    if (s0 >= (kB - 1) * D && s0 + C - 1 < n_taps) decim_steps<true>(run, h, s0, C, D, n_taps, acc);
    else decim_steps<false>(run, h, s0, C, D, n_taps, acc);
  }
  const int kt = k_blk + threadIdx.x * kB;
#pragma unroll
  for (int b = 0; b < kB; ++b)
    if (kt + b < n_out) y[(size_t) sid * y_stride + kt + b] = acc[b];
}

// next carry: virtual samples [m, m + 16 D) of every stream, into the other carry buffer
__global__ void k_decim_carry(const void *__restrict__ x, int fmt, size_t x_stride, long m,
                              const float2 *__restrict__ carry_in, float2 *__restrict__ carry_out, int L)
{
  const int q = blockIdx.x * blockDim.x + threadIdx.x, sid = blockIdx.y;
  if (q >= L) return;
  const long v = m + q;
  carry_out[(size_t) sid * L + q] = v < L ? carry_in[(size_t) sid * L + v]
                                          : sdb_ld_iq(x, (long) sid * (long) x_stride + (v - L), fmt);
}

static size_t decim_smem_bytes(int D)
{
  return (size_t) ((16 * D + 1 + 3) & ~3) * sizeof(float) + (size_t) kT * kRow * sizeof(float2);
}

static std::atomic<unsigned long long> g_decim_smem_set{ 0 };

struct sdb_decimator {
  int device = 0;
  uint32_t S = 0, D = 1;
  int fmt = SDB_FMT_F32;
  size_t max_feed = 0, out_cap = 0;
  uint32_t phase = 0;             // input samples fed so far, modulo D
  int cur = 0;                    // carry[cur] holds the last 16 D input samples of every stream
  size_t last_out = 0;            // outputs per stream of the last feed
  DevBuf<float> taps;
  DevBuf<float2> carry[2], out;
  DevBuf<unsigned char> xin;      // host feeds: input staged on the device
  Stream stream;
};

extern "C" sdb_decimator_t *sdb_decimator_new(int device, uint32_t n_streams, uint32_t decimation, int32_t input_format,
                                              size_t max_feed)
{
  if (sdb_device_count() <= 0) { g_err = "no CUDA device: sigdigger_b200 has no CPU fallback"; return nullptr; }
  if (n_streams == 0 || max_feed == 0) { g_err = "decimator: empty geometry"; return nullptr; }
  if (decimation < 1 || decimation > SDB_DECIMATION_MAX) {
    g_err = "decimation must be in [1, " + std::to_string(SDB_DECIMATION_MAX) + "], got " + std::to_string(decimation);
    return nullptr;
  }
  if (input_format < SDB_FORMAT_FLOAT32 || input_format > SDB_FORMAT_SIGNED16) { g_err = "unknown input format"; return nullptr; }
  if (max_feed > (size_t) 1 << 31) { g_err = "decimator: max_feed above 2^31 samples"; return nullptr; }
  CKP(cudaSetDevice(device));
  sdb_decimator *d = new sdb_decimator();
  d->device = device; d->S = n_streams; d->D = decimation; d->fmt = input_format; d->max_feed = max_feed;
  d->out_cap = max_feed / decimation + 1;
  const size_t L = (size_t) 16 * decimation, n_taps = L + 1;
  std::vector<float> h(n_taps);
  sdbh::taps_brickwall_lp(h.data(), (unsigned) n_taps, (float) (1.0 / (double) decimation));
  cudaError_t e = d->stream.create(cudaStreamNonBlocking);
  if (e == cudaSuccess) e = d->taps.alloc(n_taps);
  if (e == cudaSuccess) e = d->carry[0].alloc(L * n_streams);
  if (e == cudaSuccess) e = d->carry[1].alloc(L * n_streams);
  if (e == cudaSuccess) e = d->out.alloc(d->out_cap * n_streams);
  if (e == cudaSuccess) e = cudaMemcpy(d->taps, h.data(), n_taps * sizeof(float), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemset(d->carry[0], 0, L * n_streams * sizeof(float2));
  if (e == cudaSuccess && sdb_first_on_device(g_decim_smem_set))
    e = cudaFuncSetAttribute(k_decimate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) decim_smem_bytes(256));
  if (e != cudaSuccess) { g_err = std::string("decimator: ") + cudaGetErrorString(e); delete d; return nullptr; }
  return d;
}

extern "C" void sdb_decimator_destroy(sdb_decimator_t *d)
{
  if (!d) return;
  cudaSetDevice(d->device);
  cudaStreamSynchronize(d->stream);
  delete d;
}

extern "C" long sdb_decimator_feed_device(sdb_decimator_t *d, const void *x, size_t stream_stride, size_t n)
{
  if (!d || !x) return fail("null argument");
  if (n == 0 || n > d->max_feed) return fail("feed size out of range");
  if (d->S > 1 && stream_stride < n) return fail("stream stride smaller than the feed");
  CK(cudaSetDevice(d->device));
  const int D = (int) d->D, L = 16 * D;
  const int t0 = (int) ((d->D - d->phase) % d->D);                 // first output of this feed, as an input offset
  const size_t n_out = n > (size_t) t0 ? (n - (size_t) t0 + d->D - 1) / d->D : 0;
  if (n_out) {
    dim3 grid((unsigned) ((n_out + kT * kB - 1) / (kT * kB)), d->S);
    k_decimate<<<grid, kT, decim_smem_bytes(D), d->stream>>>(x, d->fmt, stream_stride, (long) n, d->carry[d->cur], D,
                                                              t0, (int) n_out, d->taps, d->out, d->out_cap);
    CK(cudaGetLastError());
  }
  k_decim_carry<<<dim3((unsigned) ((L + 255) / 256), d->S), 256, 0, d->stream>>>(x, d->fmt, stream_stride, (long) n,
                                                                                 d->carry[d->cur], d->carry[d->cur ^ 1], L);
  CK(cudaGetLastError());
  d->cur ^= 1;
  d->phase = (uint32_t) ((d->phase + n) % d->D);
  d->last_out = n_out;
  return (long) n_out;
}

extern "C" long sdb_decimator_feed_host(sdb_decimator_t *d, const void *x, size_t stream_stride, size_t n)
{
  if (!d || !x) return fail("null argument");
  if (n == 0 || n > d->max_feed) return fail("feed size out of range");
  if (d->S > 1 && stream_stride < n) return fail("stream stride smaller than the feed");
  CK(cudaSetDevice(d->device));
  const size_t bps = sdb_fmt_bytes(d->fmt);
  if (!d->xin.size() && d->xin.alloc(d->max_feed * d->S * bps) != cudaSuccess)
    return fail("out of device memory (input staging)");
  // the copy waits, in stream order, for the kernels of the previous feed to finish reading the staging buffer
  CK(cudaMemcpy2DAsync(d->xin, n * bps, x, (d->S > 1 ? stream_stride : n) * bps, n * bps, d->S, cudaMemcpyHostToDevice,
                       d->stream));
  return sdb_decimator_feed_device(d, d->xin.get(), n, n);
}

extern "C" const sdb_complex *sdb_decimator_output_device(const sdb_decimator_t *d)
{
  return d ? reinterpret_cast<const sdb_complex *>(d->out.get()) : nullptr;
}

extern "C" size_t sdb_decimator_output_stride(const sdb_decimator_t *d) { return d ? d->out_cap : 0; }

extern "C" void *sdb_decimator_stream(const sdb_decimator_t *d) { return d ? (void *) d->stream.get() : nullptr; }

extern "C" int sdb_decimator_sync(sdb_decimator_t *d)
{
  if (!d) return fail("null decimator");
  CK(cudaSetDevice(d->device));
  CK(cudaStreamSynchronize(d->stream));
  return 0;
}

extern "C" int sdb_decimator_read(sdb_decimator_t *d, sdb_complex *dst, size_t cap)
{
  if (!d || !dst) return fail("null argument");
  if (cap < d->last_out * d->S) return fail("destination too small");
  CK(cudaSetDevice(d->device));
  if (d->last_out)
    CK(cudaMemcpy2DAsync(dst, d->last_out * sizeof(float2), d->out, d->out_cap * sizeof(float2),
                         d->last_out * sizeof(float2), d->S, cudaMemcpyDeviceToHost, d->stream));
  CK(cudaStreamSynchronize(d->stream));
  return 0;
}

extern "C" int sdb_decimator_reset(sdb_decimator_t *d)
{
  if (!d) return fail("null decimator");
  CK(cudaSetDevice(d->device));
  CK(cudaMemsetAsync(d->carry[d->cur], 0, (size_t) 16 * d->D * d->S * sizeof(float2), d->stream));
  d->phase = 0; d->last_out = 0;
  return 0;
}
