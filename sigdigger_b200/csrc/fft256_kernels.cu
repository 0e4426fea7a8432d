// fft256_kernels.cu -- the 65536-point transform of BASELINE.json's headline configs, specialised:
// 65536 = 256 x 256, each 256-point transform = 16 x 16 with BOTH radix-16 butterflies held in
// registers (16 complex values per thread) and ONE shared-memory exchange between them.
//
//   pass A (k_cols256): a CTA owns 16 adjacent columns of a window: every thread issues 16 independent
//       coalesced float2 loads (128 B per thread in flight), optional window multiply, radix-16 over the
//       high row digit, twiddle W_256^(t ka), exchange, radix-16 over the low row digit, inter-pass twiddle
//       W_65536^(n2 k1) = coarse x fine (SPEC F.4) read from a [k1][n2] table tabulated once with the same
//       arithmetic, transposed coalesced store into the L2-pinned scratch.
//   pass B (k_rows256): a CTA owns 32 rows of the scratch; same two butterflies; the second one is mapped
//       so that a warp holds 32 consecutive output bins -> 128-byte PSD / compacted-spectrum stores.
//
// Same mathematics as the generic path in fft_kernels.cu (which remains for every other size); results
// are bit-identical to oracle/fft_spec.c (SPEC.md F.4).
// Replaces the forward FFTs of su_specttuner
// (Tasks/LPFTask.cpp:83-87) and of the PSD (Suscan/Messages/PSDMessage.cpp:26-39).
#include "sdb_internal.h"
#include "sdb_math.h"
#include "sdb_cpx.h"

#define C1 0.92387953251128675613f   // cos(pi/8)
#define S1 0.38268343236508977173f   // sin(pi/8)
#define R2 0.70710678118654752440f

// complex arithmetic (cadd, csub, cmulf = SPEC F.1 twiddle product, fft4): sdb_cpx.h.  The unit is compiled with -fmad=false so nothing else is contracted.

// forward 16-point DFT of v[0..15] (natural order in).  Result X[m + 4 q] is left in v[4 m + q].
static __device__ __forceinline__ void fft16(float2 (&v)[16])
{
#pragma unroll
  for (int i = 0; i < 4; ++i) fft4(v[i], v[i + 4], v[i + 8], v[i + 12]);
  // twiddles W16^(i m) on v[i + 4 m]
  v[5]  = cmulf(v[5],  make_float2(C1, -S1));      // i=1 m=1 : W^1
  v[9]  = cmulf(v[9],  make_float2(R2, -R2));      // i=1 m=2 : W^2
  v[13] = cmulf(v[13], make_float2(S1, -C1));      // i=1 m=3 : W^3
  v[6]  = cmulf(v[6],  make_float2(R2, -R2));      // i=2 m=1 : W^2
  v[10] = mul_mi(v[10]);                           // i=2 m=2 : W^4 = -i
  v[14] = cmulf(v[14], make_float2(-R2, -R2));     // i=2 m=3 : W^6
  v[7]  = cmulf(v[7],  make_float2(S1, -C1));      // i=3 m=1 : W^3
  v[11] = cmulf(v[11], make_float2(-R2, -R2));     // i=3 m=2 : W^6
  v[15] = cmulf(v[15], make_float2(-C1, S1));      // i=3 m=3 : W^9
#pragma unroll
  for (int m = 0; m < 4; ++m) fft4(v[4 * m], v[4 * m + 1], v[4 * m + 2], v[4 * m + 3]);
}
// position p = 4 m + q of fft16's output holds X[m + 4 q]
#define REV16(p) ((((p) >> 2)) | (((p) & 3) << 2))

struct Cols256K {
  const void *x; int fmt; size_t stream_stride;
  const float2 *hist; int hist_len;
  int windows_per_stream, first_window, hop, base_off, win_base;
  const float *window;
  float2 *scratch;
  const float2 *tw256;     // W_256^i
  const float2 *twfine;    // W_65536^i, i < 256
  const float2 *twpq;      // tabulated inter-pass twiddle [k1][n2]
};

#define LDC 273    // pitch of one column's [ka][17] block (odd: conflict-free across columns)

__global__ void __launch_bounds__(256, 4) k_cols256(const Cols256K p)   // 64 regs, 39 KB smem -> 4 CTAs / SM
{
  __shared__ float2 sm[16 * LDC];
  __shared__ float2 s_tw[256];
  const int tid = threadIdx.x;
  s_tw[tid] = __ldg(p.tw256 + tid);
  const int c = tid & 15, t = tid >> 4;
  const int w = p.win_base + blockIdx.y;
  const int stream = w / p.windows_per_stream;
  const int j0 = p.first_window + (w - stream * p.windows_per_stream);
  const int col = blockIdx.x * 16 + c;
  const long v0 = (long) p.base_off + (long) j0 * p.hop;
  const int fmt = p.fmt;
  const char *__restrict__ xs = reinterpret_cast<const char *>(p.x) + (size_t) stream * p.stream_stride * sdb_fmt_bytes(fmt);
  const float2 *__restrict__ hs = p.hist ? p.hist + (size_t) stream * p.hist_len : nullptr;

  float2 v[16];
  if (fmt == SDB_FMT_F32) {
    const float2 *__restrict__ xf = reinterpret_cast<const float2 *>(xs);
    if (v0 >= p.hist_len) {                         // CTA-uniform: the window lies wholly in the new samples
      const float2 *__restrict__ src = xf + (v0 - p.hist_len) + t * 256 + col;
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] = __ldg(src + j * 4096);    // row n1 = t + 16 j
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int r = t + 16 * j;
        const long vi = v0 + (long) r * 256 + col;
        v[j] = vi < p.hist_len ? __ldg(hs + vi) : __ldg(xf + (vi - p.hist_len));
      }
    }
  } else {                                          // 8 / 16-bit SDR samples: converted in the load
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int r = t + 16 * j;
      const long vi = v0 + (long) r * 256 + col;
      v[j] = vi < p.hist_len ? __ldg(hs + vi) : sdb_ld_iq(xs, vi - p.hist_len, fmt);
    }
  }
  if (p.window) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float wv = __ldg(p.window + (t + 16 * j) * 256 + col);
      v[j] = sdb_mul2(v[j], make_float2(wv, wv));
    }
  }
  fft16(v);                                         // over j: Y[t][ka], ka = REV16(position)
  __syncthreads();                                  // tables loaded
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const int ka = REV16(q);
    float2 y = v[q];
    if (ka) y = cmulf(y, s_tw[t * ka]);             // W_256^(t ka)
    sm[c * LDC + ka * 17 + t] = y;
  }
  __syncthreads();
  const int ka = t;                                 // second butterfly: thread (c, ka) gathers all t
#pragma unroll
  for (int tt = 0; tt < 16; ++tt) v[tt] = sm[c * LDC + ka * 17 + tt];
  fft16(v);                                         // over t: X[ka + 16 kb], kb = REV16(position)
  float2 *__restrict__ out = p.scratch + (size_t) blockIdx.y * 65536;
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const int kb = REV16(q);
    const int k1 = ka + 16 * kb;
    out[(size_t) k1 * 256 + col] = cmulf(v[q], __ldg(p.twpq + k1 * 256 + col));   // SPEC F.4 inter-pass twiddle
  }
}

cudaError_t sdb_launch_cols256(const SdbLaunchCtx &c, const SdbFourStep &fs, const SdbPassAArgs &a,
                               const float2 *twfine, int win_base, int n_win)
{
  Cols256K p;
  p.x = a.x; p.fmt = a.fmt; p.stream_stride = a.stream_stride; p.hist = a.hist; p.hist_len = a.hist_len;
  p.windows_per_stream = a.windows_per_stream; p.first_window = a.first_window; p.hop = a.hop;
  p.base_off = a.base_off; p.win_base = win_base; p.window = a.window; p.scratch = a.scratch;
  p.tw256 = fs.twN1; p.twfine = twfine; p.twpq = fs.twPQ;
  dim3 grid(16, n_win);
  k_cols256<<<grid, 256, 0, c.stream>>>(p);
  if (c.launch_counter) ++*c.launch_counter;
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// N = 32768 / 16384 / 8192 = N1 x 256 with N1 = 16 T, T = 8 / 4 / 2 (SPEC F.5; BASELINE configs[3] and [0]).  Pass A:
// columns of 16 T -- the same first butterfly (fft16 over the high row digit), twiddle W_N1^(t ka), exchange, then a
// T-point butterfly over the low row digit (T = 8: one radix-2 stage + two DFT4); pass B is k_rows256 with N1 rows per
// window.
// forward 8-point DFT of v[0..7] (natural order in).  Result X[kb] is left in v[4 (kb & 1) + (kb >> 1)].
static __device__ __forceinline__ void fft8(float2 (&v)[8])
{
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 a = cadd(v[i], v[i + 4]), b = csub(v[i], v[i + 4]);
    v[i] = a; v[i + 4] = b;
  }
  v[5] = cmulf(v[5], make_float2(R2, -R2));
  v[6] = mul_mi(v[6]);
  v[7] = cmulf(v[7], make_float2(-R2, -R2));
  fft4(v[0], v[1], v[2], v[3]);
  fft4(v[4], v[5], v[6], v[7]);
}
#define REV8(p) (2 * ((p) & 3) + ((p) >> 2))
// Pass A for N1 = 16 T rows, T = 8 (N = 32768), 4 (16384), 2 (8192): 128-thread CTAs that own C = 128 / T adjacent columns
// (thread = (column c, low row digit t)); the first butterfly is the 65536 kernel's fft16 over the high row digit, the
// second a T-point butterfly over the low one, 16 / T of them per thread (ka = t + T h).
template <int T>
__global__ void __launch_bounds__(128, 8) k_cols16T(const Cols256K p)
{
  constexpr int C = 128 / T;                        // columns per CTA
  constexpr int N1 = 16 * T;
  constexpr int LD = 16 * (T + 1) + 1;              // pitch of one column's [ka][T + 1] block (odd)
  __shared__ float2 sm[C * LD];
  __shared__ float2 s_tw[N1];
  const int tid = threadIdx.x;
  if (tid < N1) s_tw[tid] = __ldg(p.tw256 + tid);   // W_N1^i
  const int c = tid % C, t = tid / C;
  const int w = p.win_base + blockIdx.y;
  const int stream = w / p.windows_per_stream;
  const int j0 = p.first_window + (w - stream * p.windows_per_stream);
  const int col = blockIdx.x * C + c;
  const long v0 = (long) p.base_off + (long) j0 * p.hop;
  const int fmt = p.fmt;
  const char *__restrict__ xs = reinterpret_cast<const char *>(p.x) + (size_t) stream * p.stream_stride * sdb_fmt_bytes(fmt);
  const float2 *__restrict__ hs = p.hist ? p.hist + (size_t) stream * p.hist_len : nullptr;

  float2 v[16];
  if (fmt == SDB_FMT_F32 && v0 >= p.hist_len) {     // CTA-uniform: the window lies wholly in the new samples
    const float2 *__restrict__ src = reinterpret_cast<const float2 *>(xs) + (v0 - p.hist_len) + t * 256 + col;
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = __ldg(src + j * (T * 256));      // row n1 = t + T j
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const long vi = v0 + (long) (t + T * j) * 256 + col;
      v[j] = vi < p.hist_len ? __ldg(hs + vi)
                             : (fmt == SDB_FMT_F32 ? __ldg(reinterpret_cast<const float2 *>(xs) + (vi - p.hist_len))
                                                   : sdb_ld_iq(xs, vi - p.hist_len, fmt));
    }
  }
  if (p.window) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float wv = __ldg(p.window + (t + T * j) * 256 + col);
      v[j] = sdb_mul2(v[j], make_float2(wv, wv));
    }
  }
  fft16(v);                                         // over j: Y[t][ka], ka = REV16(position)
  __syncthreads();                                  // table loaded
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const int ka = REV16(q);
    float2 y = v[q];
    if (ka) y = cmulf(y, s_tw[t * ka]);             // W_N1^(t ka)
    sm[c * LD + ka * (T + 1) + t] = y;
  }
  __syncthreads();
  float2 *__restrict__ out = p.scratch + (size_t) blockIdx.y * (N1 * 256);
#pragma unroll
  for (int h = 0; h < 16 / T; ++h) {                // second butterfly: thread (c, ka) gathers all t
    const int ka = t + T * h;
    float2 u[8];
#pragma unroll
    for (int tt = 0; tt < T; ++tt) u[tt] = sm[c * LD + ka * (T + 1) + tt];
    if (T == 8) fft8(u);                            // X[kb] at position REV8^-1: kb = REV8(position)
    else if (T == 4) fft4(u[0], u[1], u[2], u[3]);  // natural order
    else { const float2 a = cadd(u[0], u[1]), b = csub(u[0], u[1]); u[0] = a; u[1] = b; }
#pragma unroll
    for (int q = 0; q < T; ++q) {
      const int kb = T == 8 ? REV8(q) : q;
      const int k1 = ka + 16 * kb;
      out[(size_t) k1 * 256 + col] = cmulf(u[q], __ldg(p.twpq + k1 * 256 + col));   // SPEC F.5 inter-pass twiddle
    }
  }
}

cudaError_t sdb_launch_cols128(const SdbLaunchCtx &c, const SdbFourStep &fs, const SdbPassAArgs &a, int win_base, int n_win)
{
  Cols256K p;
  p.x = a.x; p.fmt = a.fmt; p.stream_stride = a.stream_stride; p.hist = a.hist; p.hist_len = a.hist_len;
  p.windows_per_stream = a.windows_per_stream; p.first_window = a.first_window; p.hop = a.hop;
  p.base_off = a.base_off; p.win_base = win_base; p.window = a.window; p.scratch = a.scratch;
  p.tw256 = fs.twN1; p.twfine = nullptr; p.twpq = fs.twPQ;
  const int T = fs.N1 / 16;                         // 8, 4 or 2: columns per CTA = 128 / T
  dim3 grid(256 / (128 / T), n_win);
  if (T == 8)      k_cols16T<8><<<grid, 128, 0, c.stream>>>(p);
  else if (T == 4) k_cols16T<4><<<grid, 128, 0, c.stream>>>(p);
  else if (T == 2) k_cols16T<2><<<grid, 128, 0, c.stream>>>(p);
  else return cudaErrorInvalidValue;
  if (c.launch_counter) ++*c.launch_counter;
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
struct Rows256K {
  const float2 *scratch;
  float *psd; float inv_n; int shift_db;
  const int *binmap; float2 *cspec; int n_bins;
  const float2 *tw256;
  unsigned ka_mask;
};

#define LDR 273

// N1 = rows per window: 256 (N = 65536, SPEC F.4) or 128 / 64 / 32 (N = 32768 / 16384 / 8192, SPEC F.5); output bin
// k = k1 + N1 (ka + 16 kb)
template <int MODE, int N1 = 256>
__global__ void __launch_bounds__(512, 2) k_rows256(const Rows256K p)
{
  constexpr int NN = N1 * 256;
  extern __shared__ float2 smr[];                   // 32 rows x LDR
  __shared__ float2 s_tw[256];
  const int tid = threadIdx.x;
  if (tid < 256) s_tw[tid] = __ldg(p.tw256 + tid);
  const int win = blockIdx.y, k1_0 = blockIdx.x * 32;
  const float2 *__restrict__ in = p.scratch + (size_t) win * NN + (size_t) k1_0 * 256;
  {
    const int t = tid & 15, r = tid >> 4;           // 32 rows x 16 t
    float2 v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = in[(size_t) r * 256 + t + 16 * j];
    fft16(v);
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int ka = REV16(q);
      // channeliser: output bin k = k1 + 256 (ka + 16 kb); digits ka no channel touches are never formed
      if (MODE == 1 && !((p.ka_mask >> ka) & 1)) continue;
      float2 y = v[q];
      if (ka) y = cmulf(y, s_tw[t * ka]);
      smr[r * LDR + ka * 17 + t] = y;
    }
  }
  __syncthreads();
  {
    const int r = tid & 31, ka = tid >> 5;          // a warp = 32 consecutive rows = 32 consecutive bins
    if (MODE == 1 && !((p.ka_mask >> ka) & 1)) return;     // warp-uniform: this warp's 512 bins are unused
    float2 v[16];
#pragma unroll
    for (int tt = 0; tt < 16; ++tt) v[tt] = smr[r * LDR + ka * 17 + tt];
    fft16(v);
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int kb = REV16(q);
      const int k = k1_0 + r + N1 * (ka + 16 * kb);
      if (MODE == 0) {
        float pw = __fmaf_rn(v[q].x, v[q].x, v[q].y * v[q].y) * p.inv_n;
        float *__restrict__ psd = p.psd + (size_t) win * NN;
        // one-shot outputs: streaming stores, so that they do not displace the scratch / input in L2
        if (p.shift_db) { pw = 10.0f * d_log10f(pw + 1e-8f); __stcs(psd + ((k + NN / 2) & (NN - 1)), pw); }
        else __stcs(psd + k, pw);
      } else {
        const int m = __ldg(p.binmap + k);
        if (m >= 0) __stcs(p.cspec + (size_t) win * p.n_bins + m, v[q]);
      }
    }
  }
}

cudaError_t sdb_launch_rows256(const SdbLaunchCtx &c, const SdbFourStep &fs, const SdbPassBArgs &a, int mode)
{
  Rows256K p;
  p.scratch = a.scratch; p.psd = a.psd; p.inv_n = a.inv_n; p.shift_db = a.shift_db;
  p.binmap = a.binmap; p.cspec = a.cspec; p.n_bins = a.n_bins; p.tw256 = fs.twN2;
  p.ka_mask = a.ka_mask ? a.ka_mask : 0xffffu;
  const size_t smem = (size_t) 32 * LDR * sizeof(float2);
  static std::atomic<unsigned long long> attr_done{ 0 };   // one bit per device: function attributes are per context
  if (sdb_first_on_device(attr_done)) {
    cudaFuncSetAttribute(k_rows256<0, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    cudaFuncSetAttribute(k_rows256<1, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    cudaFuncSetAttribute(k_rows256<0, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    cudaFuncSetAttribute(k_rows256<1, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    cudaFuncSetAttribute(k_rows256<0, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    cudaFuncSetAttribute(k_rows256<1, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    cudaFuncSetAttribute(k_rows256<0, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    cudaFuncSetAttribute(k_rows256<1, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  }
  dim3 grid(fs.N1 / 32, a.n_windows);               // 32 rows of the scratch per CTA
#define ROWS_CASE(N1_) case N1_: if (mode == 0) k_rows256<0, N1_><<<grid, 512, smem, c.stream>>>(p); \
                                 else           k_rows256<1, N1_><<<grid, 512, smem, c.stream>>>(p); break
  switch (fs.N1) {
    ROWS_CASE(256); ROWS_CASE(128); ROWS_CASE(64); ROWS_CASE(32);
    default: return cudaErrorInvalidValue;
  }
#undef ROWS_CASE
  if (c.launch_counter) ++*c.launch_counter;
  return cudaGetLastError();
}
