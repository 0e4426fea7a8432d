// sdb_internal.h -- structures shared by the host runtime and the kernels, and the declarations the library's units
// share with each other.  Product code: nothing here includes or links oracle/.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include "sdb_iq.h"
#ifdef __cplusplus
#include <atomic>
#include <string>

// ---------------------------------------------------------------------------------------------
// error sink: the message sdb_last_error() returns (defined in engine.cu).  fail() sets it and returns -1; CK / CKP
// return -1 / nullptr from the calling function when a CUDA call fails.
// ---------------------------------------------------------------------------------------------
extern thread_local std::string g_err __attribute__((visibility("hidden")));
static inline int fail(const std::string &m) { g_err = m; return -1; }
#define CK(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { \
  g_err = std::string(#expr) + ": " + cudaGetErrorString(e__); return -1; } } while (0)
#define CKP(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { \
  g_err = std::string(#expr) + ": " + cudaGetErrorString(e__); return nullptr; } } while (0)

// ---------------------------------------------------------------------------------------------
// Device memory (or, Pinned, page-locked host memory) with one owner.  The element count is part of the buffer:
// alloc() frees the old allocation first and leaves size 0 when the new one fails, so a failed reallocation can never
// leave a stale size beside a null pointer.  Move-only; the destructor frees.
// ---------------------------------------------------------------------------------------------
template <typename T, bool Pinned = false> class DevBuf {
public:
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  DevBuf &operator=(DevBuf &&o) noexcept
  {
    if (this != &o) { release(); p_ = o.p_; n_ = o.n_; o.p_ = nullptr; o.n_ = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t alloc(size_t n)
  {
    release();
    void *p = nullptr;
    const cudaError_t e = Pinned ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T));
    if (e != cudaSuccess) { cudaGetLastError(); return e; }
    p_ = (T *) p; n_ = n;
    return cudaSuccess;
  }
  void release()
  {
    if (p_) { if (Pinned) cudaFreeHost(p_); else cudaFree(p_); }
    p_ = nullptr; n_ = 0;
  }
  size_t size() const { return n_; }
  T *get() const { return p_; }
  operator T *() const { return p_; }
private:
  T *p_ = nullptr;
  size_t n_ = 0;
};
template <typename T> using PinnedBuf = DevBuf<T, true>;

// A CUDA stream with one owner.  Move-only; the destructor destroys the stream without synchronising it, so an object
// that queues work on its streams synchronises them before it releases anything.
class Stream {
public:
  Stream() = default;
  Stream(const Stream &) = delete;
  Stream &operator=(const Stream &) = delete;
  Stream(Stream &&o) noexcept : h_(o.h_) { o.h_ = nullptr; }
  Stream &operator=(Stream &&o) noexcept
  {
    if (this != &o) { release(); h_ = o.h_; o.h_ = nullptr; }
    return *this;
  }
  ~Stream() { release(); }
  cudaError_t create(unsigned flags, int priority = 0)
  {
    release();
    cudaStream_t h = nullptr;
    const cudaError_t e = cudaStreamCreateWithPriority(&h, flags, priority);
    if (e != cudaSuccess) { cudaGetLastError(); return e; }
    h_ = h;
    return cudaSuccess;
  }
  void release() { if (h_) cudaStreamDestroy(h_); h_ = nullptr; }
  cudaStream_t get() const { return h_; }
  operator cudaStream_t() const { return h_; }
private:
  cudaStream_t h_ = nullptr;
};

// A CUDA event with one owner, which knows whether it has been recorded: wait_on() is a no-op until the first record(),
// so "the buffer this event guards has never been used" needs no flag beside it.  Move-only; the destructor destroys.
class Event {
public:
  Event() = default;
  Event(const Event &) = delete;
  Event &operator=(const Event &) = delete;
  Event(Event &&o) noexcept : h_(o.h_), recorded_(o.recorded_) { o.h_ = nullptr; o.recorded_ = false; }
  Event &operator=(Event &&o) noexcept
  {
    if (this != &o) { release(); h_ = o.h_; recorded_ = o.recorded_; o.h_ = nullptr; o.recorded_ = false; }
    return *this;
  }
  ~Event() { release(); }
  // cudaEventDefault for an event that times a span
  cudaError_t create(unsigned flags = cudaEventDisableTiming)
  {
    release();
    cudaEvent_t h = nullptr;
    const cudaError_t e = cudaEventCreateWithFlags(&h, flags);
    if (e != cudaSuccess) { cudaGetLastError(); return e; }
    h_ = h;
    return cudaSuccess;
  }
  void release() { if (h_) cudaEventDestroy(h_); h_ = nullptr; recorded_ = false; }
  cudaError_t record(cudaStream_t s)
  {
    const cudaError_t e = cudaEventRecord(h_, s);
    if (e == cudaSuccess) recorded_ = true;
    return e;
  }
  // make stream s wait for the last record (nothing to wait for before the first)
  cudaError_t wait_on(cudaStream_t s) const { return recorded_ ? cudaStreamWaitEvent(s, h_, 0) : cudaSuccess; }
  cudaEvent_t get() const { return h_; }
  operator cudaEvent_t() const { return h_; }
private:
  cudaEvent_t h_ = nullptr;
  bool recorded_ = false;
};

// cudaFuncSetAttribute applies to the CURRENT device: a process that drives several GPUs (one GUI process, two
// analyzers) must set it once per device, not once per process.  Returns true the first time on each device.
static inline bool sdb_first_on_device(std::atomic<unsigned long long> &mask)
{
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  return (mask.fetch_or(bit) & bit) == 0;
}
#endif

#define SDB_MAX_FIR      1024
#define SDB_MAX_IIR      5        // coefficients (order <= 4)
#define SDB_MAX_AGC_HIST 4096
#define SDB_EQ_LEN       10

// ---------------------------------------------------------------------------------------------
// FFT plan pieces (fft_kernels.cu)
// ---------------------------------------------------------------------------------------------
// The kernels that transform one window (the engine's transform plan picks the path from the size and the role)
enum SdbFftPath {
  SDB_FFT_SMALL_PSD,        // PSD, N <= 4096: k_small_psd, one CTA per frame
  SDB_FFT_CLUSTER,          // N = 65536: k_fft65536, both passes in one thread-block cluster
  SDB_FFT_F5,               // N = 8192 / 16384 / 32768 = N1 x 256 (SPEC F.5): k_cols16T + k_rows256 through the scratch
  SDB_FFT_STOCKHAM,         // every other size: k_pass_a + k_pass_b through the scratch
};

struct SdbFourStep {
  int path;                 // SdbFftPath
  int N, N1, N2;            // N = N1 * N2; pass A does N1-point column FFTs, pass B N2-point row FFTs
  int ka_shift;             // log2(N1): bin k = k1 + N1 (ka + 16 kb) on the cluster and F.5 paths
  const float2 *twN1;       // W_N1^i, i < N1 (forward sign)
  const float2 *twN2;
  const float2 *twN;        // W_N^i, i < N
  const float2 *twPQ;       // cluster / F.5: SPEC F.4 / F.5 inter-pass twiddle [k1][n2] = W_N1^(p>>8) x W_N^(p&255), p = n2 k1
};

struct SdbPassAArgs {
  const void   *x;          // new samples, stream 0, in format `fmt` (sdb_iq.h)
  int           fmt;
  size_t        stream_stride;      // in samples
  const float2 *hist;       // [S][hist_len] samples preceding x (may be null when hist_len == 0)
  int           hist_len;
  int           windows_per_stream; // windows handled per stream in this launch
  int           first_window;       // index of the first window (per stream) in this launch
  int           hop;                // samples between consecutive windows; window 0 starts the virtual buffer hist ++ x
  const float  *window;             // N taps or null
  float2       *scratch;            // [launch windows][N1][N2] as [k1][n2]
};

struct SdbPassBArgs {
  const float2 *scratch;
  int           n_windows;          // windows in this launch (flattened stream-major)
  // PSD epilogue
  float        *psd;                // [n_windows][N]
  float         inv_n;
  int           shift_db;
  // channeliser epilogue
  const int    *binmap;             // N entries, compact index or -1
  float2       *cspec;              // [n_windows][n_bins]
  int           n_bins;
  unsigned      ka_mask;            // bit (k / N1) & 15 set for every needed bin k (0 = all)
};

// N = 65536 (fft256_kernels.cu): every PSD frame and channeliser window of a feed in one launch, both passes fused.
// Per stream the launch holds n_psd PSD frames (hop 65536, no history) and n_chan channeliser windows
// first_chan .. first_chan + n_chan - 1 (hop 32768 over the 32768-sample history followed by x); when both are
// present, n_chan == 2 n_psd - first_chan.
struct SdbFft65536Args {
  const void   *x;                  // new samples, stream 0, in format `fmt` (sdb_iq.h)
  int           fmt;
  size_t        stream_stride;      // in samples
  int           n_streams, n_psd, n_chan, first_chan;
  // PSD frames: [S][n_psd][65536] output
  const float  *window;             // 65536 taps or null
  float        *psd;
  float         inv_n;
  int           shift_db;
  // channeliser windows: [S][n_chan][n_bins] output
  const float2 *hist;               // [S][32768]
  const int    *binmap;             // 65536 entries, compact index or -1
  float2       *cspec;
  int           n_bins;
  unsigned      ka_mask;            // bit (k >> 8) & 15 set for every needed bin k
};

// ---------------------------------------------------------------------------------------------
// channel plan (channeliser inverse side)
// ---------------------------------------------------------------------------------------------
struct SdbChannelDev {
  int    center, size, log2size, halfw, halfsz;
  // the channel's bins are the circular range [center-halfw, center+halfw) of the N-bin spectrum;
  // in the compacted spectrum they form one run (c1, L1 entries) plus, when the range wraps past
  // bin N-1, a second run starting at compact index 0.
  int    c1, L1;
  int    precise;
  float  lo_omega;          // rad / channel sample
  const float  *kh;         // 2*halfw weights k*h, ordered from bin center-halfw upwards
  const float  *xfade;      // size cross-fade weights sin^2(pi i / size)
  const float2 *tw;         // W_size^i (forward sign; conjugated for the inverse)
  size_t out_off;           // offset (complex samples) of this channel inside one stream's channel block
  size_t out_cap;           // capacity per feed
  size_t tail_off;          // offset of this channel's halfsz-sample tail inside one stream's tail block
};

// ---------------------------------------------------------------------------------------------
// inspector chains (chain_kernels.cu). Layout mirrors SPEC.md sections A, C, G, X.
// ---------------------------------------------------------------------------------------------
struct SdbChainCfg {
  int   cls;                // SDB_INSP_*
  int   have_agc, have_costas, have_pll, have_lo, have_mf;
  int   clock_type, clock_running;
  float gain2;
  // agc
  float knee, gain_slope, fixed_gain;
  unsigned hang_max, dl_size, mh_size;
  float far_, faf, sar, saf;
  // costas / pll / lo
  int   costas_kind;
  float c_a, c_b;
  int   af_n;               // arm filter coefficient count (1 = pass-through)
  float af_b[SDB_MAX_IIR], af_a[SDB_MAX_IIR];
  float pll_alpha, pll_beta;
  float lo_omega;
  // fsk / ask
  int   fsk_quad_demod;
  float fsk_rot_re, fsk_rot_im;
  int   ask_channel;
  // matched filter
  int   mf_n;
  int   mf_off;             // offset into the taps pool
  // clock
  float clk_gain, clk_alpha, clk_beta, bnor;
  float smp_period, smp_phase0;
  // decider
  int   dec_mode, dec_intervals;
  float dec_min, dec_h;
  // audio
  int   audio_demod, audio_squelch;
  float audio_volume, dc_alpha, sq_alpha, sq_thr;
  int   alpf_n;
  float alpf_b[SDB_MAX_IIR], alpf_a[SDB_MAX_IIR];
  double rs_step;
  // CMA equaliser (SPEC E)
  int   eq_type, eq_locked;
  float eq_mu;
  // per-chain state pool sizes (in floats) so the kernel can index the pools
  int   st_dl_off, st_mh_off, st_mf_off;  // offsets inside one chain's float pool
  int   st_pool;                           // floats per chain
};

struct SdbChainState {
  // agc
  float fast_level, slow_level, peak;
  unsigned hang_n, dl_ptr, mh_ptr;
  // costas
  float c_phi, c_omega, c_lock, c_yre, c_yim;
  float afx_re[SDB_MAX_IIR], afx_im[SDB_MAX_IIR], afy_re[SDB_MAX_IIR], afy_im[SDB_MAX_IIR];
  unsigned afxp, afyp;
  // pll / lo
  float p_phi, p_omega, lo_phi;
  // fsk / fm
  float prev_re, prev_im;
  // mf
  unsigned mf_ptr;
  // clock
  float k_phi, k_bnor, k_x0r, k_x0i, k_x1r, k_x1i, k_x2r, k_x2i, k_pr, k_pi;
  int   k_half;
  float s_phase, s_pr, s_pi;
  // audio
  float dc, sq_level, rs_prev;
  float al_x[SDB_MAX_IIR], al_y[SDB_MAX_IIR];
  unsigned al_xp, al_yp;
  double rs_phase;
  int   fm_primed;
  float eq_wr[SDB_EQ_LEN], eq_wi[SDB_EQ_LEN], eq_xr[SDB_EQ_LEN], eq_xi[SDB_EQ_LEN];
};

// ---------------------------------------------------------------------------------------------
// inspector spectrum sources + baud estimators (SPEC U; kernel in fft_kernels.cu)
// ---------------------------------------------------------------------------------------------
#define SDB_U5_KMIN 8
struct SdbSpectCfg {
  int   kind;               // SDB_SPECTSRC_* (0 = none)
  int   ns, logns;          // frame size
  unsigned est_mask;        // bit i = estimator i enabled
  float fs_ch;              // channel sample rate (Hz)
  const float2 *tw;         // W_ns^i
  const float  *window;     // Blackman-Harris(ns)
  size_t out_off;           // offset (floats) of this channel's spectrum inside one stream's block
};

// plan-dependent shared-memory lines of k_inspectors (chain_kernels.cu): sized from the channel plan
#define SDB_INSP_CHUNK 16          // samples per pipeline chunk (CH in chain_kernels.cu)
#define SDB_INSP_MF_RING_MAX 209   // longest matched filter served from the shared-memory ring (256 slots)
struct SdbInspDyn {
  int rb_slots;             // carrier ring slots (power of two >= longest ring-served filter - 1 + 2 chunks)
  int mf_rows;              // tap rows [t][lane] of the longest ring-served matched filter
  int agc_rows;             // floats per chain for the AGC delay line + magnitude history
  int use_eq;               // some chain runs the CMA equaliser
  unsigned long long role_lut, part_lut;   // nibble w = role / part of warp w (0 = the kernel's default placement)
};
static inline SdbInspDyn sdb_insp_dyn(const SdbChainCfg *cfgs, int n)
{
  SdbInspDyn d = { 4 * SDB_INSP_CHUNK, 1, 8, 0, 0ull, 0ull };   // the ring holds the chunks of the carrier, demod and filter steps
  for (int k = 0; k < n; ++k) {
    const SdbChainCfg &c = cfgs[k];
    if (c.have_mf && c.mf_n <= SDB_INSP_MF_RING_MAX) {        // longer filters stay in the global pool
      int need = c.mf_n - 1 + 3 * SDB_INSP_CHUNK, slots = 4 * SDB_INSP_CHUNK;
      while (slots < need) slots <<= 1;
      if (slots > d.rb_slots) d.rb_slots = slots;
      if (c.mf_n > d.mf_rows) d.mf_rows = c.mf_n;
    }
    if (c.have_agc) {
      const int need = (int) (2 * c.dl_size + c.mh_size);
      if (need <= 160 && need > d.agc_rows) d.agc_rows = need;
    }
    if (c.eq_type == 1) d.use_eq = 1;
  }
  return d;
}

#ifdef __cplusplus
#include <vector>
#include <algorithm>
#include "../../include/sigdigger_b200.h"
// CTA slot -> chain (channel-major index k * S + s) or -1.  A CTA holds chains of ONE inspector class so that its
// role warps do not diverge (a single source with a psk / fsk / ask mix would otherwise execute all three carrier
// stages in every warp); the classes with the longest recurrences come first so that their CTAs start first.  Power
// inspectors have no chain here: k_power_integrate serves them.
static inline int sdb_build_chain_map(const SdbChainCfg *cfgs, int K, int S, std::vector<int> &map)
{
  auto cost = [&](const SdbChainCfg &c) {          // rough per-sample cost order of the carrier stage
    if (c.cls == 2) return c.have_pll ? 0 : 3;     // ask (PLL: atan2 + sincos in the loop)
    if (c.cls == 0) return c.have_costas ? 1 : 3;  // psk
    if (c.cls == 3) return 2;                      // audio
    if (c.cls == 1) return 3;                      // fsk
    return 4;                                      // raw
  };
  std::vector<int> order(K);
  for (int k = 0; k < K; ++k) order[k] = k;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
    const int ca = cost(cfgs[a]) * 8 + cfgs[a].cls, cb = cost(cfgs[b]) * 8 + cfgs[b].cls;
    return ca < cb;
  });
  map.clear();
  int prev_key = -1;
  for (int idx = 0; idx < K; ++idx) {
    const int k = order[idx];
    if (cfgs[k].cls == SDB_INSP_POWER) continue;   // served by k_power_integrate
    const int key = cost(cfgs[k]) * 8 + cfgs[k].cls;
    if (key != prev_key) while (map.size() % 32) map.push_back(-1);
    prev_key = key;
    for (int s = 0; s < S; ++s) map.push_back(k * S + s);
  }
  while (map.size() % 32) map.push_back(-1);
  return (int) (map.size() / 32);
}

// One launch of k_inspectors: the CTAs [cta0, cta0 + n_ctas) of a chain map, every chain of them of inspector class
// cls, with the shared-memory lines of those chains alone.  sdb_insp_grids cuts a map from sdb_build_chain_map into
// one grid per run of CTAs of one class, in the map's order (slowest class first).
struct SdbInspGrid { int cls, cta0, n_ctas; SdbInspDyn dyn; };
static inline std::vector<SdbInspGrid> sdb_insp_grids(const SdbChainCfg *cfgs, int S, const std::vector<int> &map)
{
  std::vector<SdbInspGrid> out;
  std::vector<SdbChainCfg> run;                     // the channels of the current grid, once each
  int last_k = -1;
  auto close = [&]() { if (!out.empty()) out.back().dyn = sdb_insp_dyn(run.data(), (int) run.size()); run.clear(); };
  for (size_t q = 0; q < map.size(); q += 32) {
    const int g = map[q];                           // a CTA's first slot always holds a chain
    const int cta = (int) (q / 32), cls = cfgs[g / S].cls;
    if (out.empty() || out.back().cls != cls) { close(); out.push_back(SdbInspGrid{ cls, cta, 0, {} }); last_k = -1; }
    ++out.back().n_ctas;
    for (size_t l = q; l < q + 32; ++l)
      if (map[l] >= 0 && map[l] / S != last_k) { last_k = map[l] / S; run.push_back(cfgs[last_k]); }
  }
  close();
  return out;
}
#endif

// host-callable launchers ----------------------------------------------------------------------
struct SdbLaunchCtx {
  cudaStream_t stream;
  uint64_t    *launch_counter;
};

cudaError_t sdb_launch_pass_a_range(const SdbLaunchCtx &c, const SdbFourStep &fs, const SdbPassAArgs &a,
                                    int win_base, int n_win);
// 65536 / 32768 / 16384 / 8192 = N1 x 256 specialisations (fft256_kernels.cu)
cudaError_t sdb_launch_fft65536(const SdbLaunchCtx &c, const SdbFourStep &fs, const SdbFft65536Args &a);
cudaError_t sdb_launch_cols128(const SdbLaunchCtx &c, const SdbFourStep &fs, const SdbPassAArgs &a, int win_base, int n_win);
cudaError_t sdb_launch_rows256(const SdbLaunchCtx &c, const SdbFourStep &fs, const SdbPassBArgs &a, int mode);
// mode 0: PSD epilogue, 1: channeliser scatter
cudaError_t sdb_launch_pass_b(const SdbLaunchCtx &c, const SdbFourStep &fs, const SdbPassBArgs &a, int mode);
cudaError_t sdb_launch_hist_convert(cudaStream_t s, const void *x, int fmt, size_t stream_stride, size_t offset,
                                    float2 *hist, int hist_len, int n_streams);
cudaError_t sdb_launch_small_psd(const SdbLaunchCtx &c, int N, const float2 *tw, const void *x, int fmt,
                                 size_t stream_stride, int frames_per_stream, int n_streams,
                                 const float *window, float *psd, int shift_db);
cudaError_t sdb_launch_chan_ifft_group(const SdbLaunchCtx &c, const SdbChannelDev *chans_dev,
                                       const int *group_dev, int group_len, int size, int n_channels,
                                       int n_streams, const float2 *cspec, int n_bins, int wps,
                                       float2 *tails, size_t tail_stream_stride, float *lo_phase,
                                       float2 *chan_out, size_t chan_stream_stride, int any_precise = 1);
cudaError_t sdb_launch_sym_pack(cudaStream_t stream, const uint32_t *counts, unsigned long long *offsets, size_t chains,
                                const float2 *soft, const unsigned char *hard, size_t cap, void *out_soft,
                                void *out_hard, unsigned long long cap_total, uint64_t *launch_counter);
size_t sdb_inspector_smem_bytes(const SdbInspDyn &dyn);
// one grid of sdb_insp_grids over chain_map (from sdb_build_chain_map); the pool holds 32 * pool_stride floats per CTA
// of the whole map
cudaError_t sdb_launch_inspectors_n(const SdbLaunchCtx &c, const SdbInspGrid &grid, const SdbChainCfg *cfg_dev,
                                    int n_channels, int n_streams, const int *chain_map, SdbChainState *state,
                                    float *pool, size_t pool_stride,
                                    const float *taps_pool, const SdbChannelDev *chans_dev,
                                    const float2 *chan_in, size_t chan_stream_stride, uint32_t n_hops,
                                    float2 *soft, uint8_t *hard, uint32_t *sym_counts, size_t sym_cap, int fresh);
cudaError_t sdb_launch_spectsrc(const SdbLaunchCtx &c, const SdbSpectCfg *cfg_dev, const SdbChannelDev *chans_dev,
                                int n_channels, int n_streams, int max_ns, const float2 *chan_in,
                                size_t chan_stream_stride, uint32_t n_hops, float *spect, size_t spect_stream_stride,
                                uint32_t *spect_size, float *est, int *est_valid);
// spectsched_kernels.cu: scheduled spectrum sources / estimators (SPEC US).  One entry per scheduled channel: where
// its samples, ring and frames live (offsets inside one stream's block) and this feed's schedule.
struct SdbSchedChan {
  size_t   in_off;          // the channel's offset in a stream's channel block
  size_t   ring_off;        // its ring (Ns + 1 entries) in a stream's ring block
  size_t   frame_off;       // its first emission slot's frame (Ns + 1 samples) in a stream's frame block
  uint32_t ns1;             // Ns + 1
  uint32_t slot0;           // index of its first emission slot
  unsigned long long t0;        // channel samples before this feed (T_before)
  unsigned long long t_first;   // the feed's first emission point
  unsigned long long interval;  // I
  uint32_t n_emit;          // emissions of this feed
  uint32_t w_from, w_to;    // feed samples [w_from, w_to) go to the ring
};
cudaError_t sdb_launch_spectsched_gather(const SdbLaunchCtx &c, const SdbSchedChan *sched, const int *slot_chan,
                                         SdbChannelDev *slot_dev, int n_slots, int n_streams, const float2 *chan_in,
                                         size_t chan_stride, const float2 *ring, size_t ring_stride, float2 *frames,
                                         size_t frame_stride);
cudaError_t sdb_launch_spectsched_ring(const SdbLaunchCtx &c, const SdbSchedChan *sched, int n_sched, int n_streams,
                                       const float2 *chan_in, size_t chan_stride, float2 *ring, size_t ring_stride);
// sview_kernels.cu: frame-averaged main PSD (SPEC A); psd [S][frames][n] -> out [S][means][n], carry [S][n]
cudaError_t sdb_launch_psd_group_mean(const SdbLaunchCtx &c, const float *psd, unsigned frames, unsigned n,
                                      size_t n_streams, unsigned A, unsigned carried, unsigned means, int shift_db,
                                      float *carry, float *out);
// sview_kernels.cu: peak detectors of the main PSD (SPEC PK); psd [S][frames][n] -> out_max, out_min [S][groups][n],
// carry_max, carry_min [S][n]; n a power of two >= 16.  Internal to the library: not exported.
__attribute__((visibility("hidden")))
cudaError_t sdb_launch_psd_group_peak(const SdbLaunchCtx &c, const float *psd, unsigned frames, unsigned n,
                                      size_t n_streams, unsigned P, unsigned carried, unsigned groups, int shift_db,
                                      float *carry_max, float *carry_min, float *out_max, float *out_min);
// power_kernels.cu: the power inspector (SPEC PW).  One entry per (power channel, stream); the carry is indexed by
// `out` like the symbol rows, [S][K] over every channel.
struct SdbPowerChain {
  size_t   in_off;          // offset (complex samples) of the chain's input in a slot's channel block: s * stride + out_off
  uint32_t halfsz;          // channel samples per hop
  uint32_t out;             // output row s * K + k of soft / hard / counts, and carry entry
  unsigned long long M;     // samples per mean (>= 1)
};
struct SdbPowerCarry { double acc, c; unsigned long long n; };   // Kahan sum, its compensation, samples in the group
cudaError_t sdb_launch_power_integrate(const SdbLaunchCtx &c, const SdbPowerChain *chains, int n_chains,
                                       const float2 *chan_in, uint32_t n_hops, SdbPowerCarry *carry, float2 *soft,
                                       uint8_t *hard, uint32_t *sym_counts, size_t sym_cap);
// tasks_kernels.cu
cudaError_t sdb_launch_dc_remove(cudaStream_t st, const void *x, int fmt, size_t stream_stride, size_t n, int n_streams,
                                 float alpha, float2 *state, float2 *cur, double2 *part, float2 *out);

#ifdef __cplusplus
#include "../../include/sigdigger_b200.h"
// chdet_kernels.cu: the engine's detector pass, and the channel lists converted to Hz on the device
cudaError_t sdb_chdet_feed_stream(sdb_chdet_t *d, const float *psd_dev, uint32_t frames, size_t stream_stride,
                                  cudaStream_t stream, uint64_t *launch_counter);
cudaError_t sdb_chdet_pack_device(sdb_chdet_t *d, double samp_rate, const double *centers_dev,
                                  sdb_detected_channel *out_dev, size_t cap, int *counts_dev, cudaStream_t stream);
// chdet_kernels.cu: channel tracking across detector updates (oracle/SPEC_KT.md), one update after every detector update
struct sdb_chtrack;
sdb_chtrack *sdb_chtrack_new(int device, uint32_t n_bins, uint32_t n_streams, float beta, uint32_t hold);
void sdb_chtrack_destroy(sdb_chtrack *t);
cudaError_t sdb_chtrack_feed_stream(sdb_chtrack *t, const sdb_chdet_t *d, uint32_t frames, cudaStream_t stream,
                                    uint64_t *launch_counter);
long sdb_chtrack_read(sdb_chtrack *t, uint32_t stream, double samp_rate, double center_freq, sdb_tracked_channel *out,
                      size_t cap, uint32_t *total, uint64_t *dropped);
int  sdb_chtrack_read_all(sdb_chtrack *t, double samp_rate, const double *centers, sdb_tracked_channel *out, size_t cap,
                          uint32_t *counts, uint64_t *dropped);
// fac_kernels.cu: the FAC tab (oracle/SPEC_FC.md).  One chain per (FAC channel, stream), channel-major.
#define SDB_FAC_KINDS 4     // work units of a feed: F.2 blocks, F.3 4096-point units, statistics tiles, averaging units
struct SdbFacChan {
  uint32_t L, logL, lo, hi, ntiles;   // block size, lag window [lo, hi), its 1024-lag tiles
  uint32_t N1, N2, logN1, logN2;      // F.3 split (L >= 8192)
  float alpha; double sigma;
  uint32_t row;                       // s * K + k: the chain's row of soft / counts
  uint32_t slot_off, tile_off;        // its first block slot and first tile record; slots * ntiles records
  size_t blk_off, fac_off;            // carried block [L] (float2), averaged FAC [L / 2]
  size_t work_off, scr_off;           // per slot: [L] floats of P / v, [L] float2 of F.3 scratch (L >= 8192)
  const float2 *tw, *twN1, *twN2;     // W_L (F.2, and F.3's inter-pass twiddle), W_N1, W_N2
};
struct SdbFacState { uint32_t p; float max, min; };
struct SdbFacTile { float max, min, pre, pow; uint32_t pos, cnt; };   // pre: the feed's running maximum before it
struct SdbFacArgs {
  const SdbFacChan *chans; int n_chans;
  SdbFacState *state; float2 *blk; float *fac;
  float *work; float2 *scr; float *slot_max; SdbFacTile *tiles;
  uint32_t *offs;                     // [SDB_FAC_KINDS][n_chans + 1]: per-chain exclusive prefix sums, totals last
  uint32_t *nb;                       // blocks each chain completes in this feed
  const float2 *soft; const uint32_t *counts; size_t sym_cap;
  sdb_fac_status *status;
};
// engine.cu: the parameter checks of sdb_engine_set_fac (0, or -1 with sdb_last_error() set), shared with the analyzer
int sdb_fac_check(const sdb_fac_params *p);
// grid[k]: CTAs of the persistent launches over units of kind k (0: no chain has that kind)
cudaError_t sdb_launch_fac(const SdbLaunchCtx &c, const SdbFacArgs &a, const int grid[SDB_FAC_KINDS]);
// snr_kernels.cu: the SNR meter (oracle/SPEC_SN.md).  One descriptor per channel with the meter on; its chains are
// chain0 + s (s < n_streams), each with h and the model at hist_off + s L and its state in status[chain0 + s].
#define SDB_SNR_BINS_MIN 16u
#define SDB_SNR_BINS_MAX 1024u
struct SdbSnrChan {
  uint32_t L, K, k, chain0;           // bins, comb teeth 2^bps, channel (row s * n_channels + k), first chain
  int32_t mode;                       // SPEC D: 0 argument, 1 modulus
  float dmin, dh, alpha;              // SPEC D's min and max - min, the step size
  size_t hist_off;
};
struct SdbSnrArgs {
  const SdbSnrChan *chans; int n_chans, n_streams, n_channels; uint32_t max_L;
  const float2 *soft; const uint32_t *counts; size_t sym_cap;
  uint32_t *hist; float *model; sdb_snr_status *status;
};
// engine.cu: the parameter checks of sdb_engine_set_snr (0, or -1 with sdb_last_error() set), shared with the analyzer
int sdb_snr_check(const sdb_snr_params *p);
cudaError_t sdb_launch_snr(const SdbLaunchCtx &c, const SdbSnrArgs &a);
// engine.cu: the parameter checks of sdb_engine_set_tv (0, or -1 with sdb_last_error() set) and whether two parameter
// blocks give the same picture geometry (W, H, delay line, interlacing), shared with the analyzer
int sdb_tv_tab_check(const sdb_tv_tab_params *p);
bool sdb_tv_same_geometry(const sdb_tv_params &a, const sdb_tv_params &b);
// stream-ordered pieces of the panoramic sweep (panoramic.cu): caller-owned device buffers, no host copies, no
// default-stream work.  engine.cu:
int sdb_engine_pack_channels_device(sdb_engine_t *e, const double *centers_dev, sdb_detected_channel *out_dev, size_t cap,
                                    int *counts_dev, cudaStream_t st);
// sview_kernels.cu.  psd_dev: hop h's frame at psd_dev + h * hop_stride; psd_is_linear: the engine's linear
// natural-order PSD (the PSDMessage conversion happens inside the projection) instead of shifted dB; centers_dev: the
// hop centres on the device.  Returns 1 when the geometry needs the general kernel (histogram mode or a very wide hop):
// the caller then converts and calls with psd_is_linear = 0.
int sdb_sview_project_async(sdb_sview_t *v, cudaStream_t st, const float *psd_dev, size_t psd_size, size_t hop_stride,
                            int psd_is_linear, const double *centers_dev, size_t n_hops, int adjust_sides, int32_t *j0,
                            int32_t *nb, float *va, float *vc);
int sdb_sview_accumulate_async(sdb_sview_t *v, cudaStream_t st, const int32_t *j0, const int32_t *nb, const float *va,
                               const float *vc, size_t n_hops);
int sdb_sview_reset_async(sdb_sview_t *v, cudaStream_t st);
int sdb_psd_shift_db_async(cudaStream_t st, const float *lin_dev, float *db_dev, size_t n_frames, uint32_t psd_size);
#endif
