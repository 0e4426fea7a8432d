// engine.cu -- host runtime + C-ABI (include/sigdigger_b200.h) of the H100 analyzer engine.
//
// One engine = one channel plan applied to a batch of S independent IQ streams on one GPU.
// feed(): main PSD over every psd_size frame (four-step FFT, two kernels), channeliser forward FFT
// over half-overlapping windows with a compacting bin scatter, per-channel IFFT + cross-fade, and
// the inspector chains.  Everything is queued on one CUDA stream; results are read back on demand.
//
// This file replaces, for the hot path only, suscan's analyzer object as the reference drives it:
// suscan_analyzer_new/destroy (Suscan/Analyzer.cpp:608,636), open/set_inspector_config
// (Suscan/Analyzer.cpp:459-495), and the PSD / SAMPLES payloads (Suscan/Messages/PSDMessage.cpp:26-39,
// include/Suscan/Messages/SamplesMessage.h:33-59).  No CPU fallback exists: without a device the
// constructor fails with an error string.
#include "../../include/sigdigger_b200.h"
#include "sdb_internal.h"
#include "host_design.h"
#include "sdb_tv_steps.h"

#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <vector>
#include <cstdio>
#include <cstring>
#include <cstddef>
#include <cmath>

thread_local std::string g_err;
extern "C" const char *sdb_last_error(void) { return g_err.c_str(); }

extern "C" int sdb_device_count(void)
{
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

static bool is_pow2(unsigned v) { return v && !(v & (v - 1)); }
static int ilog2u(unsigned v) { int l = 0; while ((1u << l) < v) ++l; return l; }

struct Channel {
  sdb_channel_params p;
  unsigned center, size, width, halfw, halfsz;
  bool has_insp;
  sdb_inspector_config cfg;
  int spect_kind = 0; unsigned spect_size = 0, est_mask = 0;   // SPEC U
  uint64_t spect_interval = 0;                                    // SPEC US (0: once per feed, SPEC U.1)
  bool has_fac = false; sdb_fac_params fac{};                     // SPEC FC
  bool has_snr = false; sdb_snr_params snr{};                     // SPEC SN
  bool has_tv = false; sdb_tv_tab_params tv{};                    // SPEC TI
};

struct TimedSpan { int family; Event a, b; };
enum { FAM_COLS = 0, FAM_ROWS_PSD, FAM_ROWS_CHAN, FAM_CHAN_IFFT, FAM_INSPECTOR, FAM_PSD_AVERAGE, FAM_POWER, FAM_PSD_PEAK,
       FAM_SPECTSCHED, FAM_CHAN_TRACK, FAM_FAC, FAM_SNR, FAM_TV,
       FAM_COUNT };
static const char *kFamNames[FAM_COUNT] = { "fft_cols", "fft_rows_psd", "fft_rows_chan", "chan_ifft",
                                            "inspector", "psd_average", "power", "psd_peak", "spectsrc_sched",
                                            "chan_track", "fac", "snr", "tv" };

// SPEC PW: samples per mean of a power inspector (power.integrate-samples, 0 read as 1)
static uint64_t power_m(const sdb_inspector_config &c) { return c.power_integrate_samples ? c.power_integrate_samples : 1; }
static bool is_power(const Channel &c) { return c.has_insp && c.cfg.insp_class == SDB_INSP_POWER; }

struct ChdetDeleter { void operator()(sdb_chdet *d) const { sdb_chdet_destroy(d); } };
struct ChtrackDeleter { void operator()(sdb_chtrack *t) const { sdb_chtrack_destroy(t); } };

// Host-buffer pipeline: results are double-buffered by feed parity so that the D2H reads of feed i-1 overlap the
// kernels of feed i (three copy/compute streams).  Each event guards its slot's buffers between the streams.
struct Slot {
  float *psd = nullptr;                             // [S][frames][Np]
  // channel streams: the (latency-bound, 1-CTA-per-32-chains) inspector kernel of feed i runs on its own stream
  // while the FFT kernels of feed i+1 fill the other slot
  float2 *chan = nullptr;
  float2 *soft = nullptr; uint8_t *hard = nullptr; uint32_t *counts = nullptr;
  DevBuf<unsigned long long> sym_off;               // packed read-out: start of every chain, 16-symbol aligned
  // scheduled spectra (SPEC US): per emission slot [S][slot] spectrum (ns floats), size, estimates and validity, and
  // on the host the emission count and first t_j of each scheduled channel in this feed
  DevBuf<float> sched_spect, sched_est; DevBuf<uint32_t> sched_size; DevBuf<int> sched_valid;
  std::vector<uint32_t> sched_n; std::vector<uint64_t> sched_first;
  Event psd_ready, psd_read, sym_read, insp;
};

// A reduction over groups of G consecutive main-PSD frames: the frame-averaged PSD (SPEC A, one output: the means) or
// the peak detectors (SPEC PK, two outputs: the maxima and the minima).  Each output has a carry, the open group of
// every stream (one frame count serves all: a feed has the same frames per stream), and is double-buffered by parity.
struct FrameGroups {
  int fam, n_out;                       // timing family; outputs
  unsigned G = 0;                       // frames per group, 0: off
  DevBuf<float> carry[2];               // [output]: [S][Np]
  DevBuf<float> out[2][2];              // [feed parity][output]: [S][ceil(max_frames / G)][Np]
  unsigned count = 0;                   // frames of the open group
  size_t last = 0;                      // groups the latest feed completed
};

// Everything sdb_engine_commit builds, and the running state that exists only after a commit.  A commit builds it
// whole and hands it to the engine only on success, so a failed commit leaves nothing behind.
struct Plan {
  std::vector<DevBuf<unsigned char>> allocs;   // every device buffer of the plan (dalloc), freed with it
  std::map<unsigned, float2 *> tw;     // twiddle tables by size

  SdbFourStep fs_psd{}, fs_st{};       // transform plans (make_plan)
  float *d_window = nullptr;
  // four-step scratch of the two-kernel transforms (the F.5 and Stockham paths)
  float2 *d_scratch = nullptr; int chunk_windows = 1; size_t l2_pinned_bytes = 0;
  // Two-kernel sizes with Np == W: the PSD transforms run on their own stream, concurrently with the channeliser
  // transforms of the same group of streams (feed_device): the two kernel chains fill each other's launch gaps
  // and partial waves, and both read the same input region while it is still in L2.
  Stream psd_stream; Event ev_feed;
  float2 *d_hist = nullptr;             // [S][W/2]
  // channeliser
  int *d_binmap = nullptr; int n_bins = 0; unsigned ka_mask = 0;
  float2 *d_cspec = nullptr;
  std::vector<SdbChannelDev> h_chans; SdbChannelDev *d_chans = nullptr;
  struct Group { int size; int len; int *d_ids; int any_precise; };
  std::vector<Group> groups;
  float2 *d_tails = nullptr; size_t tail_stride = 0;
  float *d_lo_phase = nullptr;
  size_t chan_stride = 0;
  Stream insp_stream; Event ev_chan;
  Slot slot[2];
  // Host-input staging has its own parity, host_feeds: device feeds between host feeds make it differ from the feed
  // parity.  The H2D copy of feed i+1 overlaps the kernels of feed i.
  struct Stage { DevBuf<float2> xin; Event xfree; } stage[2];
  Stream h2d_stream, d2h_stream; Event ev_h2d;
  // chains
  SdbChainCfg *d_cfg = nullptr; std::vector<SdbChainCfg> h_cfg;
  SdbChainState *d_state = nullptr;
  float *d_pool = nullptr; size_t pool_stride = 0;
  int *d_chain_map = nullptr; int insp_ctas = 0; std::vector<int> h_chain_map;
  // one inspector grid per class run of the chain map, launched in the map's order on the inspector stream.  They do
  // not run concurrently: two classes' kernels on one SM fetch from two code images, and every role of both slowed
  // down (DESIGN.md section 5); the next feed's transforms fill the SMs a grid's last wave leaves free.
  std::vector<SdbInspGrid> insp_grids;
  float *d_taps = nullptr;
  size_t sym_cap = 0;
  // power inspectors (SPEC PW; power_kernels.cu): one integrator per (power channel, stream), channel-major, and the
  // partial group of every [stream][channel] (entries of other classes stay unused).  No power channel: both empty.
  DevBuf<SdbPowerChain> d_power; int n_power = 0;
  DevBuf<SdbPowerCarry> power_carry;
  // channel detector on the main PSD (SPEC K; chdet_kernels.cu)
  std::unique_ptr<sdb_chdet, ChdetDeleter> chdet;
  // channel tracking across the detector's updates (SPEC KT), when enabled
  std::unique_ptr<sdb_chtrack, ChtrackDeleter> chtrack;
  // inspector spectrum sources / estimators (SPEC U)
  std::vector<SdbSpectCfg> h_spect; SdbSpectCfg *d_spectcfg = nullptr;
  float *d_spect = nullptr; size_t spect_stride = 0; int spect_max_ns = 0;
  uint32_t *d_spect_size = nullptr; float *d_est = nullptr; int *d_est_valid = nullptr;
  // scheduled spectrum sources / estimators (SPEC US; spectsched_kernels.cu).  A scheduled channel has an empty entry
  // in the per-feed tables above and owns `slots` consecutive emission slots: k_spectsrc runs over the slots with
  // n_hops = 1, each slot's channel entry holding one frame (halfsz = Ns + 1, set by the gather) or none (0).
  struct Sched {
    int k; unsigned ns, kind, est_mask; uint64_t interval; uint32_t slot0, slots;
    size_t out0;            // slot e's spectrum at out0 + e ns in a stream's block
    uint64_t t = 0;         // channel samples since the channel started
    uint64_t v = 0;         // the ring holds c[m] for every m in [max(v, t - ns - 1), t)
  };
  std::vector<Sched> sched; std::vector<int> sched_of;   // sched_of[k]: index into sched, or -1
  std::vector<SdbSchedChan> h_sched; DevBuf<SdbSchedChan> d_sched;
  DevBuf<int> d_slot_chan; DevBuf<SdbSpectCfg> d_slot_cfg; DevBuf<SdbChannelDev> d_slot_dev;
  DevBuf<float2> d_ring, d_frames;
  int n_slots = 0, sched_max_ns = 0;
  size_t ring_stride = 0, frame_stride = 0, sched_spect_stride = 0;
  // DC removal (SDB_FLAG_DC_REMOVE, SPEC R): per-stream estimate, the estimate the current block is corrected with,
  // run sums, and the corrected float32 copy of the block the rest of the path reads
  float2 *d_dc_state = nullptr, *d_dc_cur = nullptr, *d_xdc = nullptr; double2 *d_dc_part = nullptr;
  // the FAC tab (SPEC FC; fac_kernels.cu): one chain per (FAC channel, stream), channel-major, with its running state;
  // first[k] is channel k's stream-0 chain or -1.  Per feed: its blocks' work areas, tile records and status.
  struct Fac {
    std::vector<SdbFacChan> h; std::vector<int> first;
    DevBuf<SdbFacChan> chans; DevBuf<SdbFacState> state; DevBuf<float2> blk, scr; DevBuf<float> fac, work, slot_max;
    DevBuf<SdbFacTile> tiles; DevBuf<uint32_t> offs, nb; DevBuf<sdb_fac_status> status;
    int grid[SDB_FAC_KINDS] = {0, 0, 0, 0};
  } fac;
  // the SNR meter (SPEC SN; snr_kernels.cu): one descriptor per channel with the meter on, first[k] its index or -1;
  // per (channel, stream) chain, channel-major: h and the model [L] each, and the state / status of the latest feed
  struct Snr {
    std::vector<SdbSnrChan> h; std::vector<int> first; uint32_t max_L = 0;
    DevBuf<SdbSnrChan> chans; DevBuf<uint32_t> hist; DevBuf<float> model; DevBuf<sdb_snr_status> status;
  } snr;
  // the Analog TV tab (SPEC TI; k_tv_insp in tv_kernels.cu): one descriptor per channel with the TV on, first[k] its
  // index or -1; per (channel, stream) processor, channel-major: state, delay line, row, ring, posted frame and status
  struct Tv {
    std::vector<SdbTvInspChan> h; std::vector<int> first; size_t smem = 0;
    DevBuf<SdbTvInspChan> chans; DevBuf<SdbTvState> state; DevBuf<float> delay, line, ring, post;
    DevBuf<sdb_tv_status> status;
  } tv;
  // frame averaging (SPEC A) and peak detection (SPEC PK), in the order they run
  FrameGroups avg{FAM_PSD_AVERAGE, 1}, peak{FAM_PSD_PEAK, 2};
  // running state
  unsigned feed_index = 0, host_feeds = 0;
  bool first_feed = true;               // (engines without channels keep no history)
  uint64_t n_fed = 0;                   // samples fed so far
  size_t last_frames = 0, last_hops = 0;

  // the parity of the latest feed (0 before the first) and its slot
  unsigned cur_parity() const { return feed_index ? (feed_index - 1) & 1u : 0; }
  Slot &cur() { return slot[cur_parity()]; }
  template <typename T> T *dalloc(size_t n)
  {
    DevBuf<unsigned char> b;
    if (b.alloc(std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) return nullptr;
    allocs.push_back(std::move(b));
    return (T *) allocs.back().get();
  }
  const float2 *twiddle(unsigned n)
  {
    auto it = tw.find(n);
    if (it != tw.end()) return it->second;
    std::vector<float2> h;
    sdbh::twiddle_fill(n, h);
    float2 *d = dalloc<float2>(n);
    if (!d) return nullptr;
    cudaMemcpy(d, h.data(), n * sizeof(float2), cudaMemcpyHostToDevice);
    tw[n] = d;
    return d;
  }
};

struct sdb_engine {
  sdb_engine_params prm;
  double samp_rate;
  Stream stream;
  uint64_t launches = 0;
  bool timing = false;
  std::vector<Channel> channels;
  unsigned Np = 0, W = 0;               // PSD size, channeliser window
  // channel detector parameters
  bool cd_enabled = false;
  float cd_alpha = 0, cd_gamma = 0, cd_snr = 0; unsigned cd_min_bins = 1;
  float cd_beta = 0;
  bool ct_enabled = false; unsigned ct_hold = 0;    // channel tracking (SPEC KT)
  std::unique_ptr<Plan> plan;           // set by a successful sdb_engine_commit
  // timing
  std::vector<TimedSpan> spans;
  double fam_ms[FAM_COUNT] = {0}; uint64_t fam_n[FAM_COUNT] = {0};

  void span_begin(int fam, cudaStream_t on = nullptr)
  {
    if (!timing) return;
    TimedSpan s; s.family = fam;
    s.a.create(cudaEventDefault); s.b.create(cudaEventDefault);
    s.a.record(on ? on : stream.get());
    spans.push_back(std::move(s));
  }
  void span_end(cudaStream_t on = nullptr)
  {
    if (!timing) return;
    spans.back().b.record(on ? on : stream.get());
  }
  // make the main stream wait for everything queued on the inspector stream
  cudaError_t join() { return plan ? plan->cur().insp.wait_on(stream) : cudaSuccess; }
  void collect_spans()
  {
    for (auto &s : spans) {
      float ms = 0;
      if (cudaEventElapsedTime(&ms, s.a, s.b) == cudaSuccess) { fam_ms[s.family] += ms; fam_n[s.family]++; }
    }
    spans.clear();
  }
};

// The transform plan of an N-point window for the main PSD (psd = true) or the channeliser: which kernels run
// (SdbFftPath), the split N = N1 x N2 and the tables.  This is the one place that ties transform sizes to kernels.
static bool make_plan(Plan &pl, unsigned N, bool psd, SdbFourStep *fs)
{
  *fs = SdbFourStep{};
  fs->N = (int) N;
  if (psd && N <= 4096) {
    fs->path = SDB_FFT_SMALL_PSD;
    fs->twN = pl.twiddle(N);
    return fs->twN != nullptr;
  }
  fs->path = N == 65536 ? SDB_FFT_CLUSTER
           : (N == 8192 || N == 16384 || N == 32768) ? SDB_FFT_F5 : SDB_FFT_STOCKHAM;
  const int l = ilog2u(N);
  fs->N1 = 1 << (fs->path == SDB_FFT_STOCKHAM ? l / 2 : l - 8);   // cluster and F.5: N1 x 256
  fs->N2 = (int) N / fs->N1;
  fs->ka_shift = ilog2u(fs->N1);
  fs->twN1 = pl.twiddle(fs->N1); fs->twN2 = pl.twiddle(fs->N2); fs->twN = pl.twiddle(N);
  if (!(fs->twN1 && fs->twN2 && fs->twN)) return false;
  if (fs->path == SDB_FFT_STOCKHAM) return true;
  // SPEC F.4 / F.5 inter-pass twiddle [k1][n2] = W_N1^(p >> 8) x W_N^(p & 255), p = n2 k1: the product of two table
  // look-ups, tabulated once with the arithmetic of SPEC F.1 (one rounded product + one fused multiply-add per
  // component)
  auto it = pl.tw.find(N | 1u);
  if (it != pl.tw.end()) { fs->twPQ = it->second; return true; }
  const unsigned N1 = (unsigned) fs->N1;
  std::vector<float2> c, f, pq((size_t) N);
  sdbh::twiddle_fill(N1, c); sdbh::twiddle_fill(N, f);
  for (unsigned k1 = 0; k1 < N1; ++k1)
    for (unsigned n2 = 0; n2 < 256; ++n2) {
      const unsigned p = n2 * k1;
      const float2 a = c[p >> 8], b = f[p & 255];
      pq[(size_t) k1 * 256 + n2].x = fmaf(a.x, b.x, -(a.y * b.y));
      pq[(size_t) k1 * 256 + n2].y = fmaf(a.x, b.y, a.y * b.x);
    }
  float2 *d = pl.dalloc<float2>(N);
  if (!d) return false;
  cudaMemcpy(d, pq.data(), (size_t) N * sizeof(float2), cudaMemcpyHostToDevice);
  pl.tw[N | 1u] = d;
  fs->twPQ = d;
  return true;
}

static bool uses_scratch(const SdbFourStep &fs) { return fs.path == SDB_FFT_F5 || fs.path == SDB_FFT_STOCKHAM; }

// Windows per chunk of the four-step scratch, for the largest scratch transform `big` of the engine.  Both passes of
// both two-kernel paths put the window of the chunk on grid.y, so a chunk holds at most the device's grid.y limit
// (65535 on an H100): 64 MB of 64- or 128-point channeliser windows would otherwise be 131072 or 65536 of them.
static size_t scratch_chunk_windows(const SdbFourStep &big, int device)
{
  const size_t window_bytes = (size_t) big.N * sizeof(float2);
  size_t cw = std::max<size_t>(1, ((size_t) 64 << 20) / window_bytes);
  int max_grid_y = 0;
  if (cudaDeviceGetAttribute(&max_grid_y, cudaDevAttrMaxGridDimY, device) == cudaSuccess && max_grid_y > 0)
    cw = std::min(cw, (size_t) max_grid_y);
  if (big.path != SDB_FFT_F5) return cw;
  // SPEC F.5 path: 512 KB of windows per SM is whole waves of both passes (two 32768-point windows: 32 k_cols16T
  // CTAs at 8 per SM, 8 k_rows256 CTAs at 2 per SM).  On an H100 that is 69 MB, more than its 50 MB L2 can set
  // aside for persisting lines, so the chunk is halved (whole waves still) until it fits.
  const size_t per_sm = (size_t) 512 << 10;
  int sms = 0, max_persist = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && sms > 0 &&
      (size_t) sms * per_sm <= ((size_t) 100 << 20)) {
    cw = (size_t) sms * (per_sm / window_bytes);
    cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, device);
    while (max_persist > 0 && cw % 2 == 0 && cw * window_bytes > (size_t) max_persist) cw /= 2;
  }
  return cw;
}

extern "C" sdb_engine_t *sdb_engine_new(const sdb_engine_params *p, double samp_rate)
{
  if (!p) { g_err = "null params"; return nullptr; }
  if (sdb_device_count() <= 0) { g_err = "no CUDA device: sigdigger_b200 has no CPU fallback"; return nullptr; }
  if (p->n_streams < 1) { g_err = "n_streams must be >= 1"; return nullptr; }
  if (p->psd_size && (!is_pow2(p->psd_size) || p->psd_size < 16 || p->psd_size > (1u << 20))) {
    g_err = "psd_size must be a power of two in [16, 2^20]"; return nullptr;
  }
  unsigned W = p->st_window_size ? p->st_window_size : p->psd_size;
  if (!is_pow2(W) || W < 64 || W > (1u << 20)) { g_err = "st_window_size must be a power of two in [64, 2^20]"; return nullptr; }
  if (p->input_format < SDB_FORMAT_FLOAT32 || p->input_format > SDB_FORMAT_SIGNED16) {
    g_err = "unknown input_format"; return nullptr;
  }
  CKP(cudaSetDevice(p->device));
  sdb_engine *e = new sdb_engine();
  e->prm = *p; e->samp_rate = samp_rate; e->Np = p->psd_size; e->W = W;
  if (e->stream.create(cudaStreamNonBlocking) != cudaSuccess) {
    g_err = "cudaStreamCreate failed"; delete e; return nullptr;
  }
  return e;
}

extern "C" void sdb_engine_destroy(sdb_engine_t *e)
{
  if (!e) return;
  cudaSetDevice(e->prm.device);
  cudaStreamSynchronize(e->stream);
  if (Plan *p = e->plan.get()) {
    for (cudaStream_t s : { p->insp_stream.get(), p->psd_stream.get(), p->h2d_stream.get(), p->d2h_stream.get() })
      if (s) cudaStreamSynchronize(s);
    if (p->l2_pinned_bytes) { cudaCtxResetPersistingL2Cache(); cudaGetLastError(); }
  }
  e->collect_spans();
  delete e;
}

extern "C" int sdb_inspector_config_default(sdb_inspector_config *c, int insp_class, float fs)
{
  if (!c) return fail("null config");
  memset(c, 0, sizeof(*c));
  c->insp_class = insp_class; c->fs = fs;
  c->agc_enabled = 1; c->agc_gain_db = 0.0f;
  c->costas_order = insp_class == SDB_INSP_PSK ? 2 : 0;
  c->bits_per_symbol = insp_class == SDB_INSP_PSK ? 2 : 1;
  c->loop_bw = fs * 1e-3f; c->offset = 0.0f;
  c->mf_type = 0; c->mf_rolloff = 0.35f;
  c->clock_type = 1; c->baud = fs * 0.25f; c->clock_gain = 1.0f; c->clock_phase = 0.0f; c->clock_running = 1;
  c->audio_cutoff = 5000.0f; c->audio_volume = 1.0f; c->audio_sample_rate = 44100;
  c->audio_demod = SDB_AUDIO_FM; c->agc_ts = 0.1f;
  c->eq_type = 0; c->eq_rate = 1e-3f; c->eq_locked = 0;
  // a tenth of a second of channel samples (the upstream default is not known)
  const double m = 0.1 * (double) fs;
  c->power_integrate_samples = m > 1.0 ? (uint64_t) llround(m) : 1;
  return 0;
}

extern "C" int sdb_engine_open_channel(sdb_engine_t *e, const sdb_channel_params *p, sdb_channel_info *info)
{
  if (!e || !p) return fail("null argument");
  if (e->plan) return fail("engine already committed");
  if (!(p->guard >= 1.0f) || !(p->bw > 0.0f) || p->bw > 6.28318530717958647692f * 1.0001f)
    return fail("invalid channel: guard >= 1 and 0 < bw <= 2 pi required");   // INVALID_CHANNEL
  if (!(p->f0 >= 0.0f) || p->f0 >= 6.28318530717958647692f) return fail("invalid channel: f0 must be in [0, 2 pi)");
  Channel c;
  c.p = *p; c.has_insp = false;
  sdbh::channel_geometry(e->W, p->f0, p->bw, p->guard, &c.center, &c.size, &c.width);
  c.halfw = c.width >> 1; c.halfsz = c.size >> 1;
  if (c.size > 16384) return fail("channel size > 16384 bins not supported by the shared-memory IFFT");
  memset(&c.cfg, 0, sizeof(c.cfg));
  e->channels.push_back(c);
  if (info) { info->center = c.center; info->size = c.size; info->width = c.width;
              info->decimation = (float) e->W / (float) c.size; }
  return (int) e->channels.size() - 1;
}

// channel geometry without an engine (su_specttuner_open_channel computes it before any transform exists)
extern "C" int sdb_channel_geometry(uint32_t window_size, const sdb_channel_params *p, sdb_channel_info *info)
{
  if (!p || !info) return fail("null argument");
  if (!is_pow2(window_size) || window_size < 64) return fail("window size must be a power of two >= 64");
  if (!(p->guard >= 1.0f) || !(p->bw > 0.0f) || p->bw > 6.28318530717958647692f * 1.0001f)
    return fail("invalid channel: bw must be in (0, 2 pi], guard >= 1");
  if (!(p->f0 >= 0.0f) || p->f0 >= 6.28318530717958647692f) return fail("invalid channel: f0 must be in [0, 2 pi)");
  unsigned center, size, width;
  sdbh::channel_geometry(window_size, p->f0, p->bw, p->guard, &center, &size, &width);
  info->center = center; info->size = size; info->width = width;
  info->decimation = (float) window_size / (float) size;
  return 0;
}

extern "C" int sdb_engine_set_inspector(sdb_engine_t *e, int handle, const sdb_inspector_config *cfg)
{
  if (!e || !cfg) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");   // WRONG_HANDLE
  if (e->plan) return fail("engine already committed");
  if (cfg->insp_class < SDB_INSP_PSK || cfg->insp_class > SDB_INSP_POWER) return fail("wrong kind");
  Channel &c = e->channels[handle];
  c.cfg = *cfg; c.has_insp = true;
  c.cfg.fs = (float) (e->samp_rate * (double) c.size / (double) e->W);
  return 0;
}

extern "C" int sdb_engine_set_channel_detector(sdb_engine_t *e, float alpha, float beta, float gamma, float snr,
                                               uint32_t min_bins)
{
  if (!e) return fail("null argument");
  if (e->plan) return fail("engine already committed");
  if (!e->prm.psd_size) return fail("the channel detector needs the main PSD");
  if ((e->prm.flags & SDB_FLAG_PSD_SHIFT_DB) && e->prm.psd_average < 2 && e->prm.psd_peak < 2)
    return fail("the channel detector needs a linear PSD");
  if (!(snr > 0.0f) || !(alpha >= 0.0f && alpha <= 1.0f) || !(gamma >= 0.0f && gamma <= 1.0f))
    return fail("detector parameters out of range");
  e->cd_enabled = true; e->cd_alpha = alpha; e->cd_gamma = gamma; e->cd_snr = snr; e->cd_min_bins = min_bins ? min_bins : 1;
  e->cd_beta = beta;                  // used by channel tracking only (checked at commit when tracking is on)
  return 0;
}

extern "C" int sdb_engine_set_channel_tracking(sdb_engine_t *e, uint32_t hold)
{
  if (!e) return fail("null argument");
  if (e->plan) return fail("engine already committed");
  if (!e->cd_enabled) return fail("channel tracking needs the channel detector (sdb_engine_set_channel_detector)");
  if (hold > SDB_CHTRACK_HOLD_MAX) return fail("channel tracking hold must be at most 65535 updates");
  e->ct_enabled = true; e->ct_hold = hold;
  return 0;
}

extern "C" long sdb_engine_read_channels(sdb_engine_t *e, uint32_t stream, double center_freq,
                                         sdb_detected_channel *out, size_t cap, uint32_t *total)
{
  if (!e) return fail("null argument");
  if (!e->plan || !e->plan->chdet) return fail("channel detector not enabled");
  const Plan &p = *e->plan;
  if (stream >= e->prm.n_streams) return fail("stream out of range");
  CK(cudaSetDevice(e->prm.device));
  CK(cudaStreamSynchronize(p.psd_stream ? p.psd_stream.get() : e->stream.get()));
  CK(cudaStreamSynchronize(e->stream));
  const long n = sdb_chdet_read(p.chdet.get(), stream, e->samp_rate, center_freq, out, cap, total);
  if (n < 0) return fail("channel read failed");
  return n;
}

// all streams at once: centers[S] (host), out[S][cap], counts[S]
extern "C" int sdb_engine_read_all_channels(sdb_engine_t *e, const double *centers, sdb_detected_channel *out, size_t cap,
                                            uint32_t *counts)
{
  if (!e || !centers || !out || !counts) return fail("null argument");
  if (!e->plan || !e->plan->chdet) return fail("channel detector not enabled");
  const Plan &p = *e->plan;
  CK(cudaSetDevice(e->prm.device));
  CK(cudaStreamSynchronize(p.psd_stream ? p.psd_stream.get() : e->stream.get()));
  CK(cudaStreamSynchronize(e->stream));
  if (sdb_chdet_read_all(p.chdet.get(), e->samp_rate, centers, out, cap, counts)) return fail("channel read failed");
  return 0;
}

extern "C" long sdb_engine_read_tracked_channels(sdb_engine_t *e, uint32_t stream, double center_freq,
                                                 sdb_tracked_channel *out, size_t cap, uint32_t *total, uint64_t *dropped)
{
  if (!e) return fail("null argument");
  if (!e->plan || !e->plan->chtrack) return fail("channel tracking not enabled");
  const Plan &p = *e->plan;
  if (stream >= e->prm.n_streams) return fail("stream out of range");
  if (!out && cap) return fail("null argument");
  CK(cudaSetDevice(e->prm.device));
  CK(cudaStreamSynchronize(p.psd_stream ? p.psd_stream.get() : e->stream.get()));
  CK(cudaStreamSynchronize(e->stream));
  const long n = sdb_chtrack_read(p.chtrack.get(), stream, e->samp_rate, center_freq, out, cap, total, dropped);
  if (n < 0) return fail("tracked channel read failed");
  return n;
}

extern "C" int sdb_engine_read_all_tracked_channels(sdb_engine_t *e, const double *centers, sdb_tracked_channel *out,
                                                    size_t cap, uint32_t *counts, uint64_t *dropped)
{
  if (!e || !centers || !out || !counts) return fail("null argument");
  if (!e->plan || !e->plan->chtrack) return fail("channel tracking not enabled");
  const Plan &p = *e->plan;
  CK(cudaSetDevice(e->prm.device));
  CK(cudaStreamSynchronize(p.psd_stream ? p.psd_stream.get() : e->stream.get()));
  CK(cudaStreamSynchronize(e->stream));
  if (sdb_chtrack_read_all(p.chtrack.get(), e->samp_rate, centers, out, cap, counts, dropped))
    return fail("tracked channel read failed");
  return 0;
}

static const char *kSpectNames[SDB_SPECTSRC_COUNT] = { "none", "psd", "cyclo", "fmspect", "timediff", "abstimediff",
                                                      "exp_2", "exp_4", "exp_8", "fac" };
static const char *kEstNames[SDB_ESTIMATOR_COUNT] = { "baud-fac", "baud-nonlinear" };
extern "C" const char *sdb_spectsrc_name(int id) { return id >= 0 && id < SDB_SPECTSRC_COUNT ? kSpectNames[id] : nullptr; }
extern "C" const char *sdb_estimator_name(int id) { return id >= 0 && id < SDB_ESTIMATOR_COUNT ? kEstNames[id] : nullptr; }

extern "C" int sdb_engine_set_spectrum_source(sdb_engine_t *e, int handle, int spectsrc_id, uint32_t size)
{
  if (!e) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (e->plan) return fail("engine already committed");
  if (spectsrc_id < 0 || spectsrc_id >= SDB_SPECTSRC_COUNT) return fail("unknown spectrum source");
  if (!is_pow2(size) || size < 64 || size > 4096) return fail("spectrum size must be a power of two in [64, 4096]");
  Channel &c = e->channels[handle];
  if (c.spect_size && c.spect_size != size && c.est_mask) return fail("spectrum size already fixed by an estimator");
  c.spect_kind = spectsrc_id; c.spect_size = size;
  return 0;
}

int sdb_fac_check(const sdb_fac_params *p)
{
  if (!is_pow2(p->size) || p->size < 512 || p->size > (1u << 19)) return fail("FAC size must be a power of two in [512, 2^19]");
  if (!(p->alpha >= 0.0f && p->alpha <= 1.0f)) return fail("FAC alpha must be in [0, 1]");
  if ((p->lag_lo || p->lag_hi) && !(p->lag_lo < p->lag_hi && p->lag_hi <= p->size / 2))
    return fail("FAC lag window must satisfy lag_lo < lag_hi <= size / 2");
  if (std::isnan(p->sigma)) return fail("FAC sigma must not be NaN");
  return 0;
}

extern "C" int sdb_engine_set_fac(sdb_engine_t *e, int handle, const sdb_fac_params *p)
{
  if (!e) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (e->plan) return fail("engine already committed");
  Channel &c = e->channels[handle];
  if (!p) { c.has_fac = false; return 0; }
  if (sdb_fac_check(p)) return -1;
  if (!c.has_insp || c.cfg.insp_class > SDB_INSP_ASK) return fail("the FAC needs a psk, fsk or ask inspector");
  c.fac = *p; c.has_fac = true;
  return 0;
}

extern "C" int sdb_engine_read_fac(sdb_engine_t *e, int handle, float *fac, sdb_fac_status *st)
{
  if (!e) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (!e->plan) return fail("engine not committed");
  const Plan::Fac &f = e->plan->fac;
  if (f.first.empty() || f.first[handle] < 0) return fail("the FAC is not enabled on this channel");
  const SdbFacChan &h = f.h[f.first[handle]];
  const unsigned S = e->prm.n_streams;
  CK(cudaSetDevice(e->prm.device));
  CK(e->join());
  CK(cudaStreamSynchronize(e->stream));
  if (fac) CK(cudaMemcpy(fac, f.fac.get() + h.fac_off, (size_t) S * (h.L / 2) * sizeof(float), cudaMemcpyDeviceToHost));
  if (st) CK(cudaMemcpy(st, f.status.get() + f.first[handle], S * sizeof(sdb_fac_status), cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" const float *sdb_engine_fac_device(const sdb_engine_t *e, int handle)
{
  if (!e || !e->plan || handle < 0 || handle >= (int) e->plan->fac.first.size() || e->plan->fac.first[handle] < 0)
    return nullptr;
  const Plan::Fac &f = e->plan->fac;
  return f.fac.get() + f.h[f.first[handle]].fac_off;
}

// SPEC SN: the meter's parameters
int sdb_snr_check(const sdb_snr_params *p)
{
  if (p->bins < SDB_SNR_BINS_MIN || p->bins > SDB_SNR_BINS_MAX) return fail("SNR bins must be in [16, 1024]");
  if (!(std::isfinite(p->sigma) && p->sigma > 0.0f)) return fail("SNR sigma must be finite and positive");
  if (!(std::isfinite(p->alpha) && p->alpha > 0.0f)) return fail("SNR alpha must be finite and positive");
  return 0;
}

// SN.2: K = 2^bps with bps 0 read as 1 (InspectorUI::getBps)
static uint32_t snr_K(const sdb_inspector_config &c) { return 1u << (c.bits_per_symbol ? c.bits_per_symbol : 1u); }

extern "C" int sdb_engine_set_snr(sdb_engine_t *e, int handle, const sdb_snr_params *p)
{
  if (!e) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (e->plan) return fail("engine already committed");
  Channel &c = e->channels[handle];
  if (!p) { c.has_snr = false; return 0; }
  if (sdb_snr_check(p)) return -1;
  if (!c.has_insp || c.cfg.insp_class > SDB_INSP_ASK) return fail("the SNR meter needs a psk, fsk or ask inspector");
  c.snr = *p; c.has_snr = true;
  return 0;
}

// SN.3: the state of the latest feed is the status; a reset writes sigma of every stream, in order with the feeds
extern "C" int sdb_engine_reset_snr(sdb_engine_t *e, int handle, float sigma)
{
  if (!e) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (!e->plan) return fail("engine not committed");
  const Plan::Snr &q = e->plan->snr;
  if (q.first.empty() || q.first[handle] < 0) return fail("the SNR meter is not on for this channel");
  if (!(std::isfinite(sigma) && sigma > 0.0f)) return fail("SNR sigma must be finite and positive");
  const unsigned S = e->prm.n_streams;
  std::vector<sdb_snr_status> st(S);
  sdb_snr_status *d = q.status.get() + q.h[q.first[handle]].chain0;
  CK(cudaSetDevice(e->prm.device));
  CK(e->join());
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaMemcpy(st.data(), d, S * sizeof(sdb_snr_status), cudaMemcpyDeviceToHost));
  const uint32_t K = q.h[q.first[handle]].K;
  for (auto &x : st) { x.sigma = sigma; x.snr = 1.0f / (K * sigma); }
  CK(cudaMemcpy(d, st.data(), S * sizeof(sdb_snr_status), cudaMemcpyHostToDevice));
  return 0;
}

extern "C" int sdb_engine_read_snr(sdb_engine_t *e, int handle, uint32_t *hist, float *model, sdb_snr_status *st)
{
  if (!e) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (!e->plan) return fail("engine not committed");
  const Plan::Snr &q = e->plan->snr;
  if (q.first.empty() || q.first[handle] < 0) return fail("the SNR meter is not on for this channel");
  const SdbSnrChan &h = q.h[q.first[handle]];
  const size_t n = (size_t) e->prm.n_streams * h.L;
  CK(cudaSetDevice(e->prm.device));
  CK(e->join());
  CK(cudaStreamSynchronize(e->stream));
  if (hist) CK(cudaMemcpy(hist, q.hist.get() + h.hist_off, n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  if (model) CK(cudaMemcpy(model, q.model.get() + h.hist_off, n * sizeof(float), cudaMemcpyDeviceToHost));
  if (st) CK(cudaMemcpy(st, q.status.get() + h.chain0, e->prm.n_streams * sizeof(sdb_snr_status),
                        cudaMemcpyDeviceToHost));
  return 0;
}

// SPEC TI.4: the tab's parameters, and what a running processor cannot change (TV.7)
int sdb_tv_tab_check(const sdb_tv_tab_params *p)
{
  if (!sdb_tv_params_valid(p->tv)) return fail("TV: invalid parameters (the sample rate may be too low for them)");
  return 0;
}

bool sdb_tv_same_geometry(const sdb_tv_params &a, const sdb_tv_params &b)
{
  SdbTvCfg x, y;
  sdb_tv_derive(a, x); sdb_tv_derive(b, y);
  return x.W == y.W && x.H == y.H && x.delay_len == y.delay_len && x.interlace == y.interlace;
}

// SPEC TI.1: the processor's constants and the conversion of the channel's class
static void tv_describe(const Channel &c, SdbTvInspChan &h)
{
  sdb_tv_derive(c.tv.tv, h.c);
  h.mode = c.cfg.insp_class == SDB_INSP_ASK ? 0 : 1;
  h.gain = c.tv.invert_sync ? -1.0f : 1.0f; h.dc = c.tv.dc;
}

extern "C" int sdb_engine_set_tv(sdb_engine_t *e, int handle, const sdb_tv_tab_params *p)
{
  if (!e) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (e->plan) return fail("engine already committed");
  Channel &c = e->channels[handle];
  if (!p) { c.has_tv = false; return 0; }
  if (sdb_tv_tab_check(p)) return -1;
  if (!c.has_insp || c.cfg.insp_class > SDB_INSP_ASK) return fail("the TV needs a psk, fsk or ask inspector");
  c.tv = *p; c.has_tv = true;
  return 0;
}

// SPEC TI.4: from the next feed on, in order with the feeds; the state is kept
extern "C" int sdb_engine_set_tv_params(sdb_engine_t *e, int handle, const sdb_tv_tab_params *p)
{
  if (!e || !p) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (!e->plan) return fail("engine not committed");
  Plan::Tv &q = e->plan->tv;
  if (q.first.empty() || q.first[handle] < 0) return fail("the TV is not on for this channel");
  if (sdb_tv_tab_check(p)) return -1;
  Channel &c = e->channels[handle];
  if (!sdb_tv_same_geometry(c.tv.tv, p->tv))
    return fail("TV: the picture geometry (width, height, delay line, interlacing) cannot change without a re-plan");
  SdbTvInspChan &h = q.h[q.first[handle]];
  CK(cudaSetDevice(e->prm.device));
  CK(e->join());
  CK(cudaStreamSynchronize(e->stream));
  c.tv = *p;
  tv_describe(c, h);
  CK(cudaMemcpy(q.chans.get() + q.first[handle], &h, sizeof(h), cudaMemcpyHostToDevice));
  return 0;
}

extern "C" int sdb_engine_read_tv(sdb_engine_t *e, int handle, float *frames, sdb_tv_status *st)
{
  if (!e) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (!e->plan) return fail("engine not committed");
  const Plan::Tv &q = e->plan->tv;
  if (q.first.empty() || q.first[handle] < 0) return fail("the TV is not on for this channel");
  const SdbTvInspChan &h = q.h[q.first[handle]];
  const unsigned S = e->prm.n_streams;
  CK(cudaSetDevice(e->prm.device));
  CK(e->join());
  CK(cudaStreamSynchronize(e->stream));
  if (frames) CK(cudaMemcpy(frames, q.post.get() + h.post_off, (size_t) S * h.c.H * h.c.W * sizeof(float),
                            cudaMemcpyDeviceToHost));
  if (st) CK(cudaMemcpy(st, q.status.get() + h.chain0, S * sizeof(sdb_tv_status), cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int sdb_engine_set_estimator(sdb_engine_t *e, int handle, int estimator_id, int enabled)
{
  if (!e) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (e->plan) return fail("engine already committed");
  if (estimator_id < 0 || estimator_id >= SDB_ESTIMATOR_COUNT) return fail("unknown estimator");
  Channel &c = e->channels[handle];
  if (enabled) c.est_mask |= 1u << estimator_id; else c.est_mask &= ~(1u << estimator_id);
  return 0;
}

extern "C" int sdb_engine_set_spectrum_interval(sdb_engine_t *e, int handle, uint64_t interval)
{
  if (!e) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (e->plan) return fail("engine already committed");
  Channel &c = e->channels[handle];
  if (c.spect_kind == 0 && c.est_mask == 0)
    return fail("spectrum interval on a channel without a spectrum source or estimator");
  if (interval > SDB_SPECTRUM_INTERVAL_MAX) return fail("spectrum interval must be at most 2^62 channel samples");
  c.spect_interval = interval;
  return 0;
}

static int sched_index(const Plan &p, int handle)
{
  return handle < (int) p.sched_of.size() ? p.sched_of[handle] : -1;
}
static unsigned sched_out_size(const Plan::Sched &q) { return q.kind == SDB_SPECTSRC_FAC ? q.ns / 2 : q.ns; }

// Emissions [e0, e0 + n) of scheduled channel q in the latest feed, every stream: spectra into out (rows of out_size
// floats, estimator < 0) or estimates into values / valid; stream s starts `pitch` elements after stream s - 1.
// Fenced on the feed's inspector work like the PSD reads.
static int read_sched(sdb_engine_t *e, const Plan::Sched &q, int estimator, uint32_t e0, uint32_t n, size_t pitch,
                      float *out, float *values, int32_t *valid)
{
  Plan &p = *e->plan;
  Slot &sl = p.cur();
  const unsigned S = e->prm.n_streams;
  CK(cudaSetDevice(e->prm.device));
  CK(sl.insp.wait_on(p.d2h_stream));
  const size_t slot = (size_t) q.slot0 + e0;
  for (unsigned s = 0; s < S; ++s) {
    if (estimator < 0) {
      const unsigned w = sched_out_size(q);
      CK(cudaMemcpy2DAsync(out + (size_t) s * pitch, (size_t) w * sizeof(float),
                           sl.sched_spect + (size_t) s * p.sched_spect_stride + q.out0 + (size_t) e0 * q.ns,
                           (size_t) q.ns * sizeof(float), (size_t) w * sizeof(float), n, cudaMemcpyDeviceToHost,
                           p.d2h_stream));
    } else {
      const size_t off = ((size_t) s * p.n_slots + slot) * 2 + (size_t) estimator;
      CK(cudaMemcpy2DAsync(values + (size_t) s * pitch, sizeof(float), sl.sched_est + off, 2 * sizeof(float),
                           sizeof(float), n, cudaMemcpyDeviceToHost, p.d2h_stream));
      CK(cudaMemcpy2DAsync(valid + (size_t) s * pitch, sizeof(int32_t), sl.sched_valid + off, 2 * sizeof(int),
                           sizeof(int32_t), n, cudaMemcpyDeviceToHost, p.d2h_stream));
    }
  }
  CK(cudaStreamSynchronize(p.d2h_stream));
  return 0;
}

static int sched_check(sdb_engine_t *e, int handle, int estimator, const Plan::Sched **q)
{
  if (!e->plan) return fail("engine not committed");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  const int i = sched_index(*e->plan, handle);
  if (i < 0) return fail("no spectrum interval on this channel");
  *q = &e->plan->sched[i];
  if (estimator < 0 && (*q)->kind == 0) return fail("no spectrum source on this channel");
  if (estimator >= SDB_ESTIMATOR_COUNT) return fail("unknown estimator");
  if (estimator >= 0 && !((*q)->est_mask & (1u << estimator))) return fail("estimator not enabled on this channel");
  return 0;
}

// sdb_engine_read_spectrum / _read_estimate on a scheduled channel: the feed's last emission, or none
static int read_sched_last(sdb_engine_t *e, int handle, int estimator, float *out, uint32_t *sizes, int32_t *valid)
{
  const Plan::Sched *q = nullptr;
  if (sched_check(e, handle, estimator, &q)) return -1;
  const Plan &p = *e->plan;
  const unsigned S = e->prm.n_streams;
  const uint32_t n = p.feed_index ? p.slot[(p.feed_index - 1) & 1u].sched_n[sched_index(p, handle)] : 0;
  if (n == 0) {
    for (unsigned s = 0; s < S; ++s) { if (sizes) sizes[s] = 0; if (valid) valid[s] = 0; }
    return 0;
  }
  if (estimator < 0) {
    for (unsigned s = 0; s < S; ++s) sizes[s] = sched_out_size(*q);
    return read_sched(e, *q, -1, n - 1, 1, q->ns, out, nullptr, nullptr);   // [S][size], as on a per-feed channel
  }
  return read_sched(e, *q, estimator, n - 1, 1, 1, nullptr, out, valid);
}

extern "C" long sdb_engine_read_spectra(sdb_engine_t *e, int handle, float *out, uint64_t *ends, size_t cap)
{
  if (!e || !out || !ends) return fail("null argument");
  const Plan::Sched *q = nullptr;
  if (sched_check(e, handle, -1, &q)) return -1;
  const Plan &p = *e->plan;
  if (p.feed_index == 0) return 0;
  const Slot &sl = p.slot[(p.feed_index - 1) & 1u];
  const int i = sched_index(p, handle);
  const uint32_t n = (uint32_t) std::min<size_t>(sl.sched_n[i], cap);
  for (uint32_t j = 0; j < n; ++j) ends[j] = sl.sched_first[i] + (uint64_t) j * q->interval;
  if (n && read_sched(e, *q, -1, 0, n, cap * sched_out_size(*q), out, nullptr, nullptr)) return -1;
  return (long) n;
}

extern "C" long sdb_engine_read_estimates(sdb_engine_t *e, int handle, int estimator_id, float *values, int32_t *valid,
                                          size_t cap)
{
  if (!e || !values || !valid) return fail("null argument");
  if (estimator_id < 0) return fail("unknown estimator");
  const Plan::Sched *q = nullptr;
  if (sched_check(e, handle, estimator_id, &q)) return -1;
  const Plan &p = *e->plan;
  if (p.feed_index == 0) return 0;
  const uint32_t n = (uint32_t) std::min<size_t>(p.slot[(p.feed_index - 1) & 1u].sched_n[sched_index(p, handle)], cap);
  if (n && read_sched(e, *q, estimator_id, 0, n, cap, nullptr, values, valid)) return -1;
  return (long) n;
}

extern "C" int sdb_engine_read_spectrum(sdb_engine_t *e, int handle, float *out, uint32_t *sizes)
{
  if (!e || !out || !sizes) return fail("null argument");
  if (!e->plan) return fail("engine not committed");
  const Plan &p = *e->plan;
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (sched_index(p, handle) >= 0) return read_sched_last(e, handle, -1, out, sizes, nullptr);
  if (!p.d_spect || p.h_spect[handle].kind == 0) return fail("no spectrum source on this channel");
  CK(cudaSetDevice(e->prm.device));
  CK(cudaStreamSynchronize(p.insp_stream));
  const unsigned S = e->prm.n_streams; const int K = (int) e->channels.size();
  const SdbSpectCfg &q = p.h_spect[handle];
  CK(cudaMemcpy2D(out, (size_t) q.ns * sizeof(float), p.d_spect + q.out_off, p.spect_stride * sizeof(float),
                  (size_t) q.ns * sizeof(float), S, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy2D(sizes, sizeof(uint32_t), p.d_spect_size + handle, (size_t) K * sizeof(uint32_t), sizeof(uint32_t), S,
                  cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int sdb_engine_read_estimate(sdb_engine_t *e, int handle, int estimator_id, float *values, int32_t *valid)
{
  if (!e || !values || !valid) return fail("null argument");
  if (!e->plan) return fail("engine not committed");
  const Plan &p = *e->plan;
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (estimator_id < 0 || estimator_id >= SDB_ESTIMATOR_COUNT) return fail("unknown estimator");
  if (sched_index(p, handle) >= 0) return read_sched_last(e, handle, estimator_id, values, nullptr, valid);
  if (!p.d_est || !(p.h_spect[handle].est_mask & (1u << estimator_id))) return fail("estimator not enabled on this channel");
  CK(cudaSetDevice(e->prm.device));
  CK(cudaStreamSynchronize(p.insp_stream));
  const unsigned S = e->prm.n_streams; const int K = (int) e->channels.size();
  const size_t pitch = (size_t) K * 2 * sizeof(float), off = (size_t) handle * 2 + estimator_id;
  CK(cudaMemcpy2D(values, sizeof(float), p.d_est + off, pitch, sizeof(float), S, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy2D(valid, sizeof(int32_t), p.d_est_valid + off, pitch, sizeof(int32_t), S, cudaMemcpyDeviceToHost));
  return 0;
}

// sdb_inspector_config -> SdbChainCfg (SPEC X; same derivations as the inspector constructors).  A power inspector
// keeps only its class: it has no chain (sdb_build_chain_map leaves it out).
static bool build_chain_cfg(const Channel &ch, SdbChainCfg &c, std::vector<float> &taps_pool)
{
  const sdb_inspector_config &g = ch.cfg;
  memset(&c, 0, sizeof(c));
  c.cls = ch.has_insp ? g.insp_class : SDB_INSP_RAW;
  if (c.cls == SDB_INSP_RAW || c.cls == SDB_INSP_POWER) return true;
  const float fs = g.fs;
  float bnor = g.baud / fs;
  if (bnor > 1.0f) bnor = 1.0f;
  if (!(bnor > 0.0f)) bnor = 1e-6f;
  const float T = 1.0f / bnor;
  c.bnor = bnor;
  c.gain2 = 2.0f * d_db_to_mag(g.agc_gain_db);
  c.dl_size = c.mh_size = 1;

  if (c.cls == SDB_INSP_AUDIO) {
    float tau = g.agc_ts * fs;
    if (tau < 2.0f) tau = 2.0f;
    if (g.agc_enabled) {
      sdbh::AgcDesign d = sdbh::agc_from_tau(tau, 1.0f);
      c.have_agc = 1; c.knee = d.knee; c.gain_slope = d.gain_slope; c.fixed_gain = d.fixed_gain;
      c.hang_max = d.hang_max; c.dl_size = d.dl_size; c.mh_size = d.mh_size;
      c.far_ = d.far_; c.faf = d.faf; c.sar = d.sar; c.saf = d.saf;
    }
    if (sdbh::butter_lp(4, sdbh::clampf(2.0f * g.audio_cutoff / fs, 1e-4f, 0.95f), c.alpf_b, c.alpf_a))
      c.alpf_n = 5;
    c.audio_demod = (int) g.audio_demod; c.audio_squelch = g.audio_squelch;
    c.audio_volume = g.audio_volume;
    c.dc_alpha = (float) (1.0 - exp(-1.0 / (0.05 * (double) fs)));
    c.sq_alpha = (float) (1.0 - exp(-1.0 / (0.01 * (double) fs)));
    c.sq_thr = g.audio_squelch_level;
    c.rs_step = (double) g.audio_sample_rate / (double) fs;
    float fo = g.audio_demod == SDB_AUDIO_USB ? g.offset : -g.offset;
    c.lo_omega = 3.14159265358979323846f * (2.0f * fo / fs);
    return true;
  }

  if (g.agc_enabled) {
    sdbh::AgcDesign d = sdbh::agc_from_tau(T, 1.0f);
    c.have_agc = 1; c.knee = d.knee; c.gain_slope = d.gain_slope; c.fixed_gain = d.fixed_gain;
    c.hang_max = d.hang_max; c.dl_size = d.dl_size; c.mh_size = d.mh_size;
    c.far_ = d.far_; c.faf = d.faf; c.sar = d.sar; c.saf = d.saf;
  }
  c.af_n = 1; c.af_b[0] = 1.0f; c.af_a[0] = 1.0f;
  switch (c.cls) {
    case SDB_INSP_PSK:
      if (g.costas_order > 0) {
        if (g.costas_order > 3) return false;
        c.have_costas = 1; c.costas_kind = (int) g.costas_order;
        float loop = 2.0f * g.loop_bw / fs;
        c.c_a = 3.14159265358979323846f * loop;
        c.c_b = 0.5f * c.c_a * c.c_a;
        // arm filter "order 3" = 2-pole Butterworth (Tasks/CostasRecoveryTask.cpp:41)
        if (!sdbh::butter_lp(2, sdbh::clampf(2.0f * bnor, 1e-3f, 0.95f), c.af_b, c.af_a)) return false;
        c.af_n = 3;
      } else {
        c.have_lo = 1;
        c.lo_omega = 3.14159265358979323846f * (2.0f * g.offset / fs);
      }
      break;
    case SDB_INSP_FSK: {
      float s, co;
      d_sincosf(g.fsk_phase, &s, &co);
      c.fsk_rot_re = co; c.fsk_rot_im = s;
      c.fsk_quad_demod = g.fsk_quad_demod;
      break;
    }
    case SDB_INSP_ASK:
      if (g.ask_use_pll) {
        float fc = 3.14159265358979323846f * (2.0f * g.loop_bw / fs);
        float dinv = 1.0f / (1.0f + 2.0f * 0.707f * fc + fc * fc);
        c.have_pll = 1;
        c.pll_alpha = 4.0f * fc * fc * dinv;
        c.pll_beta = 4.0f * 0.707f * fc * dinv;
      } else {
        c.have_lo = 1;
        c.lo_omega = 3.14159265358979323846f * (2.0f * g.offset / fs);
      }
      c.ask_channel = (int) g.ask_channel;
      break;
    default:
      return false;
  }
  if (g.mf_type == 1) {
    std::vector<float> h;
    unsigned n = sdbh::mf_span(T);
    sdbh::taps_rrc(h, n, T, g.mf_rolloff);
    c.have_mf = 1; c.mf_n = (int) n; c.mf_off = (int) taps_pool.size();
    taps_pool.insert(taps_pool.end(), h.begin(), h.end());
  }
  c.clock_type = (int) g.clock_type; c.clock_running = g.clock_running;
  c.clk_gain = g.clock_gain; c.clk_alpha = 2e-1f; c.clk_beta = 6e-4f * c.clk_alpha;
  c.smp_period = 1.0f / bnor; c.smp_phase0 = g.clock_phase * c.smp_period;
  if (c.cls == SDB_INSP_ASK) { c.dec_mode = 1; c.dec_min = 0.0f; c.dec_h = 1.0f - 0.0f; }
  else { c.dec_mode = 0; c.dec_min = -3.14159265358979323846f;
         c.dec_h = 3.14159265358979323846f - (-3.14159265358979323846f); }
  c.dec_intervals = 1 << g.bits_per_symbol;
  c.eq_type = (int) g.eq_type; c.eq_locked = g.eq_locked; c.eq_mu = g.eq_rate;
  if (g.eq_type > 1) return false;
  return true;
}

// Lays out the chain's state lines in its float pool (AGC delay line, magnitude history, matched-filter line) and
// returns its initial loop state: AGC levels at the -160 dB floor, Gardner phase 1/4, CMA equaliser at identity.
static SdbChainState chain_layout(SdbChainCfg &c)
{
  c.st_dl_off = 0; c.st_mh_off = 2 * (int) c.dl_size; c.st_mf_off = c.st_mh_off + (int) c.mh_size;
  c.st_pool = c.st_mf_off + 2 * c.mf_n;
  SdbChainState s;
  memset(&s, 0, sizeof(s));
  s.fast_level = s.slow_level = s.peak = -160.0f;
  s.k_phi = 0.25f; s.k_bnor = c.bnor; s.eq_wr[0] = 1.0f;
  return s;
}

// Pin the four-step scratch in L2.  Without this the streamed input and output evict it between the two passes and
// every window costs two extra HBM round trips.  Accesses of the transform streams inside the window are "persisting"
// (a set-aside part of L2 that normal traffic cannot evict); the kernels additionally mark their one-shot outputs as
// streaming (st.global.cs).  The set-aside is device-wide: only the F.5 plans claim it.
static void pin_scratch(const sdb_engine *e, Plan &p, const SdbFourStep &big)
{
  int max_persist = 0, max_window = 0;
  cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, e->prm.device);
  cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, e->prm.device);
  const size_t bytes = (size_t) p.chunk_windows * big.N * sizeof(float2);
  if (max_persist > 0 && max_window > 0) {
    const size_t set_aside = std::min(bytes, (size_t) max_persist);
    if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, set_aside) == cudaSuccess) {
      cudaStreamAttrValue av{};
      av.accessPolicyWindow.base_ptr = p.d_scratch;
      av.accessPolicyWindow.num_bytes = std::min(bytes, (size_t) max_window);
      av.accessPolicyWindow.hitRatio = (float) std::min(1.0, (double) set_aside / (double) av.accessPolicyWindow.num_bytes);
      av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
      av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
      if (cudaStreamSetAttribute(e->stream, cudaStreamAttributeAccessPolicyWindow, &av) == cudaSuccess)
        p.l2_pinned_bytes = set_aside;
      if (p.psd_stream) cudaStreamSetAttribute(p.psd_stream, cudaStreamAttributeAccessPolicyWindow, &av);
    }
    cudaGetLastError();   // the pin is an optimisation: never fail the commit because of it
  }
}

// the group size of the frame-averaged PSD (SPEC A.1) or of the peak detectors (SPEC PK.1): 0 or 1 = off, at most
// `max`, and only with a main PSD
static int check_group_size(const char *name, unsigned v, unsigned max, unsigned Np)
{
  if (v > max) return fail(std::string(name) + " must be at most " + std::to_string(max) + ", got " + std::to_string(v));
  if (v >= 2 && !Np) return fail(std::string(name) + " needs the main PSD (psd_size > 0)");
  return 0;
}

// G >= 2 turns the stage on: outputs for feeds of at most max_frames frames, and a zero carry
static int groups_commit(FrameGroups &g, unsigned G, size_t S, unsigned Np, size_t max_frames, const char *oom)
{
  if (G < 2) return 0;
  g.G = G;
  // a feed completes at most ceil(max_frames / G) groups (G - 1 carried frames + max_frames)
  const size_t max_groups = (max_frames + G - 1) / G;
  for (int k = 0; k < g.n_out; ++k) {
    if (g.out[0][k].alloc(S * max_groups * Np) || g.out[1][k].alloc(S * max_groups * Np) || g.carry[k].alloc(S * Np))
      return fail(oom);
    CK(cudaMemset(g.carry[k], 0, S * Np * sizeof(float)));
  }
  return 0;
}

// the groups of this feed's `frames` PSD frames (slot `parity`), on lc's stream
static int groups_feed(sdb_engine *e, FrameGroups &g, const SdbLaunchCtx &lc, unsigned parity, const float *psd,
                       unsigned frames, int shift_db)
{
  if (!g.G) return 0;
  const size_t S = e->prm.n_streams;
  const unsigned groups = (g.count + frames) / g.G;
  const DevBuf<float> *o = g.out[parity];
  e->span_begin(g.fam, lc.stream);
  if (g.n_out == 1)
    CK(sdb_launch_psd_group_mean(lc, psd, frames, e->Np, S, g.G, g.count, groups, shift_db, g.carry[0], o[0]));
  else
    CK(sdb_launch_psd_group_peak(lc, psd, frames, e->Np, S, g.G, g.count, groups, shift_db, g.carry[0], g.carry[1],
                                 o[0], o[1]));
  e->span_end(lc.stream);
  g.count = (g.count + frames) % g.G;
  g.last = groups;
  return 0;
}

// live re-plan: the partial group carries over when both engines group the same frames the same way
static int groups_migrate(FrameGroups &to, const FrameGroups &from, const sdb_engine *dst, const sdb_engine *src)
{
  if (!to.G || to.G != from.G || dst->Np != src->Np || dst->prm.psd_window != src->prm.psd_window) return 0;
  for (int k = 0; k < to.n_out; ++k)
    CK(cudaMemcpy(to.carry[k], from.carry[k], to.carry[k].size() * sizeof(float), cudaMemcpyDeviceToDevice));
  to.count = from.count;
  return 0;
}

// blocking read of the latest feed's groups, fenced like sdb_engine_read_psd; g: null without a plan, dst: NULL skips
static int groups_read(sdb_engine *e, const FrameGroups *g, float *dst0, float *dst1, size_t cap, const char *off)
{
  if (!g || !g->G) return fail(off);
  Plan &p = *e->plan;
  if (p.feed_index == 0) return fail("no PSD available");
  const size_t n = (size_t) e->prm.n_streams * g->last * e->Np;
  if (cap < n) return fail("destination too small");
  if (n == 0 || (!dst0 && !dst1)) return 0;
  float *const dst[2] = { dst0, dst1 };
  Slot &sl = p.cur();
  CK(cudaSetDevice(e->prm.device));
  CK(sl.psd_ready.wait_on(p.d2h_stream));
  for (int k = 0; k < g->n_out; ++k)
    if (dst[k])
      CK(cudaMemcpyAsync(dst[k], g->out[p.cur_parity()][k], n * sizeof(float), cudaMemcpyDeviceToHost, p.d2h_stream));
  CK(sl.psd_read.record(p.d2h_stream));
  CK(cudaStreamSynchronize(p.d2h_stream));
  return 0;
}

// SPEC FC: the FAC chains of every channel with the FAC on, their state (empty blocks, max = -inf, min = +inf, fac = 0)
// and per-feed work areas for the most blocks one feed can complete.  Persistent launches get at most two CTAs per SM.
static int fac_commit(sdb_engine *e, Plan &p, size_t max_hops)
{
  const unsigned S = e->prm.n_streams;
  const int K = (int) e->channels.size();
  Plan::Fac &f = p.fac;
  f.first.assign(K, -1);
  size_t blk = 0, facn = 0, work = 0, scr = 0;
  uint32_t slots_total = 0, tiles_total = 0;
  uint64_t units[SDB_FAC_KINDS] = {0, 0, 0, 0};
  for (int k = 0; k < K; ++k) {
    const Channel &c = e->channels[k];
    if (!c.has_fac) continue;
    if (!c.has_insp || c.cfg.insp_class > SDB_INSP_ASK) return fail("the FAC needs a psk, fsk or ask inspector");
    const uint32_t L = c.fac.size;
    SdbFacChan h{};
    h.L = L; h.logL = (uint32_t) ilog2u(L);
    h.lo = c.fac.lag_lo; h.hi = c.fac.lag_hi ? c.fac.lag_hi : L / 2;
    h.ntiles = (h.hi - h.lo + 1023) / 1024;
    h.alpha = c.fac.alpha; h.sigma = c.fac.sigma;
    h.tw = p.twiddle(L);
    if (L > 4096) {                      // SPEC F.3: N1 = 2^floor(l / 2)
      h.N1 = 1u << (h.logL / 2); h.N2 = L / h.N1;
      h.logN1 = (uint32_t) ilog2u(h.N1); h.logN2 = (uint32_t) ilog2u(h.N2);
      h.twN1 = p.twiddle(h.N1); h.twN2 = p.twiddle(h.N2);
      if (!h.twN1 || !h.twN2) return fail("out of device memory (FAC)");
    }
    if (!h.tw) return fail("out of device memory (FAC)");
    // a chain emits at most one symbol per channel sample (the bound the symbol rows are sized by): a feed brings at
    // most max_hops halfsz of them, and completes at most (L - 1 + that) / L blocks
    const size_t sym_max = max_hops * c.halfsz;
    const uint32_t slots = (uint32_t) ((L - 1 + sym_max) / L);
    f.first[k] = (int) f.h.size();
    for (unsigned s = 0; s < S; ++s) {
      h.row = s * (uint32_t) K + (uint32_t) k;
      h.slot_off = slots_total; h.tile_off = tiles_total;
      h.blk_off = blk; h.fac_off = facn; h.work_off = work; h.scr_off = scr;
      slots_total += slots; tiles_total += slots * h.ntiles;
      blk += L; facn += L / 2; work += (size_t) slots * L;
      if (L > 4096) scr += (size_t) slots * L;
      units[L <= 4096 ? 0 : 1] += L <= 4096 ? slots : (uint64_t) slots * (L / 4096);
      units[2] += (uint64_t) slots * h.ntiles;
      units[3] += (L / 2 + 1023) / 1024;
      f.h.push_back(h);
    }
  }
  if (f.h.empty()) return 0;
  const size_t C = f.h.size();
  if (f.chans.alloc(C) || f.state.alloc(C) || f.blk.alloc(blk) || f.fac.alloc(facn) || f.work.alloc(work) ||
      (scr && f.scr.alloc(scr)) || f.slot_max.alloc(slots_total) || f.tiles.alloc(tiles_total) ||
      f.offs.alloc(SDB_FAC_KINDS * (C + 1)) || f.nb.alloc(C) || f.status.alloc(C))
    return fail("out of device memory (FAC)");
  CK(cudaMemcpy(f.chans, f.h.data(), C * sizeof(SdbFacChan), cudaMemcpyHostToDevice));
  const std::vector<SdbFacState> st(C, SdbFacState{ 0u, -INFINITY, INFINITY });
  CK(cudaMemcpy(f.state, st.data(), C * sizeof(SdbFacState), cudaMemcpyHostToDevice));
  const std::vector<sdb_fac_status> none(C, sdb_fac_status{ 0u, 0u, -INFINITY, INFINITY, 0.0f, 0 });
  CK(cudaMemcpy(f.status, none.data(), C * sizeof(sdb_fac_status), cudaMemcpyHostToDevice));
  CK(cudaMemset(f.fac, 0, facn * sizeof(float)));
  CK(cudaMemset(f.blk, 0, blk * sizeof(float2)));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, e->prm.device));
  for (int k = 0; k < SDB_FAC_KINDS; ++k) f.grid[k] = (int) std::min<uint64_t>(units[k], 2 * (uint64_t) sms);
  return 0;
}

// SPEC FC for one feed, on the inspector stream after the chains: the blocks the feed's symbols complete
static int fac_feed(sdb_engine *e, Plan &p, Slot &sl, const SdbLaunchCtx &ictx)
{
  Plan::Fac &f = p.fac;
  if (f.h.empty()) return 0;
  SdbFacArgs a{};
  a.chans = f.chans; a.n_chans = (int) f.h.size();
  a.state = f.state; a.blk = f.blk; a.fac = f.fac; a.work = f.work; a.scr = f.scr; a.slot_max = f.slot_max;
  a.tiles = f.tiles; a.offs = f.offs; a.nb = f.nb;
  a.soft = sl.soft; a.counts = sl.counts; a.sym_cap = p.sym_cap; a.status = f.status;
  e->span_begin(FAM_FAC, ictx.stream);
  CK(sdb_launch_fac(ictx, a, f.grid));
  e->span_end(ictx.stream);
  return 0;
}

// SPEC SN.3: every channel with the meter on starts with an empty h, a zero model and sigma from its parameters
static int snr_commit(sdb_engine *e, Plan &p)
{
  const unsigned S = e->prm.n_streams;
  const int K = (int) e->channels.size();
  Plan::Snr &q = p.snr;
  q.first.assign(K, -1);
  size_t bins = 0;
  std::vector<sdb_snr_status> st;
  for (int k = 0; k < K; ++k) {
    const Channel &c = e->channels[k];
    if (!c.has_snr) continue;
    if (!c.has_insp || c.cfg.insp_class > SDB_INSP_ASK) return fail("the SNR meter needs a psk, fsk or ask inspector");
    SdbSnrChan h{};
    h.L = c.snr.bins; h.K = snr_K(c.cfg); h.k = (uint32_t) k; h.chain0 = (uint32_t) st.size();
    h.mode = c.cfg.insp_class == SDB_INSP_ASK ? 1 : 0;
    if (h.mode) { h.dmin = 0.0f; h.dh = 1.0f - 0.0f; }          // SPEC D, as build_chain_cfg sets the decider
    else { h.dmin = -3.14159265358979323846f; h.dh = 3.14159265358979323846f - (-3.14159265358979323846f); }
    h.alpha = c.snr.alpha; h.hist_off = bins;
    bins += (size_t) S * h.L;
    q.max_L = std::max(q.max_L, h.L);
    q.first[k] = (int) q.h.size();
    q.h.push_back(h);
    st.insert(st.end(), S, sdb_snr_status{ 0ull, 0u, 0u, c.snr.sigma, 1.0f / (h.K * c.snr.sigma), 0.0f });
  }
  if (q.h.empty()) return 0;
  if (q.chans.alloc(q.h.size()) || q.hist.alloc(bins) || q.model.alloc(bins) || q.status.alloc(st.size()))
    return fail("out of device memory (SNR meter)");
  CK(cudaMemcpy(q.chans, q.h.data(), q.h.size() * sizeof(SdbSnrChan), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(q.status, st.data(), st.size() * sizeof(sdb_snr_status), cudaMemcpyHostToDevice));
  CK(cudaMemset(q.hist, 0, bins * sizeof(uint32_t)));
  CK(cudaMemset(q.model, 0, bins * sizeof(float)));
  return 0;
}

// SPEC TI: every channel with the TV on starts from sdb_tv_state_init with every buffer zero
static int tv_commit(sdb_engine *e, Plan &p)
{
  const unsigned S = e->prm.n_streams;
  const int K = (int) e->channels.size();
  Plan::Tv &q = p.tv;
  q.first.assign(K, -1);
  size_t nd = 0, nl = 0, nr = 0, np = 0;
  std::vector<SdbTvState> st;
  std::vector<sdb_tv_status> status;
  for (int k = 0; k < K; ++k) {
    const Channel &c = e->channels[k];
    if (!c.has_tv) continue;
    if (!c.has_insp || c.cfg.insp_class > SDB_INSP_ASK) return fail("the TV needs a psk, fsk or ask inspector");
    if (sdb_tv_tab_check(&c.tv)) return -1;
    SdbTvInspChan h{};
    tv_describe(c, h);
    const size_t px = (size_t) h.c.H * h.c.W;
    h.k = (uint32_t) k; h.chain0 = (uint32_t) st.size();
    h.delay_off = nd; h.line_off = nl; h.ring_off = nr; h.post_off = np;
    nd += (size_t) S * h.c.delay_len; nl += (size_t) S * h.c.W; nr += (size_t) S * SDB_TV_RING * px; np += S * px;
    q.smem = std::max(q.smem, (size_t) (h.c.W + h.c.delay_len) * sizeof(float));
    q.first[k] = (int) q.h.size();
    q.h.push_back(h);
    SdbTvState s0;
    sdb_tv_state_init(h.c, s0);
    st.insert(st.end(), S, s0);
    status.insert(status.end(), S, sdb_tv_status{ 0ull, 0ull, 0u, (uint32_t) h.c.W, (uint32_t) h.c.H, s0.est_line_len,
                                                  s0.est_hsync_len, s0.agc_gain });
  }
  if (q.h.empty()) return 0;
  if (q.chans.alloc(q.h.size()) || q.state.alloc(st.size()) || q.status.alloc(st.size()) || q.delay.alloc(nd) ||
      q.line.alloc(nl) || q.ring.alloc(nr) || q.post.alloc(np))
    return fail("out of device memory (TV)");
  CK(cudaMemcpy(q.chans, q.h.data(), q.h.size() * sizeof(SdbTvInspChan), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(q.state, st.data(), st.size() * sizeof(SdbTvState), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(q.status, status.data(), status.size() * sizeof(sdb_tv_status), cudaMemcpyHostToDevice));
  CK(cudaMemset(q.delay, 0, nd * sizeof(float)));
  CK(cudaMemset(q.line, 0, nl * sizeof(float)));
  CK(cudaMemset(q.ring, 0, nr * sizeof(float)));
  CK(cudaMemset(q.post, 0, np * sizeof(float)));
  return 0;
}

// SPEC TI.1-TI.3 for one feed, on the inspector stream after the SNR meter
static int tv_feed(sdb_engine *e, Plan &p, Slot &sl, const SdbLaunchCtx &ictx)
{
  Plan::Tv &q = p.tv;
  if (q.h.empty()) return 0;
  SdbTvInspArgs a{};
  a.chans = q.chans; a.n_chans = (int) q.h.size(); a.n_streams = (int) e->prm.n_streams;
  a.n_channels = (int) e->channels.size(); a.smem = q.smem;
  a.soft = sl.soft; a.counts = sl.counts; a.sym_cap = p.sym_cap;
  a.state = q.state; a.delay = q.delay; a.line = q.line; a.ring = q.ring; a.post = q.post; a.status = q.status;
  e->span_begin(FAM_TV, ictx.stream);
  CK(sdb_launch_tv_insp(ictx, a));
  e->span_end(ictx.stream);
  return 0;
}

// SPEC SN.2 for one feed, on the inspector stream after the chains (and the power and FAC launches)
static int snr_feed(sdb_engine *e, Plan &p, Slot &sl, const SdbLaunchCtx &ictx)
{
  Plan::Snr &q = p.snr;
  if (q.h.empty()) return 0;
  SdbSnrArgs a{};
  a.chans = q.chans; a.n_chans = (int) q.h.size(); a.n_streams = (int) e->prm.n_streams;
  a.n_channels = (int) e->channels.size(); a.max_L = q.max_L;
  a.soft = sl.soft; a.counts = sl.counts; a.sym_cap = p.sym_cap;
  a.hist = q.hist; a.model = q.model; a.status = q.status;
  e->span_begin(FAM_SNR, ictx.stream);
  CK(sdb_launch_snr(ictx, a));
  e->span_end(ictx.stream);
  return 0;
}

extern "C" int sdb_engine_commit(sdb_engine_t *e)
{
  if (!e) return fail("null engine");
  if (e->plan) return fail("already committed");
  CK(cudaSetDevice(e->prm.device));
  const unsigned S = e->prm.n_streams, W = e->W, Np = e->Np;
  const int K = (int) e->channels.size();
  size_t max_feed = e->prm.max_feed;
  if (max_feed == 0) return fail("max_feed must be > 0");
  if (max_feed % (W / 2)) return fail("max_feed must be a multiple of st_window_size / 2");
  if (Np && max_feed % Np) return fail("max_feed must be a multiple of psd_size");
  const unsigned A = e->prm.psd_average, P = e->prm.psd_peak;
  if (check_group_size("psd_average", A, SDB_PSD_AVERAGE_MAX, Np) || check_group_size("psd_peak", P, SDB_PSD_PEAK_MAX, Np))
    return -1;
  // built here and handed to the engine at the end: every early return frees what was built so far
  auto plan = std::make_unique<Plan>();
  Plan &p = *plan;

  // ---- PSD plan
  if (Np) {
    std::vector<float> w;
    if (e->prm.psd_window != SDB_WINDOW_NONE) {
      sdbh::window_fill(w, Np, e->prm.psd_window);
      p.d_window = p.dalloc<float>(Np);
      if (!p.d_window) return fail("out of device memory");
      CK(cudaMemcpy(p.d_window, w.data(), Np * sizeof(float), cudaMemcpyHostToDevice));
    }
    if (!make_plan(p, Np, true, &p.fs_psd)) return fail("out of device memory");
    const size_t max_frames = max_feed / Np;
    for (Slot &sl : p.slot) {
      sl.psd = p.dalloc<float>((size_t) S * max_frames * Np);
      if (!sl.psd) return fail("out of device memory (psd)");
    }
    if (groups_commit(p.avg, A, S, Np, max_frames, "out of device memory (averaged psd)") ||
        groups_commit(p.peak, P, S, Np, max_frames, "out of device memory (psd peaks)"))
      return -1;
    if (e->cd_enabled) {
      p.chdet.reset(sdb_chdet_new(e->prm.device, Np, S, e->cd_alpha, e->cd_gamma, e->cd_snr, e->cd_min_bins));
      if (!p.chdet) return fail("out of device memory (channel detector)");
      if (e->ct_enabled) {
        if (!(e->cd_beta > 0.0f && e->cd_beta <= 1.0f)) return fail("channel tracking needs a detector beta in (0, 1]");
        p.chtrack.reset(sdb_chtrack_new(e->prm.device, Np, S, e->cd_beta, e->ct_hold));
        if (!p.chtrack) return fail("out of device memory (channel tracking)");
      }
    }
  }
  if (K > 0 && !make_plan(p, W, false, &p.fs_st)) return fail("out of device memory");
  // ---- four-step scratch of the two-kernel paths: whole waves of both passes, pinned in L2 (pin_scratch).  The
  // cluster path keeps its intermediate in the shared memory of a thread-block cluster and needs none.
  const SdbFourStep *big = nullptr;
  if (Np && uses_scratch(p.fs_psd)) big = &p.fs_psd;
  if (K > 0 && uses_scratch(p.fs_st) && (!big || p.fs_st.N > big->N)) big = &p.fs_st;
  if (big) {
    p.chunk_windows = (int) scratch_chunk_windows(*big, e->prm.device);
    p.d_scratch = p.dalloc<float2>((size_t) p.chunk_windows * big->N);
    if (!p.d_scratch) return fail("out of device memory (scratch)");
    if (Np && K > 0 && Np == W && uses_scratch(p.fs_psd)) {
      CK(p.psd_stream.create(cudaStreamNonBlocking));
      CK(p.ev_feed.create());
    }
  }
  // ---- channeliser plan
  const size_t max_hops = max_feed / (W / 2);
  if (K > 0) {
    std::vector<int> binmap(W, -1);
    std::vector<char> need(W, 0);
    for (auto &c : e->channels)
      for (unsigned i = 0; i < 2 * c.halfw; ++i) need[(c.center + W - c.halfw + i) % W] = 1;
    int nb = 0;
    // bin k = k1 + N1 (ka + 16 kb) on the cluster and F.5 paths; the Stockham passes ignore the mask
    const int ka_shift = p.fs_st.ka_shift;
    for (unsigned b = 0; b < W; ++b) if (need[b]) { binmap[b] = nb++; p.ka_mask |= 1u << ((b >> ka_shift) & 15u); }
    p.n_bins = nb;
    p.d_binmap = p.dalloc<int>(W);
    if (!p.d_binmap) return fail("out of device memory");
    CK(cudaMemcpy(p.d_binmap, binmap.data(), W * sizeof(int), cudaMemcpyHostToDevice));
    p.d_cspec = p.dalloc<float2>((size_t) S * max_hops * nb);
    p.d_hist = p.dalloc<float2>((size_t) S * (W / 2));
    if (!p.d_cspec || !p.d_hist) return fail("out of device memory (cspec)");
    CK(cudaMemset(p.d_hist, 0, (size_t) S * (W / 2) * sizeof(float2)));

    p.h_chans.resize(K);
    size_t out_off = 0, tail_off = 0;
    std::map<int, std::vector<int>> by_size;
    for (int k = 0; k < K; ++k) {
      Channel &c = e->channels[k];
      SdbChannelDev &d = p.h_chans[k];
      memset(&d, 0, sizeof(d));
      d.center = (int) c.center; d.size = (int) c.size; d.log2size = ilog2u(c.size);
      d.halfw = (int) c.halfw; d.halfsz = (int) c.halfsz;
      unsigned b0 = (c.center + W - c.halfw) % W;
      d.c1 = binmap[b0];
      d.L1 = (int) std::min<unsigned>(2 * c.halfw, W - b0);
      d.precise = c.p.precise;
      if (c.p.precise) {
        double resid = (double) c.p.f0 - 2.0 * sdbh::kPi * (double) c.center / (double) W;
        if (resid > sdbh::kPi) resid -= 2.0 * sdbh::kPi;
        float dec = (float) W / (float) c.size;
        float fnor = (float) (resid * (double) dec / sdbh::kPi);
        d.lo_omega = 3.14159265358979323846f * fnor;
      }
      std::vector<float> kh, xf;
      sdbh::channel_weights(W, c.halfw, kh);
      sdbh::xfade_fill(c.size, xf);
      float *dkh = p.dalloc<float>(kh.size()), *dxf = p.dalloc<float>(xf.size());
      if (!dkh || !dxf) return fail("out of device memory");
      CK(cudaMemcpy(dkh, kh.data(), kh.size() * sizeof(float), cudaMemcpyHostToDevice));
      CK(cudaMemcpy(dxf, xf.data(), xf.size() * sizeof(float), cudaMemcpyHostToDevice));
      d.kh = dkh; d.xfade = dxf; d.tw = p.twiddle(c.size);
      if (!d.tw) return fail("out of device memory");
      d.out_off = out_off; d.out_cap = max_hops * c.halfsz; out_off += d.out_cap;
      d.tail_off = tail_off; tail_off += c.halfsz;
      by_size[(int) c.size].push_back(k);
    }
    p.chan_stride = out_off; p.tail_stride = tail_off;
    p.d_chans = p.dalloc<SdbChannelDev>(K);
    for (Slot &sl : p.slot) sl.chan = p.dalloc<float2>((size_t) S * out_off);
    p.d_tails = p.dalloc<float2>((size_t) S * tail_off);
    p.d_lo_phase = p.dalloc<float>((size_t) S * K);
    if (!p.d_chans || !p.slot[0].chan || !p.slot[1].chan || !p.d_tails || !p.d_lo_phase)
      return fail("out of device memory (channels)");
    // The inspector kernel of feed i runs beside the transforms of feed i + 1.  Its CTAs are few and long-lived; the
    // highest priority places them as soon as SM space frees up instead of after every CTA of a transform grid
    // queued before them (the cluster path: one grid per feed) has been dispatched.
    int prio_least = 0, prio_greatest = 0;
    CK(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
    CK(p.insp_stream.create(cudaStreamNonBlocking, prio_greatest));
    CK(p.ev_chan.create());
    CK(cudaMemcpy(p.d_chans, p.h_chans.data(), K * sizeof(SdbChannelDev), cudaMemcpyHostToDevice));
    CK(cudaMemset(p.d_tails, 0, (size_t) S * tail_off * sizeof(float2)));
    CK(cudaMemset(p.d_lo_phase, 0, (size_t) S * K * sizeof(float)));
    for (auto &kv : by_size) {
      Plan::Group g; g.size = kv.first; g.len = (int) kv.second.size(); g.any_precise = 0;
      for (int id : kv.second) if (p.h_chans[id].precise) g.any_precise = 1;
      g.d_ids = p.dalloc<int>(kv.second.size());
      if (!g.d_ids) return fail("out of device memory");
      CK(cudaMemcpy(g.d_ids, kv.second.data(), kv.second.size() * sizeof(int), cudaMemcpyHostToDevice));
      p.groups.push_back(g);
    }
    // ---- inspector spectrum sources / estimators, once per feed (SPEC U) or on a schedule (SPEC US)
    {
      std::vector<SdbSpectCfg> sc(K), slot_cfg;
      std::vector<SdbChannelDev> slot_dev;
      std::vector<int> slot_chan;
      std::map<unsigned, float *> bh_windows;   // Blackman-Harris windows by size
      size_t off = 0, soff = 0, ring_off = 0, frame_off = 0; int max_ns = 0; bool any = false;
      p.sched_of.assign(K, -1);
      for (int k = 0; k < K; ++k) {
        const Channel &c = e->channels[k];
        SdbSpectCfg q;
        memset(&q, 0, sizeof(q));
        memset(&sc[k], 0, sizeof(q));          // scheduled channels keep this empty entry
        if (c.spect_kind == 0 && c.est_mask == 0) {
          if (c.spect_interval)
            return fail("spectrum interval on channel " + std::to_string(k) + ", which has no spectrum source or estimator");
          continue;
        }
        const unsigned ns = c.spect_size ? c.spect_size : 1024u;
        q.kind = c.spect_kind; q.ns = (int) ns; q.logns = ilog2u(ns); q.est_mask = c.est_mask;
        q.fs_ch = (float) (e->samp_rate * (double) c.size / (double) W);
        q.tw = p.twiddle(ns);
        if (!q.tw) return fail("out of device memory");
        auto it = bh_windows.find(ns);
        if (it == bh_windows.end()) {
          std::vector<float> w;
          sdbh::window_fill(w, ns, SDB_WINDOW_BLACKMANN_HARRIS);
          float *d = p.dalloc<float>(ns);
          if (!d) return fail("out of device memory");
          CK(cudaMemcpy(d, w.data(), ns * sizeof(float), cudaMemcpyHostToDevice));
          it = bh_windows.emplace(ns, d).first;
        }
        q.window = it->second;
        const uint64_t I = c.spect_interval;
        if (!I) {
          any = true;
          q.out_off = off; off += ns;
          max_ns = std::max(max_ns, (int) ns);
          sc[k] = q;
          continue;
        }
        // a feed emits at every multiple of I among its channel samples: at most ceil(samples / I) times
        const uint64_t n_max = (uint64_t) max_hops * c.halfsz, slots = (n_max + I - 1) / I;
        if (slots > SDB_SPECTRUM_EMITS_MAX)
          return fail("spectrum interval " + std::to_string(I) + " on channel " + std::to_string(k) + " allows " +
                      std::to_string(slots) + " emissions per feed of max_feed samples; at most " +
                      std::to_string(SDB_SPECTRUM_EMITS_MAX));
        Plan::Sched sd;
        sd.k = k; sd.ns = ns; sd.kind = (unsigned) c.spect_kind; sd.est_mask = c.est_mask; sd.interval = I;
        sd.slot0 = (uint32_t) slot_cfg.size(); sd.slots = (uint32_t) slots; sd.out0 = soff;
        SdbSchedChan h;
        memset(&h, 0, sizeof(h));
        h.in_off = p.h_chans[k].out_off; h.ring_off = ring_off; h.frame_off = frame_off;
        h.ns1 = ns + 1; h.slot0 = sd.slot0; h.interval = I;
        for (uint64_t j = 0; j < slots; ++j) {
          SdbSpectCfg qe = q;
          qe.out_off = soff + j * ns;
          slot_cfg.push_back(qe);
          SdbChannelDev d;
          memset(&d, 0, sizeof(d));
          d.out_off = frame_off + j * (ns + 1);   // halfsz: set per feed by the gather
          slot_dev.push_back(d);
          slot_chan.push_back((int) p.sched.size());
        }
        soff += slots * ns; ring_off += ns + 1; frame_off += slots * (ns + 1);
        p.sched_max_ns = std::max(p.sched_max_ns, (int) ns);
        p.sched_of[k] = (int) p.sched.size();
        p.sched.push_back(sd); p.h_sched.push_back(h);
      }
      if (!p.sched.empty()) {
        const size_t ns_ = p.sched.size();
        p.n_slots = (int) slot_cfg.size();
        p.ring_stride = ring_off; p.frame_stride = frame_off; p.sched_spect_stride = soff;
        if (p.d_sched.alloc(ns_) || p.d_slot_chan.alloc(p.n_slots) || p.d_slot_cfg.alloc(p.n_slots) ||
            p.d_slot_dev.alloc(p.n_slots) || p.d_ring.alloc((size_t) S * ring_off) ||
            p.d_frames.alloc((size_t) S * frame_off))
          return fail("out of device memory (scheduled spectra)");
        for (Slot &sl : p.slot) {
          if (sl.sched_spect.alloc((size_t) S * soff) || sl.sched_size.alloc((size_t) S * p.n_slots) ||
              sl.sched_est.alloc((size_t) S * p.n_slots * 2) || sl.sched_valid.alloc((size_t) S * p.n_slots * 2))
            return fail("out of device memory (scheduled spectra)");
          CK(cudaMemset(sl.sched_size, 0, (size_t) S * p.n_slots * sizeof(uint32_t)));
          CK(cudaMemset(sl.sched_valid, 0, (size_t) S * p.n_slots * 2 * sizeof(int)));
          sl.sched_n.assign(ns_, 0); sl.sched_first.assign(ns_, 0);
        }
        CK(cudaMemcpy(p.d_slot_chan, slot_chan.data(), slot_chan.size() * sizeof(int), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(p.d_slot_cfg, slot_cfg.data(), slot_cfg.size() * sizeof(SdbSpectCfg), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(p.d_slot_dev, slot_dev.data(), slot_dev.size() * sizeof(SdbChannelDev), cudaMemcpyHostToDevice));
        CK(cudaMemset(p.d_ring, 0, (size_t) S * ring_off * sizeof(float2)));
      }
      if (any) {
        p.spect_stride = off; p.spect_max_ns = max_ns; p.h_spect = sc;
        p.d_spectcfg = p.dalloc<SdbSpectCfg>(K);
        p.d_spect = p.dalloc<float>((size_t) S * off);
        p.d_spect_size = p.dalloc<uint32_t>((size_t) S * K);
        p.d_est = p.dalloc<float>((size_t) S * K * 2);
        p.d_est_valid = p.dalloc<int>((size_t) S * K * 2);
        if (!p.d_spectcfg || !p.d_spect || !p.d_spect_size || !p.d_est || !p.d_est_valid)
          return fail("out of device memory (spectrum sources)");
        CK(cudaMemcpy(p.d_spectcfg, sc.data(), K * sizeof(SdbSpectCfg), cudaMemcpyHostToDevice));
        CK(cudaMemset(p.d_spect_size, 0, (size_t) S * K * sizeof(uint32_t)));
        CK(cudaMemset(p.d_est_valid, 0, (size_t) S * K * 2 * sizeof(int)));
      }
    }
    // ---- chains
    p.h_cfg.resize(K);
    std::vector<float> taps_pool;
    std::vector<SdbChainState> st0(K);
    size_t pool = 1, cap = 1;
    for (int k = 0; k < K; ++k) {
      if (!build_chain_cfg(e->channels[k], p.h_cfg[k], taps_pool)) return fail("invalid inspector configuration");
      SdbChainCfg &c = p.h_cfg[k];
      st0[k] = chain_layout(c);
      pool = std::max<size_t>(pool, (size_t) c.st_pool);
      cap = std::max<size_t>(cap, max_hops * e->channels[k].halfsz);
    }
    p.pool_stride = pool; p.sym_cap = cap;
    const size_t chains = (size_t) S * K;
    p.d_cfg = p.dalloc<SdbChainCfg>(K);
    p.d_state = p.dalloc<SdbChainState>(chains);
    p.insp_ctas = sdb_build_chain_map(p.h_cfg.data(), K, (int) S, p.h_chain_map);
    p.d_chain_map = p.dalloc<int>(p.h_chain_map.size());
    if (!p.d_chain_map) return fail("out of device memory (chain map)");
    CK(cudaMemcpy(p.d_chain_map, p.h_chain_map.data(), p.h_chain_map.size() * sizeof(int), cudaMemcpyHostToDevice));
    p.insp_grids = sdb_insp_grids(p.h_cfg.data(), (int) S, p.h_chain_map);
    const size_t pool_floats = (size_t) p.insp_ctas * 32 * pool;   // per-CTA interleaved [slot][lane]
    p.d_pool = p.dalloc<float>(pool_floats);
    p.d_taps = p.dalloc<float>(taps_pool.size());
    for (Slot &sl : p.slot) {
      sl.soft = p.dalloc<float2>(chains * cap);
      sl.hard = p.dalloc<uint8_t>(chains * cap);
      sl.counts = p.dalloc<uint32_t>(chains);
      if (!sl.soft || !sl.hard || !sl.counts) return fail("out of device memory (symbols)");
      CK(cudaMemset(sl.counts, 0, chains * sizeof(uint32_t)));
    }
    if (!p.d_cfg || !p.d_state || !p.d_pool || !p.d_taps) return fail("out of device memory (chains)");
    CK(cudaMemcpy(p.d_cfg, p.h_cfg.data(), K * sizeof(SdbChainCfg), cudaMemcpyHostToDevice));
    if (!taps_pool.empty())
      CK(cudaMemcpy(p.d_taps, taps_pool.data(), taps_pool.size() * sizeof(float), cudaMemcpyHostToDevice));
    std::vector<SdbChainState> st(chains);
    for (size_t ci = 0; ci < chains; ++ci) st[ci] = st0[ci % K];
    CK(cudaMemcpy(p.d_state, st.data(), chains * sizeof(SdbChainState), cudaMemcpyHostToDevice));
    {
      // lines start empty: delay line and filter line 0, magnitude history at the -160 dB floor (SPEC A); the engine
      // never asks the kernel for a `fresh` start, so that a re-planned engine can take over running chains
      std::vector<float> hp(pool_floats, 0.0f);
      for (size_t q = 0; q < p.h_chain_map.size(); ++q) {
        const int g = p.h_chain_map[q];
        if (g < 0) continue;
        const SdbChainCfg &c = p.h_cfg[g / (int) S];
        if (!c.have_agc) continue;
        float *base = hp.data() + (q / 32) * 32 * pool + (q % 32);
        for (unsigned i = 0; i < c.mh_size; ++i) base[(size_t) (c.st_mh_off + (int) i) * 32] = -160.0f;
      }
      CK(cudaMemcpy(p.d_pool, hp.data(), pool_floats * sizeof(float), cudaMemcpyHostToDevice));
    }
    // ---- power inspectors (SPEC PW): their groups start empty
    std::vector<SdbPowerChain> pw;
    for (int k = 0; k < K; ++k)
      if (is_power(e->channels[k]))
        for (unsigned s = 0; s < S; ++s)
          pw.push_back(SdbPowerChain{ (size_t) s * p.chan_stride + p.h_chans[k].out_off, e->channels[k].halfsz,
                                      s * (uint32_t) K + (uint32_t) k, power_m(e->channels[k].cfg) });
    if (!pw.empty()) {
      if (p.d_power.alloc(pw.size()) != cudaSuccess || p.power_carry.alloc(chains) != cudaSuccess)
        return fail("out of device memory (power inspectors)");
      p.n_power = (int) pw.size();
      CK(cudaMemcpy(p.d_power, pw.data(), pw.size() * sizeof(SdbPowerChain), cudaMemcpyHostToDevice));
      CK(cudaMemset(p.power_carry, 0, chains * sizeof(SdbPowerCarry)));
    }
    if (fac_commit(e, p, max_hops)) return -1;
    if (snr_commit(e, p)) return -1;
    if (tv_commit(e, p)) return -1;
  }
  if (e->prm.flags & SDB_FLAG_DC_REMOVE) {
    p.d_dc_state = p.dalloc<float2>(S); p.d_dc_cur = p.dalloc<float2>(S);
    p.d_dc_part = p.dalloc<double2>((size_t) S * ((max_feed + 255) / 256));
    p.d_xdc = p.dalloc<float2>((size_t) S * max_feed);
    if (!p.d_dc_state || !p.d_dc_cur || !p.d_dc_part || !p.d_xdc) return fail("out of device memory (DC removal)");
    CK(cudaMemset(p.d_dc_state, 0, S * sizeof(float2)));
  }
  CK(p.h2d_stream.create(cudaStreamNonBlocking));
  CK(p.d2h_stream.create(cudaStreamNonBlocking));
  for (Slot &sl : p.slot)
    for (Event *ev : { &sl.psd_ready, &sl.psd_read, &sl.sym_read, &sl.insp }) CK(ev->create());
  for (Plan::Stage &sg : p.stage) CK(sg.xfree.create());
  CK(p.ev_h2d.create());
  if (big && big->path == SDB_FFT_F5) pin_scratch(e, p, *big);
  e->plan = std::move(plan);
  return 0;
}

// SPEC US for one feed of `hops` channeliser hops.  On the host: every scheduled channel's emission points in
// (t, t + samples] whose frame lies in the history (t_j - Ns - 1 >= v; for a channel that started, t_j >= Ns + 1) and
// the feed samples a later frame can still need, [max(t, t_next - Ns - 1), t + samples).  On the inspector stream,
// after the feed's channel samples: the frame gather, k_spectsrc over the emitted frames, the ring update.
static int sched_feed(sdb_engine *e, Plan &p, Slot &sl, const SdbLaunchCtx &ictx, uint64_t hops)
{
  const int S = (int) e->prm.n_streams;
  uint32_t total = 0;
  bool writes = false;
  for (size_t i = 0; i < p.sched.size(); ++i) {
    Plan::Sched &q = p.sched[i];
    SdbSchedChan &h = p.h_sched[i];
    const uint64_t I = q.interval, ns1 = q.ns + 1, T0 = q.t, n = hops * (uint64_t) p.h_chans[q.k].halfsz, T1 = T0 + n;
    uint64_t first = (T0 / I + 1) * I;
    if (first < q.v + ns1) first += (q.v + ns1 - first + I - 1) / I * I;
    const uint32_t cnt = first <= T1 ? (uint32_t) ((T1 - first) / I + 1) : 0;
    const uint64_t next = (T1 / I + 1) * I;
    const uint64_t a = std::min(T1, std::max(T0, next > ns1 ? next - ns1 : 0));
    h.t0 = T0; h.t_first = first; h.n_emit = cnt;
    h.w_from = (uint32_t) (a - T0); h.w_to = (uint32_t) n;
    if (a > T0) q.v = a;                   // the ring holds [a, T1) only
    q.t = T1;
    sl.sched_n[i] = cnt; sl.sched_first[i] = first;
    total += cnt;
    writes = writes || a < T1;
  }
  if (!total && !writes) return 0;
  e->span_begin(FAM_SPECTSCHED, ictx.stream);
  CK(cudaMemcpyAsync(p.d_sched, p.h_sched.data(), p.h_sched.size() * sizeof(SdbSchedChan), cudaMemcpyHostToDevice,
                     ictx.stream));
  if (total) {
    CK(sdb_launch_spectsched_gather(ictx, p.d_sched, p.d_slot_chan, p.d_slot_dev, p.n_slots, S, sl.chan, p.chan_stride,
                                    p.d_ring, p.ring_stride, p.d_frames, p.frame_stride));
    CK(sdb_launch_spectsrc(ictx, p.d_slot_cfg, p.d_slot_dev, p.n_slots, S, p.sched_max_ns, p.d_frames, p.frame_stride,
                           1u, sl.sched_spect, p.sched_spect_stride, sl.sched_size, sl.sched_est, sl.sched_valid));
  }
  if (writes)
    CK(sdb_launch_spectsched_ring(ictx, p.d_sched, (int) p.sched.size(), S, sl.chan, p.chan_stride, p.d_ring,
                                  p.ring_stride));
  e->span_end(ictx.stream);
  return 0;
}

extern "C" int sdb_engine_feed_device(sdb_engine_t *e, const sdb_complex *xv, size_t stride, size_t n)
{
  if (!e || !xv) return fail("null argument");
  if (!e->plan) return fail("engine not committed");
  Plan &p = *e->plan;
  const unsigned S = e->prm.n_streams, W = e->W, Np = e->Np;
  const int K = (int) e->channels.size();
  if (n == 0 || n > e->prm.max_feed) return fail("feed size out of range");
  if (Np && n % Np) return fail("feed size must be a multiple of psd_size");
  if (K && n % (W / 2)) return fail("feed size must be a multiple of st_window_size / 2");
  CK(cudaSetDevice(e->prm.device));
  const void *x = reinterpret_cast<const void *>(xv);
  int fmt = e->prm.input_format | ((e->prm.flags & SDB_FLAG_IQ_REVERSE) ? SDB_FMT_SWAP : 0);
  if (p.d_xdc) {
    // SPEC R: the block is corrected with the estimate of the blocks before it; everything downstream reads the
    // corrected float32 copy (format conversion and I/Q swap happen in this pass)
    const float alpha = (float) (1.0 - exp(-(double) n / (e->samp_rate * 0.1)));
    CK(sdb_launch_dc_remove(e->stream, x, fmt, stride, n, (int) S, alpha, p.d_dc_state, p.d_dc_cur, p.d_dc_part,
                            p.d_xdc));
    e->launches += 3;
    x = p.d_xdc; fmt = SDB_FMT_F32; stride = n;
  }
  SdbLaunchCtx ctx{ e->stream, &e->launches };
  // with frame averaging or peak detection the flag applies to their group outputs: the transforms keep the per-frame
  // PSD linear
  const int groups_db = (e->prm.flags & SDB_FLAG_PSD_SHIFT_DB) ? 1 : 0;
  const int shift_db = p.avg.G || p.peak.G ? 0 : groups_db;
  Slot &sl = p.slot[p.feed_index & 1u];     // result buffers of this feed

  const int frames = Np ? (int) (n / Np) : 0;
  // the SPEC A means, then the SPEC PK extremes of this feed, on the stream of its PSD transforms after the last one
  auto frame_groups = [&](const SdbLaunchCtx &lc) -> int {
    return groups_feed(e, p.avg, lc, p.feed_index & 1u, sl.psd, (unsigned) frames, groups_db) ||
           groups_feed(e, p.peak, lc, p.feed_index & 1u, sl.psd, (unsigned) frames, groups_db);
  };
  // SPEC KT: the tracking update of this feed, on the detector's stream right after it
  auto chan_track = [&](cudaStream_t on) -> int {
    e->span_begin(FAM_CHAN_TRACK, on);
    CK(sdb_chtrack_feed_stream(p.chtrack.get(), p.chdet.get(), (uint32_t) frames, on, &e->launches));
    e->span_end(on);
    return 0;
  };
  const int H = K ? (int) (n / (W / 2)) : 0;
  const int first = (K && p.first_feed) ? 1 : 0;
  const int wps = K ? H - first : 0;
  // arguments of the two-kernel transforms: PSD frames (hop Np, no history) and channeliser windows (hop W / 2 over
  // the W / 2-sample history followed by x)
  SdbPassAArgs psd_a{}, chan_a{};
  psd_a.x = chan_a.x = x; psd_a.fmt = chan_a.fmt = fmt; psd_a.stream_stride = chan_a.stream_stride = stride;
  psd_a.windows_per_stream = frames; psd_a.hop = (int) Np; psd_a.window = p.d_window;
  chan_a.hist = p.d_hist; chan_a.hist_len = (int) (W / 2);
  chan_a.windows_per_stream = wps; chan_a.first_window = first; chan_a.hop = (int) (W / 2);
  SdbPassBArgs psd_b{}, chan_b{};
  psd_b.shift_db = shift_db;
  chan_b.binmap = p.d_binmap; chan_b.cspec = p.d_cspec; chan_b.n_bins = p.n_bins; chan_b.ka_mask = p.ka_mask;
  if (Np) {
    p.last_frames = frames;
    psd_b.psd = sl.psd; psd_b.inv_n = 1.0f / (float) Np;
  }
  // windows [w0, w0 + cw) of the flattened [stream][window] order through scratch region `scr`; pass B is timed as
  // family `fam_b` (FAM_ROWS_PSD: PSD epilogue, FAM_ROWS_CHAN: channeliser scatter)
  auto chunk = [&](const SdbLaunchCtx &lc, const SdbFourStep &fs, SdbPassAArgs a, SdbPassBArgs b, int fam_b, int w0,
                   int cw, float2 *scr) -> int {
    const int mode = fam_b == FAM_ROWS_CHAN ? 1 : 0;
    const bool f5 = fs.path == SDB_FFT_F5;
    a.scratch = scr;
    b.scratch = scr; b.n_windows = cw;
    if (mode) b.cspec += (size_t) w0 * b.n_bins;
    else      b.psd += (size_t) w0 * fs.N;
    e->span_begin(FAM_COLS, lc.stream);
    if (f5) CK(sdb_launch_cols128(lc, fs, a, w0, cw));
    else    CK(sdb_launch_pass_a_range(lc, fs, a, w0, cw));
    e->span_end(lc.stream);
    e->span_begin(fam_b, lc.stream);
    if (f5) CK(sdb_launch_rows256(lc, fs, b, mode));
    else    CK(sdb_launch_pass_b(lc, fs, b, mode));
    e->span_end(lc.stream);
    return 0;
  };

  // Stream groups: G whole streams per step, PSD frames on psd_stream and channeliser windows on the main stream,
  // each with its own part of the pinned scratch (G * (frames + wps) windows <= chunk_windows).  The largest group
  // that fits the pinned scratch is the fastest (cfg2, 2048 streams: 12 streams 64.7 GS/s, 9 streams -- whole waves
  // for either kernel alone -- 63.1, 8: 60.2, 6: 54.2; the two chains overlap, so wave quantisation of a single
  // launch does not matter).
  const int G = p.psd_stream && wps > 0 ? std::min(p.chunk_windows / (frames + wps), (int) S) : 0;
  if (G >= 1) {
    // timing mode (sdb_engine_timing): every kernel on the main stream, so that the CUDA-event spans are the
    // kernels' own durations and not those of two chains sharing the SMs
    SdbLaunchCtx pctx{ e->timing ? e->stream.get() : p.psd_stream.get(), &e->launches };
    CK(p.ev_feed.record(e->stream));              // the input is valid from here on
    CK(p.ev_feed.wait_on(p.psd_stream));
    CK(sl.psd_read.wait_on(p.psd_stream));        // async read of feed i-2
    float2 *scr_psd = p.d_scratch, *scr_ch = p.d_scratch + (size_t) G * frames * Np;
    for (int s0 = 0; s0 < (int) S; s0 += G) {
      const int g = std::min(G, (int) S - s0);
      if (chunk(pctx, p.fs_psd, psd_a, psd_b, FAM_ROWS_PSD, s0 * frames, g * frames, scr_psd)) return -1;
      if (chunk(ctx, p.fs_st, chan_a, chan_b, FAM_ROWS_CHAN, s0 * wps, g * wps, scr_ch)) return -1;
    }
    if (p.chdet) CK(sdb_chdet_feed_stream(p.chdet.get(), sl.psd, (uint32_t) frames, (size_t) frames * Np, p.psd_stream,
                                          &e->launches));
    if (p.chtrack && chan_track(p.psd_stream)) return -1;
    if (frame_groups(pctx)) return -1;
    CK(sl.psd_ready.record(p.psd_stream));
    CK(sl.psd_ready.wait_on(e->stream));          // the main stream stays the engine's timeline
  } else {
    CK(sl.psd_read.wait_on(e->stream));           // async read of feed i-2
    // ---- cluster-path PSD frames and channeliser windows: one launch, both passes fused, ordered by stream
    const bool fused_psd = Np && p.fs_psd.path == SDB_FFT_CLUSTER, fused_chan = K && p.fs_st.path == SDB_FFT_CLUSTER;
    if ((fused_psd && frames > 0) || (fused_chan && wps > 0)) {
      const SdbFourStep &fs = fused_psd ? p.fs_psd : p.fs_st;
      SdbFft65536Args f{};
      f.x = x; f.fmt = fmt; f.stream_stride = stride; f.n_streams = (int) S;
      f.n_psd = fused_psd ? frames : 0; f.n_chan = fused_chan ? wps : 0; f.first_chan = first;
      f.window = p.d_window; f.psd = sl.psd; f.inv_n = 1.0f / (float) fs.N; f.shift_db = shift_db;
      f.hist = p.d_hist; f.binmap = p.d_binmap; f.cspec = p.d_cspec; f.n_bins = p.n_bins; f.ka_mask = p.ka_mask;
      e->span_begin(FAM_COLS);
      CK(sdb_launch_fft65536(ctx, fs, f));
      e->span_end();
    }
    // ---- main PSD
    if (Np) {
      if (p.fs_psd.path == SDB_FFT_SMALL_PSD) {
        e->span_begin(FAM_ROWS_PSD);
        CK(sdb_launch_small_psd(ctx, (int) Np, p.fs_psd.twN, x, fmt, stride, frames, (int) S, p.d_window,
                                sl.psd, shift_db));
        e->span_end();
      } else if (!fused_psd) {
        const int total = frames * (int) S;
        for (int w0 = 0; w0 < total; w0 += p.chunk_windows)
          if (chunk(ctx, p.fs_psd, psd_a, psd_b, FAM_ROWS_PSD, w0, std::min(p.chunk_windows, total - w0),
                    p.d_scratch)) return -1;
      }
      if (p.chdet) CK(sdb_chdet_feed_stream(p.chdet.get(), sl.psd, (uint32_t) frames, (size_t) frames * Np, e->stream,
                                            &e->launches));
      if (p.chtrack && chan_track(e->stream)) return -1;
      if (frame_groups(ctx)) return -1;
      CK(sl.psd_ready.record(e->stream));
    }
    // ---- channeliser forward transforms
    if (K && wps > 0 && !fused_chan) {
      const int total = wps * (int) S;
      for (int w0 = 0; w0 < total; w0 += p.chunk_windows)
        if (chunk(ctx, p.fs_st, chan_a, chan_b, FAM_ROWS_CHAN, w0, std::min(p.chunk_windows, total - w0),
                  p.d_scratch)) return -1;
    }
  }
  // ---- per-channel inverse transforms + inspectors
  if (K) {
    p.last_hops = wps > 0 ? wps : 0;
    if (wps > 0) {
      CK(sl.insp.wait_on(e->stream));             // the slot was last read by the inspector launch of feed i-2
      e->span_begin(FAM_CHAN_IFFT);
      for (auto &g : p.groups)
        CK(sdb_launch_chan_ifft_group(ctx, p.d_chans, g.d_ids, g.len, g.size, K, (int) S, p.d_cspec,
                                      p.n_bins, wps, p.d_tails, p.tail_stride, p.d_lo_phase, sl.chan,
                                      p.chan_stride, g.any_precise));
      e->span_end();
      CK(p.ev_chan.record(e->stream));
      CK(p.ev_chan.wait_on(p.insp_stream));
      CK(sl.sym_read.wait_on(p.insp_stream));
      SdbLaunchCtx ictx{ e->timing ? e->stream.get() : p.insp_stream.get(), &e->launches };
      if (p.d_spectcfg)
        CK(sdb_launch_spectsrc(ictx, p.d_spectcfg, p.d_chans, K, (int) S, p.spect_max_ns, sl.chan,
                               p.chan_stride, (uint32_t) wps, p.d_spect, p.spect_stride, p.d_spect_size,
                               p.d_est, p.d_est_valid));
      if (!p.sched.empty() && sched_feed(e, p, sl, ictx, (uint64_t) wps)) return -1;
      if (!p.insp_grids.empty()) {                // (every channel a power inspector: no chain)
        e->span_begin(FAM_INSPECTOR, ictx.stream);
        for (const SdbInspGrid &g : p.insp_grids)
          CK(sdb_launch_inspectors_n(ictx, g, p.d_cfg, K, (int) S, p.d_chain_map, p.d_state, p.d_pool, p.pool_stride,
                                     p.d_taps, p.d_chans, sl.chan, p.chan_stride, (uint32_t) wps, sl.soft, sl.hard,
                                     sl.counts, p.sym_cap, 0));
        e->span_end(ictx.stream);
      }
      if (p.n_power) {
        e->span_begin(FAM_POWER, ictx.stream);
        CK(sdb_launch_power_integrate(ictx, p.d_power, p.n_power, sl.chan, (uint32_t) wps, p.power_carry, sl.soft,
                                      sl.hard, sl.counts, p.sym_cap));
        e->span_end(ictx.stream);
      }
      if (fac_feed(e, p, sl, ictx)) return -1;
      if (snr_feed(e, p, sl, ictx)) return -1;
      if (tv_feed(e, p, sl, ictx)) return -1;
      CK(sl.insp.record(ictx.stream));
    } else {
      std::fill(sl.sched_n.begin(), sl.sched_n.end(), 0u);   // no channel samples: no emission
      CK(sl.sym_read.wait_on(p.insp_stream));
      CK(cudaMemsetAsync(sl.counts, 0, (size_t) S * K * sizeof(uint32_t), p.insp_stream));
      if (fac_feed(e, p, sl, SdbLaunchCtx{ p.insp_stream.get(), &e->launches })) return -1;   // (a status of no blocks)
      if (snr_feed(e, p, sl, SdbLaunchCtx{ p.insp_stream.get(), &e->launches })) return -1;   // (a status of no step)
      if (tv_feed(e, p, sl, SdbLaunchCtx{ p.insp_stream.get(), &e->launches })) return -1;    // (no frame completed)
      CK(sl.insp.record(p.insp_stream));
    }
    // keep the last half window of every stream as history for the next feed
    if (fmt == SDB_FMT_F32)
      CK(cudaMemcpy2DAsync(p.d_hist, (W / 2) * sizeof(float2), reinterpret_cast<const float2 *>(x) + (n - W / 2),
                           stride * sizeof(float2), (W / 2) * sizeof(float2), S, cudaMemcpyDeviceToDevice, e->stream));
    else
      CK(sdb_launch_hist_convert(e->stream, x, fmt, stride, n - W / 2, p.d_hist, (int) (W / 2), (int) S));
    p.first_feed = false;
  }
  ++p.feed_index;
  p.n_fed += n;
  return 0;
}

extern "C" int sdb_engine_feed_host(sdb_engine_t *e, const sdb_complex *x, size_t stride, size_t n)
{
  if (!e || !x) return fail("null argument");
  if (!e->plan) return fail("engine not committed");
  Plan &p = *e->plan;
  if (n == 0 || n > e->prm.max_feed) return fail("feed size out of range");
  CK(cudaSetDevice(e->prm.device));
  const unsigned S = e->prm.n_streams;
  Plan::Stage &sg = p.stage[p.host_feeds & 1u];
  const size_t bps = sdb_fmt_bytes(e->prm.input_format);
  if (!sg.xin.size() && sg.xin.alloc((size_t) S * e->prm.max_feed) != cudaSuccess)
    return fail("out of device memory (input staging)");
  // H2D on its own stream into this staging buffer, as soon as the kernels of host feed i-2 are done with it;
  // the kernels of this feed wait for the copy.  Copies of consecutive feeds overlap compute.
  CK(sg.xfree.wait_on(p.h2d_stream));
  if (stride == n)
    CK(cudaMemcpyAsync(sg.xin, x, (size_t) S * n * bps, cudaMemcpyHostToDevice, p.h2d_stream));
  else
    CK(cudaMemcpy2DAsync(sg.xin, n * bps, x, stride * bps, n * bps, S, cudaMemcpyHostToDevice, p.h2d_stream));
  CK(p.ev_h2d.record(p.h2d_stream));
  CK(p.ev_h2d.wait_on(e->stream));
  int rc = sdb_engine_feed_device(e, reinterpret_cast<const sdb_complex *>(sg.xin.get()), n, n);
  if (rc) return rc;
  CK(sg.xfree.record(e->stream));
  ++p.host_feeds;
  return 0;
}

extern "C" int sdb_engine_sync(sdb_engine_t *e)
{
  if (!e) return fail("null engine");
  CK(cudaSetDevice(e->prm.device));
  CK(e->join());
  CK(cudaStreamSynchronize(e->stream));
  if (e->plan) {
    CK(cudaStreamSynchronize(e->plan->d2h_stream));
    CK(cudaStreamSynchronize(e->plan->h2d_stream));
  }
  e->collect_spans();
  return 0;
}

// Queue a dependency: work submitted to the engine stream after this call starts only once the
// inspector kernels of all previous feeds have finished (they run on a second stream so that the
// next feed's FFT kernels overlap them).  Use before recording an event that should cover a feed.
extern "C" int sdb_engine_join(sdb_engine_t *e)
{
  if (!e) return fail("null engine");
  CK(cudaSetDevice(e->prm.device));
  CK(e->join());
  return 0;
}

extern "C" size_t sdb_engine_psd_frames(const sdb_engine_t *e) { return e && e->plan ? e->plan->last_frames : 0; }
extern "C" const float *sdb_engine_psd_device(const sdb_engine_t *e) { return e && e->plan ? e->plan->cur().psd : nullptr; }

extern "C" int sdb_engine_read_psd(sdb_engine_t *e, float *dst, size_t cap)
{
  if (!e || !dst) return fail("null argument");
  if (sdb_engine_read_psd_async(e, dst, cap)) return -1;
  CK(cudaStreamSynchronize(e->plan->d2h_stream));
  return 0;
}

extern "C" size_t sdb_engine_psd_average_frames(const sdb_engine_t *e) { return e && e->plan ? e->plan->avg.last : 0; }
extern "C" const float *sdb_engine_psd_average_device(const sdb_engine_t *e)
{
  return e && e->plan ? e->plan->avg.out[e->plan->cur_parity()][0].get() : nullptr;
}

extern "C" int sdb_engine_read_psd_average(sdb_engine_t *e, float *dst, size_t cap)
{
  if (!e || !dst) return fail("null argument");
  return groups_read(e, e->plan ? &e->plan->avg : nullptr, dst, nullptr, cap, "PSD averaging not enabled");
}

extern "C" size_t sdb_engine_psd_peak_groups(const sdb_engine_t *e) { return e && e->plan ? e->plan->peak.last : 0; }
extern "C" const float *sdb_engine_psd_peak_device(const sdb_engine_t *e, int which)
{
  if (!e || !e->plan || (which != 0 && which != 1)) return nullptr;
  return e->plan->peak.out[e->plan->cur_parity()][which].get();
}

extern "C" int sdb_engine_read_psd_peak(sdb_engine_t *e, float *max_dst, float *min_dst, size_t cap)
{
  if (!e) return fail("null argument");
  return groups_read(e, e->plan ? &e->plan->peak : nullptr, max_dst, min_dst, cap, "PSD peak detection not enabled");
}

// Asynchronous variants: the copy is queued on the engine's D2H stream behind the kernels that produce
// the data; the next feed may be submitted immediately (results are double-buffered by feed parity, a
// buffer is reused two feeds later and its writer waits for this copy).  dst should be pinned memory and
// must stay valid until sdb_engine_sync().
extern "C" int sdb_engine_read_psd_async(sdb_engine_t *e, float *dst, size_t cap)
{
  if (!e || !dst) return fail("null argument");
  if (!e->plan || !e->Np || e->plan->feed_index == 0) return fail("no PSD available");
  Plan &p = *e->plan;
  const size_t n = (size_t) e->prm.n_streams * p.last_frames * e->Np;
  if (cap < n) return fail("destination too small");
  Slot &sl = p.cur();
  CK(cudaSetDevice(e->prm.device));
  CK(sl.psd_ready.wait_on(p.d2h_stream));
  CK(cudaMemcpyAsync(dst, sl.psd, n * sizeof(float), cudaMemcpyDeviceToHost, p.d2h_stream));
  CK(sl.psd_read.record(p.d2h_stream));
  return 0;
}

extern "C" long sdb_engine_read_channel(sdb_engine_t *e, uint32_t stream, int handle, sdb_complex *dst, size_t cap)
{
  if (!e || !dst) return fail("null argument");
  if (handle < 0 || handle >= (int) e->channels.size()) return fail("wrong handle");
  if (stream >= e->prm.n_streams) return fail("stream out of range");
  if (!e->plan) return fail("engine not committed");
  Plan &p = *e->plan;
  const SdbChannelDev &d = p.h_chans[handle];
  size_t n = p.last_hops * (size_t) d.halfsz;
  if (n > cap) n = cap;
  CK(cudaSetDevice(e->prm.device));
  CK(cudaMemcpyAsync(dst, p.cur().chan + (size_t) stream * p.chan_stride + d.out_off, n * sizeof(float2),
                     cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return (long) n;
}

extern "C" long sdb_engine_read_symbols(sdb_engine_t *e, uint32_t stream, int handle, sdb_complex *soft,
                                        uint8_t *hard, size_t cap)
{
  if (!e) return fail("null argument");
  const int K = (int) e->channels.size();
  if (handle < 0 || handle >= K) return fail("wrong handle");
  if (stream >= e->prm.n_streams) return fail("stream out of range");
  if (!e->plan) return fail("engine not committed");
  Plan &p = *e->plan;
  const Slot &sl = p.cur();
  const size_t chain = (size_t) stream * K + handle;
  uint32_t cnt = 0;
  CK(cudaSetDevice(e->prm.device));
  CK(e->join());
  CK(cudaMemcpyAsync(&cnt, sl.counts + chain, sizeof(cnt), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  size_t n = cnt;
  if (n > cap) n = cap;
  if (soft) CK(cudaMemcpyAsync(soft, sl.soft + chain * p.sym_cap, n * sizeof(float2), cudaMemcpyDeviceToHost, e->stream));
  if (hard) CK(cudaMemcpyAsync(hard, sl.hard + chain * p.sym_cap, n, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return (long) n;
}

extern "C" int sdb_engine_read_all_symbols(sdb_engine_t *e, uint32_t *counts, sdb_complex *soft, uint8_t *hard,
                                           size_t cap)
{
  if (!e || !counts) return fail("null argument");
  const size_t chains = (size_t) e->prm.n_streams * e->channels.size();
  if (chains == 0) return 0;
  if (sdb_engine_read_all_symbols_async(e, counts, soft, hard, cap)) return -1;
  CK(cudaStreamSynchronize(e->plan->d2h_stream));
  return 0;
}

extern "C" int sdb_engine_read_all_symbols_async(sdb_engine_t *e, uint32_t *counts, sdb_complex *soft,
                                                 uint8_t *hard, size_t cap)
{
  if (!e || !counts) return fail("null argument");
  const size_t chains = (size_t) e->prm.n_streams * e->channels.size();
  if (chains == 0) return 0;
  if (!e->plan || e->plan->feed_index == 0) return fail("no symbols available");
  Plan &p = *e->plan;
  Slot &sl = p.cur();
  CK(cudaSetDevice(e->prm.device));
  // everything queued so far on the inspector stream (including this feed's launch or its count reset)
  CK(sl.insp.wait_on(p.d2h_stream));
  CK(cudaMemcpyAsync(counts, sl.counts, chains * sizeof(uint32_t), cudaMemcpyDeviceToHost, p.d2h_stream));
  const size_t w = std::min(cap, p.sym_cap);
  if (soft) CK(cudaMemcpy2DAsync(soft, cap * sizeof(float2), sl.soft, p.sym_cap * sizeof(float2),
                                 w * sizeof(float2), chains, cudaMemcpyDeviceToHost, p.d2h_stream));
  if (hard) CK(cudaMemcpy2DAsync(hard, cap, sl.hard, p.sym_cap, w, chains, cudaMemcpyDeviceToHost, p.d2h_stream));
  CK(sl.sym_read.record(p.d2h_stream));
  return 0;
}

// destination of a device-written read: device memory as is, pinned / registered host memory through its device
// alias; anything else cannot be written by a kernel and is refused
static int device_writable(void *p, void **dev, const char *what)
{
  *dev = nullptr;
  if (!p) return 0;
  if (((uintptr_t) p & 15u) != 0) return fail(std::string("packed symbol read: ") + what + " must be 16-byte aligned");
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return fail(std::string("packed symbol read: ") + what + " is not pinned host or device memory"); }
  if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) { *dev = p; return 0; }
  if (at.type == cudaMemoryTypeHost && at.devicePointer) { *dev = at.devicePointer; return 0; }
  return fail(std::string("packed symbol read: ") + what + " must be pinned (cudaHostAlloc / cudaHostRegister) host "
              "memory or device memory: the GPU writes it directly");
}

extern "C" int sdb_engine_read_symbols_packed_async(sdb_engine_t *e, uint32_t *counts, uint64_t *offsets,
                                                    sdb_complex *soft, uint8_t *hard, size_t cap_total)
{
  if (!e || !counts || !offsets) return fail("null argument");
  const size_t chains = (size_t) e->prm.n_streams * e->channels.size();
  if (chains == 0) return 0;
  if (!e->plan || e->plan->feed_index == 0) return fail("no symbols available");
  Plan &p = *e->plan;
  Slot &sl = p.cur();
  CK(cudaSetDevice(e->prm.device));
  void *dsoft = nullptr, *dhard = nullptr;
  if (device_writable(soft, &dsoft, "soft") || device_writable(hard, &dhard, "hard")) return -1;
  if (!sl.sym_off.size() && sl.sym_off.alloc(chains + 1) != cudaSuccess)
    return fail("out of device memory (symbol offsets)");
  CK(sl.insp.wait_on(p.d2h_stream));
  CK(sdb_launch_sym_pack(p.d2h_stream, sl.counts, sl.sym_off, chains, sl.soft, sl.hard,
                         p.sym_cap, dsoft, dhard, (unsigned long long) cap_total, &e->launches));
  CK(cudaMemcpyAsync(counts, sl.counts, chains * sizeof(uint32_t), cudaMemcpyDeviceToHost, p.d2h_stream));
  CK(cudaMemcpyAsync(offsets, sl.sym_off, (chains + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, p.d2h_stream));
  CK(sl.sym_read.record(p.d2h_stream));
  return 0;
}

extern "C" int sdb_engine_read_symbols_packed(sdb_engine_t *e, uint32_t *counts, uint64_t *offsets, sdb_complex *soft,
                                              uint8_t *hard, size_t cap_total)
{
  if (sdb_engine_read_symbols_packed_async(e, counts, offsets, soft, hard, cap_total)) return -1;
  if (e->plan) CK(cudaStreamSynchronize(e->plan->d2h_stream));   // (no chains: an engine may read before its commit)
  return 0;
}

extern "C" const uint32_t *sdb_engine_symbol_counts_device(const sdb_engine_t *e)
{
  return e && e->plan ? e->plan->cur().counts : nullptr;
}
extern "C" size_t sdb_engine_symbol_capacity(const sdb_engine_t *e) { return e && e->plan ? e->plan->sym_cap : 0; }
extern "C" void *sdb_engine_stream(const sdb_engine_t *e) { return e ? (void *) e->stream.get() : nullptr; }
extern "C" uint64_t sdb_engine_launch_count(const sdb_engine_t *e) { return e ? e->launches : 0; }
extern "C" void sdb_engine_timing(sdb_engine_t *e, int enable)
{
  if (!e) return;
  e->timing = enable != 0;
  for (int i = 0; i < FAM_COUNT; ++i) { e->fam_ms[i] = 0; e->fam_n[i] = 0; }
}

extern "C" int sdb_engine_kernel_time(sdb_engine_t *e, const char *family, double *avg_ms, uint64_t *launches)
{
  if (!e || !family) return fail("null argument");
  for (int i = 0; i < FAM_COUNT; ++i)
    if (!strcmp(family, kFamNames[i])) {
      if (avg_ms) *avg_ms = e->fam_n[i] ? e->fam_ms[i] / (double) e->fam_n[i] : 0.0;
      if (launches) *launches = e->fam_n[i];
      return 0;
    }
  return fail("unknown kernel family");
}

// ---- take over the running state of another engine (live re-plan: suscan keeps every inspector that stays open
// ---- running when one is opened, closed or reconfigured, Suscan/Analyzer.cpp:459-537).  Channels are matched by
// ---- their parameters (f0, bw, guard, precise), first come first served: a matched channel keeps its cross-fade
// ---- tail and LO phase; if its inspector class and the sizes of its state lines are unchanged it also keeps the
// ---- loop state of every chain (AGC, Costas / PLL, matched-filter line, Gardner, CMA...), whatever else of its
// ---- configuration changed (loop bandwidths, gains, thresholds take effect at this block boundary).
// SPEC SN.4: a channel that keeps its inspector class and L keeps h, the model and the state while its inspector
// configuration is unchanged field by field; otherwise h is cleared (the new plan's h is empty) and sigma kept, and it
// restarts at 1/8 when bps changed.  alpha is the new descriptor's.  Anything else keeps the new plan's fresh start.
static bool same_inspector_config(const sdb_inspector_config &a, const sdb_inspector_config &b)
{
  return !memcmp(&a, &b, offsetof(sdb_inspector_config, eq_locked) + sizeof a.eq_locked) &&
         a.power_integrate_samples == b.power_integrate_samples;
}

static int snr_migrate(Plan &to, const Plan &from, const Channel &cn, const Channel &co, int kn, int ko, unsigned S)
{
  const int qn = to.snr.first.empty() ? -1 : to.snr.first[kn], qo = from.snr.first.empty() ? -1 : from.snr.first[ko];
  if (qn < 0 || qo < 0 || cn.cfg.insp_class != co.cfg.insp_class || cn.snr.bins != co.snr.bins) return 0;
  const SdbSnrChan &hn = to.snr.h[qn], &ho = from.snr.h[qo];
  std::vector<sdb_snr_status> st(S);
  CK(cudaMemcpy(st.data(), from.snr.status.get() + ho.chain0, S * sizeof(sdb_snr_status), cudaMemcpyDeviceToHost));
  if (same_inspector_config(cn.cfg, co.cfg)) {
    const size_t n = (size_t) S * hn.L;
    CK(cudaMemcpy(to.snr.hist.get() + hn.hist_off, from.snr.hist.get() + ho.hist_off, n * sizeof(uint32_t),
                  cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(to.snr.model.get() + hn.hist_off, from.snr.model.get() + ho.hist_off, n * sizeof(float),
                  cudaMemcpyDeviceToDevice));
  } else {
    std::vector<sdb_snr_status> fresh(S);
    CK(cudaMemcpy(fresh.data(), to.snr.status.get() + hn.chain0, S * sizeof(sdb_snr_status), cudaMemcpyDeviceToHost));
    const bool bps_changed = cn.cfg.bits_per_symbol != co.cfg.bits_per_symbol;
    for (unsigned s = 0; s < S; ++s) {
      const float sigma = bps_changed ? 1.f / 8.f : st[s].sigma;
      st[s] = fresh[s];
      st[s].sigma = sigma; st[s].snr = 1.0f / (hn.K * sigma);
    }
  }
  CK(cudaMemcpy(to.snr.status.get() + hn.chain0, st.data(), S * sizeof(sdb_snr_status), cudaMemcpyHostToDevice));
  return 0;
}

// SPEC TI.5: a channel that keeps its class and the picture geometry keeps the whole processor; its new descriptor
// (parameters, invert_sync, dc) applies from the next feed
static int tv_migrate(Plan &to, const Plan &from, const Channel &cn, const Channel &co, int kn, int ko, unsigned S)
{
  const int qn = to.tv.first.empty() ? -1 : to.tv.first[kn], qo = from.tv.first.empty() ? -1 : from.tv.first[ko];
  if (qn < 0 || qo < 0 || cn.cfg.insp_class != co.cfg.insp_class || !sdb_tv_same_geometry(cn.tv.tv, co.tv.tv)) return 0;
  const SdbTvInspChan &hn = to.tv.h[qn], &ho = from.tv.h[qo];
  const size_t px = (size_t) hn.c.H * hn.c.W;
  CK(cudaMemcpy(to.tv.state.get() + hn.chain0, from.tv.state.get() + ho.chain0, S * sizeof(SdbTvState),
                cudaMemcpyDeviceToDevice));
  CK(cudaMemcpy(to.tv.status.get() + hn.chain0, from.tv.status.get() + ho.chain0, S * sizeof(sdb_tv_status),
                cudaMemcpyDeviceToDevice));
  CK(cudaMemcpy(to.tv.delay.get() + hn.delay_off, from.tv.delay.get() + ho.delay_off,
                (size_t) S * hn.c.delay_len * sizeof(float), cudaMemcpyDeviceToDevice));
  CK(cudaMemcpy(to.tv.line.get() + hn.line_off, from.tv.line.get() + ho.line_off, (size_t) S * hn.c.W * sizeof(float),
                cudaMemcpyDeviceToDevice));
  CK(cudaMemcpy(to.tv.ring.get() + hn.ring_off, from.tv.ring.get() + ho.ring_off, S * SDB_TV_RING * px * sizeof(float),
                cudaMemcpyDeviceToDevice));
  CK(cudaMemcpy(to.tv.post.get() + hn.post_off, from.tv.post.get() + ho.post_off, S * px * sizeof(float),
                cudaMemcpyDeviceToDevice));
  return 0;
}

static int migrate_impl(sdb_engine_t *dst, sdb_engine_t *src, const std::vector<int> &old_of_new)
{
  CK(cudaSetDevice(dst->prm.device));
  if (sdb_engine_sync(src)) return -1;
  Plan &to = *dst->plan;
  const Plan &from = *src->plan;
  const unsigned S = dst->prm.n_streams, W = dst->W;
  const int Kn = (int) dst->channels.size(), Ko = (int) src->channels.size();
  if (to.d_hist && from.d_hist)
    CK(cudaMemcpy(to.d_hist, from.d_hist, (size_t) S * (W / 2) * sizeof(float2), cudaMemcpyDeviceToDevice));
  if (to.d_dc_state && from.d_dc_state)
    CK(cudaMemcpy(to.d_dc_state, from.d_dc_state, S * sizeof(float2), cudaMemcpyDeviceToDevice));
  // the partial SPEC A and SPEC PK groups
  if (groups_migrate(to.avg, from.avg, dst, src) || groups_migrate(to.peak, from.peak, dst, src)) return -1;
  // an engine that had no channel so far kept no input history: its first window starts with this feed
  to.first_feed = from.d_hist ? from.first_feed : true;
  to.n_fed = from.n_fed;
  auto slot_of = [](const Plan &p, int chain_g) {
    for (size_t q = 0; q < p.h_chain_map.size(); ++q) if (p.h_chain_map[q] == chain_g) return (long) q;
    return -1L;
  };
  for (int kn = 0; kn < Kn; ++kn) {
    const int ko = kn < (int) old_of_new.size() ? old_of_new[kn] : -1;
    if (ko < 0 || ko >= Ko) continue;
    const Channel &cn = dst->channels[kn], &co = src->channels[ko];
    const SdbChannelDev &dn = to.h_chans[kn], &dold = from.h_chans[ko];
    const bool same_channel = co.p.f0 == cn.p.f0 && co.p.bw == cn.p.bw && co.p.guard == cn.p.guard &&
                              co.p.precise == cn.p.precise && co.size == cn.size && co.center == cn.center;
    if (same_channel && !from.first_feed) {
      CK(cudaMemcpy2D(to.d_tails + dn.tail_off, to.tail_stride * sizeof(float2), from.d_tails + dold.tail_off,
                      from.tail_stride * sizeof(float2), (size_t) cn.halfsz * sizeof(float2), S, cudaMemcpyDeviceToDevice));
      CK(cudaMemcpy2D(to.d_lo_phase + kn, (size_t) Kn * sizeof(float), from.d_lo_phase + ko, (size_t) Ko * sizeof(float),
                      sizeof(float), S, cudaMemcpyDeviceToDevice));
      // SPEC US: the channel's sample count and ring go on while both schedule it with the same Ns, whatever its
      // kind, estimators or interval
      const int qn = sched_index(to, kn), qo = sched_index(from, ko);
      if (qn >= 0 && qo >= 0 && to.sched[qn].ns == from.sched[qo].ns) {
        const SdbSchedChan &hn = to.h_sched[qn], &ho = from.h_sched[qo];
        CK(cudaMemcpy2D(to.d_ring.get() + hn.ring_off, to.ring_stride * sizeof(float2), from.d_ring.get() + ho.ring_off,
                        from.ring_stride * sizeof(float2), (size_t) hn.ns1 * sizeof(float2), S, cudaMemcpyDeviceToDevice));
        to.sched[qn].t = from.sched[qo].t; to.sched[qn].v = from.sched[qo].v;
      }
    }
    // SPEC FC: the FAC goes on while the channel keeps its inspector class, block size and channel rate
    const int fn = to.fac.first.empty() ? -1 : to.fac.first[kn], fo = from.fac.first.empty() ? -1 : from.fac.first[ko];
    if (fn >= 0 && fo >= 0 && cn.cfg.insp_class == co.cfg.insp_class && cn.fac.size == co.fac.size &&
        cn.cfg.fs == co.cfg.fs) {
      const size_t L = cn.fac.size;
      CK(cudaMemcpy(to.fac.state.get() + fn, from.fac.state.get() + fo, S * sizeof(SdbFacState), cudaMemcpyDeviceToDevice));
      CK(cudaMemcpy(to.fac.blk.get() + to.fac.h[fn].blk_off, from.fac.blk.get() + from.fac.h[fo].blk_off,
                    S * L * sizeof(float2), cudaMemcpyDeviceToDevice));
      CK(cudaMemcpy(to.fac.fac.get() + to.fac.h[fn].fac_off, from.fac.fac.get() + from.fac.h[fo].fac_off,
                    S * (L / 2) * sizeof(float), cudaMemcpyDeviceToDevice));
    }
    if (snr_migrate(to, from, cn, co, kn, ko, S)) return -1;
    if (tv_migrate(to, from, cn, co, kn, ko, S)) return -1;
    if (!cn.has_insp || !co.has_insp) continue;
    if (is_power(cn) || is_power(co)) {
      // SPEC PW: the partial group goes on while the inspector stays a power inspector with the same M
      if (is_power(cn) && is_power(co) && power_m(cn.cfg) == power_m(co.cfg))
        CK(cudaMemcpy2D(to.power_carry + kn, (size_t) Kn * sizeof(SdbPowerCarry), from.power_carry + ko,
                        (size_t) Ko * sizeof(SdbPowerCarry), sizeof(SdbPowerCarry), S, cudaMemcpyDeviceToDevice));
      continue;
    }
    const SdbChainCfg &a = to.h_cfg[kn], &b = from.h_cfg[ko];
    if (a.cls != b.cls || a.have_agc != b.have_agc || a.dl_size != b.dl_size || a.mh_size != b.mh_size ||
        a.have_mf != b.have_mf || a.mf_n != b.mf_n || a.af_n != b.af_n || a.alpf_n != b.alpf_n ||
        a.have_costas != b.have_costas || a.have_pll != b.have_pll || a.eq_type != b.eq_type ||
        a.clock_type != b.clock_type)
      continue;                                            // structural change: this inspector restarts
    CK(cudaMemcpy2D(to.d_state + kn, (size_t) Kn * sizeof(SdbChainState), from.d_state + ko,
                    (size_t) Ko * sizeof(SdbChainState), sizeof(SdbChainState), S, cudaMemcpyDeviceToDevice));
    // clock.baud is a parameter AND the start value of the Gardner loop's own estimate: a new baud restarts it
    if (a.bnor != b.bnor) {
      std::vector<SdbChainState> st(S);
      CK(cudaMemcpy2D(st.data(), sizeof(SdbChainState), to.d_state + kn, (size_t) Kn * sizeof(SdbChainState),
                      sizeof(SdbChainState), S, cudaMemcpyDeviceToHost));
      for (auto &q : st) q.k_bnor = a.bnor;
      CK(cudaMemcpy2D(to.d_state + kn, (size_t) Kn * sizeof(SdbChainState), st.data(), sizeof(SdbChainState),
                      sizeof(SdbChainState), S, cudaMemcpyHostToDevice));
    }
    const size_t rows = (size_t) std::min(a.st_pool, b.st_pool);
    for (unsigned s = 0; s < S; ++s) {
      const long qn = slot_of(to, kn * (int) S + (int) s), qo = slot_of(from, ko * (int) S + (int) s);
      if (qn < 0 || qo < 0) continue;
      float *pd = to.d_pool + (size_t) (qn / 32) * 32 * to.pool_stride + (qn % 32);
      const float *ps = from.d_pool + (size_t) (qo / 32) * 32 * from.pool_stride + (qo % 32);
      CK(cudaMemcpy2D(pd, 32 * sizeof(float), ps, 32 * sizeof(float), sizeof(float), rows, cudaMemcpyDeviceToDevice));
    }
  }
  return 0;
}

static int migrate_check(sdb_engine_t *dst, sdb_engine_t *src)
{
  if (!dst || !src) return fail("null engine");
  if (!dst->plan || !src->plan) return fail("both engines must be committed");
  if (dst->prm.n_streams != src->prm.n_streams || dst->W != src->W || dst->prm.device != src->prm.device)
    return fail("engines differ in streams / window / device");
  return 0;
}

// can dst continue src (same streams, window, device)?  PSD size, window function, flags and feed size may differ
extern "C" int sdb_engine_same_geometry(const sdb_engine_t *a, const sdb_engine_t *b)
{
  return a && b && a->prm.n_streams == b->prm.n_streams && a->W == b->W && a->prm.device == b->prm.device;
}

extern "C" int sdb_engine_migrate(sdb_engine_t *dst, sdb_engine_t *src)
{
  if (migrate_check(dst, src)) return -1;
  const int Kn = (int) dst->channels.size(), Ko = (int) src->channels.size();
  std::vector<int> map(Kn, -1);
  std::vector<char> used(Ko, 0);
  for (int kn = 0; kn < Kn; ++kn) {
    const Channel &cn = dst->channels[kn];
    for (int k = 0; k < Ko; ++k) {
      const Channel &co = src->channels[k];
      if (!used[k] && co.p.f0 == cn.p.f0 && co.p.bw == cn.p.bw && co.p.guard == cn.p.guard &&
          co.p.precise == cn.p.precise) { map[kn] = k; used[k] = 1; break; }
    }
  }
  return migrate_impl(dst, src, map);
}

extern "C" int sdb_engine_migrate_map(sdb_engine_t *dst, sdb_engine_t *src, const int32_t *old_of_new, size_t n)
{
  if (migrate_check(dst, src)) return -1;
  if (!old_of_new && n) return fail("null map");
  std::vector<int> map(old_of_new, old_of_new + n);
  return migrate_impl(dst, src, map);
}

// Offline inspector over `batch` captured channel-rate buffers (what the GUI's TimeWindow / SamplerDialog
// do block-wise on the CPU, Components/TimeWindow.cpp:1571-2183): one GPU chain per buffer.
extern "C" long sdb_task_inspector(const sdb_inspector_config *cfg, const sdb_complex *src, size_t n,
                                   size_t batch, sdb_complex *soft, uint8_t *hard, uint32_t *counts, size_t cap)
{
  if (!cfg || !src || !counts || n == 0 || batch == 0) return fail("invalid argument");
  if (cfg->insp_class == SDB_INSP_POWER) return fail("invalid inspector configuration: the power class has no chain");
  if (sdb_device_count() <= 0) return fail("no CUDA device: sigdigger_b200 has no CPU fallback");
  Channel ch; memset(&ch.p, 0, sizeof(ch.p));
  ch.center = 0; ch.size = 2; ch.width = 2; ch.halfw = 1; ch.halfsz = 1; ch.has_insp = true; ch.cfg = *cfg;
  SdbChainCfg c; std::vector<float> taps;
  if (!build_chain_cfg(ch, c, taps)) return fail("invalid inspector configuration");
  const std::vector<SdbChainState> st(batch, chain_layout(c));
  const size_t pool = (size_t) std::max(1, c.st_pool);
  SdbChannelDev cd; memset(&cd, 0, sizeof(cd)); cd.halfsz = 1; cd.out_off = 0;
  std::vector<int> map;
  const int n_ctas = sdb_build_chain_map(&c, 1, (int) batch, map);
  const std::vector<SdbInspGrid> grids = sdb_insp_grids(&c, (int) batch, map);   // (one class: one grid)
  const size_t pool_floats = (size_t) n_ctas * 32 * pool;
  DevBuf<float2> d_src, d_soft; DevBuf<uint8_t> d_hard; DevBuf<uint32_t> d_cnt; DevBuf<SdbChainCfg> d_cfg;
  DevBuf<SdbChainState> d_st; DevBuf<float> d_pool, d_taps; DevBuf<SdbChannelDev> d_cd; DevBuf<int> d_map;
  CK(d_src.alloc(n * batch)); CK(d_soft.alloc(cap * batch)); CK(d_hard.alloc(cap * batch)); CK(d_cnt.alloc(batch));
  CK(d_map.alloc(map.size()));
  CK(cudaMemcpy(d_map, map.data(), map.size() * sizeof(int), cudaMemcpyHostToDevice));
  CK(d_cfg.alloc(1)); CK(d_st.alloc(batch)); CK(d_pool.alloc(pool_floats));
  CK(d_taps.alloc(std::max<size_t>(1, taps.size()))); CK(d_cd.alloc(1));
  CK(cudaMemcpy(d_src, src, n * batch * sizeof(float2), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_cfg, &c, sizeof(c), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_st, st.data(), batch * sizeof(SdbChainState), cudaMemcpyHostToDevice));
  CK(cudaMemset(d_pool, 0, pool_floats * sizeof(float)));
  if (!taps.empty()) CK(cudaMemcpy(d_taps, taps.data(), taps.size() * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_cd, &cd, sizeof(cd), cudaMemcpyHostToDevice));
  SdbLaunchCtx ctx{ 0, nullptr };
  // every chain is "stream s, channel 0"; chan_stream_stride = n
  for (const SdbInspGrid &g : grids)
    CK(sdb_launch_inspectors_n(ctx, g, d_cfg, 1, (int) batch, d_map, d_st, d_pool, pool, d_taps, d_cd, d_src, n,
                               (uint32_t) n, d_soft, d_hard, d_cnt, cap, 1));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(counts, d_cnt, batch * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  if (soft) CK(cudaMemcpy(soft, d_soft, cap * batch * sizeof(float2), cudaMemcpyDeviceToHost));
  if (hard) CK(cudaMemcpy(hard, d_hard, cap * batch, cudaMemcpyDeviceToHost));
  return 0;
}

// channel lists of the last feed, converted to Hz on the device (sdb_engine_read_all_channels without the host)
int sdb_engine_pack_channels_device(sdb_engine_t *e, const double *centers_dev, sdb_detected_channel *out_dev, size_t cap,
                                    int *counts_dev, cudaStream_t st)
{
  if (!e || !e->plan || !e->plan->chdet) return fail("channel detector not enabled");
  CK(sdb_chdet_pack_device(e->plan->chdet.get(), e->samp_rate, centers_dev, out_dev, cap, counts_dev, st));
  return 0;
}
