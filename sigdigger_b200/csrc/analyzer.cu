// analyzer.cu -- suscan-style asynchronous analyzer on top of the engine: a worker thread pulls IQ from a
// source, runs the engine block by block and posts heap-allocated messages on a FIFO that the caller
// drains with sdb_analyzer_read(); requests (open / set id / set config / close / set params) are queued
// and answered in order with messages carrying the caller's req_id.
//
// This is SURVEY.md section 8(a) row a18 + the command half of section 8(b), i.e. what the reference's
// Suscan::Analyzer wrapper drives:
//   suscan_analyzer_new / read / dispose_message / req_halt / destroy   Suscan/Analyzer.cpp:608, :111-115, :63-103, :321, :625-638
//   suscan_analyzer_open_ex_async                                      Suscan/Analyzer.cpp:459-484
//   suscan_analyzer_set_inspector_id_async / _config_async / close     Suscan/Analyzer.cpp:486-537
//   suscan_analyzer_set_params_async                                   Suscan/Analyzer.cpp:219-227
//   open handshake OPEN -> SET_ID                                      Suscan/AnalyzerRequestTracker.cpp:138-157
//   message payload fields                                             Suscan/Messages/PSDMessage.cpp:30-112,
//                                                                      include/Suscan/Messages/SamplesMessage.h:33-59,
//                                                                      Suscan/Messages/InspectorMessage.cpp:28-71
// Differences stated openly: the channel plan is rebuilt at a block boundary whenever an inspector is
// opened, closed or reconfigured, which restarts the loops of the inspectors that stay open (suscan keeps
// them running); one source per analyzer; no estimators / spectrum sources (section 8(f)).
#include "sdb_internal.h"

#include <algorithm>
#include <cmath>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include <sys/time.h>

namespace {

struct Cmd {
  enum Kind { OPEN, SET_ID, SET_CONFIG, CLOSE, SET_PARAMS, SET_SPECTRUM, ESTIMATOR_CMD, SET_IQ_REVERSE, SET_THROTTLE, SET_WATERMARK,
              SET_FREQ, SET_BANDWIDTH, SEEK, SET_HOP_RANGE, SET_REL_BW, SET_BUFFERING, SET_STRATEGY,
              SET_PARTITIONING, SET_HISTORY, REPLAY, SET_DC_REMOVE, SET_FAC, SET_SNR, RESET_SNR, SET_TV } kind;
  double value2 = 0;
  uint32_t req_id = 0;
  uint32_t aux_id = 0; int enabled = 0;       // spectrum source id / estimator id + enable flag
  double value = 0;                           // the request's number: rate, watermark, size, position, frequency...
  int32_t handle = -1;
  int32_t parent = -1;                        // open_ex: handle of the inspector whose channel is the input
  uint32_t inspector_id = 0;
  std::string cls;
  sdb_sigutils_channel channel{};
  int precise = 0;
  sdb_inspector_config cfg{};
  sdb_analyzer_params params{};
  sdb_fac_params fac{};                       // SET_FAC (enabled: on)
  sdb_snr_params snr{};                       // SET_SNR (enabled: on); RESET_SNR: sigma
  sdb_tv_tab_params tv{};                     // SET_TV (enabled: on)
};

struct Insp {
  int32_t handle;
  bool open;
  bool has_id;
  uint32_t inspector_id;
  int cls;
  sdb_sigutils_channel channel;
  int precise;
  sdb_inspector_config cfg;
  int engine_handle;      // handle inside the current engine, -1 if not mapped
  float fs, bandwidth, lo;
  int32_t parent;         // -1 = fed by the baseband; else sub-carrier inspector on that inspector's channel
  uint32_t size;          // channel IFFT size (samples per two hops) in the engine that feeds it
  uint32_t spectsrc_id;   // 0 = none (index 0 of the GUI's combo)
  uint32_t est_mask;
  uint32_t spect_size;    // frame size chosen at rebuild time (0 = too few channel samples per block)
  bool spect_sched;       // emitting on the spectrum_update_int schedule (SPEC US) instead of once per block
  bool fac_on;            // the FAC tab (SPEC FC) with these parameters
  sdb_fac_params fac;
  bool snr_on;            // the SNR meter (SPEC SN) with these parameters
  sdb_snr_params snr;
  bool snr_reset;         // a reset to snr_reset_sigma waits for the next block boundary
  float snr_reset_sigma;
  bool tv_on;             // the Analog TV tab (SPEC TI) with these parameters
  sdb_tv_tab_params tv;
  bool tv_live;           // a change of tv that keeps the geometry waits for the next block boundary
};

// class names in SDB_INSP_* order, as requests and inspector messages carry them
const char *const kClassNames[] = { "psk", "fsk", "ask", "audio", "raw", "power" };

int class_id(const std::string &c)
{
  for (int k = SDB_INSP_PSK; k <= SDB_INSP_POWER; ++k)
    if (c == kClassNames[k]) return k;
  return -1;
}

// a sigutils channel (Hz, relative to the input's centre) as channeliser parameters at the input rate in_rate
sdb_channel_params channel_params(const sdb_sigutils_channel &ch, double in_rate, int precise)
{
  sdb_channel_params cp;
  cp.f0 = (float) (2.0 * 3.14159265358979323846 * fmod(ch.fc / in_rate + 1.0, 1.0));
  cp.bw = (float) (2.0 * 3.14159265358979323846 * (ch.f_hi - ch.f_lo) / in_rate);
  cp.guard = 1.0f; cp.precise = precise;
  return cp;
}

struct EngineDeleter { void operator()(sdb_engine_t *e) const { sdb_engine_destroy(e); } };
struct DecimatorDeleter { void operator()(sdb_decimator_t *d) const { sdb_decimator_destroy(d); } };
using EnginePtr = std::unique_ptr<sdb_engine_t, EngineDeleter>;

}  // namespace

struct sdb_analyzer {
  sdb_analyzer_params params;
  sdb_source_config src;
  size_t src_pos = 0;
  // output queue (suscan_mq): MPSC FIFO of (type, payload)
  std::mutex mq_m;
  std::condition_variable mq_cv;
  std::deque<std::pair<uint32_t, void *>> mq;
  // command queue
  std::mutex cmd_m;
  std::deque<Cmd> cmds;
  bool halt_req = false;
  std::thread worker;
  std::vector<Insp> insps;
  EnginePtr eng;
  // Sub-carrier inspection (GenericInspector.cpp:502-525: openInspectorTab(..., parent = this handle)): every
  // inspector with open children -- at any depth: a sub-carrier inspector can be a parent itself -- gets an engine
  // whose input is its channel stream and whose channeliser window equals its channel size, so that one parent hop
  // is exactly one child hop.  Children have inspector chains, spectrum sources and estimators like any other.
  struct Sub { int32_t parent; EnginePtr eng; };
  std::vector<Sub> subs;
  // the engine that runs inspector i's chain: the analyzer's own for a baseband inspector, its parent's
  // sub-carrier engine otherwise
  sdb_engine_t *engine_of(const Insp &i) const
  {
    if (i.parent < 0) return eng.get();
    for (auto &sb : subs) if (sb.parent == i.parent) return sb.eng.get();
    return nullptr;
  }
  bool plan_dirty = true;
  size_t block = 0;                               // samples per block at the analysis rate
  // source decimation (SPEC L, suscan_source_config_set_average): each block reads block * decim source samples and
  // the decimator brings them to `rate`.  It belongs to the analyzer, not to an engine, so that re-plans keep its carry.
  uint32_t decim = 1;
  double rate = 0;                                // analysis sample rate: src.samp_rate / decim
  std::unique_ptr<sdb_decimator_t, DecimatorDeleter> dec;
  std::vector<sdb_complex> raw;                   // one block of source samples in their native format
  std::vector<sdb_complex> buf;                   // one block at `rate` on the host (a sweep's hops in wide mode)
  std::vector<sdb_complex> drop;                  // samples a sweep reads and discards after a retune
  std::vector<float> psd;
  std::vector<sdb_complex> soft;
  std::vector<uint8_t> hard;
  std::chrono::steady_clock::time_point t0;       // start of the worker loop, for the measured rate
  uint32_t exit_type = SDB_WORKER_MSG_TYPE_HALT;  // the status that ends the worker, set by stop()
  std::atomic<double> measured_rate{ 0.0 };   // written by the worker, read by sdb_analyzer_get_measured_samp_rate
  uint64_t total_samples = 0;
  std::atomic<uint64_t> total_samples_pub{ 0 };   // copy for readers on other threads
  // Guards insps against readers on other threads (sdb_analyzer_get_inspector_config).  The worker changes insps
  // under it in handle_cmds; outside it, it writes only fields that no other thread reads (the engine mapping and
  // geometry set by rebuild).
  std::mutex insp_m;
  double psd_credit = 0;
  // the baseband engine's frame-group stage, SPEC A's means or SPEC PK's extremes: G frames per group (< 2: off), N,
  // the window function, whether G was clamped, whether the minima are posted, and the frames of the engine's open group
  // (its carry survives a re-plan exactly when the kind, G, N and the window stay, see sdb_engine_migrate)
  struct PsdGroups {
    enum Kind { NONE, MEAN, PEAK } kind = NONE;
    uint32_t G = 0, N = 0; int32_t window = 0; bool clamped = false, neg = false;
    uint64_t frames = 0;
  } psd_groups;
  // source-side options of the worker loop (Suscan/Analyzer.cpp:117-135, 229-244; SourceWidget.cpp:1156-1184)
  bool iq_reverse = false, dc_remove = false;
  double throttle = 0;                                  // samples / s, 0 = as fast as the source delivers
  std::chrono::steady_clock::time_point throttle_t0; uint64_t throttle_s0 = 0;
  // history ring + replay (suscan_analyzer_set_history_size / _replay, Suscan/Analyzer.cpp:157-167;
  // Default/Source/SourceWidget.cpp:1070-1073, 1206, 1508)
  std::vector<sdb_complex> hist; size_t hist_start = 0, hist_fill = 0, replay_pos = 0;
  bool replaying = false, replay_wrapped = false; int looped = 0;
  struct BbFilter { sdb_baseband_filter_fn fn; void *priv; int64_t prio; };
  std::vector<BbFilter> bb_filters;

  Insp *open_insp(int32_t handle)
  {
    return handle >= 0 && handle < (int32_t) insps.size() && insps[handle].open ? &insps[handle] : nullptr;
  }
  // bytes per IQ pair of what source_read() delivers: float32 from a read callback, else the capture's own format
  size_t src_bytes() const { return src.read ? 8 : sdb_fmt_bytes(src.input_format); }
  // the blocks the analyzer sees are float32 (baseband filters and the history need that)
  bool f32_src() const { return src.read || src.input_format == SDB_FORMAT_FLOAT32 || dec; }

  void post(uint32_t type, void *payload)
  {
    std::lock_guard<std::mutex> l(mq_m);
    mq.emplace_back(type, payload);
    mq_cv.notify_one();
  }
  void post_status(uint32_t type, int code, const char *msg)
  {
    sdb_analyzer_status_msg *m = (sdb_analyzer_status_msg *) calloc(1, sizeof(*m));
    m->code = code;
    m->err_msg = msg ? strdup(msg) : nullptr;
    post(type, m);
  }
  // the steps of the worker return true to go on, or stop(): false, with the status that ends the worker
  bool stop(uint32_t type) { exit_type = type; return false; }
  bool init_failure()
  {
    post_status(SDB_ANALYZER_MESSAGE_TYPE_SOURCE_INIT, SDB_ANALYZER_INIT_FAILURE, sdb_last_error());
    return stop(SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR);
  }
  // ts: signal time of the first sample of the frame, in seconds
  void post_psd(int64_t fc, double samp_rate, const float *data, size_t n, double ts, int looped_, uint64_t history)
  {
    sdb_analyzer_psd_msg *m = (sdb_analyzer_psd_msg *) calloc(1, sizeof(*m));
    m->fc = fc; m->samp_rate = (float) samp_rate; m->measured_samp_rate = (float) measured_rate.load();
    gettimeofday(&m->rt_time, nullptr);
    m->timestamp.tv_sec = (time_t) ts; m->timestamp.tv_usec = (suseconds_t) ((ts - floor(ts)) * 1e6);
    m->looped = looped_; m->history_size = history;
    m->psd_size = n;
    m->psd_data = (float *) malloc(n * sizeof(float));
    memcpy(m->psd_data, data, n * sizeof(float));
    post(SDB_ANALYZER_MESSAGE_TYPE_PSD, m);
  }
  // an inspector message with the fields every kind carries; the caller fills the rest and posts it
  static sdb_analyzer_inspector_msg *inspector_msg(int kind, int32_t handle, uint32_t inspector_id, const char *cls)
  {
    sdb_analyzer_inspector_msg *m = (sdb_analyzer_inspector_msg *) calloc(1, sizeof(*m));
    m->kind = kind; m->handle = handle; m->inspector_id = inspector_id; m->class_name = strdup(cls);
    return m;
  }
  // the reply to request c: about inspector i, or (i null) an error that echoes the request
  void post_inspector(int kind, const Cmd &c, const Insp *i)
  {
    sdb_analyzer_inspector_msg *m = i ? inspector_msg(kind, i->handle, i->inspector_id, kClassNames[i->cls])
                                      : inspector_msg(kind, c.handle, c.inspector_id, c.cls.c_str());
    m->req_id = c.req_id;
    if (i) { m->channel = i->channel; m->config = i->cfg; m->fs = (float) rate; m->equiv_fs = i->fs;
             m->bandwidth = i->bandwidth; m->lo = i->lo; m->spectsrc_id = i->spectsrc_id; }
    else m->channel = c.channel;
    m->spectsrc_count = SDB_SPECTSRC_COUNT - 1; m->estimator_count = SDB_ESTIMATOR_COUNT;
    if (kind == SDB_INSPECTOR_MSGKIND_ESTIMATOR) { m->estimator_id = c.aux_id; m->enabled = c.enabled; }
    post(SDB_ANALYZER_MESSAGE_TYPE_INSPECTOR, m);
  }
  double chan_credit = 0;

  // SAMPLES batches: suscan flushes an inspector's sample buffer once it holds `watermark` samples
  // (suscan_analyzer_set_inspector_watermark_async, Suscan/Analyzer.cpp:527-537; the audio path asks for half a
  // playback buffer, Default/Audio/AudioProcessor.cpp:745-747).  watermark 0 = one batch per block.
  struct Pending { std::vector<sdb_complex> soft; std::vector<uint8_t> hard; uint64_t watermark = 0; };
  std::map<int32_t, Pending> pending;
  void deliver(const Insp &i, const sdb_complex *s, const uint8_t *h, size_t n, bool flush)
  {
    Pending &p = pending[i.handle];
    p.soft.insert(p.soft.end(), s, s + n);
    p.hard.insert(p.hard.end(), h, h + n);
    if (p.soft.empty() || (!flush && p.soft.size() < p.watermark)) return;
    sdb_analyzer_sample_batch_msg *m = (sdb_analyzer_sample_batch_msg *) calloc(1, sizeof(*m));
    m->inspector_id = i.inspector_id; m->sample_count = (uint64_t) p.soft.size();
    m->samples = (sdb_complex *) malloc(p.soft.size() * sizeof(sdb_complex));
    m->symbols = (uint8_t *) malloc(p.hard.size());
    memcpy(m->samples, p.soft.data(), p.soft.size() * sizeof(sdb_complex));
    memcpy(m->symbols, p.hard.data(), p.hard.size());
    p.soft.clear(); p.hard.clear();
    post(SDB_ANALYZER_MESSAGE_TYPE_SAMPLES, m);
  }

  // Plans one engine level: the baseband (parent -1, with the channel detector) or the children of inspector
  // `parent`, whose channel stream at in_rate is the input.  Every open inspector of the level gets a channel, in
  // handle order; one whose channel cannot be opened stays unmapped.  After the commit the engine takes over the
  // running state of `old` where the geometry allows (old_handle: each inspector's handle in the engines being
  // replaced).  Returns null when the engine cannot be created or committed; sdb_last_error() says why.
  EnginePtr plan_level(const sdb_engine_params &ep, double in_rate, int32_t parent, const std::vector<int> &old_handle,
                       sdb_engine_t *old)
  {
    EnginePtr e(sdb_engine_new(&ep, in_rate));
    if (!e) return nullptr;
    const size_t hops_per_block = block / (params.detector_params.window_size / 2);
    std::vector<int32_t> old_of_new;
    for (auto &i : insps) {
      if (!i.open || i.parent != parent) continue;
      const sdb_channel_params cp = channel_params(i.channel, in_rate, i.precise);
      sdb_channel_info info;
      const int h = sdb_engine_open_channel(e.get(), &cp, &info);
      if (h < 0) continue;
      i.engine_handle = h; i.size = info.size;
      old_of_new.push_back(old_handle[(size_t) i.handle]);
      i.fs = (float) (in_rate / info.decimation);
      i.bandwidth = (float) (i.channel.f_hi - i.channel.f_lo); i.lo = (float) i.channel.fc;
      sdb_engine_set_inspector(e.get(), h, &i.cfg);
      if (i.fac_on) sdb_engine_set_fac(e.get(), h, &i.fac);      // (checked when requested; the class cannot change)
      if (i.snr_on) sdb_engine_set_snr(e.get(), h, &i.snr);      // (likewise)
      if (i.tv_on) sdb_engine_set_tv(e.get(), h, &i.tv);         // (likewise)
      // spectrum source / estimators: the largest frame (<= 4096) a steady-state block can fill (SPEC U.1)
      i.spect_size = 0; i.spect_sched = false;
      if ((i.spectsrc_id || i.est_mask) && params.spectrum_update_int > 0) {
        // SPEC US: 4096-point frames every spectrum_update_int of channel time, whatever the block size.  An interval
        // shorter than a block allows (more than SDB_SPECTRUM_EMITS_MAX emissions in one feed, which the engine
        // refuses) is raised to the shortest that fits: emitting as often as possible beats stopping the session.
        const uint32_t W = ep.st_window_size ? ep.st_window_size : ep.psd_size;
        const uint64_t n_max = (uint64_t) (ep.max_feed / (W / 2)) * (info.size / 2);
        const double I_min = (double) std::max<uint64_t>(1, (n_max + SDB_SPECTRUM_EMITS_MAX - 1) / SDB_SPECTRUM_EMITS_MAX);
        const double I = std::min(std::max(I_min, std::floor((double) params.spectrum_update_int * (double) i.fs + 0.5)),
                                  (double) SDB_SPECTRUM_INTERVAL_MAX);
        i.spect_size = 4096; i.spect_sched = true;
        sdb_engine_set_spectrum_source(e.get(), h, (int) i.spectsrc_id, 4096);
        for (int k = 0; k < SDB_ESTIMATOR_COUNT; ++k)
          if (i.est_mask & (1u << k)) sdb_engine_set_estimator(e.get(), h, k, 1);
        sdb_engine_set_spectrum_interval(e.get(), h, (uint64_t) I);
      } else if (i.spectsrc_id || i.est_mask) {
        const size_t n_ch = hops_per_block * (info.size / 2);
        uint32_t ns = 4096;
        while (ns >= 64 && (size_t) ns + 1 > n_ch) ns >>= 1;
        if (ns >= 64) {
          i.spect_size = ns;
          sdb_engine_set_spectrum_source(e.get(), h, (int) i.spectsrc_id, ns);
          for (int k = 0; k < SDB_ESTIMATOR_COUNT; ++k)
            if (i.est_mask & (1u << k)) sdb_engine_set_estimator(e.get(), h, k, 1);
        }
      }
    }
    if (parent < 0 && params.channel_update_int > 0)
      sdb_engine_set_channel_detector(e.get(), params.detector_params.alpha, params.detector_params.beta,
                                      params.detector_params.gamma,
                                      params.detector_params.snr > 0 ? params.detector_params.snr : 4.0f, 2);
    if (parent < 0 && params.channel_update_int > 0 && params.channel_hold_int > 0) {
      // SPEC KT: one tracking update per block, so the hold in seconds becomes whole blocks
      const double h = std::ceil((double) params.channel_hold_int * rate / (double) block);
      if (sdb_engine_set_channel_tracking(e.get(), (uint32_t) std::min<double>(h, SDB_CHTRACK_HOLD_MAX))) return nullptr;
    }
    if (sdb_engine_commit(e.get())) return nullptr;
    if (old && sdb_engine_same_geometry(e.get(), old))
      sdb_engine_migrate_map(e.get(), old, old_of_new.data(), old_of_new.size());
    return e;
  }

  // (re)plan the engines from the open inspectors at a block boundary.  A new engine takes over the running state of
  // the one it replaces (sdb_engine_migrate_map): input history, DC estimate, and for every inspector that stays open
  // its cross-fade tail, LO phase and loop state -- opening, closing, retuning or reconfiguring ONE inspector leaves
  // the sample streams of the others untouched (suscan keeps them running too, Suscan/Analyzer.cpp:459-537).  The old
  // engines are released only once every new level has migrated from them.  Returns false when the baseband engine
  // cannot be planned (sdb_last_error() says why).
  bool rebuild()
  {
    EnginePtr old = std::move(eng);
    std::vector<Sub> old_subs; old_subs.swap(subs);
    std::vector<int> old_handle(insps.size(), -1);
    for (size_t q = 0; q < insps.size(); ++q) { old_handle[q] = insps[q].engine_handle; insps[q].engine_handle = -1; }
    sdb_engine_params ep;
    memset(&ep, 0, sizeof(ep));
    ep.n_streams = 1;
    ep.psd_size = (uint32_t) params.detector_params.window_size;
    ep.psd_window = params.detector_params.window;
    ep.st_window_size = 0;
    ep.max_feed = (uint32_t) block;
    ep.device = src.device;
    ep.flags = (iq_reverse ? SDB_FLAG_IQ_REVERSE : 0) | (dc_remove ? SDB_FLAG_DC_REMOVE : 0);
    ep.input_format = src.read || dec ? SDB_FORMAT_FLOAT32 : src.input_format;
    // the whole frames of one psd_update_int, clamped to [1, max]; *clamped says whether the clamp changed them
    auto interval_frames = [&](uint32_t max, bool *clamped) {
      const double want = (double) params.psd_update_int * rate / (double) ep.psd_size;
      const long long r = want > 0 ? llround(std::min(want, 1e12)) : 0;
      const uint32_t f = (uint32_t) std::min<long long>(std::max<long long>(r, 1), max);
      *clamped = (long long) f != r;
      return f;
    };
    // a peak detector takes precedence over averaging (SPEC PK.5); G = 1: every frame is a group of its own
    const bool peaks = params.psd_detector != SDB_PSD_DETECTOR_DEFAULT;
    PsdGroups g;
    g.kind = peaks ? PsdGroups::PEAK : params.psd_average ? PsdGroups::MEAN : PsdGroups::NONE;
    if (g.kind != PsdGroups::NONE) g.G = interval_frames(peaks ? SDB_PSD_PEAK_MAX : SDB_PSD_AVERAGE_MAX, &g.clamped);
    g.N = ep.psd_size; g.window = ep.psd_window;
    g.neg = params.psd_detector == SDB_PSD_DETECTOR_NEG_PEAK;
    (peaks ? ep.psd_peak : ep.psd_average) = g.G;
    const PsdGroups &o = psd_groups;
    if (old && g.kind == o.kind && g.G == o.G && g.N == o.N && g.window == o.window) g.frames = o.frames;
    psd_groups = g;
    eng = plan_level(ep, rate, -1, old_handle, old.get());
    if (!eng) return false;
    // sub-carrier engines: one per inspector that has open children, parents before children (an inspector's handle
    // is larger than its parent's, so one pass in handle order visits every parent after it was planned itself).
    // Every level runs the same number of hops per block: a child's window is its parent's channel size.
    const size_t hops_per_block = block / (ep.psd_size / 2);
    for (const Insp &p : insps) {
      if (!p.open || p.engine_handle < 0 || p.size < 16) continue;
      if (std::none_of(insps.begin(), insps.end(), [&](const Insp &c) { return c.open && c.parent == p.handle; }))
        continue;
      sdb_engine_params sp;
      memset(&sp, 0, sizeof(sp));
      sp.n_streams = 1; sp.psd_size = 0; sp.st_window_size = p.size;
      sp.max_feed = (uint32_t) (hops_per_block * (p.size / 2));
      sp.device = src.device; sp.input_format = SDB_FORMAT_FLOAT32;
      sdb_engine_t *old_sub = nullptr;
      for (auto &os : old_subs) if (os.parent == p.handle) old_sub = os.eng.get();
      EnginePtr se = plan_level(sp, (double) p.fs, p.handle, old_handle, old_sub);
      if (se) subs.push_back(Sub{ p.handle, std::move(se) });
      else for (auto &c : insps) if (c.open && c.parent == p.handle) c.engine_handle = -1;
    }
    plan_dirty = false;
    return true;
  }

  void handle_cmds()
  {
    std::deque<Cmd> todo;
    { std::lock_guard<std::mutex> l(cmd_m); todo.swap(cmds); }
    std::lock_guard<std::mutex> il(insp_m);
    for (auto &c : todo) {
      switch (c.kind) {
        case Cmd::OPEN: {
          int cls = class_id(c.cls);
          double bw = c.channel.f_hi - c.channel.f_lo;
          if (cls < 0) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_KIND, c, nullptr); break; }
          // the input of the new inspector: the baseband, or (sub-carrier inspection) the channel of `parent`
          double in_rate = rate;
          uint32_t in_window = (uint32_t) params.detector_params.window_size;
          if (c.parent >= 0) {
            const Insp *p = open_insp(c.parent);
            if (!p || p->size < 16) {
              Cmd w = c; w.handle = c.parent;
              post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_HANDLE, w, nullptr); break;
            }
            in_rate = (double) p->fs; in_window = p->size;
          }
          if (!(bw > 0) || bw > in_rate || fabs(c.channel.fc) > in_rate / 2) {
            post_inspector(SDB_INSPECTOR_MSGKIND_INVALID_CHANNEL, c, nullptr); break;
          }
          // geometry -> equivalent rate, needed for the default config the OPEN reply carries; the engine's
          // shared-memory channel IFFT takes at most 16384 bins
          const sdb_channel_params cp = channel_params(c.channel, in_rate, c.precise);
          sdb_channel_info info;
          if (sdb_channel_geometry(in_window, &cp, &info) || info.size > 16384) {
            post_inspector(SDB_INSPECTOR_MSGKIND_INVALID_CHANNEL, c, nullptr); break;
          }
          Insp i;
          memset(&i, 0, sizeof(i));
          i.handle = (int32_t) insps.size(); i.open = true; i.has_id = false; i.cls = cls; i.channel = c.channel;
          i.precise = c.precise; i.engine_handle = -1; i.parent = c.parent;
          i.fs = (float) (in_rate / info.decimation);
          i.size = info.size;
          i.bandwidth = (float) bw; i.lo = (float) c.channel.fc;
          sdb_inspector_config_default(&i.cfg, cls, i.fs);
          i.cfg.clock_running = 0;       // "by default ... no samples are being delivered" (manual p.62)
          insps.push_back(i);
          plan_dirty = true;
          post_inspector(SDB_INSPECTOR_MSGKIND_OPEN, c, &insps.back());
          break;
        }
        case Cmd::SET_ID:
        case Cmd::SET_CONFIG:
        case Cmd::SET_SPECTRUM:
        case Cmd::ESTIMATOR_CMD:
        case Cmd::SET_FAC:
        case Cmd::SET_SNR:
        case Cmd::RESET_SNR:
        case Cmd::SET_TV:
        case Cmd::CLOSE: {
          Insp *ip = open_insp(c.handle);
          if (!ip) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_HANDLE, c, nullptr); break; }
          Insp &i = *ip;
          if (c.kind == Cmd::SET_SPECTRUM) {
            if (c.aux_id >= (uint32_t) SDB_SPECTSRC_COUNT) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_OBJECT, c, nullptr); break; }
            i.spectsrc_id = c.aux_id; plan_dirty = true;
            post_inspector(SDB_INSPECTOR_MSGKIND_SPECTRUM, c, &i);     // acknowledgement: no spectrum_data yet
          } else if (c.kind == Cmd::ESTIMATOR_CMD) {
            if (c.aux_id >= (uint32_t) SDB_ESTIMATOR_COUNT) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_OBJECT, c, nullptr); break; }
            if (c.enabled) i.est_mask |= 1u << c.aux_id; else i.est_mask &= ~(1u << c.aux_id);
            plan_dirty = true;
            post_inspector(SDB_INSPECTOR_MSGKIND_ESTIMATOR, c, &i);    // acknowledgement: value follows per block
          } else if (c.kind == Cmd::SET_FAC) {
            if (c.enabled && i.cls > SDB_INSP_ASK) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_KIND, c, nullptr); break; }
            if (c.enabled && sdb_fac_check(&c.fac)) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_OBJECT, c, nullptr); break; }
            i.fac_on = c.enabled != 0; i.fac = c.fac; plan_dirty = true;
            post_inspector(SDB_INSPECTOR_MSGKIND_FAC, c, &i);         // acknowledgement: data follows per block
          } else if (c.kind == Cmd::SET_SNR) {
            if (c.enabled && i.cls > SDB_INSP_ASK) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_KIND, c, nullptr); break; }
            if (c.enabled && sdb_snr_check(&c.snr)) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_OBJECT, c, nullptr); break; }
            i.snr_on = c.enabled != 0; i.snr = c.snr; i.snr_reset = false; plan_dirty = true;
            post_inspector(SDB_INSPECTOR_MSGKIND_SNR, c, &i);         // acknowledgement: data follows per block
          } else if (c.kind == Cmd::RESET_SNR) {
            if (!i.snr_on || !(std::isfinite(c.snr.sigma) && c.snr.sigma > 0.0f)) {
              post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_OBJECT, c, nullptr); break;
            }
            i.snr_reset = true; i.snr_reset_sigma = c.snr.sigma;      // no re-plan: applied before the next block
            post_inspector(SDB_INSPECTOR_MSGKIND_SNR, c, &i);
          } else if (c.kind == Cmd::SET_TV) {
            if (c.enabled && i.cls > SDB_INSP_ASK) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_KIND, c, nullptr); break; }
            if (c.enabled && sdb_tv_tab_check(&c.tv)) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_OBJECT, c, nullptr); break; }
            // SPEC TI.4: the same geometry while on is a live change at the next block boundary; anything else re-plans
            if (c.enabled && i.tv_on && sdb_tv_same_geometry(i.tv.tv, c.tv.tv)) i.tv_live = true;
            else { i.tv_on = c.enabled != 0; i.tv_live = false; plan_dirty = true; }
            i.tv = c.tv;
            post_inspector(SDB_INSPECTOR_MSGKIND_TV, c, &i);          // acknowledgement: frames follow per block
          } else if (c.kind == Cmd::SET_ID) {
            i.inspector_id = c.inspector_id; i.has_id = true;
            post_inspector(SDB_INSPECTOR_MSGKIND_SET_ID, c, &i);
          } else if (c.kind == Cmd::SET_CONFIG) {
            if (c.cfg.insp_class != i.cls) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_KIND, c, nullptr); break; }
            i.cfg = c.cfg; plan_dirty = true;
            post_inspector(SDB_INSPECTOR_MSGKIND_SET_CONFIG, c, &i);
          } else {
            i.open = false; plan_dirty = true;
            // sub-carrier inspectors go with it, to any depth (handles grow with the order of opening: one pass)
            for (auto &ch : insps) if (ch.open && ch.parent >= 0 && !insps[ch.parent].open) ch.open = false;
            post_inspector(SDB_INSPECTOR_MSGKIND_CLOSE, c, &i);
          }
          break;
        }
        case Cmd::SET_WATERMARK:
          if (!open_insp(c.handle)) { post_inspector(SDB_INSPECTOR_MSGKIND_WRONG_HANDLE, c, nullptr); break; }
          pending[c.handle].watermark = (uint64_t) c.value;
          break;
        case Cmd::SET_HISTORY:
          hist.assign((size_t) c.value, sdb_complex{ 0.0f, 0.0f });
          hist_start = hist_fill = replay_pos = 0; replaying = false; looped = 0;
          break;
        case Cmd::REPLAY:
          replaying = c.enabled != 0 && hist_fill > 0;
          replay_pos = 0; looped = 0; replay_wrapped = false;
          break;
        case Cmd::SET_HOP_RANGE:
          if (c.value <= c.value2) { hop_min = c.value; hop_max = c.value2; hop_index = 0; }
          break;
        case Cmd::SET_REL_BW:
          if (c.value > 0) rel_bw = (float) (c.value > 1 ? 1 : c.value);
          break;
        case Cmd::SET_BUFFERING: buffering = (uint64_t) c.value; break;
        case Cmd::SET_STRATEGY: strategy = c.enabled; hop_index = 0; break;
        case Cmd::SET_PARTITIONING: partitioning = c.enabled; break;
        case Cmd::SEEK:       // suscan_analyzer_seek (Suscan/Analyzer.cpp:151-155): in-memory captures only
          if (!src.read && src.data && c.value >= 0) {
            const double p = c.value * src.samp_rate;
            src_pos = p >= (double) src.length ? src.length : (size_t) p;
          }
          break;
        case Cmd::SET_FREQ:
        case Cmd::SET_BANDWIDTH: {
          // "overridable" setters (Suscan/Analyzer.cpp:509-526): no reply; the latest value wins.  The channel is
          // re-planned at the next block boundary (see the a18 limits in DESIGN.md).
          Insp *ip = open_insp(c.handle);
          if (!ip) break;
          Insp &i = *ip;
          const double in_rate = i.parent >= 0 ? (double) insps[i.parent].fs : rate;
          if (c.kind == Cmd::SET_FREQ) {
            if (fabs(c.value) > in_rate / 2) break;
            i.channel.fc = c.value; i.lo = (float) c.value;
          } else {
            if (!(c.value > 0) || c.value > in_rate) break;
            i.channel.f_lo = -0.5 * c.value; i.channel.f_hi = 0.5 * c.value; i.channel.bw = (float) c.value;
            i.bandwidth = (float) c.value;
          }
          plan_dirty = true;
          break;
        }
        case Cmd::SET_IQ_REVERSE:
          if (iq_reverse != (c.enabled != 0)) { iq_reverse = c.enabled != 0; plan_dirty = true; }
          break;
        case Cmd::SET_DC_REMOVE:
          if (dc_remove != (c.enabled != 0)) { dc_remove = c.enabled != 0; plan_dirty = true; }
          break;
        case Cmd::SET_THROTTLE:
          throttle = c.value > 0 ? c.value : 0;
          throttle_t0 = std::chrono::steady_clock::now(); throttle_s0 = total_samples;   // pace from here on
          break;
        case Cmd::SET_PARAMS: {
          params = c.params; plan_dirty = true;
          hop_min = params.min_freq; hop_max = params.max_freq; hop_index = 0;
          sdb_analyzer_params *m = (sdb_analyzer_params *) malloc(sizeof(*m));
          *m = params;
          post(SDB_ANALYZER_MESSAGE_TYPE_PARAMS, m);
          break;
        }
      }
    }
  }

  long source_read(sdb_complex *dst, size_t n)
  {
    if (src.read) return src.read(src.priv, dst, n);
    if (!src.data) return -1;
    // in-memory capture in its native sample format (bps bytes per IQ pair); dst is a byte buffer of n * 8
    const size_t bps = src_bytes();
    const unsigned char *base = reinterpret_cast<const unsigned char *>(src.data);
    unsigned char *out = reinterpret_cast<unsigned char *>(dst);
    size_t got = 0;
    while (got < n) {
      if (src_pos >= src.length) { if (!src.loop) break; src_pos = 0; }
      size_t take = std::min(n - got, src.length - src_pos);
      memcpy(out + got * bps, base + src_pos * bps, take * bps);
      got += take; src_pos += take;
    }
    return (long) got;
  }

  // ---------------------------------------------------------------------------------------------------------
  // SUSCAN_ANALYZER_MODE_WIDE_SPECTRUM: the panoramic scanner's analyzer (Panoramic/Scanner.cpp:296-372, 419-523):
  // retune, drop `buffering` samples (tuner round trip), take one window, post its PSD with the hop's centre; the GUI
  // stitches the hops (SpectrumView).  Hops are independent, so HB of them go through the engine as HB streams.
  // Hop plan (own definition, the upstream one is not in the reference): step = rel_bw fs; PROGRESSIVE: centres
  // min + step/2 + i step while the hop still starts below max, then wrap; STOCHASTIC: uniform in [min, max] from a
  // 32-bit LCG, snapped to the progressive grid when the partitioning is DISCRETE.  min == max: one centre.
  // ---------------------------------------------------------------------------------------------------------
  double hop_min = 0, hop_max = 0; float rel_bw = 0.5f; uint64_t buffering = 0;
  int strategy = SDB_SWEEP_STRATEGY_PROGRESSIVE, partitioning = SDB_SPECTRUM_PARTITIONING_DISCRETE;
  uint64_t hop_index = 0; uint32_t lcg = 0x5167D166u;
  double next_hop()
  {
    const double step = (double) rel_bw * src.samp_rate;
    if (!(hop_max > hop_min) || !(step > 0)) return hop_min;
    const uint64_t n_grid = (uint64_t) ceil((hop_max - hop_min) / step);
    if (strategy == SDB_SWEEP_STRATEGY_PROGRESSIVE) {
      const uint64_t i = hop_index++ % (n_grid ? n_grid : 1);
      return hop_min + 0.5 * step + (double) i * step;
    }
    lcg = lcg * 1664525u + 1013904223u;
    const double u = (double) (lcg >> 8) / 16777216.0;
    if (partitioning == SDB_SPECTRUM_PARTITIONING_DISCRETE) {
      uint64_t i = (uint64_t) (u * (double) n_grid);
      if (i >= n_grid) i = n_grid - 1;
      return hop_min + 0.5 * step + (double) i * step;
    }
    return hop_min + u * (hop_max - hop_min);
  }

  // one sweep of HB hops
  bool sweep()
  {
    const size_t HB = 16, N = (size_t) params.detector_params.window_size;
    if (plan_dirty) {
      eng.reset();
      sdb_engine_params ep;
      memset(&ep, 0, sizeof(ep));
      ep.n_streams = (uint32_t) HB; ep.psd_size = (uint32_t) N; ep.psd_window = params.detector_params.window;
      ep.max_feed = (uint32_t) N; ep.device = src.device;
      ep.flags = iq_reverse ? SDB_FLAG_IQ_REVERSE : 0;
      ep.input_format = src.read ? SDB_FORMAT_FLOAT32 : src.input_format;   // in-memory captures keep their format
      eng.reset(sdb_engine_new(&ep, src.samp_rate));
      if (!eng || sdb_engine_commit(eng.get())) return init_failure();
      plan_dirty = false;
    }
    // hops are packed back to back in the source's native sample format: bps bytes per IQ pair
    const size_t bps = src_bytes();
    double fcs[HB];
    buf.resize(HB * N);
    unsigned char *bytes = reinterpret_cast<unsigned char *>(buf.data());
    size_t got_hops = 0;
    bool eos = false, err = false;
    for (size_t h = 0; h < HB && !eos && !err; ++h) {
      fcs[h] = next_hop();
      if (src.set_frequency && src.set_frequency(src.priv, fcs[h]) != 0) { err = true; break; }
      for (uint64_t left = buffering; left > 0 && !eos && !err;) {          // the tuner's round trip
        const size_t take = (size_t) std::min<uint64_t>(left, 65536);
        drop.resize(take);
        const long g = source_read(drop.data(), take);
        if (g < 0) err = true; else if ((size_t) g < take) eos = true;
        left -= take;
      }
      if (eos || err) break;
      const long g = source_read(reinterpret_cast<sdb_complex *>(bytes + h * N * bps), N);
      if (g < 0) err = true; else if ((size_t) g < N) eos = true; else ++got_hops;
    }
    if (err) return stop(SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR);
    if (got_hops) {
      for (size_t h = got_hops; h < HB; ++h)
        memset(bytes + h * N * bps, src.input_format == SDB_FORMAT_UNSIGNED8 && !src.read ? 0x80 : 0, N * bps);
      if (sdb_engine_feed_host(eng.get(), buf.data(), N, N) || sdb_engine_sync(eng.get()))
        return stop(SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR);
      psd.resize(HB * N);
      if (sdb_engine_read_psd(eng.get(), psd.data(), psd.size())) return stop(SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR);
      for (size_t h = 0; h < got_hops; ++h) post_psd((int64_t) llround(fcs[h]), src.samp_rate, &psd[h * N], N, 0, 0, 0);
      total_samples += got_hops * (N + buffering);
    }
    if (eos) return stop(SDB_ANALYZER_MESSAGE_TYPE_EOS);
    return true;
  }

  // ---------------------------------------------------------------------------------------------------------
  // SUSCAN_ANALYZER_MODE_CHANNEL: one block per step
  // ---------------------------------------------------------------------------------------------------------
  // one block into buf, or left in the decimator's device output (on_device)
  bool read_block(bool &on_device)
  {
    if (replaying && hist_fill > 0) {
      // suscan_analyzer_replay: the source is paused and the history ring is played back, oldest sample first
      for (size_t i = 0; i < block; ++i) {
        if (replay_pos == 0 && replay_wrapped) looped = 1;         // playing the ring for the second time
        buf[i] = hist[(hist_start + replay_pos) % hist.size()];
        if (++replay_pos >= hist_fill) { replay_pos = 0; replay_wrapped = true; }
      }
      return true;
    }
    long got;
    if (dec) {
      // SPEC L: block * decim source samples in their native format -> block float32 samples at `rate`.  Baseband
      // filters and the history see the decimated samples on the host; otherwise the engine reads them in place.
      const long g = source_read(raw.data(), block * decim);
      got = g < 0 ? g : g / (long) decim;
      if (got == (long) block) {
        if (sdb_decimator_feed_host(dec.get(), raw.data(), raw.size(), block * decim) != (long) block)
          return stop(SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR);
        bool host = !hist.empty();
        { std::lock_guard<std::mutex> l(cmd_m); host = host || !bb_filters.empty(); }
        if (!host) {
          if (sdb_decimator_sync(dec.get())) return stop(SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR);
          on_device = true;
        } else if (sdb_decimator_read(dec.get(), buf.data(), buf.size())) {
          return stop(SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR);
        }
      }
    } else {
      got = source_read(buf.data(), block);
    }
    if (got == (long) block && f32_src() && !hist.empty()) {       // suscan_analyzer_set_history_size: keep the tail
      for (size_t i = 0; i < block; ++i) {
        hist[(hist_start + hist_fill) % hist.size()] = buf[i];
        if (hist_fill < hist.size()) ++hist_fill; else hist_start = (hist_start + 1) % hist.size();
      }
    }
    if (got < 0) return stop(SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR);
    if ((size_t) got < block) return stop(SDB_ANALYZER_MESSAGE_TYPE_EOS);   // partial tail blocks are dropped
    return true;
  }

  // baseband filters see (and may rewrite) every float32 block before the analyzer does, in registration order;
  // with decimation the block and the offset are at the decimated rate
  bool run_filters(bool &on_device)
  {
    if (!f32_src()) return true;
    const std::vector<BbFilter> fl = [&] { std::lock_guard<std::mutex> l(cmd_m); return bb_filters; }();
    if (on_device && !fl.empty()) {                  // a filter registered while the block was being read
      if (sdb_decimator_read(dec.get(), buf.data(), buf.size())) return stop(SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR);
      on_device = false;
    }
    for (auto &f : fl) f.fn(f.priv, this, buf.data(), (uint64_t) block, total_samples / decim);
    return true;
  }

  bool feed(bool on_device)
  {
    const int fed = on_device ? sdb_engine_feed_device(eng.get(), sdb_decimator_output_device(dec.get()), block, block)
                              : sdb_engine_feed_host(eng.get(), buf.data(), block, block);
    if (fed || sdb_engine_sync(eng.get())) return stop(SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR);
    total_samples += block * decim;                   // source samples
    total_samples_pub.store(total_samples);
    return true;
  }

  void pace()
  {
    if (throttle > 0) {                                // suscan_analyzer_set_throttle_async: pace to `throttle` samples/s
      const double due = (double) (total_samples - throttle_s0) / throttle;
      const double now = std::chrono::duration<double>(std::chrono::steady_clock::now() - throttle_t0).count();
      if (due > now) std::this_thread::sleep_for(std::chrono::duration<double>(due - now));
    }
    double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    measured_rate.store(el > 0 ? (double) total_samples / el : 0);
  }

  // PSD messages at psd_update_int cadence of SIGNAL time (coverage = N / (fs * interval)).  Internal to the library:
  // hidden, so that the compiler's choice not to inline it adds no export.
  __attribute__((visibility("hidden"))) void publish_psd()
  {
    const size_t N = (size_t) params.detector_params.window_size, frames = block / N;
    // the extremes (SPEC PK) or the means (SPEC A) of the groups the block completed, G frames each
    PsdGroups &pg = psd_groups;
    if (pg.G >= 2) {
      const bool peaks = pg.kind == PsdGroups::PEAK;
      const size_t groups = peaks ? sdb_engine_psd_peak_groups(eng.get()) : sdb_engine_psd_average_frames(eng.get());
      // group j of the block starts j G - carried frames after the block's first (earlier blocks hold its start when
      // that is negative).  Unless G was clamped a group lasts exactly the interval the credit is measured against, so
      // every group is posted.
      const uint64_t carried = pg.frames;
      pg.frames = (pg.frames + frames) % pg.G;
      psd.resize(groups * N);
      if (groups && (peaks ? sdb_engine_read_psd_peak(eng.get(), pg.neg ? nullptr : psd.data(),
                                                      pg.neg ? psd.data() : nullptr, psd.size())
                           : sdb_engine_read_psd_average(eng.get(), psd.data(), psd.size())))
        return;
      const double per_group = (double) pg.G * (double) N / rate;
      const double interval = pg.clamped ? (double) params.psd_update_int : per_group;
      const int64_t block_start = (int64_t) (total_samples - block * decim);
      for (size_t j = 0; j < groups; ++j) {
        psd_credit += per_group;
        if (psd_credit + 1e-12 >= interval) {
          psd_credit = fmod(psd_credit, interval);
          const int64_t first = (int64_t) (j * pg.G) - (int64_t) carried;
          post_psd((int64_t) src.freq, rate, &psd[j * N], N,
                   (double) (block_start + first * (int64_t) (N * decim)) / src.samp_rate, looped, (uint64_t) hist_fill);
        }
      }
      return;
    }
    psd.resize(frames * N);
    if (sdb_engine_read_psd(eng.get(), psd.data(), psd.size())) return;
    const double per_frame = (double) N / rate;
    for (size_t f = 0; f < frames; ++f) {
      psd_credit += per_frame;
      if (psd_credit + 1e-12 >= params.psd_update_int) {
        psd_credit = params.psd_update_int > 0 ? fmod(psd_credit, params.psd_update_int) : 0;
        post_psd((int64_t) src.freq, rate, &psd[f * N], N,
                 (double) (total_samples - block * decim + f * N * decim) / src.samp_rate, looped, (uint64_t) hist_fill);
      }
    }
  }

  void deliver_symbols(sdb_engine_t *e, const Insp &i, size_t cap)
  {
    if (!i.has_id || i.engine_handle < 0) return;
    soft.resize(cap); hard.resize(cap);
    long n = sdb_engine_read_symbols(e, 0, i.engine_handle, soft.data(), hard.data(), cap);
    if (n > 0) deliver(i, soft.data(), hard.data(), (size_t) n, false);
  }

  // sample batches, keyed by the caller-chosen inspector_id
  // sub-carrier inspectors: the parent's channel samples of this block through the child engine.  `subs` is in
  // parent-before-child order (rebuild), so a nested parent's engine has been fed by the time it is read.
  void publish_symbols()
  {
    for (auto &sb : subs) {
      const Insp &p = insps[sb.parent];
      sdb_engine_t *host = engine_of(p);
      if (!p.open || p.engine_handle < 0 || !host) continue;
      std::vector<sdb_complex> ch(block);
      long nch = sdb_engine_read_channel(host, 0, p.engine_handle, ch.data(), ch.size());
      if (nch <= 0) continue;
      if (sdb_engine_feed_host(sb.eng.get(), ch.data(), (size_t) nch, (size_t) nch) || sdb_engine_sync(sb.eng.get())) continue;
      for (auto &i : insps) if (i.open && i.parent == p.handle) deliver_symbols(sb.eng.get(), i, (size_t) nch);
    }
    for (auto &i : insps) if (i.open && i.parent < 0) deliver_symbols(eng.get(), i, block);
  }

  void post_spectrum(const Insp &i, const float *sp, uint32_t n)
  {
    sdb_analyzer_inspector_msg *m = inspector_msg(SDB_INSPECTOR_MSGKIND_SPECTRUM, i.handle, i.inspector_id,
                                                  kClassNames[i.cls]);
    m->spectsrc_id = i.spectsrc_id; m->spectrum_size = n; m->samp_rate = (uint64_t) i.fs;
    m->fs = (float) rate; m->equiv_fs = i.fs;
    m->spectrum_data = (float *) malloc(n * sizeof(float));
    memcpy(m->spectrum_data, sp, n * sizeof(float));
    post(SDB_ANALYZER_MESSAGE_TYPE_INSPECTOR, m);
  }
  void post_estimate(const Insp &i, int e, float v)
  {
    sdb_analyzer_inspector_msg *m = inspector_msg(SDB_INSPECTOR_MSGKIND_ESTIMATOR, i.handle, i.inspector_id,
                                                  kClassNames[i.cls]);
    m->estimator_id = (uint32_t) e; m->enabled = 1; m->value = v;
    post(SDB_ANALYZER_MESSAGE_TYPE_INSPECTOR, m);
  }

  // SPEC US: every emission of the block, in t_j order: its spectrum, then its valid estimates.  The read buffers
  // (sched_*) are kept across blocks: they grow once, and a block without emissions copies nothing.
  std::vector<float> sched_sp, sched_vals[SDB_ESTIMATOR_COUNT];
  std::vector<int32_t> sched_ok[SDB_ESTIMATOR_COUNT];
  std::vector<uint64_t> sched_ends;
  void publish_scheduled(sdb_engine_t *ie, const Insp &i)
  {
    const size_t cap = SDB_SPECTRUM_EMITS_MAX;
    const uint32_t w = i.spectsrc_id == SDB_SPECTSRC_FAC ? i.spect_size / 2 : i.spect_size;
    std::vector<float> &sp = sched_sp, *vals = sched_vals;
    std::vector<int32_t> *ok = sched_ok;
    std::vector<uint64_t> &ends = sched_ends;
    if (ends.size() < cap) ends.resize(cap);
    long n = -1;
    if (i.spectsrc_id) {
      if (sp.size() < cap * w) sp.resize(cap * w);
      n = sdb_engine_read_spectra(ie, i.engine_handle, sp.data(), ends.data(), cap);
      if (n < 0) return;
    }
    for (int e = 0; e < SDB_ESTIMATOR_COUNT; ++e) {
      if (!(i.est_mask & (1u << e))) continue;
      if (vals[e].size() < cap) { vals[e].resize(cap); ok[e].resize(cap); }
      const long m = sdb_engine_read_estimates(ie, i.engine_handle, e, vals[e].data(), ok[e].data(), cap);
      if (m < 0) return;
      n = m;
    }
    for (long j = 0; j < n; ++j) {
      if (i.spectsrc_id) post_spectrum(i, sp.data() + (size_t) j * w, w);
      for (int e = 0; e < SDB_ESTIMATOR_COUNT; ++e)
        if ((i.est_mask & (1u << e)) && ok[e][j]) post_estimate(i, e, vals[e][j]);
    }
  }

  // kind=SPECTRUM / kind=ESTIMATOR inspector messages (one per block that filled a frame, or on the schedule)
  void publish_spectra()
  {
    for (auto &i : insps) {
      sdb_engine_t *ie = engine_of(i);
      if (!i.open || i.engine_handle < 0 || !i.spect_size || !ie) continue;
      if (i.spect_sched) { publish_scheduled(ie, i); continue; }
      if (i.spectsrc_id) {
        std::vector<float> sp(i.spect_size);
        uint32_t emitted = 0;
        if (sdb_engine_read_spectrum(ie, i.engine_handle, sp.data(), &emitted) == 0 && emitted)
          post_spectrum(i, sp.data(), emitted);
      }
      for (int e = 0; e < SDB_ESTIMATOR_COUNT; ++e) {
        if (!(i.est_mask & (1u << e))) continue;
        float v = 0; int32_t ok = 0;
        if (sdb_engine_read_estimate(ie, i.engine_handle, e, &v, &ok) == 0 && ok) post_estimate(i, e, v);
      }
    }
  }

  // kind=FAC inspector messages (SPEC FC): one per block that completed a FAC block, after the block's SAMPLES
  std::vector<float> fac_buf;
  void publish_fac()
  {
    for (auto &i : insps) {
      sdb_engine_t *ie = engine_of(i);
      if (!i.open || !i.fac_on || i.engine_handle < 0 || !ie) continue;
      sdb_fac_status st;
      fac_buf.resize(i.fac.size / 2);
      if (sdb_engine_read_fac(ie, i.engine_handle, fac_buf.data(), &st) || !st.blocks) continue;
      sdb_analyzer_inspector_msg *m = inspector_msg(SDB_INSPECTOR_MSGKIND_FAC, i.handle, i.inspector_id,
                                                    kClassNames[i.cls]);
      m->spectrum_size = fac_buf.size(); m->samp_rate = (uint64_t) i.fs;
      m->fs = (float) rate; m->equiv_fs = i.fs; m->fac = st;
      m->spectrum_data = (float *) malloc(fac_buf.size() * sizeof(float));
      memcpy(m->spectrum_data, fac_buf.data(), fac_buf.size() * sizeof(float));
      post(SDB_ANALYZER_MESSAGE_TYPE_INSPECTOR, m);
    }
  }

  // SPEC SN.3: the resets requested since the last block, on the engines that run the next one
  void apply_snr_resets()
  {
    for (auto &i : insps) {
      if (!i.snr_reset) continue;
      i.snr_reset = false;
      sdb_engine_t *ie = engine_of(i);
      if (i.open && i.snr_on && i.engine_handle >= 0 && ie) sdb_engine_reset_snr(ie, i.engine_handle, i.snr_reset_sigma);
    }
  }

  // SPEC TI.4: the live changes requested since the last block, on the engines that run the next one
  void apply_tv_params()
  {
    for (auto &i : insps) {
      if (!i.tv_live) continue;
      i.tv_live = false;
      sdb_engine_t *ie = engine_of(i);
      if (i.open && i.tv_on && i.engine_handle >= 0 && ie) sdb_engine_set_tv_params(ie, i.engine_handle, &i.tv);
    }
  }

  // kind=TV inspector messages (SPEC TI.3): one per block whose feed completed a frame, after the block's SAMPLES, FAC
  // and SNR messages
  void publish_tv()
  {
    for (auto &i : insps) {
      sdb_engine_t *ie = engine_of(i);
      if (!i.open || !i.tv_on || i.engine_handle < 0 || !ie) continue;
      sdb_tv_status st;
      if (sdb_engine_read_tv(ie, i.engine_handle, nullptr, &st) || !st.completed) continue;
      const size_t px = (size_t) st.width * st.height;
      float *frame = (float *) malloc(px * sizeof(float));
      if (!frame || sdb_engine_read_tv(ie, i.engine_handle, frame, nullptr)) { free(frame); continue; }
      sdb_analyzer_inspector_msg *m = inspector_msg(SDB_INSPECTOR_MSGKIND_TV, i.handle, i.inspector_id,
                                                    kClassNames[i.cls]);
      m->samp_rate = (uint64_t) i.fs; m->fs = (float) rate; m->equiv_fs = i.fs;
      m->tv = st; m->tv_frame = frame;
      post(SDB_ANALYZER_MESSAGE_TYPE_INSPECTOR, m);
    }
  }

  // kind=SNR inspector messages (SPEC SN): one per block in which the meter stepped, after the block's SAMPLES
  std::vector<float> snr_model;
  std::vector<uint32_t> snr_hist;
  void publish_snr()
  {
    for (auto &i : insps) {
      sdb_engine_t *ie = engine_of(i);
      if (!i.open || !i.snr_on || i.engine_handle < 0 || !ie) continue;
      sdb_snr_status st;
      snr_model.resize(i.snr.bins); snr_hist.resize(i.snr.bins);
      if (sdb_engine_read_snr(ie, i.engine_handle, snr_hist.data(), snr_model.data(), &st) || !st.stepped) continue;
      sdb_analyzer_inspector_msg *m = inspector_msg(SDB_INSPECTOR_MSGKIND_SNR, i.handle, i.inspector_id,
                                                    kClassNames[i.cls]);
      m->spectrum_size = snr_model.size(); m->samp_rate = (uint64_t) i.fs;
      m->fs = (float) rate; m->equiv_fs = i.fs; m->snr = st;
      m->spectrum_data = (float *) malloc(snr_model.size() * sizeof(float));
      memcpy(m->spectrum_data, snr_model.data(), snr_model.size() * sizeof(float));
      m->snr_histogram = (uint32_t *) malloc(snr_hist.size() * sizeof(uint32_t));
      memcpy(m->snr_histogram, snr_hist.data(), snr_hist.size() * sizeof(uint32_t));
      post(SDB_ANALYZER_MESSAGE_TYPE_INSPECTOR, m);
    }
  }

  // MESSAGE_TYPE_CHANNEL at channel_update_int cadence of signal time
  void publish_channels()
  {
    if (!(params.channel_update_int > 0)) return;
    chan_credit += (double) block / rate;
    if (chan_credit + 1e-12 >= params.channel_update_int) {
      chan_credit = fmod(chan_credit, params.channel_update_int);
      std::vector<sdb_detected_channel> ch(256);
      uint32_t total = 0;
      if (params.channel_hold_int > 0) {
        // SPEC KT: the tracked list, and each track as a sigutils_channel with its smoothed S0
        std::vector<sdb_tracked_channel> tr(256);
        const long nc = sdb_engine_read_tracked_channels(eng.get(), 0, src.freq, tr.data(), tr.size(), &total, nullptr);
        if (nc < 0) return;
        for (long i = 0; i < nc; ++i) {
          sdb_detected_channel &c = ch[i];
          const sdb_tracked_channel &t = tr[i];
          c.fc = t.fc; c.f_lo = t.f_lo; c.f_hi = t.f_hi; c.bw = t.bw; c.snr = t.snr; c.S0 = t.S0; c.N0 = t.N0;
          c.bin_lo = t.bin_lo; c.bin_hi = t.bin_hi;
        }
        sdb_analyzer_channel_msg *m = (sdb_analyzer_channel_msg *) calloc(1, sizeof(*m));
        m->channel_count = (uint32_t) nc;
        m->channel_list = (sdb_detected_channel *) malloc(std::max<long>(1, nc) * sizeof(sdb_detected_channel));
        memcpy(m->channel_list, ch.data(), (size_t) nc * sizeof(sdb_detected_channel));
        m->tracked_list = (sdb_tracked_channel *) malloc(std::max<long>(1, nc) * sizeof(sdb_tracked_channel));
        memcpy(m->tracked_list, tr.data(), (size_t) nc * sizeof(sdb_tracked_channel));
        post(SDB_ANALYZER_MESSAGE_TYPE_CHANNEL, m);
        return;
      }
      long nc = sdb_engine_read_channels(eng.get(), 0, src.freq, ch.data(), ch.size(), &total);
      if (nc >= 0) {
        sdb_analyzer_channel_msg *m = (sdb_analyzer_channel_msg *) calloc(1, sizeof(*m));
        m->channel_count = (uint32_t) nc;
        m->channel_list = (sdb_detected_channel *) malloc(std::max<long>(1, nc) * sizeof(sdb_detected_channel));
        memcpy(m->channel_list, ch.data(), (size_t) nc * sizeof(sdb_detected_channel));
        post(SDB_ANALYZER_MESSAGE_TYPE_CHANNEL, m);
      }
    }
  }

  // re-plan, read, baseband filters, feed, pacing, then the block's messages
  bool step()
  {
    const size_t N = (size_t) params.detector_params.window_size;
    if (block % N) block = std::max<size_t>(N, (block / N) * N);     // after a PARAMS change
    if (buf.size() != block) buf.resize(block);
    if (decim > 1 && raw.size() < block * decim) {    // first block, or a PARAMS change that grew the block
      dec.reset();
      raw.resize(block * decim);
      dec.reset(sdb_decimator_new(src.device, 1, decim, src.read ? SDB_FORMAT_FLOAT32 : src.input_format, raw.size()));
      if (!dec) return init_failure();
    }
    if (plan_dirty && !rebuild()) return init_failure();
    apply_snr_resets();
    apply_tv_params();
    bool on_device = false;                      // the decimated block is only in the decimator's device output
    if (!read_block(on_device) || !run_filters(on_device) || !feed(on_device)) return false;
    pace();
    publish_psd();
    publish_symbols();
    publish_fac();
    publish_snr();
    publish_tv();
    publish_spectra();
    publish_channels();
    return true;
  }

  void run()
  {
    // the mode is the one the analyzer was created with: a later SET_PARAMS does not switch it
    const bool wide = params.mode == SDB_ANALYZER_MODE_WIDE_SPECTRUM;
    sdb_source_info *si = (sdb_source_info *) calloc(1, sizeof(*si));
    si->source_samp_rate = (uint64_t) src.samp_rate; si->effective_samp_rate = (uint64_t) rate;
    si->frequency = src.freq; si->seekable = !wide && !src.read;
    post(SDB_ANALYZER_MESSAGE_TYPE_SOURCE_INFO, si);
    if (wide) { hop_min = params.min_freq; hop_max = params.max_freq; }
    t0 = std::chrono::steady_clock::now();
    for (;;) {
      { std::lock_guard<std::mutex> l(cmd_m); if (halt_req) break; }
      handle_cmds();
      if (!(wide ? sweep() : step())) break;
    }
    for (auto &i : insps)                                // what the watermark still holds back goes out with the end
      if (i.has_id && pending.count(i.handle)) deliver(i, nullptr, nullptr, 0, true);
    subs.clear(); eng.reset(); dec.reset();              // released before the exit status is posted
    post_status(exit_type, 0, exit_type == SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR ? sdb_last_error() : nullptr);
  }
};

extern "C" sdb_analyzer_t *sdb_analyzer_new(const sdb_analyzer_params *params, const sdb_source_config *src)
{
  if (!params || !src) return nullptr;
  if (sdb_device_count() <= 0) return nullptr;   // sdb_last_error() is set by the engine on first use; no CPU fallback
  const uint64_t N = params->detector_params.window_size;
  if (N < 16 || (N & (N - 1)) || !(src->samp_rate > 0) || (!src->read && !src->data)) return nullptr;
  if (src->input_format < SDB_FORMAT_FLOAT32 || src->input_format > SDB_FORMAT_SIGNED16) return nullptr;
  if (params->psd_detector < SDB_PSD_DETECTOR_DEFAULT || params->psd_detector > SDB_PSD_DETECTOR_NEG_PEAK) {
    fail("psd_detector must be SDB_PSD_DETECTOR_DEFAULT, _POS_PEAK or _NEG_PEAK, got " +
         std::to_string(params->psd_detector));
    return nullptr;
  }
  if (!(params->spectrum_update_int >= 0.0f) || !std::isfinite(params->spectrum_update_int)) {
    fail("spectrum_update_int must be a finite number of seconds >= 0");
    return nullptr;
  }
  if (!(params->channel_hold_int >= 0.0f) || !std::isfinite(params->channel_hold_int)) {
    fail("channel_hold_int must be a finite number of seconds >= 0");
    return nullptr;
  }
  const uint32_t D = src->decimation ? src->decimation : 1;
  if (D > SDB_DECIMATION_MAX) {
    fail("source decimation must be at most " + std::to_string(SDB_DECIMATION_MAX) + ", got " + std::to_string(D));
    return nullptr;
  }
  // a wide-spectrum hop would carry the decimator's history across a retune
  if (D > 1 && params->mode == SDB_ANALYZER_MODE_WIDE_SPECTRUM) {
    fail("source decimation is not supported in wide-spectrum mode");
    return nullptr;
  }
  sdb_analyzer *a = new sdb_analyzer();
  a->params = *params;
  a->src = *src;
  a->decim = D;
  a->rate = src->samp_rate / (double) D;
  size_t blk = src->read_size ? src->read_size : (size_t) N * 8;
  blk = std::max<size_t>(N, (blk / N) * N);
  a->block = blk;
  a->worker = std::thread([a] { a->run(); });
  return a;
}

extern "C" void *sdb_analyzer_read(sdb_analyzer_t *a, uint32_t *type)
{
  if (!a) return nullptr;
  std::unique_lock<std::mutex> l(a->mq_m);
  a->mq_cv.wait(l, [a] { return !a->mq.empty(); });
  auto m = a->mq.front();
  a->mq.pop_front();
  if (type) *type = m.first;
  return m.second;
}

extern "C" void *sdb_analyzer_read_timeout(sdb_analyzer_t *a, uint32_t *type, unsigned timeout_ms)
{
  if (!a) return nullptr;
  std::unique_lock<std::mutex> l(a->mq_m);
  if (!a->mq_cv.wait_for(l, std::chrono::milliseconds(timeout_ms), [a] { return !a->mq.empty(); })) {
    if (type) *type = 0xfffffffeu;
    return nullptr;
  }
  auto m = a->mq.front();
  a->mq.pop_front();
  if (type) *type = m.first;
  return m.second;
}

extern "C" void sdb_analyzer_dispose_message(uint32_t type, void *ptr)
{
  if (!ptr) return;
  switch (type) {
    case SDB_ANALYZER_MESSAGE_TYPE_PSD:
      free(((sdb_analyzer_psd_msg *) ptr)->psd_data); break;
    case SDB_ANALYZER_MESSAGE_TYPE_SAMPLES:
      free(((sdb_analyzer_sample_batch_msg *) ptr)->samples);
      free(((sdb_analyzer_sample_batch_msg *) ptr)->symbols); break;
    case SDB_ANALYZER_MESSAGE_TYPE_INSPECTOR:
      free(((sdb_analyzer_inspector_msg *) ptr)->class_name);
      free(((sdb_analyzer_inspector_msg *) ptr)->spectrum_data);
      free(((sdb_analyzer_inspector_msg *) ptr)->snr_histogram);
      free(((sdb_analyzer_inspector_msg *) ptr)->tv_frame); break;
    case SDB_ANALYZER_MESSAGE_TYPE_CHANNEL:
      free(((sdb_analyzer_channel_msg *) ptr)->channel_list);
      free(((sdb_analyzer_channel_msg *) ptr)->tracked_list); break;
    case SDB_ANALYZER_MESSAGE_TYPE_EOS:
    case SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR:
    case SDB_ANALYZER_MESSAGE_TYPE_SOURCE_INIT:
    case SDB_WORKER_MSG_TYPE_HALT:
      free(((sdb_analyzer_status_msg *) ptr)->err_msg); break;
    default: break;
  }
  free(ptr);
}

extern "C" void sdb_analyzer_req_halt(sdb_analyzer_t *a)
{
  if (!a) return;
  std::lock_guard<std::mutex> l(a->cmd_m);
  a->halt_req = true;
}

extern "C" void sdb_analyzer_destroy(sdb_analyzer_t *a)
{
  if (!a) return;
  sdb_analyzer_req_halt(a);
  if (a->worker.joinable()) a->worker.join();
  for (auto &m : a->mq) sdb_analyzer_dispose_message(m.first, m.second);
  delete a;
}

static int push_cmd(sdb_analyzer_t *a, Cmd &&c)
{
  if (!a) return -1;
  std::lock_guard<std::mutex> l(a->cmd_m);
  a->cmds.push_back(std::move(c));
  return 0;
}

extern "C" int sdb_analyzer_open_ex_async(sdb_analyzer_t *a, const char *class_name, const sdb_sigutils_channel *ch,
                                          int precise, int32_t parent, uint32_t req_id)
{
  if (!class_name || !ch) return -1;
  if (parent < -1) return -1;
  // parent >= 0: sub-carrier inspection (Default/GenericInspector/GenericInspector.cpp:502-525); the channel is
  // given relative to the parent's channel centre, at the parent's equivalent sample rate
  Cmd c; c.kind = Cmd::OPEN; c.req_id = req_id; c.cls = class_name; c.channel = *ch; c.precise = precise;
  c.parent = parent;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_inspector_id_async(sdb_analyzer_t *a, int32_t handle, uint32_t inspector_id, uint32_t req_id)
{
  Cmd c; c.kind = Cmd::SET_ID; c.req_id = req_id; c.handle = handle; c.inspector_id = inspector_id;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_inspector_config_async(sdb_analyzer_t *a, int32_t handle, const sdb_inspector_config *cfg,
                                                       uint32_t req_id)
{
  if (!cfg) return -1;
  Cmd c; c.kind = Cmd::SET_CONFIG; c.req_id = req_id; c.handle = handle; c.cfg = *cfg;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_close_async(sdb_analyzer_t *a, int32_t handle, uint32_t req_id)
{
  Cmd c; c.kind = Cmd::CLOSE; c.req_id = req_id; c.handle = handle;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_inspector_watermark_async(sdb_analyzer_t *a, int32_t handle, uint64_t watermark,
                                                          uint32_t req_id)
{
  Cmd c; c.kind = Cmd::SET_WATERMARK; c.req_id = req_id; c.handle = handle; c.value = (double) watermark;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_history_size(sdb_analyzer_t *a, uint64_t samples)
{
  if (samples > (1ull << 31)) return -1;
  Cmd c; c.kind = Cmd::SET_HISTORY; c.value = (double) samples;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_replay(sdb_analyzer_t *a, int enabled)
{
  Cmd c; c.kind = Cmd::REPLAY; c.enabled = enabled;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_hop_range(sdb_analyzer_t *a, double min_freq, double max_freq)
{
  if (min_freq > max_freq) return -1;
  Cmd c; c.kind = Cmd::SET_HOP_RANGE; c.value = min_freq; c.value2 = max_freq;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_rel_bandwidth(sdb_analyzer_t *a, float rel_bw)
{
  Cmd c; c.kind = Cmd::SET_REL_BW; c.value = rel_bw;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_buffering_size(sdb_analyzer_t *a, uint64_t samples)
{
  Cmd c; c.kind = Cmd::SET_BUFFERING; c.value = (double) samples;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_sweep_strategy(sdb_analyzer_t *a, int strategy)
{
  if (strategy != SDB_SWEEP_STRATEGY_STOCHASTIC && strategy != SDB_SWEEP_STRATEGY_PROGRESSIVE) return -1;
  Cmd c; c.kind = Cmd::SET_STRATEGY; c.enabled = strategy;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_spectrum_partitioning(sdb_analyzer_t *a, int partitioning)
{
  if (partitioning != SDB_SPECTRUM_PARTITIONING_DISCRETE && partitioning != SDB_SPECTRUM_PARTITIONING_CONTINUOUS) return -1;
  Cmd c; c.kind = Cmd::SET_PARTITIONING; c.enabled = partitioning;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_seek(sdb_analyzer_t *a, const struct timeval *pos)
{
  if (!a || !pos || a->src.read || !a->src.data) return -1;      // seekable sources only (source_info.seekable)
  Cmd c; c.kind = Cmd::SEEK; c.value = (double) pos->tv_sec + 1e-6 * (double) pos->tv_usec;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_inspector_freq_overridable(sdb_analyzer_t *a, int32_t handle, double freq)
{
  Cmd c; c.kind = Cmd::SET_FREQ; c.handle = handle; c.value = freq;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_inspector_bandwidth_overridable(sdb_analyzer_t *a, int32_t handle, double bw)
{
  Cmd c; c.kind = Cmd::SET_BANDWIDTH; c.handle = handle; c.value = bw;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_dc_remove(sdb_analyzer_t *a, int enabled)
{
  Cmd c; c.kind = Cmd::SET_DC_REMOVE; c.enabled = enabled;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_iq_reverse(sdb_analyzer_t *a, int enabled)
{
  Cmd c; c.kind = Cmd::SET_IQ_REVERSE; c.enabled = enabled;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_throttle_async(sdb_analyzer_t *a, uint64_t samp_rate, uint32_t req_id)
{
  Cmd c; c.kind = Cmd::SET_THROTTLE; c.req_id = req_id; c.value = (double) samp_rate;
  return push_cmd(a, std::move(c));
}
// suscan_analyzer_register_baseband_filter_with_prio (Suscan/Analyzer.cpp:137-143): filters run in ascending priority
// value, registration order among equals; the plain registration uses priority 0
extern "C" int sdb_analyzer_register_baseband_filter_prio(sdb_analyzer_t *a, sdb_baseband_filter_fn fn, void *priv,
                                                          int64_t prio)
{
  if (!a || !fn) return -1;
  std::lock_guard<std::mutex> l(a->cmd_m);
  auto it = a->bb_filters.begin();
  while (it != a->bb_filters.end() && it->prio <= prio) ++it;
  a->bb_filters.insert(it, { fn, priv, prio });
  return 0;
}
extern "C" int sdb_analyzer_register_baseband_filter(sdb_analyzer_t *a, sdb_baseband_filter_fn fn, void *priv)
{
  return sdb_analyzer_register_baseband_filter_prio(a, fn, priv, 0);
}
// signal time of the source in seconds since its start (suscan_analyzer_get_source_time, Suscan/Analyzer.cpp:145-149)
extern "C" double sdb_analyzer_get_source_time(const sdb_analyzer_t *a)
{
  return a ? (double) a->total_samples_pub.load() / a->src.samp_rate : 0.0;
}
// current configuration of an open inspector (what a GET_CONFIG reply would carry); -1 if the handle is not open
extern "C" int sdb_analyzer_get_inspector_config(sdb_analyzer_t *a, int32_t handle, sdb_inspector_config *cfg)
{
  if (!a || !cfg) return -1;
  std::lock_guard<std::mutex> l(a->insp_m);
  const Insp *i = a->open_insp(handle);
  if (!i) return -1;
  *cfg = i->cfg;
  return 0;
}
extern "C" int sdb_analyzer_inspector_set_spectrum_async(sdb_analyzer_t *a, int32_t handle, uint32_t spectsrc_id,
                                                         uint32_t req_id)
{
  Cmd c; c.kind = Cmd::SET_SPECTRUM; c.req_id = req_id; c.handle = handle; c.aux_id = spectsrc_id;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_inspector_set_fac_async(sdb_analyzer_t *a, int32_t handle, const sdb_fac_params *p,
                                                    uint32_t req_id)
{
  Cmd c; c.kind = Cmd::SET_FAC; c.req_id = req_id; c.handle = handle;
  c.enabled = p ? 1 : 0;
  if (p) c.fac = *p;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_inspector_set_snr_async(sdb_analyzer_t *a, int32_t handle, const sdb_snr_params *p,
                                                    uint32_t req_id)
{
  Cmd c; c.kind = Cmd::SET_SNR; c.req_id = req_id; c.handle = handle;
  c.enabled = p ? 1 : 0;
  if (p) c.snr = *p;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_inspector_reset_snr_async(sdb_analyzer_t *a, int32_t handle, float sigma, uint32_t req_id)
{
  Cmd c; c.kind = Cmd::RESET_SNR; c.req_id = req_id; c.handle = handle; c.snr.sigma = sigma;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_inspector_set_tv_async(sdb_analyzer_t *a, int32_t handle, const sdb_tv_tab_params *p,
                                                   uint32_t req_id)
{
  Cmd c; c.kind = Cmd::SET_TV; c.req_id = req_id; c.handle = handle;
  c.enabled = p ? 1 : 0;
  if (p) c.tv = *p;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_inspector_estimator_cmd_async(sdb_analyzer_t *a, int32_t handle, uint32_t estimator_id,
                                                          int enabled, uint32_t req_id)
{
  Cmd c; c.kind = Cmd::ESTIMATOR_CMD; c.req_id = req_id; c.handle = handle; c.aux_id = estimator_id; c.enabled = enabled;
  return push_cmd(a, std::move(c));
}
extern "C" int sdb_analyzer_set_params_async(sdb_analyzer_t *a, const sdb_analyzer_params *p, uint32_t req_id)
{
  if (!p) return -1;
  const uint64_t N = p->detector_params.window_size;
  if (N < 16 || (N & (N - 1))) return -1;
  if (p->psd_detector < SDB_PSD_DETECTOR_DEFAULT || p->psd_detector > SDB_PSD_DETECTOR_NEG_PEAK) return -1;
  if (!(p->spectrum_update_int >= 0.0f) || !std::isfinite(p->spectrum_update_int)) return -1;
  if (!(p->channel_hold_int >= 0.0f) || !std::isfinite(p->channel_hold_int)) return -1;
  Cmd c; c.kind = Cmd::SET_PARAMS; c.req_id = req_id; c.params = *p;
  return push_cmd(a, std::move(c));
}
extern "C" uint64_t sdb_analyzer_get_samp_rate(const sdb_analyzer_t *a) { return a ? (uint64_t) a->rate : 0; }
extern "C" float sdb_analyzer_get_measured_samp_rate(const sdb_analyzer_t *a) { return a ? (float) a->measured_rate.load() : 0; }
