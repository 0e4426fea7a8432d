// reference_tu.cpp -- test translation unit for the drop-in boundary (SURVEY.md 8(b)).
//
// Qt-free restatement of the CALLING code of the reference, compiled against include/sigutils/*.h and
// include/analyzer/*.h and linked with libsigutils.so / libsuscan.so (tests/test_gpu_shim.py builds it with g++):
//   * CostasTask      -- the constructor / work() pair of Tasks/CostasRecoveryTask.cpp:36-61 with the member layout of
//                        include/CostasRecoveryTask.h:29-41 (`su_costas_t costas = su_costas_INITIALIZER`), plus the
//                        PLL, AGC, carrier-xlator, Gardner (WaveSampler FREQUENCY path) and LPF (specttuner) tasks in
//                        the same shape (Tasks/PLLSyncTask.cpp:36,53-56, Tasks/AGCTask.cpp:41-53,70-73,
//                        Tasks/CarrierXlator.cpp:36-37,57-60, Tasks/WaveSampler.cpp:60-66,188-205, Tasks/LPFTask.cpp:52-107);
//   * AnalyzerSession -- Suscan/Analyzer.cpp:63-115 (reader loop, std::thread in place of QThread), :459-495
//                        (open_ex / set_inspector_config / set_inspector_id), :601-638 (construction with a
//                        caller-owned suscan_mq, halt, join, destroy) and the OPEN -> SET_ID handshake of
//                        Suscan/AnalyzerRequestTracker.cpp:138-157;
//   * mq / messages   -- Suscan/MQ.cpp:28-43 (caller-owned queue: init, read, finalize), the shared_ptr deleter of
//                        Suscan/Message.cpp:46 and the getters of Suscan/Messages/SamplesMessage.cpp and
//                        StatusMessage.cpp (a status message is disposed as SUSCAN_ANALYZER_MESSAGE_TYPE_INTERNAL).
// Every sigutils / suscan call below is written as the reference writes it; only the Qt scaffolding is gone.
#include <sigutils/types.h>
#include <sigutils/sampling.h>
#include <sigutils/ncqo.h>
#include <sigutils/pll.h>
#include <sigutils/agc.h>
#include <sigutils/clock.h>
#include <sigutils/iir.h>
#include <sigutils/taps.h>
#include <sigutils/specttuner.h>
#include <sigutils/tvproc.h>
#include <analyzer/analyzer.h>

#include <algorithm>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>
#include <string.h>

#define SU_ATTEMPT(expr) do { if (!(expr)) throw std::runtime_error(#expr); } while (0)   // include/Suscan/Compat.h:28-36
#define BLOCK_LENGTH 4096

// ---------------------------------------------------------------------------------------------- Tasks/
class CostasTask {
  const SUCOMPLEX *origin = nullptr;
  SUCOMPLEX *destination = nullptr;
  size_t length, p = 0;
  su_costas_t costas = su_costas_INITIALIZER;
  bool costasInitialized = false;
public:
  CostasTask(const SUCOMPLEX *data, SUCOMPLEX *destination, size_t length, SUFLOAT tau, SUFLOAT loopbw,
             enum sigutils_costas_kind kind)
  {
    SUFLOAT bw = 1. / tau;
    this->origin = data; this->destination = destination; this->length = length;
    SU_ATTEMPT(su_costas_init(&this->costas, kind, 0, bw, 3, loopbw));
    this->costasInitialized = true;
  }
  bool work(void)
  {
    size_t amount = this->length - this->p;
    size_t p = this->p;
    if (amount > BLOCK_LENGTH) amount = BLOCK_LENGTH;
    while (amount--) {
      this->destination[p] = su_costas_feed(&this->costas, this->origin[p]);
      ++p;
    }
    this->p = p;
    return this->p < this->length;
  }
  // the same block through the device twin: state in, state out
  bool workBulk(void)
  {
    size_t amount = this->length - this->p;
    if (amount > BLOCK_LENGTH) amount = BLOCK_LENGTH;
    SU_ATTEMPT(su_costas_feed_bulk(&this->costas, this->origin + this->p, this->destination + this->p, amount));
    this->p += amount;
    return this->p < this->length;
  }
  ~CostasTask() { if (this->costasInitialized) su_costas_finalize(&this->costas); }
};

extern "C" int tu_costas_task(const SUCOMPLEX *data, SUCOMPLEX *dst, size_t n, float tau, float loopbw, int kind, int bulk)
{
  try {
    CostasTask t(data, dst, n, tau, loopbw, (enum sigutils_costas_kind) kind);
    if (bulk) while (t.workBulk()) ; else while (t.work()) ;
    return 0;
  } catch (std::exception &) { return -1; }
}

extern "C" int tu_pll_task(const SUCOMPLEX *data, SUCOMPLEX *dst, size_t n, float bw, int bulk)
{
  su_pll_t pll = su_pll_INITIALIZER;
  if (!su_pll_init(&pll, 0, bw)) return -1;
  size_t p = 0;
  while (p < n) {
    size_t amount = n - p > BLOCK_LENGTH ? BLOCK_LENGTH : n - p;
    if (bulk) { if (!su_pll_track_bulk(&pll, data + p, dst + p, amount)) return -1; p += amount; }
    else while (amount--) { dst[p] = su_pll_track(&pll, data[p]); ++p; }
  }
  su_pll_finalize(&pll);
  return 0;
}

extern "C" int tu_agc_task(const SUCOMPLEX *data, SUCOMPLEX *dst, size_t n, float tau)
{
  su_agc_t agc = su_agc_INITIALIZER;
  struct su_agc_params agc_params = su_agc_params_INITIALIZER;
#define AGC_FAST_RISE_FRAC (2 * 3.9062e-1)           // Tasks/AGCTask.cpp:22-28
  agc_params.fast_rise_t = tau * AGC_FAST_RISE_FRAC;
  agc_params.fast_fall_t = tau * (2 * AGC_FAST_RISE_FRAC);
  agc_params.slow_rise_t = tau * (10 * AGC_FAST_RISE_FRAC);
  agc_params.slow_fall_t = tau * (10 * (2 * AGC_FAST_RISE_FRAC));
  agc_params.hang_max    = tau * (AGC_FAST_RISE_FRAC * 5);
  if (!su_agc_init(&agc, &agc_params)) return -1;
  for (size_t p = 0; p < n; ++p) dst[p] = su_agc_feed(&agc, data[p]);
  su_agc_finalize(&agc);
  return 0;
}

extern "C" int tu_xlate_task(const SUCOMPLEX *data, SUCOMPLEX *dst, size_t n, float relFreq, float phase, int bulk)
{
  su_ncqo_t ncqo;
  su_ncqo_init(&ncqo, -relFreq);
  su_ncqo_set_phase(&ncqo, -phase);
  if (bulk) return su_ncqo_mix_bulk(&ncqo, data, dst, n) ? 0 : -1;
  for (size_t p = 0; p < n; ++p) dst[p] = data[p] * su_ncqo_read(&ncqo);
  return 0;
}

// WaveSampler, Gardner branch, FREQUENCY space: quadrature demodulation inside the feed loop
extern "C" long tu_gardner_task(const SUCOMPLEX *data, size_t n, float loopGain, float bnor, SUCOMPLEX *out, size_t cap)
{
  su_clock_detector_t cd = su_clock_detector_INITIALIZER;
  if (su_clock_detector_init(&cd, loopGain, bnor, BLOCK_LENGTH) == -1) return -1;
  SUCOMPLEX prev = 0, x;
  size_t p = 0; long total = 0;
  std::vector<SUCOMPLEX> block(BLOCK_LENGTH);
  while (p < n) {
    size_t amount = n - p > BLOCK_LENGTH ? BLOCK_LENGTH : n - p;
    while (amount--) {
      x = data[p++];
      su_clock_detector_feed(&cd, x * SU_C_CONJ(prev));
      prev = x;
    }
    SUSDIFF count = su_clock_detector_read(&cd, block.data(), BLOCK_LENGTH);
    for (SUSDIFF i = 0; i < count && (size_t) total < cap; ++i) out[total++] = block[(size_t) i];
  }
  su_clock_detector_finalize(&cd);
  return total;
}

// LPFTask: specttuner as a low-pass filter, output length == input length (flush with zeros)
struct LpfTask {
  su_specttuner_t *stuner = nullptr;
  su_specttuner_channel_t *schan = nullptr;
  SUCOMPLEX *destination; size_t length, q = 0;
  static SUBOOL onData(const struct sigutils_specttuner_channel *, void *privdata, const SUCOMPLEX *data, SUSCOUNT size)
  {
    LpfTask *task = reinterpret_cast<LpfTask *>(privdata);
    size_t avail = task->length - task->q;
    if (size > avail) size = avail;
    memcpy(task->destination + task->q, data, size * sizeof(SUCOMPLEX));
    task->q += size;
    return SU_TRUE;
  }
};
extern "C" int tu_lpf_task(const SUCOMPLEX *data, SUCOMPLEX *dst, size_t n, float bw)
{
  struct sigutils_specttuner_params params = sigutils_specttuner_params_INITIALIZER;
  struct sigutils_specttuner_channel_params cparams = sigutils_specttuner_channel_params_INITIALIZER;
  LpfTask task; task.destination = dst; task.length = n;
  if (!(task.stuner = su_specttuner_new(&params))) return -1;
  cparams.f0       = 0;
  cparams.bw       = SU_NORM2ANG_FREQ(bw);
  cparams.guard    = 2 * PI / cparams.bw;
  cparams.privdata = &task;
  cparams.on_data  = LpfTask::onData;
  if (!(task.schan = su_specttuner_open_channel(task.stuner, &cparams))) return -1;
  size_t p = 0;
  while (p < n) {
    size_t amount = n - p > BLOCK_LENGTH ? BLOCK_LENGTH : n - p;
    if (!su_specttuner_feed_bulk(task.stuner, data + p, amount)) return -1;
    p += amount;
  }
  std::vector<SUCOMPLEX> zeros(2048, SUCOMPLEX(0, 0));
  while (task.q < n)
    if (!su_specttuner_feed_bulk(task.stuner, zeros.data(), zeros.size())) return -1;
  su_specttuner_destroy(task.stuner);
  return 0;
}

// ---------------------------------------------------------------------------------------------- TV tab worker
// TVProcessorWorker (Default/GenericInspector/TVProcessorWorker.cpp): start() :200-209, setParams() :220-239,
// work() :120-151 with its frame acknowledgement window, returnFrame() :212-218, stop() :172-184 -- the Qt signal
// `frame` is a callback here, and the display acknowledges every frame at once (TVProcessorTab::onTVProcessorFrame,
// TVProcessorTab.cpp:657-663: acknowledgeFrame + tvProcessorDisposeFrame).
#define TV_PROCESSOR_WORKER_MAX_NACK_FRAMES   100
#define TV_PROCESSOR_WORKER_MIN_NACK_RESTART   50
#define TV_PROCESSOR_MAX_PENDING_FRAMES       120
class TVWorker {
  struct sigutils_tv_processor_params defaultParams;
  su_tv_processor_t *processor = nullptr;
  bool blocked = false;
  SUSCOUNT frameCount = 0, maxProcessingBlock = 0, frameAck = 0;
public:
  std::vector<std::vector<SUFLOAT>> frames;      // what the display received
  int width = 0, height = 0;
  ~TVWorker() { stop(); }
  bool start(void)
  {
    if (processor == nullptr) processor = su_tv_processor_new(&defaultParams);
    return processor != nullptr;
  }
  void stop(void)
  {
    if (processor != nullptr) {
      su_tv_processor_destroy(processor);
      processor = nullptr; frameAck = 0; frameCount = 0; blocked = false;
    }
  }
  bool setParams(sigutils_tv_processor_params params)
  {
    bool success = false;
    if (processor != nullptr) {
      if (su_tv_processor_set_params(processor, &params)) success = true;
    } else {
      success = true;
    }
    if (success) {
      defaultParams = params;
      maxProcessingBlock = static_cast<SUSCOUNT>(TV_PROCESSOR_MAX_PENDING_FRAMES * params.line_len * params.frame_lines);
    }
    return success;
  }
  void onFrame(struct sigutils_tv_frame_buffer *frame)
  {
    ++frameAck;                                   // acknowledgeFrame
    width = frame->width; height = frame->height;
    frames.emplace_back(frame->buffer, frame->buffer + (size_t) frame->width * frame->height);
    if (processor != nullptr) su_tv_processor_return_frame(processor, frame);   // returnFrame
    else su_tv_frame_buffer_destroy(frame);
  }
  void work(const SUFLOAT *samples, SUSCOUNT size)
  {
    SUSCOUNT currAck, diff;
    bool frameSent = false;
    if (processor != nullptr) {
      if (size > maxProcessingBlock) size = maxProcessingBlock;
      while (size-- > 0) {
        if (su_tv_processor_feed(processor, *samples++)) {
          if (!frameSent) {
            currAck = frameAck;
            if (currAck > frameCount) frameCount = currAck;
            diff = frameCount - currAck;
            if (blocked) blocked = diff > TV_PROCESSOR_WORKER_MIN_NACK_RESTART;
            else blocked = diff > TV_PROCESSOR_WORKER_MAX_NACK_FRAMES;
            if (!blocked) {
              ++frameCount;
              onFrame(su_tv_processor_take_frame(processor));
              frameSent = true;
            }
          }
        }
      }
    }
  }
};

// feeds `n` samples in blocks of `block` (one work() call per pushed buffer, TVProcessorWorker::process :188-198);
// out: up to cap frames of height x width.  Returns the number of frames the display received, -1 on a refused start.
extern "C" long tu_tv_worker(const struct sigutils_tv_processor_params *params, const SUFLOAT *x, size_t n, size_t block,
                             SUFLOAT *out, size_t cap, int *width, int *height)
{
  TVWorker w;
  if (!w.setParams(*params) || !w.start()) return -1;
  for (size_t p = 0; p < n; p += block) w.work(x + p, std::min(block, n - p));
  *width = w.width; *height = w.height;
  const size_t px = (size_t) w.width * w.height;
  for (size_t f = 0; f < w.frames.size() && f < cap; ++f) memcpy(out + f * px, w.frames[f].data(), px * sizeof(SUFLOAT));
  return (long) w.frames.size();
}

// ---------------------------------------------------------------------------------------------- Suscan::Analyzer
class AnalyzerSession {
  struct suscan_mq mq;
  suscan_analyzer_t *instance = nullptr;
  std::thread asyncThread;
  std::mutex m; std::condition_variable cv;
  bool finished = false;
  uint32_t exitType = 0;
public:
  std::vector<SUCOMPLEX> samples; std::vector<uint8_t> symbols;
  std::vector<float> lastPsd; size_t psdCount = 0;
  SUHANDLE handle = -1; uint32_t inspectorId = 0x5167u; bool opened = false, idSet = false, configAcked = false;
  float equivFs = 0; int openKind = -1;

  void run()   // AsyncThread::run
  {
    void *data = nullptr;
    uint32_t type = 0;
    bool running = true;
    do {
      type = -1;
      data = suscan_analyzer_read(this->instance, &type);
      switch (type) {
        case SUSCAN_ANALYZER_MESSAGE_TYPE_SOURCE_INFO:
        case SUSCAN_ANALYZER_MESSAGE_TYPE_INSPECTOR:
        case SUSCAN_ANALYZER_MESSAGE_TYPE_PSD:
        case SUSCAN_ANALYZER_MESSAGE_TYPE_SAMPLES:
        case SUSCAN_ANALYZER_MESSAGE_TYPE_SOURCE_INIT:
        case SUSCAN_ANALYZER_MESSAGE_TYPE_INTERNAL:
        case SUSCAN_ANALYZER_MESSAGE_TYPE_PARAMS:
          this->captureMessage(type, data);
          break;
        case SUSCAN_WORKER_MSG_TYPE_HALT:
        case SUSCAN_ANALYZER_MESSAGE_TYPE_EOS:
        case SUSCAN_ANALYZER_MESSAGE_TYPE_READ_ERROR:
          running = false;
          suscan_analyzer_dispose_message(type, data);
          break;
        default:
          suscan_analyzer_dispose_message(type, data);
          data = nullptr;
      }
    } while (running);
    std::lock_guard<std::mutex> l(m);
    finished = true; exitType = type;
    cv.notify_all();
  }

  void captureMessage(uint32_t type, void *data)
  {
    std::unique_lock<std::mutex> l(m);
    if (type == SUSCAN_ANALYZER_MESSAGE_TYPE_PSD) {
      struct suscan_analyzer_psd_msg *msg = (struct suscan_analyzer_psd_msg *) data;
      lastPsd.assign(msg->psd_data, msg->psd_data + msg->psd_size);
      ++psdCount;
    } else if (type == SUSCAN_ANALYZER_MESSAGE_TYPE_SAMPLES) {
      struct suscan_analyzer_sample_batch_msg *msg = (struct suscan_analyzer_sample_batch_msg *) data;
      if (msg->inspector_id == inspectorId) {
        samples.insert(samples.end(), msg->samples, msg->samples + msg->sample_count);
        if (msg->symbols) symbols.insert(symbols.end(), msg->symbols, msg->symbols + msg->sample_count);
      }
    } else if (type == SUSCAN_ANALYZER_MESSAGE_TYPE_INSPECTOR) {
      struct suscan_analyzer_inspector_msg *msg = (struct suscan_analyzer_inspector_msg *) data;
      switch (msg->kind) {
        case SUSCAN_ANALYZER_INSPECTOR_MSGKIND_OPEN:            // AnalyzerRequestTracker.cpp:138-151
          handle = msg->handle; equivFs = msg->equiv_fs; opened = true; openKind = (int) msg->kind;
          l.unlock();
          suscan_analyzer_set_inspector_id_async(this->instance, msg->handle, inspectorId, 1001);
          l.lock();
          break;
        case SUSCAN_ANALYZER_INSPECTOR_MSGKIND_SET_ID: idSet = true; break;
        case SUSCAN_ANALYZER_INSPECTOR_MSGKIND_SET_CONFIG: configAcked = true; break;
        default: openKind = (int) msg->kind; break;
      }
    }
    cv.notify_all();
    l.unlock();
    suscan_analyzer_dispose_message(type, data);
  }

  AnalyzerSession(const struct suscan_analyzer_params &params, suscan_source_config_t *config)
  {
    SU_ATTEMPT(suscan_mq_init(&mq));
    SU_ATTEMPT(this->instance = suscan_analyzer_new(&params, config, &mq));
    this->asyncThread = std::thread([this] { this->run(); });
  }

  void openEx(std::string const &inspClass, SUFREQ fc, SUFREQ fLow, SUFREQ fHigh, bool precise, SUHANDLE parent, uint32_t id)
  {
    struct sigutils_channel c_ch = sigutils_channel_INITIALIZER;
    c_ch.fc   = fc;
    c_ch.ft   = 0;
    c_ch.f_lo = fLow;
    c_ch.f_hi = fHigh;
    c_ch.bw   = (SUFLOAT) (fHigh - fLow);
    SU_ATTEMPT(suscan_analyzer_open_ex_async(this->instance, inspClass.c_str(), &c_ch, precise ? SU_TRUE : SU_FALSE,
                                             parent, id));
  }
  void setInspectorConfig(SUHANDLE h, const suscan_config_t *cfg, uint32_t id)
  {
    SU_ATTEMPT(suscan_analyzer_set_inspector_config_async(this->instance, h, cfg, id));
  }
  template <typename F> bool waitFor(F pred, int ms = 20000)
  {
    std::unique_lock<std::mutex> l(m);
    return cv.wait_for(l, std::chrono::milliseconds(ms), [&] { return pred() || finished; }) && pred();
  }
  bool waitFinished(int ms = 60000)
  {
    std::unique_lock<std::mutex> l(m);
    return cv.wait_for(l, std::chrono::milliseconds(ms), [&] { return finished; });
  }
  uint32_t exitReason() { return exitType; }

  ~AnalyzerSession()
  {
    if (this->instance != nullptr) {
      suscan_analyzer_req_halt(this->instance);
      if (this->asyncThread.joinable()) this->asyncThread.join();
      suscan_analyzer_destroy(this->instance);
      this->instance = nullptr;
    }
    suscan_mq_finalize(&mq);
  }
};

// A source back-end that hands out one block per permission, so that the test knows at which block boundary every
// request took effect (requests are handled between blocks, as in suscan's worker loop)
struct GatedSource {
  const SUCOMPLEX *iq; size_t n, pos = 0;
  std::mutex m; std::condition_variable cv, cvp; size_t allowed = 0, calls = 0; bool parked = false;
  void release(size_t blocks) { std::lock_guard<std::mutex> l(m); allowed = blocks; cv.notify_all(); }
  // the analyzer's worker handles requests, THEN reads: once it is parked in read() a request sent now takes effect
  // after the block about to be released -- without this the test raced the worker's request loop
  void waitParked(void) { std::unique_lock<std::mutex> l(m); cvp.wait(l, [this] { return parked && !(calls < allowed); }); }
  static SUSDIFF read(void *priv, SUCOMPLEX *dst, SUSCOUNT max)
  {
    GatedSource *g = reinterpret_cast<GatedSource *>(priv);
    std::unique_lock<std::mutex> l(g->m);
    if (!(g->calls < g->allowed)) {
      g->parked = true; g->cvp.notify_all();
      g->cv.wait(l, [g] { return g->calls < g->allowed; });
      g->parked = false;
    }
    ++g->calls;
    size_t take = g->n - g->pos < max ? g->n - g->pos : (size_t) max;
    memcpy(dst, g->iq + g->pos, take * sizeof(SUCOMPLEX));
    g->pos += take;
    return (SUSDIFF) take;
  }
};

// One PSK inspection session with the reference's handshake: open -> (OPEN) -> set_id -> (SET_ID) -> set_config ->
// (SET_CONFIG).  Block 1 runs without inspector, the channel exists from block 2, the configuration is live from
// block 4.  Returns the number of soft symbols (< 0: failure code).
extern "C" long tu_analyzer_session(const SUCOMPLEX *iq, size_t n, unsigned samp_rate, unsigned fft_size,
                                    size_t block, double fc, double bw, float baud, float loop_bw, SUCOMPLEX *soft,
                                    uint8_t *hard, size_t cap, float *psd_out, unsigned long *psd_count)
{
  try {
    struct suscan_analyzer_params params = suscan_analyzer_params_INITIALIZER;
    params.mode = SUSCAN_ANALYZER_MODE_CHANNEL;
    params.detector_params.window_size = fft_size;
    params.detector_params.window = SU_CHANNEL_DETECTOR_WINDOW_BLACKMANN_HARRIS;
    params.psd_update_int = 0;          // every frame
    params.channel_update_int = 0;
    GatedSource gate; gate.iq = iq; gate.n = n;
    suscan_source_config_t *config = suscan_source_config_new("file", SUSCAN_SOURCE_FORMAT_RAW_FLOAT32);
    suscan_source_config_set_samp_rate(config, samp_rate);
    suscan_source_config_set_freq(config, 100000000);
    SU_ATTEMPT(suscan_source_config_set_read_callback(config, GatedSource::read, &gate));
    suscan_source_config_set_read_size(config, (SUSCOUNT) block);
    long result;
    {
      AnalyzerSession s(params, config);
      gate.waitParked();                                          // block 1 runs without inspector
      s.openEx("psk", fc, -bw / 2, bw / 2, false, -1, 1000);
      gate.release(1);
      if (!s.waitFor([&] { return s.opened; })) return -2;       // captureMessage answers with set_inspector_id
      gate.release(2);
      if (!s.waitFor([&] { return s.idSet; })) return -3;
      suscan_config_t *cfg = suscan_inspector_config_new("psk", s.equivFs);
      SU_ATTEMPT(suscan_config_set_integer(cfg, "afc.costas-order", SUSCAN_INSPECTOR_CARRIER_CONTROL_COSTAS_4));
      SU_ATTEMPT(suscan_config_set_integer(cfg, "afc.bits-per-symbol", 2));
      SU_ATTEMPT(suscan_config_set_float(cfg, "afc.loop-bw", loop_bw));
      SU_ATTEMPT(suscan_config_set_integer(cfg, "mf.type", SUSCAN_INSPECTOR_MATCHED_FILTER_MANUAL));
      SU_ATTEMPT(suscan_config_set_float(cfg, "mf.roll-off", 0.35f));
      SU_ATTEMPT(suscan_config_set_integer(cfg, "clock.type", SUSCAN_INSPECTOR_BAUDRATE_CONTROL_GARDNER));
      SU_ATTEMPT(suscan_config_set_float(cfg, "clock.baud", baud));
      SU_ATTEMPT(suscan_config_set_float(cfg, "clock.gain", 0.1f));
      SU_ATTEMPT(suscan_config_set_bool(cfg, "clock.running", SU_TRUE));
      gate.waitParked();                                          // block 3 still runs the default configuration
      s.setInspectorConfig(s.handle, cfg, 1002);
      suscan_config_destroy(cfg);
      gate.release(3);
      if (!s.waitFor([&] { return s.configAcked; })) return -4;
      gate.release((size_t) -1);
      if (!s.waitFinished()) return -5;
      if (s.exitReason() != SUSCAN_ANALYZER_MESSAGE_TYPE_EOS) return -6;
      result = (long) s.samples.size();
      for (size_t i = 0; i < s.samples.size() && i < cap; ++i) { soft[i] = s.samples[i]; if (i < s.symbols.size()) hard[i] = s.symbols[i]; }
      if (psd_out && !s.lastPsd.empty()) memcpy(psd_out, s.lastPsd.data(), s.lastPsd.size() * sizeof(float));
      if (psd_count) *psd_count = s.psdCount;
    }
    suscan_source_config_destroy(config);
    return result;
  } catch (std::exception &) { return -1; }
}

// A SAMPLES batch posted with suscan_mq_write comes back through the caller-owned queue and is released by the
// message deleter.  Returns the sample count (< 0: failure code).
extern "C" long tu_mq_samples(const SUCOMPLEX *samples, unsigned long n, unsigned inspector_id, SUCOMPLEX *out,
                              unsigned *id_out)
{
  struct suscan_mq mq;
  if (!suscan_mq_init(&mq)) return -3;
  auto *m = (struct suscan_analyzer_sample_batch_msg *) calloc(1, sizeof(struct suscan_analyzer_sample_batch_msg));
  m->inspector_id = inspector_id; m->sample_count = n;
  m->samples = (SUCOMPLEX *) malloc(n * sizeof(SUCOMPLEX));
  memcpy(m->samples, samples, n * sizeof(SUCOMPLEX));
  long ret = -1;
  if (!suscan_mq_write(&mq, SUSCAN_ANALYZER_MESSAGE_TYPE_SAMPLES, m)) {
    suscan_analyzer_dispose_message(SUSCAN_ANALYZER_MESSAGE_TYPE_SAMPLES, m);
  } else {
    uint32_t type = 0;
    void *p = suscan_mq_read(&mq, &type);
    std::shared_ptr<void> msg(p, [=](void *ptr) { suscan_analyzer_dispose_message(type, ptr); });
    if (type != SUSCAN_ANALYZER_MESSAGE_TYPE_SAMPLES || p != m) {
      ret = -2;
    } else {
      auto *s = static_cast<struct suscan_analyzer_sample_batch_msg *>(p);
      *id_out = s->inspector_id;
      memcpy(out, s->samples, s->sample_count * sizeof(SUCOMPLEX));
      ret = (long) s->sample_count;
    }
  }
  suscan_mq_finalize(&mq);
  return ret;
}

// StatusMessage: code and text (empty for a NULL err_msg), disposed by the deleter.  Returns the code.
extern "C" int tu_status_message(int code, const char *text, char *text_out, size_t cap)
{
  auto *m = (struct suscan_analyzer_status_msg *) calloc(1, sizeof(struct suscan_analyzer_status_msg));
  m->code = code; m->err_msg = text ? strdup(text) : nullptr;
  std::shared_ptr<void> msg(m, [](void *ptr) { suscan_analyzer_dispose_message(SUSCAN_ANALYZER_MESSAGE_TYPE_INTERNAL, ptr); });
  const std::string s = m->err_msg == nullptr ? "" : m->err_msg;
  strncpy(text_out, s.c_str(), cap - 1); text_out[cap - 1] = 0;
  return m->code;
}
