// power_tu.cpp -- TEST INFRASTRUCTURE.  The RMS tab's use of the "power" inspector class through the suscan names
// (include/analyzer/*.h, libsuscan.so): suscan_analyzer_open_async("power"), a bag from suscan_inspector_config_new
// with power.integrate-samples written by suscan_config_set_integer (the path Suscan::Config::set(name, uint64_t)
// takes, Default/RMSInspector/RMSInspector.cpp:404-416, 438-439), suscan_analyzer_set_inspector_config_async and the
// SAMPLES messages, whose real parts are the power readings (:562-563).
#include <analyzer/analyzer.h>

#include <condition_variable>
#include <mutex>
#include <string.h>

namespace {
// A source whose first read waits until the test has queued its requests, so that they all take effect at the end of
// block 1: the inspector runs from block 2 on.
struct Gate {
  const SUCOMPLEX *iq; size_t n, pos = 0;
  std::mutex m; std::condition_variable cv;
  bool parked = false, go = false;
  static SUSDIFF read(void *priv, SUCOMPLEX *dst, SUSCOUNT max)
  {
    Gate *g = reinterpret_cast<Gate *>(priv);
    {
      std::unique_lock<std::mutex> l(g->m);
      g->parked = true; g->cv.notify_all();
      g->cv.wait(l, [g] { return g->go; });
    }
    const size_t take = g->n - g->pos < max ? g->n - g->pos : (size_t) max;
    memcpy(dst, g->iq + g->pos, take * sizeof(SUCOMPLEX));
    g->pos += take;
    return (SUSDIFF) take;
  }
};
}  // namespace

// -> the number of power readings written to out (real parts of the SAMPLES), or < 0 on failure
extern "C" long tu_power_session(const SUCOMPLEX *iq, size_t n, unsigned samp_rate, unsigned fft_size, size_t block,
                                 double fc, double bw, uint64_t integrate_samples, float *out, size_t cap)
{
  struct suscan_analyzer_params params = suscan_analyzer_params_INITIALIZER;
  params.mode = SUSCAN_ANALYZER_MODE_CHANNEL;
  params.detector_params.window_size = fft_size;
  params.detector_params.window = SU_CHANNEL_DETECTOR_WINDOW_BLACKMANN_HARRIS;
  params.psd_update_int = 0;
  params.channel_update_int = 0;
  Gate gate; gate.iq = iq; gate.n = n;
  suscan_source_config_t *config = suscan_source_config_new("file", SUSCAN_SOURCE_FORMAT_RAW_FLOAT32);
  suscan_source_config_set_samp_rate(config, samp_rate);
  if (!suscan_source_config_set_read_callback(config, Gate::read, &gate)) return -1;
  suscan_source_config_set_read_size(config, (SUSCOUNT) block);
  struct suscan_mq mq;
  if (!suscan_mq_init(&mq)) return -2;
  suscan_analyzer_t *a = suscan_analyzer_new(&params, config, &mq);
  if (!a) return -3;
  {
    std::unique_lock<std::mutex> l(gate.m);
    gate.cv.wait(l, [&] { return gate.parked; });
  }
  struct sigutils_channel ch = sigutils_channel_INITIALIZER;
  ch.fc = fc; ch.f_lo = -bw / 2; ch.f_hi = bw / 2; ch.bw = (SUFLOAT) bw;
  long result = 0;
  suscan_config_t *cfg = suscan_inspector_config_new("power", 1.0f);
  if (!cfg || !suscan_analyzer_open_async(a, "power", &ch, 1) ||
      !suscan_config_set_integer(cfg, "power.integrate-samples", integrate_samples) ||
      !suscan_analyzer_set_inspector_config_async(a, 0, cfg, 2) || !suscan_analyzer_set_inspector_id_async(a, 0, 0x77u, 3))
    result = -4;
  if (cfg) suscan_config_destroy(cfg);
  {
    std::lock_guard<std::mutex> l(gate.m);
    gate.go = true; gate.cv.notify_all();
  }
  for (bool done = false; !done;) {
    uint32_t type = 0;
    void *p = suscan_analyzer_read(a, &type);
    if (type == SUSCAN_ANALYZER_MESSAGE_TYPE_SAMPLES && result >= 0) {
      const struct suscan_analyzer_sample_batch_msg *s = (const struct suscan_analyzer_sample_batch_msg *) p;
      for (SUSCOUNT i = 0; i < s->sample_count; ++i) {
        if (SU_C_IMAG(s->samples[i]) != 0 || s->symbols[i] != 0) { result = -5; break; }
        if ((size_t) result < cap) out[result] = SU_C_REAL(s->samples[i]);
        ++result;
      }
    } else if (type == SUSCAN_ANALYZER_MESSAGE_TYPE_EOS || type == SUSCAN_ANALYZER_MESSAGE_TYPE_READ_ERROR) {
      if (type != SUSCAN_ANALYZER_MESSAGE_TYPE_EOS && result >= 0) result = -6;
      done = true;
    }
    suscan_analyzer_dispose_message(type, p);
  }
  suscan_analyzer_destroy(a);
  suscan_mq_finalize(&mq);
  suscan_source_config_destroy(config);
  return result;
}
