// spectsched_tu.cpp -- TEST INFRASTRUCTURE.  The inspector tab's spectrum through the suscan names (include/analyzer/
// *.h, libsuscan.so): suscan_analyzer_open_async, suscan_analyzer_inspector_set_spectrum_async (the GUI's spectrum
// source combo, Suscan/Analyzer.cpp:539-548) and the kind = SPECTRUM inspector messages.  The shim runs the analyzer
// with the GUI's 100 ms spectrum period.  Three inspectors from block 2 on: a "raw" one (handle 0) whose SAMPLES are
// the channel stream, a "psk" one on the same channel (handle 1) and a wide "psk" one (handle 2), both with the "psd"
// source.
#include <analyzer/analyzer.h>

#include <condition_variable>
#include <mutex>
#include <string.h>

namespace {
// A source whose first read waits until the test has queued its requests, so that they all take effect at the end of
// block 1.
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

// raw[raw_cap]: the raw inspector's samples; narrow[narrow_cap][4096]: the narrow channel's spectra; counts[0..2] =
// raw samples, narrow spectra, wide spectra (all counted past the caps); sizes[0..1] = the narrow and wide spectrum
// sizes seen (0 = none; -1 = sizes differ).  Returns 0, or < 0 on failure.
extern "C" int tu_spectrum_session(const SUCOMPLEX *iq, size_t n, unsigned samp_rate, unsigned fft_size, size_t block,
                                   double fc_narrow, double bw_narrow, double fc_wide, double bw_wide, SUCOMPLEX *raw,
                                   size_t raw_cap, float *narrow, size_t narrow_cap, uint64_t *counts, int64_t *sizes)
{
  struct suscan_analyzer_params params = suscan_analyzer_params_INITIALIZER;
  params.mode = SUSCAN_ANALYZER_MODE_CHANNEL;
  params.detector_params.window_size = fft_size;
  params.detector_params.window = SU_CHANNEL_DETECTOR_WINDOW_BLACKMANN_HARRIS;
  params.psd_update_int = 1;
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
  struct sigutils_channel nc = sigutils_channel_INITIALIZER, wc = sigutils_channel_INITIALIZER;
  nc.fc = fc_narrow; nc.f_lo = -bw_narrow / 2; nc.f_hi = bw_narrow / 2; nc.bw = (SUFLOAT) bw_narrow;
  wc.fc = fc_wide; wc.f_lo = -bw_wide / 2; wc.f_hi = bw_wide / 2; wc.bw = (SUFLOAT) bw_wide;
  int result = 0;
  const uint32_t psd = 1;      // index 1 of the GUI's source combo ("psd"; 0 is "none")
  if (!suscan_analyzer_open_async(a, "raw", &nc, 1) || !suscan_analyzer_open_async(a, "psk", &nc, 2) ||
      !suscan_analyzer_open_async(a, "psk", &wc, 3) || !suscan_analyzer_set_inspector_id_async(a, 0, 0x70u, 4) ||
      !suscan_analyzer_set_inspector_id_async(a, 1, 0x71u, 5) || !suscan_analyzer_set_inspector_id_async(a, 2, 0x72u, 6) ||
      !suscan_analyzer_inspector_set_spectrum_async(a, 1, psd, 7) || !suscan_analyzer_inspector_set_spectrum_async(a, 2, psd, 8))
    result = -4;
  {
    std::lock_guard<std::mutex> l(gate.m);
    gate.go = true; gate.cv.notify_all();
  }
  counts[0] = counts[1] = counts[2] = 0;
  sizes[0] = sizes[1] = 0;
  auto note = [](int64_t &seen, SUSCOUNT size) { if (seen == 0) seen = (int64_t) size; else if (seen != (int64_t) size) seen = -1; };
  for (bool done = false; !done;) {
    uint32_t type = 0;
    void *p = suscan_analyzer_read(a, &type);
    if (type == SUSCAN_ANALYZER_MESSAGE_TYPE_SAMPLES) {
      const struct suscan_analyzer_sample_batch_msg *s = (const struct suscan_analyzer_sample_batch_msg *) p;
      if (s->inspector_id == 0x70u)
        for (SUSCOUNT i = 0; i < s->sample_count; ++i, ++counts[0])
          if (counts[0] < raw_cap) raw[counts[0]] = s->samples[i];
    } else if (type == SUSCAN_ANALYZER_MESSAGE_TYPE_INSPECTOR) {
      const struct suscan_analyzer_inspector_msg *m = (const struct suscan_analyzer_inspector_msg *) p;
      if (m->kind == SUSCAN_ANALYZER_INSPECTOR_MSGKIND_SPECTRUM && m->spectrum_data && m->spectrum_size) {
        if (m->inspector_id == 0x71u) {
          note(sizes[0], m->spectrum_size);
          if (counts[1] < narrow_cap && m->spectrum_size == 4096)
            memcpy(narrow + counts[1] * 4096, m->spectrum_data, 4096 * sizeof(float));
          ++counts[1];
        } else if (m->inspector_id == 0x72u) {
          note(sizes[1], m->spectrum_size);
          ++counts[2];
        }
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
