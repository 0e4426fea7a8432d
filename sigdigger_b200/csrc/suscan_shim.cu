// suscan_shim.cu -- libsuscan.so: the suscan names the reference's Suscan::Analyzer wrapper calls
// (include/analyzer/*.h; Suscan/Analyzer.cpp:111-638, Suscan/MQ.cpp:25-44, Suscan/Config.cpp, Suscan/Source.cpp) on
// top of sdb_analyzer_* (include/sigdigger_b200.h).  Pure host glue: the caller-owned message queue, the typed
// key / value bag of the inspector configuration, the source configuration object, and a pump thread that turns
// the sdb messages into the suscan payload structs the reference dereferences.  All computation is behind
// sdb_analyzer_new (GPU only; suscan_analyzer_new returns NULL without a device).
#include "../../include/sigdigger_b200.h"
#include <analyzer/analyzer.h>
#include <analyzer/version.h>

#include <condition_variable>
#include <chrono>
#include <deque>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include <math.h>
#include <stdlib.h>
#include <string.h>

// ---------------------------------------------------------------------------------------------- message queue
namespace {
struct MqImpl {
  std::mutex m;
  std::condition_variable cv;
  std::deque<std::pair<uint32_t, void *>> q;
};
char *dupstr(const char *s) { if (!s) return nullptr; size_t n = strlen(s) + 1; char *p = (char *) malloc(n); memcpy(p, s, n); return p; }
}  // namespace

extern "C" {

unsigned int suscan_abi_version(void) { return 1; }
const char *suscan_api_version(void) { return "0.3.0"; }
const char *suscan_pkgversion(void) { return "0.3.0-sigdigger_b200"; }

SUBOOL suscan_mq_init(struct suscan_mq *mq) { if (!mq) return SU_FALSE; mq->impl = new MqImpl(); return SU_TRUE; }
void suscan_mq_finalize(struct suscan_mq *mq)
{
  if (!mq || !mq->impl) return;
  delete (MqImpl *) mq->impl;        // payloads still queued belong to whoever knows their type: the analyzer drains first
  mq->impl = nullptr;
}
SUBOOL suscan_mq_write(struct suscan_mq *mq, uint32_t type, void *priv)
{
  MqImpl *i = (MqImpl *) mq->impl;
  std::lock_guard<std::mutex> l(i->m);
  i->q.emplace_back(type, priv);
  i->cv.notify_all();
  return SU_TRUE;
}
SUBOOL suscan_mq_write_urgent(struct suscan_mq *mq, uint32_t type, void *priv)
{
  MqImpl *i = (MqImpl *) mq->impl;
  std::lock_guard<std::mutex> l(i->m);
  i->q.emplace_front(type, priv);
  i->cv.notify_all();
  return SU_TRUE;
}
void *suscan_mq_read(struct suscan_mq *mq, uint32_t *type)
{
  MqImpl *i = (MqImpl *) mq->impl;
  std::unique_lock<std::mutex> l(i->m);
  i->cv.wait(l, [i] { return !i->q.empty(); });
  auto e = i->q.front(); i->q.pop_front();
  if (type) *type = e.first;
  return e.second;
}
void *suscan_mq_read_w_type(struct suscan_mq *mq, uint32_t type)
{
  MqImpl *i = (MqImpl *) mq->impl;
  std::unique_lock<std::mutex> l(i->m);
  for (;;) {
    for (auto it = i->q.begin(); it != i->q.end(); ++it)
      if (it->first == type) { void *p = it->second; i->q.erase(it); return p; }
    i->cv.wait(l);
  }
}
SUBOOL suscan_mq_poll(struct suscan_mq *mq, uint32_t *type, void **priv)
{
  MqImpl *i = (MqImpl *) mq->impl;
  std::lock_guard<std::mutex> l(i->m);
  if (i->q.empty()) return SU_FALSE;
  auto e = i->q.front(); i->q.pop_front();
  if (type) *type = e.first;
  if (priv) *priv = e.second;
  return SU_TRUE;
}
SUBOOL suscan_mq_timedread(struct suscan_mq *mq, uint32_t *type, void **priv, unsigned int timeout_ms)
{
  MqImpl *i = (MqImpl *) mq->impl;
  std::unique_lock<std::mutex> l(i->m);
  if (!i->cv.wait_for(l, std::chrono::milliseconds(timeout_ms), [i] { return !i->q.empty(); })) return SU_FALSE;
  auto e = i->q.front(); i->q.pop_front();
  if (type) *type = e.first;
  if (priv) *priv = e.second;
  return SU_TRUE;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------- config bag
// Vocabulary: SURVEY.md 8(b) "Inspector config vocabulary" (Default/GenericInspector/InspectorCtl/*.cpp,
// Default/Audio/AudioProcessor.cpp:257-265).  kind: i integer, f float, b bool.
namespace {
struct KeyDef { const char *name; char kind; const char *desc; };
const KeyDef kGain[] = { { "agc.enabled", 'b', "Automatic gain control" }, { "agc.gain", 'f', "Manual gain (dB)" } };
const KeyDef kAfc[] = { { "afc.costas-order", 'i', "Constellation order (Costas loop)" },
                        { "afc.bits-per-symbol", 'i', "Bits per symbol" },
                        { "afc.offset", 'f', "Carrier offset (Hz)" }, { "afc.loop-bw", 'f', "Loop bandwidth (Hz)" } };
const KeyDef kFsk[] = { { "fsk.bits-per-symbol", 'i', "Bits per FSK tone" }, { "fsk.phase", 'f', "Quadrature demodulator phase" },
                        { "fsk.quad-demod", 'b', "Use traditional argument-based quadrature demodulator" } };
const KeyDef kAsk[] = { { "ask.bits-per-symbol", 'i', "Bits per ASK level" }, { "ask.use-pll", 'b', "Center carrier using PLL" },
                        { "ask.offset", 'f', "Carrier offset (Hz)" }, { "ask.loop-bw", 'f', "PLL cutoff frequency (Hz)" },
                        { "ask.channel", 'i', "Demodulated channel" } };
const KeyDef kMf[] = { { "mf.type", 'i', "Matched filter configuration" }, { "mf.roll-off", 'f', "Roll-off factor" } };
const KeyDef kEq[] = { { "equalizer.type", 'i', "Equalizer configuration" }, { "equalizer.rate", 'f', "Equalizer update rate" },
                       { "equalizer.locked", 'b', "Equalizer has corrected channel distortion" } };
const KeyDef kClock[] = { { "clock.type", 'i', "Clock recovery method" }, { "clock.baud", 'f', "Symbol rate (baud)" },
                          { "clock.gain", 'f', "Gardner's algorithm loop gain" }, { "clock.phase", 'f', "Symbol phase" },
                          { "clock.running", 'b', "Clock recovery is running" } };
const KeyDef kAudio[] = { { "audio.volume", 'f', "Audio gain" }, { "audio.cutoff", 'f', "Audio low pass filter" },
                          { "audio.sample-rate", 'i', "Audio sample rate" }, { "audio.demodulator", 'i', "Analog demodulator to use" },
                          { "audio.squelch", 'b', "Enable squelch" }, { "audio.squelch-level", 'f', "Squelch level" },
                          { "agc.ts", 'f', "AGC time scale" } };
// the RMS tool (Default/RMSInspector/RMSInspector.cpp:404-416, 438-439): Suscan::Config::set(name, uint64_t)
const KeyDef kPower[] = { { "power.integrate-samples", 'i', "Samples per integrated power reading" } };
template <size_t N> void add(std::vector<KeyDef> &v, const KeyDef (&k)[N]) { v.insert(v.end(), k, k + N); }

std::vector<KeyDef> keys_of(int cls)
{
  std::vector<KeyDef> v;
  switch (cls) {
    case SDB_INSP_PSK: add(v, kGain); add(v, kAfc); add(v, kMf); add(v, kEq); add(v, kClock); break;
    case SDB_INSP_FSK: add(v, kGain); add(v, kFsk); add(v, kMf); add(v, kClock); break;
    case SDB_INSP_ASK: add(v, kGain); add(v, kAsk); add(v, kMf); add(v, kClock); break;
    case SDB_INSP_AUDIO: add(v, kGain); add(v, kAudio); break;
    case SDB_INSP_POWER: add(v, kPower); break;
    default: break;
  }
  return v;
}
int class_of(const char *n)
{
  if (!n) return -1;
  if (!strcmp(n, "psk")) return SDB_INSP_PSK;
  if (!strcmp(n, "fsk")) return SDB_INSP_FSK;
  if (!strcmp(n, "ask")) return SDB_INSP_ASK;
  if (!strcmp(n, "audio")) return SDB_INSP_AUDIO;
  if (!strcmp(n, "raw")) return SDB_INSP_RAW;
  if (!strcmp(n, "power")) return SDB_INSP_POWER;
  return -1;
}
const char *kClassNames[] = { "psk", "fsk", "ask", "audio", "raw", "power" };
constexpr int kClasses = sizeof(kClassNames) / sizeof(kClassNames[0]);

// one immutable descriptor per class, built on first use
const suscan_config_desc_t *desc_of(int cls)
{
  static std::mutex m;
  static suscan_config_desc_t *descs[kClasses] = {};
  if (cls < 0 || cls >= kClasses) return nullptr;
  std::lock_guard<std::mutex> l(m);
  if (!descs[cls]) {
    auto keys = keys_of(cls);
    suscan_config_desc_t *d = (suscan_config_desc_t *) calloc(1, sizeof(*d));
    d->global_name = dupstr(kClassNames[cls]);
    d->field_count = (unsigned) keys.size();
    d->field_list = (struct suscan_field **) calloc(keys.size() ? keys.size() : 1, sizeof(*d->field_list));
    for (size_t i = 0; i < keys.size(); ++i) {
      struct suscan_field *f = (struct suscan_field *) calloc(1, sizeof(*f));
      f->type = keys[i].kind == 'f' ? SUSCAN_FIELD_TYPE_FLOAT : keys[i].kind == 'b' ? SUSCAN_FIELD_TYPE_BOOLEAN
                                                                                    : SUSCAN_FIELD_TYPE_INTEGER;
      f->optional = SU_TRUE; f->name = dupstr(keys[i].name); f->desc = dupstr(keys[i].desc);
      d->field_list[i] = f;
    }
    descs[cls] = d;
  }
  return descs[cls];
}
}  // namespace

extern "C" {

suscan_config_t *suscan_config_new(const suscan_config_desc_t *desc)
{
  if (!desc) return nullptr;
  suscan_config_t *c = (suscan_config_t *) calloc(1, sizeof(*c));
  c->desc = desc;
  c->values = (struct suscan_field_value **) calloc(desc->field_count ? desc->field_count : 1, sizeof(*c->values));
  for (unsigned i = 0; i < desc->field_count; ++i) {
    c->values[i] = (struct suscan_field_value *) calloc(1, sizeof(struct suscan_field_value));
    c->values[i]->field = desc->field_list[i];
  }
  return c;
}
suscan_config_t *suscan_config_dup(const suscan_config_t *config)
{
  if (!config) return nullptr;
  suscan_config_t *c = suscan_config_new(config->desc);
  for (unsigned i = 0; i < config->desc->field_count; ++i) *c->values[i] = *config->values[i];
  return c;
}
void suscan_config_destroy(suscan_config_t *config)
{
  if (!config) return;
  for (unsigned i = 0; i < config->desc->field_count; ++i) free(config->values[i]);
  free(config->values);
  free(config);
}
struct suscan_field_value *suscan_config_get_value(const suscan_config_t *cfg, const char *name)
{
  if (!cfg || !name) return nullptr;
  for (unsigned i = 0; i < cfg->desc->field_count; ++i)
    if (!strcmp(cfg->desc->field_list[i]->name, name)) return cfg->values[i];
  return nullptr;
}
SUBOOL suscan_config_set_integer(suscan_config_t *cfg, const char *name, uint64_t value)
{
  struct suscan_field_value *v = suscan_config_get_value(cfg, name);
  if (!v || v->field->type != SUSCAN_FIELD_TYPE_INTEGER) return SU_FALSE;
  v->as_int = value; v->set = SU_TRUE;
  return SU_TRUE;
}
SUBOOL suscan_config_set_float(suscan_config_t *cfg, const char *name, SUFLOAT value)
{
  struct suscan_field_value *v = suscan_config_get_value(cfg, name);
  if (!v || v->field->type != SUSCAN_FIELD_TYPE_FLOAT) return SU_FALSE;
  v->as_float = value; v->set = SU_TRUE;
  return SU_TRUE;
}
SUBOOL suscan_config_set_bool(suscan_config_t *cfg, const char *name, SUBOOL value)
{
  struct suscan_field_value *v = suscan_config_get_value(cfg, name);
  if (!v || v->field->type != SUSCAN_FIELD_TYPE_BOOLEAN) return SU_FALSE;
  v->as_bool = value ? SU_TRUE : SU_FALSE; v->set = SU_TRUE;
  return SU_TRUE;
}
SUBOOL suscan_config_set_string(suscan_config_t *cfg, const char *name, const char *value)
{
  struct suscan_field_value *v = suscan_config_get_value(cfg, name);
  if (!v || !value || (v->field->type != SUSCAN_FIELD_TYPE_STRING && v->field->type != SUSCAN_FIELD_TYPE_FILE)) return SU_FALSE;
  strncpy(v->as_string, value, sizeof(v->as_string) - 1); v->set = SU_TRUE;
  return SU_TRUE;
}
SUBOOL suscan_config_desc_has_prefix(const suscan_config_desc_t *desc, const char *prefix)
{
  if (!desc || !prefix) return SU_FALSE;
  const size_t n = strlen(prefix);
  for (unsigned i = 0; i < desc->field_count; ++i)
    if (!strncmp(desc->field_list[i]->name, prefix, n) && desc->field_list[i]->name[n] == '.') return SU_TRUE;
  return SU_FALSE;
}
SUBOOL suscan_config_str_to_bool(const char *s, SUBOOL deflt)
{
  if (!s) return deflt;
  if (!strcasecmp(s, "true") || !strcasecmp(s, "yes") || !strcasecmp(s, "on") || !strcmp(s, "1")) return SU_TRUE;
  if (!strcasecmp(s, "false") || !strcasecmp(s, "no") || !strcasecmp(s, "off") || !strcmp(s, "0")) return SU_FALSE;
  return deflt;
}

}  // extern "C"

namespace {
// typed struct <-> bag
void bag_from_cfg(suscan_config_t *b, const sdb_inspector_config &c)
{
  suscan_config_set_bool(b, "agc.enabled", c.agc_enabled); suscan_config_set_float(b, "agc.gain", c.agc_gain_db);
  suscan_config_set_integer(b, "afc.costas-order", c.costas_order);
  suscan_config_set_integer(b, "afc.bits-per-symbol", c.bits_per_symbol);
  suscan_config_set_float(b, "afc.offset", c.offset); suscan_config_set_float(b, "afc.loop-bw", c.loop_bw);
  suscan_config_set_integer(b, "fsk.bits-per-symbol", c.bits_per_symbol);
  suscan_config_set_float(b, "fsk.phase", c.fsk_phase); suscan_config_set_bool(b, "fsk.quad-demod", c.fsk_quad_demod);
  suscan_config_set_integer(b, "ask.bits-per-symbol", c.bits_per_symbol);
  suscan_config_set_bool(b, "ask.use-pll", c.ask_use_pll); suscan_config_set_float(b, "ask.offset", c.offset);
  suscan_config_set_float(b, "ask.loop-bw", c.loop_bw); suscan_config_set_integer(b, "ask.channel", c.ask_channel);
  suscan_config_set_integer(b, "mf.type", c.mf_type); suscan_config_set_float(b, "mf.roll-off", c.mf_rolloff);
  suscan_config_set_integer(b, "equalizer.type", c.eq_type); suscan_config_set_float(b, "equalizer.rate", c.eq_rate);
  suscan_config_set_bool(b, "equalizer.locked", c.eq_locked);
  suscan_config_set_integer(b, "clock.type", c.clock_type); suscan_config_set_float(b, "clock.baud", c.baud);
  suscan_config_set_float(b, "clock.gain", c.clock_gain); suscan_config_set_float(b, "clock.phase", c.clock_phase);
  suscan_config_set_bool(b, "clock.running", c.clock_running);
  suscan_config_set_float(b, "audio.volume", c.audio_volume); suscan_config_set_float(b, "audio.cutoff", c.audio_cutoff);
  suscan_config_set_integer(b, "audio.sample-rate", c.audio_sample_rate);
  suscan_config_set_integer(b, "audio.demodulator", c.audio_demod);
  suscan_config_set_bool(b, "audio.squelch", c.audio_squelch);
  suscan_config_set_float(b, "audio.squelch-level", c.audio_squelch_level);
  suscan_config_set_float(b, "agc.ts", c.agc_ts);
  suscan_config_set_integer(b, "power.integrate-samples", c.power_integrate_samples);
}
void cfg_from_bag(sdb_inspector_config &c, const suscan_config_t *b)
{
  auto F = [&](const char *k, float &dst) { auto *v = suscan_config_get_value(b, k); if (v) dst = v->as_float; };
  auto I = [&](const char *k, uint32_t &dst) { auto *v = suscan_config_get_value(b, k); if (v) dst = (uint32_t) v->as_int; };
  auto B = [&](const char *k, int32_t &dst) { auto *v = suscan_config_get_value(b, k); if (v) dst = v->as_bool ? 1 : 0; };
  B("agc.enabled", c.agc_enabled); F("agc.gain", c.agc_gain_db);
  I("afc.costas-order", c.costas_order); I("afc.bits-per-symbol", c.bits_per_symbol);
  F("afc.offset", c.offset); F("afc.loop-bw", c.loop_bw);
  I("fsk.bits-per-symbol", c.bits_per_symbol); F("fsk.phase", c.fsk_phase); B("fsk.quad-demod", c.fsk_quad_demod);
  I("ask.bits-per-symbol", c.bits_per_symbol); B("ask.use-pll", c.ask_use_pll); F("ask.offset", c.offset);
  F("ask.loop-bw", c.loop_bw); I("ask.channel", c.ask_channel);
  I("mf.type", c.mf_type); F("mf.roll-off", c.mf_rolloff);
  I("equalizer.type", c.eq_type); F("equalizer.rate", c.eq_rate); B("equalizer.locked", c.eq_locked);
  I("clock.type", c.clock_type); F("clock.baud", c.baud); F("clock.gain", c.clock_gain); F("clock.phase", c.clock_phase);
  B("clock.running", c.clock_running);
  F("audio.volume", c.audio_volume); F("audio.cutoff", c.audio_cutoff); I("audio.sample-rate", c.audio_sample_rate);
  I("audio.demodulator", c.audio_demod); B("audio.squelch", c.audio_squelch); F("audio.squelch-level", c.audio_squelch_level);
  F("agc.ts", c.agc_ts);
  if (auto *v = suscan_config_get_value(b, "power.integrate-samples")) c.power_integrate_samples = v->as_int;
}
}  // namespace

extern "C" {

suscan_config_t *suscan_inspector_config_new(const char *class_name, SUFLOAT equiv_fs)
{
  const int cls = class_of(class_name);
  if (cls < 0) return nullptr;
  suscan_config_t *b = suscan_config_new(desc_of(cls));
  sdb_inspector_config c;
  sdb_inspector_config_default(&c, cls, equiv_fs);
  c.clock_running = 0;                 // "by default ... no samples are being delivered" (manual p.62)
  bag_from_cfg(b, c);
  return b;
}

static const struct suscan_spectsrc_class kSpectsrc[] = {
  { "psd", "Power spectral density" }, { "cyclo", "Cyclostationary analysis" }, { "fmspect", "FM spectrum" },
  { "timediff", "Time derivative" }, { "abstimediff", "Absolute value of time derivative" },
  { "exp_2", "Signal exponentiation (2)" }, { "exp_4", "Signal exponentiation (4)" }, { "exp_8", "Signal exponentiation (8)" },
  { "fac", "Fast autocorrelation" } };
static const struct suscan_estimator_class kEstim[] = {
  { "baud-fac", "Fast autocorrelation", "clock.baud" }, { "baud-nonlinear", "Non-linear baud estimator", "clock.baud" } };
const struct suscan_spectsrc_class *suscan_spectsrc_class_lookup(const char *name)
{
  for (auto &c : kSpectsrc) if (name && !strcmp(c.name, name)) return &c;
  return nullptr;
}
const struct suscan_estimator_class *suscan_estimator_class_lookup(const char *name)
{
  for (auto &c : kEstim) if (name && !strcmp(c.name, name)) return &c;
  return nullptr;
}

SUBOOL suscan_sigutils_init(int mode) { (void) mode; return SU_TRUE; }
SUBOOL suscan_init_sources(void) { return SU_TRUE; }
SUBOOL suscan_init_estimators(void) { return SU_TRUE; }
SUBOOL suscan_init_spectsrcs(void) { return SU_TRUE; }
SUBOOL suscan_init_inspectors(void) { return SU_TRUE; }

void suscan_source_info_init(struct suscan_source_info *i) { memset(i, 0, sizeof(*i)); }
SUBOOL suscan_source_info_init_copy(struct suscan_source_info *d, const struct suscan_source_info *s)
{
  *d = *s;
  d->antenna = dupstr(s->antenna);
  d->gain_list = nullptr; d->gain_count = 0; d->antenna_list = nullptr; d->antenna_count = 0;   // none on this path
  return SU_TRUE;
}
void suscan_source_info_finalize(struct suscan_source_info *i) { free(i->antenna); memset(i, 0, sizeof(*i)); }

}  // extern "C"

// ---------------------------------------------------------------------------------------------- source config
struct suscan_source_config {
  std::string type = "file", label = SUSCAN_SOURCE_DEFAULT_NAME, path;
  enum suscan_source_format format = SUSCAN_SOURCE_FORMAT_AUTO;
  SUFREQ freq = SUSCAN_SOURCE_DEFAULT_FREQ, lnb = 0;
  unsigned int samp_rate = SUSCAN_SOURCE_DEFAULT_SAMP_RATE, average = 1;
  SUFLOAT bandwidth = SUSCAN_SOURCE_DEFAULT_BANDWIDTH, ppm = 0;
  SUBOOL loop = SU_FALSE, dc_remove = SU_FALSE, iq_balance = SU_FALSE;
  struct timeval start = { 0, 0 };
  std::map<std::string, std::string> params;
  const void *mem = nullptr; SUSCOUNT mem_len = 0;
  suscan_source_read_fn read_fn = nullptr; void *read_priv = nullptr;
  int gpu = 0; SUSCOUNT read_size = 0;
};

extern "C" {

suscan_source_config_t *suscan_source_config_new(const char *type, enum suscan_source_format format)
{
  suscan_source_config_t *c = new suscan_source_config();
  if (type) c->type = type;
  c->format = format;
  return c;
}
suscan_source_config_t *suscan_source_config_clone(const suscan_source_config_t *c) { return c ? new suscan_source_config(*c) : nullptr; }
void suscan_source_config_destroy(suscan_source_config_t *c) { delete c; }
SUBOOL suscan_source_config_set_type_format(suscan_source_config_t *c, const char *type, enum suscan_source_format f)
{ if (!c || !type) return SU_FALSE; c->type = type; c->format = f; return SU_TRUE; }
const char *suscan_source_config_get_type(const suscan_source_config_t *c) { return c->type.c_str(); }
enum suscan_source_format suscan_source_config_get_format(const suscan_source_config_t *c) { return c->format; }
SUBOOL suscan_source_config_set_label(suscan_source_config_t *c, const char *l) { c->label = l ? l : ""; return SU_TRUE; }
const char *suscan_source_config_get_label(const suscan_source_config_t *c) { return c->label.c_str(); }
SUBOOL suscan_source_config_set_path(suscan_source_config_t *c, const char *p) { c->path = p ? p : ""; return SU_TRUE; }
const char *suscan_source_config_get_path(const suscan_source_config_t *c) { return c->path.empty() ? nullptr : c->path.c_str(); }
void suscan_source_config_set_freq(suscan_source_config_t *c, SUFREQ f) { c->freq = f; }
SUFREQ suscan_source_config_get_freq(const suscan_source_config_t *c) { return c->freq; }
void suscan_source_config_set_lnb_freq(suscan_source_config_t *c, SUFREQ f) { c->lnb = f; }
SUFREQ suscan_source_config_get_lnb_freq(const suscan_source_config_t *c) { return c->lnb; }
void suscan_source_config_set_samp_rate(suscan_source_config_t *c, unsigned int r) { c->samp_rate = r; }
unsigned int suscan_source_config_get_samp_rate(const suscan_source_config_t *c) { return c->samp_rate; }
void suscan_source_config_set_average(suscan_source_config_t *c, unsigned int a) { c->average = a ? a : 1; }
unsigned int suscan_source_config_get_average(const suscan_source_config_t *c) { return c->average; }
void suscan_source_config_set_bandwidth(suscan_source_config_t *c, SUFLOAT bw) { c->bandwidth = bw; }
SUFLOAT suscan_source_config_get_bandwidth(const suscan_source_config_t *c) { return c->bandwidth; }
void suscan_source_config_set_loop(suscan_source_config_t *c, SUBOOL l) { c->loop = l; }
SUBOOL suscan_source_config_get_loop(const suscan_source_config_t *c) { return c->loop; }
void suscan_source_config_set_dc_remove(suscan_source_config_t *c, SUBOOL d) { c->dc_remove = d; }
SUBOOL suscan_source_config_get_dc_remove(const suscan_source_config_t *c) { return c->dc_remove; }
void suscan_source_config_set_iq_balance(suscan_source_config_t *c, SUBOOL d) { c->iq_balance = d; }
SUBOOL suscan_source_config_get_iq_balance(const suscan_source_config_t *c) { return c->iq_balance; }
void suscan_source_config_set_ppm(suscan_source_config_t *c, SUFLOAT p) { c->ppm = p; }
SUFLOAT suscan_source_config_get_ppm(const suscan_source_config_t *c) { return c->ppm; }
void suscan_source_config_set_start_time(suscan_source_config_t *c, struct timeval tv) { c->start = tv; }
void suscan_source_config_get_start_time(const suscan_source_config_t *c, struct timeval *tv) { if (tv) *tv = c->start; }
SUBOOL suscan_source_config_set_param(suscan_source_config_t *c, const char *k, const char *v)
{ if (!k || !v) return SU_FALSE; c->params[k] = v; return SU_TRUE; }
const char *suscan_source_config_get_param(const suscan_source_config_t *c, const char *k)
{ auto it = c->params.find(k ? k : ""); return it == c->params.end() ? nullptr : it->second.c_str(); }
void suscan_source_config_clear_params(suscan_source_config_t *c) { c->params.clear(); }
SUBOOL suscan_source_config_is_seekable(const suscan_source_config_t *c) { return c->type == "file" || c->mem ? SU_TRUE : SU_FALSE; }
SUBOOL suscan_source_config_is_real_time(const suscan_source_config_t *c) { return c->type == "file" || c->mem || c->read_fn ? SU_FALSE : SU_TRUE; }
SUBOOL suscan_source_config_file_is_valid(const suscan_source_config_t *c)
{
  if (c->path.empty()) return SU_FALSE;
  sdb_capture_info info;
  sdb_capture_t *cap = sdb_capture_open(c->path.c_str(), SDB_CONTAINER_AUTO, -1, &info);
  if (!cap) return SU_FALSE;
  sdb_capture_close(cap);
  return SU_TRUE;
}
SUBOOL suscan_source_config_set_memory(suscan_source_config_t *c, const void *data, SUSCOUNT length)
{ c->mem = data; c->mem_len = length; return SU_TRUE; }
SUBOOL suscan_source_config_set_read_callback(suscan_source_config_t *c, suscan_source_read_fn fn, void *priv)
{ c->read_fn = fn; c->read_priv = priv; return SU_TRUE; }
void suscan_source_config_set_gpu(suscan_source_config_t *c, int device) { c->gpu = device; }
void suscan_source_config_set_read_size(suscan_source_config_t *c, SUSCOUNT samples) { c->read_size = samples; }

}  // extern "C"

// ---------------------------------------------------------------------------------------------- analyzer
struct suscan_analyzer {
  sdb_analyzer_t *a = nullptr;
  struct suscan_mq *mq = nullptr;
  std::thread pump;
  sdb_capture_t *cap = nullptr;
  suscan_source_config cfg;
  struct suscan_source_info info;
  std::mutex m;
  std::map<int32_t, int> handle_class;               // handle -> SDB_INSP_* (from the OPEN replies)
  struct Bb { suscan_analyzer_baseband_filter_func_t fn; void *priv; suscan_analyzer *self; int64_t prio; };
  std::vector<Bb *> bbs;
  // tonegen source state
  double tg_phase = 0, tg_omega = 0; float tg_amp = 1, tg_noise = 0; uint32_t tg_lcg = 0x5167D166u;
};

namespace {

long cb_read(void *priv, sdb_complex *dst, size_t max)
{
  suscan_analyzer *a = (suscan_analyzer *) priv;
  return (long) a->cfg.read_fn(a->cfg.read_priv, reinterpret_cast<SUCOMPLEX *>(dst), max);
}
long cb_tonegen(void *priv, sdb_complex *dst, size_t max)
{
  // "tonegen" source (Default/SourceConfig/ToneGenSourcePage.cpp:81-87, 125-126): one complex tone at the centre
  // (offset 0) of amplitude `signal` dB over uniform noise of `noise` dB
  suscan_analyzer *a = (suscan_analyzer *) priv;
  for (size_t i = 0; i < max; ++i) {
    a->tg_lcg = a->tg_lcg * 1664525u + 1013904223u; const float u1 = (float) (a->tg_lcg >> 8) / 16777216.0f - 0.5f;
    a->tg_lcg = a->tg_lcg * 1664525u + 1013904223u; const float u2 = (float) (a->tg_lcg >> 8) / 16777216.0f - 0.5f;
    dst[i].re = a->tg_amp * (float) cos(a->tg_phase) + a->tg_noise * u1;
    dst[i].im = a->tg_amp * (float) sin(a->tg_phase) + a->tg_noise * u2;
    a->tg_phase += a->tg_omega;
    if (a->tg_phase > 6.283185307179586) a->tg_phase -= 6.283185307179586;
  }
  return (long) max;
}
int bb_trampoline(void *priv, sdb_analyzer_t *, sdb_complex *samples, uint64_t length, uint64_t offset)
{
  suscan_analyzer::Bb *b = (suscan_analyzer::Bb *) priv;
  return b->fn(b->priv, b->self, reinterpret_cast<SUCOMPLEX *>(samples), length, offset) ? 1 : 0;
}

struct sigutils_channel to_su_channel(const sdb_sigutils_channel &c)
{
  struct sigutils_channel r = sigutils_channel_INITIALIZER;
  r.fc = c.fc; r.ft = c.ft; r.f_lo = c.f_lo; r.f_hi = c.f_hi; r.bw = c.bw;
  return r;
}

// sdb message -> suscan payload (ownership of the sdb message is consumed)
void *convert(suscan_analyzer *sa, uint32_t type, void *p)
{
  switch (type) {
    case SDB_ANALYZER_MESSAGE_TYPE_PSD: {
      sdb_analyzer_psd_msg *s = (sdb_analyzer_psd_msg *) p;
      struct suscan_analyzer_psd_msg *m = (struct suscan_analyzer_psd_msg *) calloc(1, sizeof(*m));
      m->fc = s->fc; m->inspector_id = s->inspector_id; m->timestamp = s->timestamp; m->rt_time = s->rt_time;
      m->looped = s->looped; m->history_size = s->history_size; m->samp_rate = s->samp_rate;
      m->measured_samp_rate = s->measured_samp_rate; m->psd_size = s->psd_size;
      m->psd_data = s->psd_data; s->psd_data = nullptr;          // the bins move, no copy
      sdb_analyzer_dispose_message(type, s);
      return m;
    }
    case SDB_ANALYZER_MESSAGE_TYPE_SAMPLES: {
      sdb_analyzer_sample_batch_msg *s = (sdb_analyzer_sample_batch_msg *) p;
      struct suscan_analyzer_sample_batch_msg *m = (struct suscan_analyzer_sample_batch_msg *) calloc(1, sizeof(*m));
      m->inspector_id = s->inspector_id; m->sample_count = s->sample_count;
      m->samples = reinterpret_cast<SUCOMPLEX *>(s->samples); m->symbols = s->symbols;
      s->samples = nullptr; s->symbols = nullptr;
      sdb_analyzer_dispose_message(type, s);
      return m;
    }
    case SDB_ANALYZER_MESSAGE_TYPE_INSPECTOR: {
      sdb_analyzer_inspector_msg *s = (sdb_analyzer_inspector_msg *) p;
      struct suscan_analyzer_inspector_msg *m = (struct suscan_analyzer_inspector_msg *) calloc(1, sizeof(*m));
      static const int kinds[] = { SUSCAN_ANALYZER_INSPECTOR_MSGKIND_OPEN, SUSCAN_ANALYZER_INSPECTOR_MSGKIND_SET_ID,
                                   SUSCAN_ANALYZER_INSPECTOR_MSGKIND_GET_CONFIG, SUSCAN_ANALYZER_INSPECTOR_MSGKIND_SET_CONFIG,
                                   SUSCAN_ANALYZER_INSPECTOR_MSGKIND_ESTIMATOR, SUSCAN_ANALYZER_INSPECTOR_MSGKIND_SPECTRUM,
                                   SUSCAN_ANALYZER_INSPECTOR_MSGKIND_CLOSE, SUSCAN_ANALYZER_INSPECTOR_MSGKIND_INVALID_CHANNEL,
                                   SUSCAN_ANALYZER_INSPECTOR_MSGKIND_WRONG_HANDLE, SUSCAN_ANALYZER_INSPECTOR_MSGKIND_WRONG_OBJECT,
                                   SUSCAN_ANALYZER_INSPECTOR_MSGKIND_WRONG_KIND };
      m->kind = (enum suscan_analyzer_inspector_msgkind) kinds[s->kind];
      m->inspector_id = s->inspector_id; m->req_id = s->req_id; m->handle = s->handle;
      m->class_name = dupstr(s->class_name);
      m->channel = to_su_channel(s->channel);
      m->fs = (unsigned) s->fs; m->equiv_fs = s->equiv_fs; m->bandwidth = s->bandwidth; m->lo = s->lo;
      m->estimator_id = s->estimator_id; m->enabled = s->enabled; m->value = s->value;
      m->spectsrc_id = s->spectsrc_id; m->spectrum_size = s->spectrum_size; m->samp_rate = s->samp_rate;
      m->spectrum_data = s->spectrum_data; s->spectrum_data = nullptr;
      const int cls = class_of(s->class_name);
      if (s->kind == SDB_INSPECTOR_MSGKIND_OPEN || s->kind == SDB_INSPECTOR_MSGKIND_SET_CONFIG ||
          s->kind == SDB_INSPECTOR_MSGKIND_GET_CONFIG) {
        if (cls >= 0) { m->config = suscan_config_new(desc_of(cls)); bag_from_cfg(m->config, s->config); }
        m->spectsrc_count = sizeof(kSpectsrc) / sizeof(kSpectsrc[0]);
        m->spectsrc_list = (char **) calloc(m->spectsrc_count, sizeof(char *));
        for (unsigned i = 0; i < m->spectsrc_count; ++i) m->spectsrc_list[i] = dupstr(kSpectsrc[i].name);
        m->estimator_count = sizeof(kEstim) / sizeof(kEstim[0]);
        m->estimator_list = (char **) calloc(m->estimator_count, sizeof(char *));
        for (unsigned i = 0; i < m->estimator_count; ++i) m->estimator_list[i] = dupstr(kEstim[i].name);
      }
      if (s->kind == SDB_INSPECTOR_MSGKIND_OPEN && cls >= 0) {
        std::lock_guard<std::mutex> l(sa->m);
        sa->handle_class[s->handle] = cls;
      }
      sdb_analyzer_dispose_message(type, s);
      return m;
    }
    case SDB_ANALYZER_MESSAGE_TYPE_CHANNEL: {
      sdb_analyzer_channel_msg *s = (sdb_analyzer_channel_msg *) p;
      struct suscan_analyzer_channel_msg *m = (struct suscan_analyzer_channel_msg *) calloc(1, sizeof(*m));
      m->channel_count = s->channel_count;
      m->channel_list = (struct sigutils_channel **) calloc(s->channel_count ? s->channel_count : 1, sizeof(void *));
      for (unsigned i = 0; i < s->channel_count; ++i) {
        struct sigutils_channel *c = (struct sigutils_channel *) calloc(1, sizeof(*c));
        const sdb_detected_channel &d = s->channel_list[i];
        c->fc = d.fc; c->f_lo = d.f_lo; c->f_hi = d.f_hi; c->bw = (SUFLOAT) d.bw; c->snr = d.snr; c->S0 = d.S0; c->N0 = d.N0;
        // channel tracking (SPEC KT) is off unless sdb_analyzer_params.channel_hold_int is set, which
        // suscan_analyzer_params has no field for; with it on, each track's age and present fill the fields of the
        // same names
        if (s->tracked_list) { c->age = s->tracked_list[i].age; c->present = s->tracked_list[i].present; }
        m->channel_list[i] = c;
      }
      sdb_analyzer_dispose_message(type, s);
      return m;
    }
    case SDB_ANALYZER_MESSAGE_TYPE_SOURCE_INFO: {
      sdb_source_info *s = (sdb_source_info *) p;
      struct suscan_source_info *m = (struct suscan_source_info *) calloc(1, sizeof(*m));
      *m = sa->info;
      m->antenna = nullptr;
      m->source_samp_rate = s->source_samp_rate; m->effective_samp_rate = s->effective_samp_rate;
      m->measured_samp_rate = s->measured_samp_rate; m->frequency = s->frequency; m->seekable = s->seekable;
      sdb_analyzer_dispose_message(type, s);
      return m;
    }
    case SDB_ANALYZER_MESSAGE_TYPE_PARAMS: {
      sdb_analyzer_params *s = (sdb_analyzer_params *) p;
      struct suscan_analyzer_params *m = (struct suscan_analyzer_params *) calloc(1, sizeof(*m));
      struct suscan_analyzer_params def = suscan_analyzer_params_INITIALIZER;
      *m = def;
      m->mode = (enum suscan_analyzer_mode) s->mode;
      m->detector_params.window_size = s->detector_params.window_size;
      m->detector_params.window = (enum sigutils_channel_detector_window) s->detector_params.window;
      m->detector_params.alpha = s->detector_params.alpha; m->detector_params.beta = s->detector_params.beta;
      m->detector_params.gamma = s->detector_params.gamma; m->detector_params.snr = s->detector_params.snr;
      m->channel_update_int = s->channel_update_int; m->psd_update_int = s->psd_update_int;
      m->min_freq = s->min_freq; m->max_freq = s->max_freq;
      sdb_analyzer_dispose_message(type, s);
      return m;
    }
    default: {   // status-like: SOURCE_INIT, EOS, READ_ERROR, HALT
      sdb_analyzer_status_msg *s = (sdb_analyzer_status_msg *) p;
      struct suscan_analyzer_status_msg *m = (struct suscan_analyzer_status_msg *) calloc(1, sizeof(*m));
      if (s) { m->code = s->code; m->err_msg = s->err_msg; s->err_msg = nullptr; sdb_analyzer_dispose_message(type, s); }
      m->sender = sa;
      return m;
    }
  }
}

sdb_analyzer_params to_sdb_params(const struct suscan_analyzer_params *p)
{
  sdb_analyzer_params q;
  memset(&q, 0, sizeof(q));
  q.mode = p->mode;
  q.detector_params.window_size = p->detector_params.window_size;
  q.detector_params.window = p->detector_params.window;
  q.detector_params.alpha = p->detector_params.alpha; q.detector_params.beta = p->detector_params.beta;
  q.detector_params.gamma = p->detector_params.gamma; q.detector_params.snr = p->detector_params.snr;
  q.channel_update_int = p->channel_update_int; q.psd_update_int = p->psd_update_int;
  q.min_freq = p->min_freq; q.max_freq = p->max_freq;
  // the inspector spectrum's 100 ms update period (Default/GenericInspector/InspectorUI.cpp:971-975)
  q.spectrum_update_int = 0.1f;
  return q;
}

}  // namespace

extern "C" {

suscan_analyzer_t *suscan_analyzer_new(const struct suscan_analyzer_params *params, suscan_source_config_t *config,
                                       struct suscan_mq *mq)
{
  if (!params || !config || !mq || !mq->impl) return nullptr;
  if (sdb_device_count() <= 0) return nullptr;            // GPU only
  suscan_analyzer *sa = new suscan_analyzer();
  sa->mq = mq; sa->cfg = *config;
  suscan_source_info_init(&sa->info);
  sdb_source_config sc;
  memset(&sc, 0, sizeof(sc));
  // `average` is the source decimation (SPEC L): the analyzer reads samp_rate and runs at samp_rate / average
  sc.samp_rate = (double) config->samp_rate;
  sc.decimation = config->average ? config->average : 1;
  sc.freq = config->freq; sc.read_size = (size_t) config->read_size; sc.device = config->gpu;
  sc.loop = config->loop ? 1 : 0;
  static const int fmt_of[] = { -1, SDB_FORMAT_FLOAT32, SDB_FORMAT_UNSIGNED8, SDB_FORMAT_SIGNED16, SDB_FORMAT_SIGNED8, -1, -1 };
  if (config->read_fn) {
    sc.read = cb_read; sc.priv = sa; sc.input_format = SDB_FORMAT_FLOAT32;
  } else if (config->mem) {
    sc.data = (const sdb_complex *) config->mem; sc.length = (size_t) config->mem_len;
    sc.input_format = fmt_of[config->format] >= 0 ? fmt_of[config->format] : SDB_FORMAT_FLOAT32;
  } else if (config->type == "file") {
    sdb_capture_info info;
    const int container = config->format == SUSCAN_SOURCE_FORMAT_WAV ? SDB_CONTAINER_WAV
                          : config->format == SUSCAN_SOURCE_FORMAT_SIGMF ? SDB_CONTAINER_SIGMF
                          : config->format == SUSCAN_SOURCE_FORMAT_AUTO ? SDB_CONTAINER_AUTO : SDB_CONTAINER_RAW;
    sa->cap = sdb_capture_open(config->path.c_str(), container, fmt_of[config->format], &info);
    if (!sa->cap) { delete sa; return nullptr; }
    sc.data = (const sdb_complex *) sdb_capture_data(sa->cap); sc.length = (size_t) info.n_samples;
    sc.input_format = info.sample_format;
    if (info.samp_rate > 0 && (info.container != SDB_CONTAINER_RAW || (info.guessed & SDB_CAPTURE_GUESS_SAMP_RATE)))
      sc.samp_rate = info.samp_rate;
    if (info.frequency != 0) sc.freq = info.frequency;
  } else if (config->type == "tonegen") {
    const char *sg = suscan_source_config_get_param(config, "signal"), *nz = suscan_source_config_get_param(config, "noise");
    sa->tg_amp = powf(10.0f, (sg ? (float) atof(sg) : -20.0f) * 0.05f);
    sa->tg_noise = powf(10.0f, (nz ? (float) atof(nz) : -70.0f) * 0.05f);
    sc.read = cb_tonegen; sc.priv = sa; sc.input_format = SDB_FORMAT_FLOAT32;
  } else {
    delete sa; return nullptr;                            // device back-ends are outside this path
  }
  sa->info.permissions = SUSCAN_ANALYZER_PERM_ALL & ~(SUSCAN_ANALYZER_PERM_SET_GAIN | SUSCAN_ANALYZER_PERM_SET_ANTENNA |
                                                      SUSCAN_ANALYZER_PERM_SET_AGC | SUSCAN_ANALYZER_PERM_SET_PPM);
  sa->info.source_samp_rate = (SUSCOUNT) sc.samp_rate;
  sa->info.effective_samp_rate = (SUSCOUNT) (sc.samp_rate / (double) sc.decimation);
  sa->info.frequency = sc.freq; sa->info.freq_min = -3e11; sa->info.freq_max = 3e11; sa->info.lnb = config->lnb;
  sa->info.bandwidth = config->bandwidth; sa->info.dc_remove = config->dc_remove;
  sa->info.seekable = (sc.data != nullptr) ? SU_TRUE : SU_FALSE;
  sa->info.source_start = config->start;
  sdb_analyzer_params sp = to_sdb_params(params);
  sa->a = sdb_analyzer_new(&sp, &sc);
  if (!sa->a) { if (sa->cap) sdb_capture_close(sa->cap); delete sa; return nullptr; }
  sa->pump = std::thread([sa] {
    for (;;) {
      uint32_t type = 0;
      void *p = sdb_analyzer_read(sa->a, &type);
      suscan_mq_write(sa->mq, type, convert(sa, type, p));
      if (type == SDB_WORKER_MSG_TYPE_HALT || type == SDB_ANALYZER_MESSAGE_TYPE_EOS ||
          type == SDB_ANALYZER_MESSAGE_TYPE_READ_ERROR)
        break;
    }
  });
  return sa;
}

void suscan_analyzer_destroy(suscan_analyzer_t *sa)
{
  if (!sa) return;
  sdb_analyzer_req_halt(sa->a);
  if (sa->pump.joinable()) sa->pump.join();
  sdb_analyzer_destroy(sa->a);
  // whatever the caller did not read is disposed here; the queue itself belongs to the caller (Suscan/MQ.cpp:31-44)
  uint32_t type; void *p;
  while (suscan_mq_poll(sa->mq, &type, &p)) suscan_analyzer_dispose_message(type, p);
  if (sa->cap) sdb_capture_close(sa->cap);
  for (auto *b : sa->bbs) delete b;
  delete sa;
}

void *suscan_analyzer_read(suscan_analyzer_t *sa, uint32_t *type) { return suscan_mq_read(sa->mq, type); }
void *suscan_analyzer_read_timeout(suscan_analyzer_t *sa, uint32_t *type, unsigned int timeout_ms)
{
  void *p = nullptr;
  if (!suscan_mq_timedread(sa->mq, type, &p, timeout_ms)) { if (type) *type = 0xfffffffeu; return nullptr; }
  return p;
}

void suscan_analyzer_dispose_message(uint32_t type, void *ptr)
{
  if (!ptr) return;
  switch (type) {
    case SUSCAN_ANALYZER_MESSAGE_TYPE_PSD: free(((struct suscan_analyzer_psd_msg *) ptr)->psd_data); break;
    case SUSCAN_ANALYZER_MESSAGE_TYPE_SAMPLES:
      free(((struct suscan_analyzer_sample_batch_msg *) ptr)->samples);
      free(((struct suscan_analyzer_sample_batch_msg *) ptr)->symbols); break;
    case SUSCAN_ANALYZER_MESSAGE_TYPE_INSPECTOR: {
      struct suscan_analyzer_inspector_msg *m = (struct suscan_analyzer_inspector_msg *) ptr;
      free(m->class_name); free(m->spectrum_data); free(m->signal_name);
      if (m->config) suscan_config_destroy(m->config);
      for (unsigned i = 0; i < m->spectsrc_count; ++i) free(m->spectsrc_list[i]);
      for (unsigned i = 0; i < m->estimator_count; ++i) free(m->estimator_list[i]);
      free(m->spectsrc_list); free(m->estimator_list);
      break;
    }
    case SUSCAN_ANALYZER_MESSAGE_TYPE_CHANNEL: {
      struct suscan_analyzer_channel_msg *m = (struct suscan_analyzer_channel_msg *) ptr;
      for (unsigned i = 0; i < m->channel_count; ++i) free(m->channel_list[i]);
      free(m->channel_list);
      break;
    }
    case SUSCAN_ANALYZER_MESSAGE_TYPE_SOURCE_INFO: free(((struct suscan_source_info *) ptr)->antenna); break;
    case SUSCAN_ANALYZER_MESSAGE_TYPE_PARAMS: break;
    default: free(((struct suscan_analyzer_status_msg *) ptr)->err_msg); break;
  }
  free(ptr);
}

void suscan_analyzer_req_halt(suscan_analyzer_t *sa) { if (sa) sdb_analyzer_req_halt(sa->a); }
SUSCOUNT suscan_analyzer_get_samp_rate(const suscan_analyzer_t *sa) { return sa ? sdb_analyzer_get_samp_rate(sa->a) : 0; }
SUFLOAT suscan_analyzer_get_measured_samp_rate(const suscan_analyzer_t *sa) { return sa ? sdb_analyzer_get_measured_samp_rate(sa->a) : 0; }
void suscan_analyzer_get_source_time(const suscan_analyzer_t *sa, struct timeval *tv)
{
  if (!tv) return;
  const double t = sa ? sdb_analyzer_get_source_time(sa->a) : 0.0;
  tv->tv_sec = sa->info.source_start.tv_sec + (time_t) t;
  tv->tv_usec = (suseconds_t) ((t - floor(t)) * 1e6);
}
struct suscan_source_info *suscan_analyzer_get_source_info(const suscan_analyzer_t *sa)
{ return sa ? const_cast<struct suscan_source_info *>(&sa->info) : nullptr; }

// tuner-side setters: a capture has no tuner; the values are recorded so that SOURCE_INFO reflects them
SUBOOL suscan_analyzer_set_freq(suscan_analyzer_t *sa, SUFREQ freq, SUFREQ lnb) { sa->info.frequency = freq; sa->info.lnb = lnb; return SU_TRUE; }
SUBOOL suscan_analyzer_set_gain(suscan_analyzer_t *, const char *, SUFLOAT) { return SU_FALSE; }
SUBOOL suscan_analyzer_set_antenna(suscan_analyzer_t *, const char *) { return SU_FALSE; }
SUBOOL suscan_analyzer_set_bw(suscan_analyzer_t *sa, SUFLOAT bw) { sa->info.bandwidth = bw; return SU_TRUE; }
SUBOOL suscan_analyzer_set_ppm(suscan_analyzer_t *, SUFLOAT) { return SU_FALSE; }
SUBOOL suscan_analyzer_set_agc(suscan_analyzer_t *, SUBOOL) { return SU_FALSE; }
SUBOOL suscan_analyzer_set_dc_remove(suscan_analyzer_t *sa, SUBOOL r)
{ sa->info.dc_remove = r; return sdb_analyzer_set_dc_remove(sa->a, r ? 1 : 0) == 0 ? SU_TRUE : SU_FALSE; }
SUBOOL suscan_analyzer_set_iq_reverse(suscan_analyzer_t *sa, SUBOOL r)
{ sa->info.iq_reverse = r; return sdb_analyzer_set_iq_reverse(sa->a, r ? 1 : 0) == 0 ? SU_TRUE : SU_FALSE; }
SUBOOL suscan_analyzer_set_hop_range(suscan_analyzer_t *sa, SUFREQ lo, SUFREQ hi) { return sdb_analyzer_set_hop_range(sa->a, lo, hi) == 0; }
SUBOOL suscan_analyzer_set_rel_bandwidth(suscan_analyzer_t *sa, SUFLOAT r) { return sdb_analyzer_set_rel_bandwidth(sa->a, r) == 0; }
SUBOOL suscan_analyzer_set_buffering_size(suscan_analyzer_t *sa, SUSCOUNT n) { return sdb_analyzer_set_buffering_size(sa->a, n) == 0; }
SUBOOL suscan_analyzer_set_sweep_stratrgy(suscan_analyzer_t *sa, enum suscan_analyzer_sweep_strategy s)
{ return sdb_analyzer_set_sweep_strategy(sa->a, (int) s) == 0; }
SUBOOL suscan_analyzer_set_spectrum_partitioning(suscan_analyzer_t *sa, enum suscan_analyzer_spectrum_partitioning p)
{ return sdb_analyzer_set_spectrum_partitioning(sa->a, (int) p) == 0; }
SUBOOL suscan_analyzer_set_history_size(suscan_analyzer_t *sa, SUSCOUNT n) { return sdb_analyzer_set_history_size(sa->a, n) == 0; }
SUBOOL suscan_analyzer_seek(suscan_analyzer_t *sa, const struct timeval *pos) { return sdb_analyzer_seek(sa->a, pos) == 0; }
SUBOOL suscan_analyzer_replay(suscan_analyzer_t *sa, SUBOOL r) { return sdb_analyzer_replay(sa->a, r ? 1 : 0) == 0; }
SUBOOL suscan_analyzer_set_throttle_async(suscan_analyzer_t *sa, SUSCOUNT rate, uint32_t req_id)
{ return sdb_analyzer_set_throttle_async(sa->a, rate, req_id) == 0; }
SUBOOL suscan_analyzer_set_params_async(suscan_analyzer_t *sa, const struct suscan_analyzer_params *p, uint32_t req_id)
{
  if (!p) return SU_FALSE;
  sdb_analyzer_params q = to_sdb_params(p);
  return sdb_analyzer_set_params_async(sa->a, &q, req_id) == 0;
}
SUBOOL suscan_analyzer_register_baseband_filter_with_prio(suscan_analyzer_t *sa, suscan_analyzer_baseband_filter_func_t fn,
                                                          void *privdata, int64_t prio)
{
  if (!sa || !fn) return SU_FALSE;
  suscan_analyzer::Bb *b = new suscan_analyzer::Bb{ fn, privdata, sa, prio };
  sa->bbs.push_back(b);
  return sdb_analyzer_register_baseband_filter_prio(sa->a, bb_trampoline, b, prio) == 0;
}
SUBOOL suscan_analyzer_register_baseband_filter(suscan_analyzer_t *sa, suscan_analyzer_baseband_filter_func_t fn, void *privdata)
{ return suscan_analyzer_register_baseband_filter_with_prio(sa, fn, privdata, 0); }

SUBOOL suscan_analyzer_open_ex_async(suscan_analyzer_t *sa, const char *class_name, const struct sigutils_channel *ch,
                                     SUBOOL precise, SUHANDLE parent, uint32_t req_id)
{
  if (!sa || !class_name || !ch) return SU_FALSE;
  sdb_sigutils_channel c;
  c.fc = ch->fc; c.ft = ch->ft; c.f_lo = ch->f_lo; c.f_hi = ch->f_hi; c.bw = ch->bw;
  return sdb_analyzer_open_ex_async(sa->a, class_name, &c, precise ? 1 : 0, parent, req_id) == 0;
}
SUBOOL suscan_analyzer_open_async(suscan_analyzer_t *sa, const char *class_name, const struct sigutils_channel *ch, uint32_t req_id)
{ return suscan_analyzer_open_ex_async(sa, class_name, ch, SU_FALSE, -1, req_id); }
SUBOOL suscan_analyzer_close_async(suscan_analyzer_t *sa, SUHANDLE h, uint32_t req_id) { return sdb_analyzer_close_async(sa->a, h, req_id) == 0; }
SUBOOL suscan_analyzer_set_inspector_id_async(suscan_analyzer_t *sa, SUHANDLE h, uint32_t id, uint32_t req_id)
{ return sdb_analyzer_set_inspector_id_async(sa->a, h, id, req_id) == 0; }
SUBOOL suscan_analyzer_set_inspector_config_async(suscan_analyzer_t *sa, SUHANDLE h, const suscan_config_t *config, uint32_t req_id)
{
  if (!sa || !config) return SU_FALSE;
  // the bag is applied on top of the inspector's current configuration (keys the bag does not carry keep their value)
  sdb_inspector_config c;
  int cls = class_of(config->desc->global_name);
  if (cls < 0) { std::lock_guard<std::mutex> l(sa->m); auto it = sa->handle_class.find(h); cls = it == sa->handle_class.end() ? -1 : it->second; }
  if (cls < 0) cls = SDB_INSP_PSK;
  if (sdb_analyzer_get_inspector_config(sa->a, h, &c)) sdb_inspector_config_default(&c, cls, 1.0f);
  c.insp_class = cls;
  cfg_from_bag(c, config);
  return sdb_analyzer_set_inspector_config_async(sa->a, h, &c, req_id) == 0;
}
SUBOOL suscan_analyzer_set_inspector_watermark_async(suscan_analyzer_t *sa, SUHANDLE h, SUSCOUNT wm, uint32_t req_id)
{ return sdb_analyzer_set_inspector_watermark_async(sa->a, h, wm, req_id) == 0; }
SUBOOL suscan_analyzer_set_inspector_freq_overridable(suscan_analyzer_t *sa, SUHANDLE h, SUFREQ f)
{ return sdb_analyzer_set_inspector_freq_overridable(sa->a, h, f) == 0; }
SUBOOL suscan_analyzer_set_inspector_bandwidth_overridable(suscan_analyzer_t *sa, SUHANDLE h, SUFLOAT bw)
{ return sdb_analyzer_set_inspector_bandwidth_overridable(sa->a, h, bw) == 0; }
SUBOOL suscan_analyzer_inspector_set_spectrum_async(suscan_analyzer_t *sa, SUHANDLE h, uint32_t id, uint32_t req_id)
{ return sdb_analyzer_inspector_set_spectrum_async(sa->a, h, id, req_id) == 0; }
SUBOOL suscan_analyzer_inspector_estimator_cmd_async(suscan_analyzer_t *sa, SUHANDLE h, uint32_t id, SUBOOL en, uint32_t req_id)
{ return sdb_analyzer_inspector_estimator_cmd_async(sa->a, h, id, en ? 1 : 0, req_id) == 0; }

}  // extern "C"
