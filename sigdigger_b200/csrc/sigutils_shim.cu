// sigutils_shim.cu -- libsigutils.so: the sigutils names the reference's Tasks/ and wrappers call
// (include/sigutils/*.h), implemented on top of this repo's C-ABI (include/sigdigger_b200.h).
//
//   * bulk entry points (su_specttuner_feed_bulk, su_*_bulk) run on the GPU through sdb_engine_* / sdb_task_*;
//   * per-sample entry points (su_costas_feed, su_pll_track, su_agc_feed, su_ncqo_read, su_clock_detector_feed,
//     su_iir_filt_feed) are per-sample calls BY ABI -- `destination[p] = su_costas_feed(&costas, origin[p])`,
//     Tasks/CostasRecoveryTask.cpp:58-61 -- and cannot be kernel launches: they execute, on the caller's thread, the
//     very step functions the kernels execute (sdb_chain_steps.h, host + device), so a Tasks/ loop over them is
//     bit-identical to the corresponding bulk device pass (tests/test_gpu_shim.py).  They are not a fallback for the
//     hot path: the analyzer, the inspectors and the channeliser exist only on the GPU.
//
// Built with nvcc as host code (-Xcompiler -ffp-contract=off: one rounding per operator, as on the device).
#include "../../include/sigdigger_b200.h"
#include <sigutils/types.h>
#include <sigutils/sampling.h>
#include <sigutils/ncqo.h>
#include <sigutils/iir.h>
#include <sigutils/pll.h>
#include <sigutils/agc.h>
#include <sigutils/clock.h>
#include <sigutils/taps.h>
#include <sigutils/specttuner.h>
#include <sigutils/version.h>
#include <sigutils/tvproc.h>

#include "sdb_chain_steps.h"
#include "sdb_tv_steps.h"
#include "host_design.h"

#include <stdlib.h>
#include <string.h>
#include <vector>

static inline float2 to_f2(SUCOMPLEX x) { return make_float2(x.real(), x.imag()); }
static inline SUCOMPLEX to_su(float2 v) { return SUCOMPLEX(v.x, v.y); }
static const sdb_complex *as_sdb(const SUCOMPLEX *p) { return reinterpret_cast<const sdb_complex *>(p); }
static sdb_complex *as_sdb(SUCOMPLEX *p) { return reinterpret_cast<sdb_complex *>(p); }

extern "C" {

SUBOOL su_lib_gen_wisdom(void) { return SU_TRUE; }
unsigned int sigutils_abi_version(void) { return 1; }
const char *sigutils_api_version(void) { return "0.3.0"; }
const char *sigutils_pkgversion(void) { return "0.3.0-sigdigger_b200"; }

// ------------------------------------------------------------------------------------------------ ncqo (SPEC N)
void su_ncqo_init(su_ncqo_t *o, SUFLOAT fnor) { o->phi = 0.0f; o->fnor = fnor; o->omega = 3.14159265358979323846f * fnor; }
void su_ncqo_set_phase(su_ncqo_t *o, SUFLOAT phi)
{
  o->phi = phi - TWOPI_F * floorf(phi / TWOPI_F);
  if (o->phi >= TWOPI_F) o->phi = 0.0f;     // rounding guard
}
SUFLOAT su_ncqo_get_phase(const su_ncqo_t *o) { return o->phi; }
void su_ncqo_inc_phase(su_ncqo_t *o, SUFLOAT d) { o->phi = wrap_once(o->phi + d); }
void su_ncqo_set_freq(su_ncqo_t *o, SUFLOAT fnor) { o->fnor = fnor; o->omega = 3.14159265358979323846f * fnor; }
void su_ncqo_set_angfreq(su_ncqo_t *o, SUFLOAT omega) { o->omega = omega; o->fnor = omega / 3.14159265358979323846f; }
void su_ncqo_inc_angfreq(su_ncqo_t *o, SUFLOAT d) { o->omega = o->omega + d; o->fnor = o->omega / 3.14159265358979323846f; }
SUFLOAT su_ncqo_get_freq(const su_ncqo_t *o) { return o->fnor; }
SUFLOAT su_ncqo_get_angfreq(const su_ncqo_t *o) { return o->omega; }
SUCOMPLEX su_ncqo_read(su_ncqo_t *o) { return to_su(ncqo_read(o->phi, o->omega)); }
SUBOOL su_ncqo_mix_bulk(su_ncqo_t *o, const SUCOMPLEX *src, SUCOMPLEX *dst, SUSCOUNT n)
{
  // sdb_task_carrier_xlate mirrors CarrierXlator (init(-relFreq), set_phase(-phase)): pass the negated values back
  if (sdb_task_carrier_xlate(as_sdb(src), as_sdb(dst), (size_t) n, 1, -o->fnor, -o->phi)) return SU_FALSE;
  for (SUSCOUNT i = 0; i < n; ++i) o->phi = wrap_once(o->phi + o->omega);     // the phase the n reads leave behind
  return SU_TRUE;
}

// ------------------------------------------------------------------------------------------------ filters (SPEC I)
SUBOOL su_iir_filt_init(su_iir_filt_t *f, SUSCOUNT y_size, const SUFLOAT *a, SUSCOUNT x_size, const SUFLOAT *b)
{
  memset(f, 0, sizeof(*f));
  if (x_size < 1 || x_size > 1024) return SU_FALSE;
  f->x_size = (unsigned) x_size; f->y_size = (unsigned) y_size;
  f->b = (SUFLOAT *) malloc(sizeof(SUFLOAT) * x_size);
  f->x = (SUCOMPLEX *) calloc(x_size, sizeof(SUCOMPLEX));
  if (y_size > 0) {
    f->a = (SUFLOAT *) malloc(sizeof(SUFLOAT) * y_size);
    f->y = (SUCOMPLEX *) calloc(y_size, sizeof(SUCOMPLEX));
    memcpy(f->a, a, sizeof(SUFLOAT) * y_size);
  }
  memcpy(f->b, b, sizeof(SUFLOAT) * x_size);
  f->gain = 1.0f;
  return SU_TRUE;
}
SUBOOL su_iir_rrc_init(su_iir_filt_t *f, SUSCOUNT n, SUFLOAT T, SUFLOAT beta)
{
  std::vector<float> h;
  if (n < 1 || n > 1024) return SU_FALSE;
  sdbh::taps_rrc(h, (unsigned) n, T, beta);
  return su_iir_filt_init(f, 0, nullptr, n, h.data());
}
SUBOOL su_iir_bwlpf_init(su_iir_filt_t *f, SUSCOUNT order, SUFLOAT fc)
{
  float b[17], a[17];
  if (order < 1 || order > 4 || !sdbh::butter_lp((unsigned) order, fc, b, a)) return SU_FALSE;
  return su_iir_filt_init(f, order + 1, a, order + 1, b);
}
SUBOOL su_iir_brickwall_lp_init(su_iir_filt_t *f, SUSCOUNT n, SUFLOAT fc)
{
  if (n < 1 || n > 1024) return SU_FALSE;
  std::vector<float> h((size_t) n);
  su_taps_brickwall_lp_init(h.data(), fc, n);
  return su_iir_filt_init(f, 0, nullptr, n, h.data());
}
// SPEC I.1: single accumulator per component, ascending i, feed-forward part first, fused terms
SUCOMPLEX su_iir_filt_feed(su_iir_filt_t *f, SUCOMPLEX x)
{
  float ar = 0.0f, ai = 0.0f;
  unsigned i, p;
  f->x[f->x_ptr] = x;
  p = f->x_ptr;
  for (i = 0; i < f->x_size; ++i) {
    ar = fmaf(f->b[i], f->x[p].real(), ar);
    ai = fmaf(f->b[i], f->x[p].imag(), ai);
    p = p == 0 ? f->x_size - 1 : p - 1;
  }
  f->x_ptr = f->x_ptr + 1 == f->x_size ? 0 : f->x_ptr + 1;
  if (f->y_size > 1) {
    p = f->y_ptr;
    for (i = 1; i < f->y_size; ++i) {
      ar = fmaf(-f->a[i], f->y[p].real(), ar);
      ai = fmaf(-f->a[i], f->y[p].imag(), ai);
      p = p == 0 ? f->y_size - 1 : p - 1;
    }
    f->y_ptr = f->y_ptr + 1 == f->y_size ? 0 : f->y_ptr + 1;
    f->y[f->y_ptr] = SUCOMPLEX(ar, ai);
  }
  f->curr_y = SUCOMPLEX(ar, ai);
  return f->curr_y;
}
void su_iir_filt_feed_bulk(su_iir_filt_t *f, const SUCOMPLEX *x, SUCOMPLEX *y, SUSCOUNT len)
{
  for (SUSCOUNT i = 0; i < len; ++i) y[i] = su_iir_filt_feed(f, x[i]);
}
SUCOMPLEX su_iir_filt_get(const su_iir_filt_t *f) { return f->curr_y; }
void su_iir_filt_reset(su_iir_filt_t *f)
{
  if (f->x) memset(f->x, 0, sizeof(SUCOMPLEX) * f->x_size);
  if (f->y) memset(f->y, 0, sizeof(SUCOMPLEX) * f->y_size);
  f->x_ptr = f->y_ptr = 0; f->curr_y = 0;
}
void su_iir_filt_set_gain(su_iir_filt_t *f, SUFLOAT gain) { f->gain = gain; }
void su_iir_filt_finalize(su_iir_filt_t *f)
{
  free(f->a); free(f->b); free(f->x); free(f->y);
  memset(f, 0, sizeof(*f));
}

// ------------------------------------------------------------------------------------------------ PLL, Costas (SPEC C)
SUBOOL su_pll_init(su_pll_t *p, SUFLOAT fhint, SUFLOAT fc)
{
  memset(p, 0, sizeof(*p));
  const float w = 3.14159265358979323846f * fc;
  const float dinv = 1.0f / (1.0f + 2.0f * 0.707f * w + w * w);
  p->alpha = 4.0f * w * w * dinv;
  p->beta = 4.0f * 0.707f * w * dinv;
  p->phi = 0.0f; p->omega = 3.14159265358979323846f * fhint;
  return SU_TRUE;
}
SUCOMPLEX su_pll_track(su_pll_t *p, SUCOMPLEX x)
{
  p->a = to_su(pll_step(p->alpha, p->beta, p->phi, p->omega, to_f2(x)));
  return p->a;
}
SUBOOL su_pll_track_bulk(su_pll_t *p, const SUCOMPLEX *x, SUCOMPLEX *y, SUSCOUNT n)
{
  // device pass from the object's state (sdb_task_pll_ex restarts at (phi, omega) and returns the final pair)
  float st[2] = { p->phi, p->omega };
  if (sdb_task_pll_state(as_sdb(x), as_sdb(y), (size_t) n, p->alpha, p->beta, st)) return SU_FALSE;
  p->phi = st[0]; p->omega = st[1];
  if (n) p->a = y[n - 1];
  return SU_TRUE;
}
void su_pll_finalize(su_pll_t *p) { (void) p; }

static inline CostasK *ck_of(su_costas_t *c) { return reinterpret_cast<CostasK *>(&c->kind); }
static inline CostasS *cs_of(su_costas_t *c) { return reinterpret_cast<CostasS *>(&c->phi); }
static_assert(sizeof(CostasK) == sizeof(int) * 2 + sizeof(float) * (2 + 2 * SDB_MAX_IIR), "CostasK layout");
static_assert(sizeof(CostasS) == sizeof(float) * (5 + 4 * SDB_MAX_IIR), "CostasS layout");
static_assert(offsetof(su_costas_t, phi) - offsetof(su_costas_t, kind) == sizeof(CostasK), "su_costas_t packs K then S");
static_assert(SU_PLL_MAX_IIR == SDB_MAX_IIR, "arm filter size");

SUBOOL su_costas_init(su_costas_t *c, enum sigutils_costas_kind kind, SUFLOAT fhint, SUFLOAT arm_bw,
                      unsigned int arm_order, SUFLOAT loop_bw)
{
  memset(c, 0, sizeof(*c));
  if (kind < SU_COSTAS_KIND_NONE || kind > SU_COSTAS_KIND_8PSK) return SU_FALSE;
  c->kind = (int) kind;
  c->a = 3.14159265358979323846f * loop_bw;
  c->b = 0.5f * c->a * c->a;
  c->af_n = 1; c->af_b[0] = 1.0f; c->af_a[0] = 1.0f;
  if (arm_order >= 2) {
    // "order 3" at the call site (Tasks/CostasRecoveryTask.cpp:41) = 3 coefficients = 2-pole Butterworth
    const unsigned poles = arm_order - 1 > 4 ? 4 : arm_order - 1;
    if (!sdbh::butter_lp(poles, arm_bw, c->af_b, c->af_a)) return SU_FALSE;
    c->af_n = (int) poles + 1;
  }
  c->omega = 3.14159265358979323846f * fhint;
  return SU_TRUE;
}
SUCOMPLEX su_costas_feed(su_costas_t *c, SUCOMPLEX x)
{
  c->y = to_su(costas_step(*ck_of(c), *cs_of(c), to_f2(x)));
  return c->y;
}
SUBOOL su_costas_feed_bulk(su_costas_t *c, const SUCOMPLEX *x, SUCOMPLEX *y, SUSCOUNT n)
{
  if (sdb_task_costas_state(as_sdb(x), as_sdb(y), (size_t) n, &c->kind, sizeof(CostasK), &c->phi, sizeof(CostasS)))
    return SU_FALSE;
  if (n) c->y = y[n - 1];
  return SU_TRUE;
}
void su_costas_set_kind(su_costas_t *c, enum sigutils_costas_kind kind) { c->kind = (int) kind; }
void su_costas_set_loop_bw(su_costas_t *c, SUFLOAT loop_bw)
{
  c->a = 3.14159265358979323846f * loop_bw;
  c->b = 0.5f * c->a * c->a;
}
void su_costas_finalize(su_costas_t *c) { (void) c; }

// ------------------------------------------------------------------------------------------------ AGC (SPEC A)
SUBOOL su_agc_init(su_agc_t *g, const struct su_agc_params *p)
{
  memset(g, 0, sizeof(*g));
  if (p->delay_line_size < 1 || p->mag_history_size < 1 || p->delay_line_size > SDB_MAX_AGC_HIST ||
      p->mag_history_size > SDB_MAX_AGC_HIST)
    return SU_FALSE;
  g->delay_line = (SUFLOAT *) calloc(2 * (size_t) p->delay_line_size, sizeof(SUFLOAT));
  g->mag_history = (SUFLOAT *) malloc(sizeof(SUFLOAT) * p->mag_history_size);
  if (!g->delay_line || !g->mag_history) { free(g->delay_line); free(g->mag_history); return SU_FALSE; }
  for (unsigned i = 0; i < p->mag_history_size; ++i) g->mag_history[i] = -160.0f;
  g->delay_line_size = p->delay_line_size; g->mag_history_size = p->mag_history_size;
  g->knee = p->threshold;
  const float slope = p->slope_factor * 1e-2f;
  g->slope_m1 = slope - 1.0f;
  g->fixed_gain = d_db_to_mag(g->knee * (slope - 1.0f));
  g->hang_max = p->hang_max;
  g->fast_alpha_rise = sdbh::alpha_of(p->fast_rise_t); g->fast_alpha_fall = sdbh::alpha_of(p->fast_fall_t);
  g->slow_alpha_rise = sdbh::alpha_of(p->slow_rise_t); g->slow_alpha_fall = sdbh::alpha_of(p->slow_fall_t);
  g->fast_level = g->slow_level = g->peak = -160.0f;
  g->enabled = SU_TRUE;
  return SU_TRUE;
}
SUCOMPLEX su_agc_feed(su_agc_t *g, SUCOMPLEX x)
{
  AgcK k; AgcS s;
  k.knee = g->knee; k.slope_m1 = g->slope_m1; k.fixed_gain = g->fixed_gain;
  k.far_ = g->fast_alpha_rise; k.faf = g->fast_alpha_fall; k.sar = g->slow_alpha_rise; k.saf = g->slow_alpha_fall;
  k.hang_max = g->hang_max; k.dl_size = g->delay_line_size; k.mh_size = g->mag_history_size;
  s.fast = g->fast_level; s.slow = g->slow_level; s.peak = g->peak;
  s.hang_n = g->hang_n; s.dl_ptr = g->delay_line_ptr; s.mh_ptr = g->mag_history_ptr;
  const float2 y = agc_step<1>(k, s, g->delay_line, g->mag_history, to_f2(x));
  g->fast_level = s.fast; g->slow_level = s.slow; g->peak = s.peak;
  g->hang_n = s.hang_n; g->delay_line_ptr = s.dl_ptr; g->mag_history_ptr = s.mh_ptr;
  return to_su(y);
}
void su_agc_finalize(su_agc_t *g)
{
  free(g->delay_line); free(g->mag_history);
  memset(g, 0, sizeof(*g));
}

// ------------------------------------------------------------------------------------------------ clock (SPEC G, D)
int su_clock_detector_init(su_clock_detector_t *cd, SUFLOAT loop_gain, SUFLOAT bhint, SUSCOUNT bufsiz)
{
  memset(cd, 0, sizeof(*cd));
  if (bufsiz < 1) return -1;
  cd->buf = (SUCOMPLEX *) malloc(sizeof(SUCOMPLEX) * bufsiz);
  if (!cd->buf) return -1;
  cd->buf_size = bufsiz;
  cd->alpha = 2e-1f; cd->beta = 6e-4f * cd->alpha;
  cd->bnor = bhint; cd->bmin = 0.0f; cd->bmax = 1.0f;
  cd->phi = 0.25f; cd->gain = loop_gain;
  return 0;
}
void su_clock_detector_set_baud(su_clock_detector_t *cd, SUFLOAT bnor) { cd->bnor = bnor; }
SUBOOL su_clock_detector_set_bnor_limits(su_clock_detector_t *cd, SUFLOAT lo, SUFLOAT hi)
{
  if (lo > hi) return SU_FALSE;
  cd->bmin = lo; cd->bmax = hi;
  return SU_TRUE;
}
void su_clock_detector_feed(su_clock_detector_t *cd, SUCOMPLEX x)
{
  ClockS s;
  s.phi = cd->phi; s.bnor = cd->bnor; s.x0r = cd->x0r; s.x0i = cd->x0i; s.x1r = cd->x1r; s.x1i = cd->x1i;
  s.x2r = cd->x2r; s.x2i = cd->x2i; s.pr = cd->pr; s.pi = cd->pi; s.half = cd->half;
  float2 out;
  const bool produced = clock_step(cd->gain, cd->alpha, cd->beta, s, to_f2(x), out);
  cd->phi = s.phi; cd->bnor = s.bnor; cd->x0r = s.x0r; cd->x0i = s.x0i; cd->x1r = s.x1r; cd->x1i = s.x1i;
  cd->x2r = s.x2r; cd->x2i = s.x2i; cd->pr = s.pr; cd->pi = s.pi; cd->half = s.half;
  if (produced && cd->buf_avail < cd->buf_size) cd->buf[cd->buf_avail++] = to_su(out);
}
SUSDIFF su_clock_detector_read(su_clock_detector_t *cd, SUCOMPLEX *buf, SUSCOUNT size)
{
  const SUSCOUNT n = cd->buf_avail < size ? cd->buf_avail : size;
  memcpy(buf, cd->buf, sizeof(SUCOMPLEX) * n);
  if (n < cd->buf_avail) memmove(cd->buf, cd->buf + n, sizeof(SUCOMPLEX) * (cd->buf_avail - n));
  cd->buf_avail -= n;
  return (SUSDIFF) n;
}
void su_clock_detector_finalize(su_clock_detector_t *cd)
{
  free(cd->buf);
  memset(cd, 0, sizeof(*cd));
}

SUBOOL su_sampler_init(su_sampler_t *s, SUFLOAT bnor)
{
  memset(s, 0, sizeof(*s));
  return su_sampler_set_rate(s, bnor);
}
SUBOOL su_sampler_set_rate(su_sampler_t *s, SUFLOAT bnor)
{
  s->bnor = bnor;
  s->period = bnor > 0.0f ? 1.0f / bnor : 0.0f;
  s->phase0 = s->phase0_rel * s->period;
  return SU_TRUE;
}
void su_sampler_set_phase(su_sampler_t *s, SUFLOAT phase_rel) { s->phase0_rel = phase_rel; s->phase0 = phase_rel * s->period; }
SUBOOL su_sampler_feed(su_sampler_t *s, SUCOMPLEX *sample)
{
  float pr = s->prev.real(), pi = s->prev.imag();
  float2 out;
  const bool got = sampler_step(s->period, s->phase0, s->phase, pr, pi, to_f2(*sample), out);
  s->prev = SUCOMPLEX(pr, pi);
  if (got) *sample = to_su(out);
  return got ? SU_TRUE : SU_FALSE;
}
void su_sampler_finalize(su_sampler_t *s) { (void) s; }

// ------------------------------------------------------------------------------------------------ taps (SPEC W, I)
static void window_apply(SUFLOAT *h, SUCOMPLEX *hc, SUSCOUNT size, int type)
{
  std::vector<float> w;
  sdbh::window_fill(w, (unsigned) size, type);
  for (SUSCOUNT i = 0; i < size; ++i) {
    if (h) h[i] = h[i] * w[i];
    if (hc) hc[i] = SUCOMPLEX(hc[i].real() * w[i], hc[i].imag() * w[i]);
  }
}
void su_taps_apply_hamming(SUFLOAT *h, SUSCOUNT n) { window_apply(h, nullptr, n, SDB_WINDOW_HAMMING); }
void su_taps_apply_hann(SUFLOAT *h, SUSCOUNT n) { window_apply(h, nullptr, n, SDB_WINDOW_HANN); }
void su_taps_apply_flat_top(SUFLOAT *h, SUSCOUNT n) { window_apply(h, nullptr, n, SDB_WINDOW_FLAT_TOP); }
void su_taps_apply_blackmann_harris(SUFLOAT *h, SUSCOUNT n) { window_apply(h, nullptr, n, SDB_WINDOW_BLACKMANN_HARRIS); }
void su_taps_apply_hamming_complex(SUCOMPLEX *h, SUSCOUNT n) { window_apply(nullptr, h, n, SDB_WINDOW_HAMMING); }
void su_taps_apply_hann_complex(SUCOMPLEX *h, SUSCOUNT n) { window_apply(nullptr, h, n, SDB_WINDOW_HANN); }
void su_taps_apply_flat_top_complex(SUCOMPLEX *h, SUSCOUNT n) { window_apply(nullptr, h, n, SDB_WINDOW_FLAT_TOP); }
void su_taps_apply_blackmann_harris_complex(SUCOMPLEX *h, SUSCOUNT n) { window_apply(nullptr, h, n, SDB_WINDOW_BLACKMANN_HARRIS); }
void su_taps_rrc_init(SUFLOAT *h, SUFLOAT T, SUFLOAT beta, SUSCOUNT size)
{
  std::vector<float> t;
  sdbh::taps_rrc(t, (unsigned) size, T, beta);
  memcpy(h, t.data(), sizeof(float) * size);
}
void su_taps_brickwall_lp_init(SUFLOAT *h, SUFLOAT fc, SUSCOUNT n)
{
  sdbh::taps_brickwall_lp(h, (unsigned) n, fc);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ specttuner (SPEC S)
// One sdb engine (one stream, no PSD) per tuner.  The channel plan is committed at the first feed after an
// open / close; a re-plan keeps the running channels' cross-fade tails (sdb_engine_migrate).
struct sigutils_specttuner {
  sigutils_specttuner_params params;
  std::vector<su_specttuner_channel_t *> channels;
  sdb_engine_t *eng = nullptr;
  bool dirty = true;
  std::vector<SUCOMPLEX> pending;        // input not yet forming a whole hop
  std::vector<SUCOMPLEX> out;
  size_t max_hops = 64;
};

static bool st_replan(su_specttuner_t *st)
{
  sdb_engine_params ep;
  memset(&ep, 0, sizeof(ep));
  ep.n_streams = 1; ep.psd_size = 0; ep.st_window_size = (uint32_t) st->params.window_size;
  ep.max_feed = (uint32_t) (st->max_hops * st->params.window_size / 2);
  int dev = 0; cudaGetDevice(&dev); ep.device = dev;
  sdb_engine_t *ne = sdb_engine_new(&ep, 1.0);
  if (!ne) return false;
  for (auto *ch : st->channels) {
    sdb_channel_params cp;
    cp.f0 = ch->params.f0; cp.bw = ch->params.bw; cp.guard = ch->params.guard; cp.precise = ch->params.precise;
    sdb_channel_info info;
    const int h = sdb_engine_open_channel(ne, &cp, &info);
    if (h < 0) { sdb_engine_destroy(ne); return false; }
    ch->index = h;
  }
  if (sdb_engine_commit(ne)) { sdb_engine_destroy(ne); return false; }
  if (st->eng) {
    sdb_engine_migrate(ne, st->eng);       // history + tails of the channels that stay (same f0 / bw / guard)
    sdb_engine_destroy(st->eng);
  }
  st->eng = ne; st->dirty = false;
  return true;
}

extern "C" {

su_specttuner_t *su_specttuner_new(const struct sigutils_specttuner_params *params)
{
  if (!params || params->window_size < 64 || (params->window_size & (params->window_size - 1))) return nullptr;
  if (sdb_device_count() <= 0) return nullptr;      // no CPU path
  su_specttuner_t *st = new sigutils_specttuner();
  st->params = *params;
  return st;
}

su_specttuner_channel_t *su_specttuner_open_channel(su_specttuner_t *st,
                                                    const struct sigutils_specttuner_channel_params *p)
{
  if (!st || !p) return nullptr;
  sdb_channel_info info;
  sdb_channel_params cp;
  cp.f0 = p->f0; cp.bw = p->bw; cp.guard = p->guard; cp.precise = p->precise;
  if (sdb_channel_geometry((uint32_t) st->params.window_size, &cp, &info)) return nullptr;
  su_specttuner_channel_t *ch = (su_specttuner_channel_t *) calloc(1, sizeof(*ch));
  ch->params = *p;
  ch->index = -1;
  ch->k = 1.0f / (float) st->params.window_size;
  ch->decimation = info.decimation;
  ch->center = info.center; ch->size = info.size; ch->width = info.width;
  ch->halfw = info.width / 2; ch->halfsz = info.size / 2;
  st->channels.push_back(ch);
  st->dirty = true;
  return ch;
}

SUBOOL su_specttuner_close_channel(su_specttuner_t *st, su_specttuner_channel_t *channel)
{
  if (!st) return SU_FALSE;
  for (size_t i = 0; i < st->channels.size(); ++i)
    if (st->channels[i] == channel) {
      st->channels.erase(st->channels.begin() + (long) i);
      free(channel);
      st->dirty = true;
      return SU_TRUE;
    }
  return SU_FALSE;
}

SUSCOUNT su_specttuner_get_channel_count(const su_specttuner_t *st) { return st ? st->channels.size() : 0; }
SUFLOAT su_specttuner_channel_get_decimation(const su_specttuner_channel_t *ch) { return ch ? ch->decimation : 0; }

SUBOOL su_specttuner_feed_bulk(su_specttuner_t *st, const SUCOMPLEX *buf, SUSCOUNT size)
{
  if (!st || (!buf && size)) return SU_FALSE;
  const size_t hop = (size_t) st->params.window_size / 2;
  st->pending.insert(st->pending.end(), buf, buf + size);
  size_t done = 0;
  while (st->pending.size() - done >= hop) {
    if (st->dirty && !st_replan(st)) return SU_FALSE;
    size_t hops = (st->pending.size() - done) / hop;
    if (hops > st->max_hops) hops = st->max_hops;
    if (sdb_engine_feed_host(st->eng, as_sdb(st->pending.data() + done), hops * hop, hops * hop) ||
        sdb_engine_sync(st->eng))
      return SU_FALSE;
    done += hops * hop;
    for (auto *ch : st->channels) {
      if (!ch->params.on_data) continue;
      st->out.resize(hops * ch->halfsz);
      const long n = sdb_engine_read_channel(st->eng, 0, ch->index, as_sdb(st->out.data()), st->out.size());
      if (n < 0) return SU_FALSE;
      // one callback per hop, as su_specttuner does (size / 2 samples each)
      for (long o = 0; o + (long) ch->halfsz <= n; o += ch->halfsz)
        if (!ch->params.on_data(ch, ch->params.privdata, st->out.data() + o, ch->halfsz)) {
          st->pending.erase(st->pending.begin(), st->pending.begin() + (long) done);
          return SU_FALSE;
        }
    }
  }
  st->pending.erase(st->pending.begin(), st->pending.begin() + (long) done);
  return SU_TRUE;
}

void su_specttuner_destroy(su_specttuner_t *st)
{
  if (!st) return;
  for (auto *ch : st->channels) free(ch);
  if (st->eng) sdb_engine_destroy(st->eng);
  delete st;
}


// ---------------------------------------------------------------------------------------------------------
// <sigutils/tvproc.h>: the TV tab's processor, per-sample on the caller's thread (TVProcessorWorker::work)
// ---------------------------------------------------------------------------------------------------------
struct sigutils_tv_processor {
  struct sigutils_tv_processor_params prm;
  SdbTvCfg cfg; SdbTvState st;
  std::vector<float> delay, line, ring;          // ring: SDB_TV_RING frames of H x W
  struct sigutils_tv_frame_buffer *pool = nullptr;
};

void su_tv_processor_params_pal(struct sigutils_tv_processor_params *p, SUFLOAT samp_rate) { if (p) sdb_tv_preset(*p, samp_rate, true); }
void su_tv_processor_params_ntsc(struct sigutils_tv_processor_params *p, SUFLOAT samp_rate) { if (p) sdb_tv_preset(*p, samp_rate, false); }

su_tv_processor_t *su_tv_processor_new(const struct sigutils_tv_processor_params *p)
{
  if (!p || !sdb_tv_params_valid(*p)) return nullptr;
  su_tv_processor_t *t = new sigutils_tv_processor();
  t->prm = *p;
  sdb_tv_derive(*p, t->cfg);
  sdb_tv_state_init(t->cfg, t->st);
  t->delay.assign((size_t) t->cfg.delay_len, 0.0f);
  t->line.assign((size_t) t->cfg.W, 0.0f);
  t->ring.assign((size_t) SDB_TV_RING * t->cfg.W * t->cfg.H, 0.0f);
  return t;
}

SUBOOL su_tv_processor_set_params(su_tv_processor_t *t, const struct sigutils_tv_processor_params *p)
{
  if (!t || !p || !sdb_tv_params_valid(*p)) return SU_FALSE;
  SdbTvCfg c; sdb_tv_derive(*p, c);
  if (c.W != t->cfg.W || c.delay_len != t->cfg.delay_len || c.H != t->cfg.H || c.interlace != t->cfg.interlace)
    return SU_FALSE;                             // the caller stops / starts the processor for a new geometry
  t->prm = *p; t->cfg = c;
  return SU_TRUE;
}

SUBOOL su_tv_processor_feed(su_tv_processor_t *t, SUFLOAT x)
{
  int row = -1, slot = 0;
  const int flags = sdb_tv_step(t->cfg, t->st, t->delay.data(), t->line.data(), x, &row, &slot);
  if (flags & SDB_TV_LINE_DONE) {
    const size_t W = (size_t) t->cfg.W;
    if (row >= 0) memcpy(t->ring.data() + ((size_t) slot * t->cfg.H + (size_t) row) * W, t->line.data(), W * sizeof(float));
    memset(t->line.data(), 0, W * sizeof(float));
  }
  return (flags & SDB_TV_FRAME_DONE) ? SU_TRUE : SU_FALSE;
}

// the frame completed last, as a buffer the caller owns until su_tv_processor_return_frame / su_tv_frame_buffer_destroy
struct sigutils_tv_frame_buffer *su_tv_processor_take_frame(su_tv_processor_t *t)
{
  if (!t || t->st.frames == 0) return nullptr;
  const size_t px = (size_t) t->cfg.W * t->cfg.H;
  struct sigutils_tv_frame_buffer *f = t->pool;
  if (f) t->pool = f->next;
  else {
    f = (struct sigutils_tv_frame_buffer *) calloc(1, sizeof(*f));
    if (!f) return nullptr;
    f->buffer = (SUFLOAT *) malloc(px * sizeof(SUFLOAT));
    if (!f->buffer) { free(f); return nullptr; }
  }
  f->width = t->cfg.W; f->height = t->cfg.H; f->next = nullptr;
  memcpy(f->buffer, t->ring.data() + (size_t) ((t->st.frames - 1) % SDB_TV_RING) * px, px * sizeof(SUFLOAT));
  return f;
}

void su_tv_frame_buffer_destroy(struct sigutils_tv_frame_buffer *f)
{
  if (!f) return;
  free(f->buffer); free(f);
}

void su_tv_processor_return_frame(su_tv_processor_t *t, struct sigutils_tv_frame_buffer *f)
{
  if (!f) return;
  if (!t || f->width != t->cfg.W || f->height != t->cfg.H) { su_tv_frame_buffer_destroy(f); return; }
  f->next = t->pool; t->pool = f;
}

void su_tv_processor_destroy(su_tv_processor_t *t)
{
  if (!t) return;
  while (t->pool) { struct sigutils_tv_frame_buffer *n = t->pool->next; su_tv_frame_buffer_destroy(t->pool); t->pool = n; }
  delete t;
}

// test hooks (tests/test_oracle_tv.py): estimates and the picture in progress
void sdb_shim_tv_estimates(const su_tv_processor_t *t, float *line_len, float *hsync_len, float *gain, unsigned long long *frames)
{ *line_len = t->st.est_line_len; *hsync_len = t->st.est_hsync_len; *gain = t->st.agc_gain; *frames = t->st.frames; }

}  // extern "C"
