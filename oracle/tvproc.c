/* tvproc.c -- ORACLE (test infrastructure, never linked into the product): analog-TV processor, SPEC.md section TV.
 *
 * Restates what the reference drives through sigutils' su_tv_processor_* calls
 * (Default/GenericInspector/TVProcessorWorker.cpp:120-151 feed / take_frame loop, :186-239 start / setParams;
 * parameter block sigutils_tv_processor_params as filled at Default/GenericInspector/TVProcessorTab.cpp:549-597;
 * input conversion TVProcessorTab::feed, :601-620).  The processor itself lives in BatchDrake/sigutils (master,
 * unpinned, absent from the reference, no vectors): PARITY UNPINNED for the recurrence -- SPEC TV is this
 * project's statement of it.  What pins this file is tests/tv_stmt.py, an exact statement written from the SPEC text
 * alone (tests/test_tv_stmt.py: bit for bit over a table of scenes), and behaviour (tests/test_oracle_tv.py: locks on
 * a synthetic composite signal at a non-integer line length, recovers the picture, follows a line-rate offset).  The
 * input conversion is in the reference and is restated value by value (sdo_tv_feed_transform).
 *
 * Plain C, one IEEE binary32 operation per source operation (built -O2 -ffp-contract=off). */
#include "sd_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

static float tv_alpha(float tau) { return 1.0f - expf(-1.0f / tau); }            /* SU_SPLPF_ALPHA */

/* TV.0: the GUI's presets (su_tv_processor_params_pal / _ntsc, TVProcessorTab.cpp:629,633); times -> samples */
static void tv_common(sdo_tv_params *p)
{
  p->enable_sync = 1; p->reverse = 0; p->interlace = 1; p->enable_agc = 1; p->x_off = 0; p->dominance = 1;
  p->frame_spacing = 0; p->enable_comb = 1; p->comb_reverse = 0;
  p->t_tol = 1e-1f; p->l_tol = 1e-1f; p->g_tol = 1e-1f;
  p->hsync_huge_err = .25f; p->hsync_max_err = 1e-2f; p->hsync_min_err = .5e-2f;
  p->hsync_len_tau = 9.5f; p->line_len_tau = 1e3f; p->agc_tau = 1e-5f;
  p->hsync_fast_track_tau = 9.5f; p->hsync_slow_track_tau = 1e3f;
}
void sdo_tv_params_pal(sdo_tv_params *p, float fs)
{
  tv_common(p);
  p->frame_lines = 625; p->hsync_len = fs * 4e-6f; p->vsync_len = fs * 2e-6f; p->line_len = fs * 64e-6f;
  p->vsync_odd_trigger = 5;
}
void sdo_tv_params_ntsc(sdo_tv_params *p, float fs)
{
  tv_common(p);
  p->frame_lines = 525; p->hsync_len = fs * 4.749e-6f; p->vsync_len = fs * 2.375e-6f; p->line_len = fs * 63.556e-6f;
  p->vsync_odd_trigger = 6;
}

int sdo_tv_params_valid(const sdo_tv_params *p)
{
  if (!(p->line_len >= 8.0f) || !(p->line_len < (float) SDO_TV_MAX_W + 1.0f)) return 0;
  if (!(p->hsync_len >= 1.0f) || !(p->hsync_len < 0.5f * p->line_len) || !(p->vsync_len >= 1.0f)) return 0;
  if (p->frame_lines < 2 || p->frame_lines > SDO_TV_MAX_H) return 0;
  if (!(p->frame_spacing >= 0.0f && p->frame_spacing < 1.0f)) return 0;
  if (!(p->t_tol > 0 && p->t_tol < 1) || !(p->l_tol > 0 && p->l_tol < 1) || !(p->g_tol > 0 && p->g_tol < 1)) return 0;
  if (!(p->hsync_len_tau > 0) || !(p->line_len_tau > 0) || !(p->agc_tau > 0) || !(p->hsync_fast_track_tau > 0) ||
      !(p->hsync_slow_track_tau > 0))
    return 0;
  return 1;
}

struct sdo_tv {
  sdo_tv_params p;
  int W, H, delay_len;
  float thr, agc_alpha, pulse_alpha, hsync_len_alpha, line_len_alpha, fast_alpha, slow_alpha;
  float *delay, *line, *ring;                   /* ring: SDO_TV_RING frames of H x W */
  uint64_t ptr, sync_start, last_hsync, last_short, frames;
  int field_x, field_y, parity, field_lines, row, delay_ptr;
  float dec, gain, line_max, agc_accum, pulse, est_hsync, est_line, ll_accum;
  unsigned agc_lines, ll_count, vs_count, lines_since_vs;
  int sync_found, have_last_hsync, slow;
};

static int tv_row(const sdo_tv *t, int fy, int parity)
{
  const int row = t->p.interlace ? 2 * fy + (parity ^ (t->p.dominance ? 0 : 1)) : fy;
  return row >= 0 && row < t->H ? row : -1;
}

/* TV.1: derived constants */
static void tv_derive(sdo_tv *t)
{
  const sdo_tv_params *p = &t->p;
  float pt = p->hsync_len / 20.0f;
  if (pt < 1.0f) pt = 1.0f;
  t->thr = 1.0f - p->l_tol;
  t->agc_alpha = tv_alpha(p->agc_tau); t->pulse_alpha = tv_alpha(pt);
  t->hsync_len_alpha = tv_alpha(p->hsync_len_tau); t->line_len_alpha = tv_alpha(p->line_len_tau);
  t->fast_alpha = tv_alpha(p->hsync_fast_track_tau); t->slow_alpha = tv_alpha(p->hsync_slow_track_tau);
}

sdo_tv *sdo_tv_new(const sdo_tv_params *p)
{
  if (!p || !sdo_tv_params_valid(p)) return NULL;
  sdo_tv *t = calloc(1, sizeof(*t));
  if (!t) return NULL;
  t->p = *p;
  t->W = (int) floorf(p->line_len); t->H = (int) p->frame_lines; t->delay_len = (int) ceilf(p->line_len);
  tv_derive(t);
  t->delay = calloc((size_t) t->delay_len, sizeof(float));
  t->line = calloc((size_t) t->W, sizeof(float));
  t->ring = calloc((size_t) SDO_TV_RING * t->W * t->H, sizeof(float));
  if (!t->delay || !t->line || !t->ring) { sdo_tv_destroy(t); return NULL; }
  t->field_lines = p->interlace ? (t->H + 1) / 2 : t->H;
  t->row = tv_row(t, 0, 0);
  t->gain = 1.0f; t->est_hsync = p->hsync_len; t->est_line = p->line_len;
  t->lines_since_vs = 0x7fffffffu;
  return t;
}

void sdo_tv_destroy(sdo_tv *t)
{
  if (!t) return;
  free(t->delay); free(t->line); free(t->ring); free(t);
}

/* su_tv_processor_set_params: geometry (line_len, frame_lines, interlace) is fixed at creation; the rest is live */
int sdo_tv_set_params(sdo_tv *t, const sdo_tv_params *p)
{
  if (!t || !p || !sdo_tv_params_valid(p)) return 0;
  if ((int) floorf(p->line_len) != t->W || (int) ceilf(p->line_len) != t->delay_len || (int) p->frame_lines != t->H ||
      !p->interlace != !t->p.interlace)
    return 0;
  t->p = *p;
  tv_derive(t);
  return 1;
}

void sdo_tv_geometry(const sdo_tv *t, int *w, int *h) { *w = t->W; *h = t->H; }
uint64_t sdo_tv_frames(const sdo_tv *t) { return t->frames; }
const float *sdo_tv_frame(const sdo_tv *t, uint64_t frame_no)
{
  return t->ring + (size_t) (frame_no % SDO_TV_RING) * t->W * t->H;
}
void sdo_tv_estimates(const sdo_tv *t, float *line_len, float *hsync_len, float *gain)
{
  *line_len = t->est_line; *hsync_len = t->est_hsync; *gain = t->gain;
}

static void tv_set_xf(sdo_tv *t, float xf)
{
  const float fl = floorf(xf);
  t->field_x = (int) fl; t->dec = xf - fl;
}

/* su_tv_processor_feed (TVProcessorWorker.cpp:133): one sample; non-zero when a frame was completed */
int sdo_tv_feed(sdo_tv *t, float x)
{
  const sdo_tv_params *p = &t->p;
  int frame_done = 0;
  /* TV.2 */
  if (p->enable_comb) {
    const float prev = t->delay[t->delay_ptr];
    t->delay[t->delay_ptr] = x;
    if (++t->delay_ptr == t->delay_len) t->delay_ptr = 0;
    x = 0.5f * (p->comb_reverse ? x - prev : x + prev);
  }
  /* TV.3 */
  if (x > t->line_max) t->line_max = x;
  const float xg = p->enable_agc ? t->gain * x : x;
  /* TV.4 */
  t->pulse = t->pulse + t->pulse_alpha * (xg - t->pulse);
  /* TV.5 */
  if (p->enable_sync) {
    const int up = t->pulse > t->thr;
    if (!t->sync_found) {
      if (up) { t->sync_found = 1; t->sync_start = t->ptr; }
    } else if (!up) {
      const float len = (float) (t->ptr - t->sync_start);
      t->sync_found = 0;
      if (fabsf(len - t->est_hsync) <= p->t_tol * t->est_hsync) {
        if (t->have_last_hsync) {
          const float dl = (float) (t->sync_start - t->last_hsync);
          if (fabsf(dl - t->est_line) <= p->g_tol * t->est_line) { t->ll_accum = t->ll_accum + dl; ++t->ll_count; }
        }
        t->have_last_hsync = 1; t->last_hsync = t->sync_start;
        t->est_hsync = t->est_hsync + t->hsync_len_alpha * (len - t->est_hsync);
        {
          float xf = (float) t->field_x + t->dec;
          const float L = t->est_line;
          float err = (0.5f * t->est_hsync + p->x_off) - (xf - 0.5f * len);
          float rel;
          if (err > 0.5f * L) err = err - L; else if (err < -0.5f * L) err = err + L;
          rel = fabsf(err) / L;
          if (rel > p->hsync_max_err) t->slow = 0; else if (rel < p->hsync_min_err) t->slow = 1;
          if (rel > p->hsync_huge_err) xf = xf + err;
          else xf = xf + (t->slow ? t->slow_alpha : t->fast_alpha) * err;
          if (xf < 0.0f) xf = xf + L;
          tv_set_xf(t, xf);
        }
      } else {
        t->have_last_hsync = 0;
        if (fabsf(len - p->vsync_len) <= 2.0f * p->t_tol * p->vsync_len) {
          const float age = (float) (t->sync_start - t->last_short);
          if (t->vs_count > 0 && fabsf(age - 0.5f * t->est_line) <= 2.0f * p->t_tol * t->est_line) ++t->vs_count;
          else t->vs_count = 1;
          t->last_short = t->sync_start;
          if (t->vs_count == p->vsync_odd_trigger && t->lines_since_vs >= (unsigned) (t->field_lines / 2)) {
            const int early = t->field_y < t->field_lines / 2;
            t->lines_since_vs = 0;
            if (p->interlace) {
              const float pos = ((float) t->field_x + t->dec) - 0.5f * len;
              const int mid = fabsf(pos - 0.5f * t->est_line) < 0.25f * t->est_line;
              const int next = mid ? 1 : 0;
              t->parity = early ? next : next ^ 1;
              t->field_lines = t->parity == 0 ? (t->H + 1) / 2 : t->H / 2;
            }
            t->field_y = early ? -1 : t->field_lines - 1;
          }
        } else {
          t->vs_count = 0;
        }
      }
    }
  }
  /* TV.6 */
  {
    const float val = p->reverse ? xg : 1.0f - xg;
    const int n = t->field_x;
    const float d = t->dec;
    float xf;
    if (n >= 0 && n < t->W) t->line[n] = t->line[n] + (1.0f - d) * val;
    if (n + 1 >= 0 && n + 1 < t->W) t->line[n + 1] = d * val;
    ++t->field_x;
    xf = (float) t->field_x + t->dec;
    if (xf >= t->est_line) {
      if (t->row >= 0)
        memcpy(t->ring + ((size_t) (t->frames % SDO_TV_RING) * t->H + (size_t) t->row) * t->W, t->line,
               (size_t) t->W * sizeof(float));
      memset(t->line, 0, (size_t) t->W * sizeof(float));
      xf = xf - t->est_line;
      t->agc_accum = t->agc_accum + t->line_max; ++t->agc_lines; t->line_max = 0.0f;
      if (t->lines_since_vs < 0x7fffffffu) ++t->lines_since_vs;
      if (++t->field_y >= t->field_lines) {
        t->field_y = 0;
        if (p->enable_agc && t->agc_lines > 0 && t->agc_accum > 0.0f)
          t->gain = t->gain + t->agc_alpha * ((float) t->agc_lines / t->agc_accum - t->gain);
        t->agc_accum = 0.0f; t->agc_lines = 0;
        if (t->ll_count > 0) {
          t->est_line = t->est_line + t->line_len_alpha * (t->ll_accum / (float) t->ll_count - t->est_line);
          t->ll_accum = 0.0f; t->ll_count = 0;
        }
        frame_done = 1;
        if (p->interlace) {
          t->parity ^= 1;
          t->field_lines = t->parity == 0 ? (t->H + 1) / 2 : t->H / 2;
          frame_done = t->parity == 0;
        }
        if (frame_done) { ++t->frames; xf = xf - p->frame_spacing * t->est_line; }
      }
      tv_set_xf(t, xf);
      t->row = tv_row(t, t->field_y, t->parity);
    }
  }
  ++t->ptr;
  return frame_done;
}

size_t sdo_tv_feed_bulk(sdo_tv *t, const float *x, size_t n)
{
  size_t done = 0;
  for (size_t i = 0; i < n; ++i) done += (size_t) sdo_tv_feed(t, x[i]);
  return done;
}

/* TVProcessorTab::feed (Default/GenericInspector/TVProcessorTab.cpp:601-620): k |x| + dc, or k arg(x) / pi + dc.
 * mode 0 = Decider::MODULUS, 1 = ARGUMENT.  arg via the SPEC M atan2 (libm's differs in the last ulp). */
void sdo_tv_feed_transform(const sdo_cpx *x, size_t n, int mode, float k, float dc, float *out)
{
  for (size_t i = 0; i < n; ++i) {
    if (mode == 0) out[i] = k * sqrtf(x[i].re * x[i].re + x[i].im * x[i].im) + dc;
    else out[i] = k * sdo_atan2f(x[i].im, x[i].re) / 3.14159265358979323846f + dc;
  }
}
