/*
 * snr.c -- ORACLE (test infrastructure). The inspector's SNR meter, SPEC_SN.md.  The Y.7 step is sdo_snr_feed of
 * tasks.c, driven with this meter's histogram.
 */
#include "snr.h"
#include <stdlib.h>
#include <string.h>
#include <math.h>

static unsigned snr_K(unsigned bps) { return 1u << (bps ? bps : 1u); }

static void snr_fresh(sdo_snrm *m, float sigma)
{
  memset(m->h, 0, m->L * sizeof(unsigned));
  memset(m->model, 0, m->L * sizeof(float));
  m->est.sigma = sigma; m->est.delta = 0.f;
  memset(&m->st, 0, sizeof m->st);
  m->st.sigma = sigma; m->st.snr = 1.f / (m->K * sigma);
}

int sdo_snrm_init(sdo_snrm *m, int insp_class, unsigned L, unsigned bps, float sigma, float alpha)
{
  memset(m, 0, sizeof *m);
  if (insp_class < 0 || insp_class > 2 || L < 16 || L > 1024) return -1;
  m->L = L; m->bps = bps; m->K = snr_K(bps);
  m->mode = insp_class == 2 ? SDO_DECIDE_MODULUS : SDO_DECIDE_ARGUMENT;
  m->h = calloc(L, sizeof(unsigned)); m->model = calloc(L, sizeof(float));
  sdo_snr_init(&m->est);
  m->est.intervals = m->K; m->est.alpha = alpha;
  snr_fresh(m, sigma);
  return 0;
}

void sdo_snrm_free(sdo_snrm *m)
{
  free(m->h); free(m->model);
  sdo_snr_free(&m->est);
  memset(m, 0, sizeof *m);
}

/* SN.1: D's expression with L for 2^bps; the argument clamps s = L (v = pi) into the last bin, the modulus drops
 * s >= L; NaN is never counted */
unsigned sdo_snrm_bin(int mode, unsigned L, sdo_cpx x)
{
  const float fL = (float) L;
  float v, s;
  if (mode == SDO_DECIDE_ARGUMENT) {
    v = sdo_atan2f(x.im, x.re);
    s = floorf((v - -SDO_PI_F) / (SDO_PI_F - -SDO_PI_F) * fL);
    if (isnan(s)) return L;
    return s < fL ? (unsigned) s : L - 1;
  }
  v = sdo_cabsf(x);
  s = floorf((v - 0.0f) / (1.0f - 0.0f) * fL);
  return s < fL ? (unsigned) s : L;
}

void sdo_snrm_feed(sdo_snrm *m, const sdo_cpx *x, unsigned n)
{
  unsigned i, b;
  int halve = 0;
  unsigned long long sum = 0;
  if (n == 0) { m->st.stepped = 0; return; }
  for (i = 0; i < n; ++i)
    if ((b = sdo_snrm_bin(m->mode, m->L, x[i])) < m->L) ++m->h[b];
  for (i = 0; i < m->L; ++i) halve |= m->h[i] >= 0x80000000u;
  for (i = 0; i < m->L; ++i) {
    if (halve) m->h[i] >>= 1;
    sum += m->h[i];
  }
  m->est.intervals = m->K;
  sdo_snr_feed(&m->est, m->h, m->L);
  memcpy(m->model, m->est.hi, m->L * sizeof(float));
  m->st.counted = sum; m->st.steps += 1; m->st.stepped = 1;
  m->st.sigma = m->est.sigma; m->st.snr = 1.f / (m->K * m->est.sigma); m->st.delta = m->est.delta;
}

void sdo_snrm_reset(sdo_snrm *m, float sigma)
{
  m->est.sigma = sigma;
  m->st.sigma = sigma; m->st.snr = 1.f / (m->K * sigma);
}

void sdo_snrm_replan(sdo_snrm *m, int same_cfg, unsigned bps, float alpha)
{
  m->est.alpha = alpha;
  if (same_cfg) return;
  {
    const float sigma = bps != m->bps ? 1.f / 8.f : m->est.sigma;
    m->bps = bps; m->K = snr_K(bps);
    snr_fresh(m, sigma);
  }
}
