/*
 * decimate.c -- ORACLE (test infrastructure). Source decimation (SPEC_L.md): the FIR decimator behind the source
 * config's `average` (Suscan/Source.cpp:195-201, 419-425; Settings/ProfileConfigTab.cpp:622-638).
 *
 * Compile with -ffp-contract=off: every term below is one explicit fmaf, in ascending tap order.
 */
#include "decimate.h"
#include <stdlib.h>
#include <string.h>
#include <math.h>

/* SPEC Q: native sample formats, exact in binary32 */
static sdo_cpx load_iq(const void *x, size_t j, int fmt)
{
  sdo_cpx v;
  if (fmt == SDO_FMT_U8) {
    const unsigned char *p = (const unsigned char *) x + 2 * j;
    v.re = ((float) p[0] - 128.0f) * (1.0f / 128.0f); v.im = ((float) p[1] - 128.0f) * (1.0f / 128.0f);
  } else if (fmt == SDO_FMT_S8) {
    const signed char *p = (const signed char *) x + 2 * j;
    v.re = (float) p[0] * (1.0f / 128.0f); v.im = (float) p[1] * (1.0f / 128.0f);
  } else if (fmt == SDO_FMT_S16) {
    const short *p = (const short *) x + 2 * j;
    v.re = (float) p[0] * (1.0f / 32768.0f); v.im = (float) p[1] * (1.0f / 32768.0f);
  } else {
    v = ((const sdo_cpx *) x)[j];
  }
  return v;
}

int sdo_decimate_init(sdo_decimate *d, unsigned D)
{
  memset(d, 0, sizeof(*d));
  if (D < 1 || D > SDO_DECIM_MAX) return -1;
  d->D = D; d->n = 16 * D + 1;
  d->h = (float *) malloc(sizeof(float) * d->n);
  d->hist = (sdo_cpx *) calloc(16 * D, sizeof(sdo_cpx));
  if (!d->h || !d->hist) { sdo_decimate_free(d); return -1; }
  sdo_taps_brickwall_lp(d->h, d->n, (float) (1.0 / (double) D));
  return 0;
}

void sdo_decimate_free(sdo_decimate *d)
{
  free(d->h); free(d->hist);
  memset(d, 0, sizeof(*d));
}

void sdo_decimate_reset(sdo_decimate *d)
{
  memset(d->hist, 0, sizeof(sdo_cpx) * 16 * d->D);
  d->phase = 0;
}

/* y[k] = sum_{i=0}^{n-1} h_i x[kD - i], x[j < 0] = 0: one accumulator per component from 0, ascending i, one fmaf per
 * term (SPEC I.1's convention).  Outputs fall on the input indices that are multiples of D; `phase` is the global
 * input index of the next sample modulo D and `hist` the last 16 D inputs, oldest first, so the result does not
 * depend on how the input is split into feeds.  Returns the number of outputs written to y. */
size_t sdo_decimate_feed(sdo_decimate *d, const void *x, int fmt, size_t m, sdo_cpx *y)
{
  const unsigned D = d->D, L = 16 * D;
  size_t j, out = 0;
  sdo_cpx *buf = (sdo_cpx *) malloc(sizeof(sdo_cpx) * (L + m));    /* hist ++ converted input */
  memcpy(buf, d->hist, sizeof(sdo_cpx) * L);
  for (j = 0; j < m; ++j) buf[L + j] = load_iq(x, j, fmt);
  for (j = (D - d->phase) % D; j < m; j += D) {
    const sdo_cpx *xn = buf + L + j;                                 /* x[kD] */
    sdo_cpx acc = { 0.0f, 0.0f };
    unsigned i;
    for (i = 0; i < d->n; ++i) {
      acc.re = fmaf(d->h[i], xn[-(long) i].re, acc.re);
      acc.im = fmaf(d->h[i], xn[-(long) i].im, acc.im);
    }
    y[out++] = acc;
  }
  memcpy(d->hist, buf + m, sizeof(sdo_cpx) * L);
  d->phase = (unsigned) ((d->phase + m) % D);
  free(buf);
  return out;
}
