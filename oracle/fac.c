/* ORACLE (test infrastructure): SPEC FC, the inspector's FAC tab.  See fac.h and SPEC_FC.md. */
#include "fac.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

int sdo_fac_init(sdo_fac *f, unsigned L, float alpha, unsigned lo, unsigned hi, double sigma)
{
  memset(f, 0, sizeof(*f));
  if (L < 512 || L > (1u << 19) || (L & (L - 1))) return -1;
  if (lo == 0 && hi == 0) hi = L / 2;
  if (!(lo < hi && hi <= L / 2)) return -1;
  f->L = L; f->lo = lo; f->hi = hi; f->alpha = alpha; f->sigma = sigma;
  f->max = -INFINITY; f->min = INFINITY;
  f->blk = (sdo_cpx *) calloc(L, sizeof(sdo_cpx));
  f->fac = (float *) calloc(L / 2, sizeof(float));
  f->v = (float *) calloc(L / 2, sizeof(float));
  /* FC.1: F.2 up to 4096 points, F.3 (kind 1) above, whatever sdo_spec_plan_init picks for 8192 .. 65536 */
  if (sdo_spec_plan_init(&f->plan, L, 0)) return -1;
  if (L > 4096 && f->plan.kind != 1) {
    unsigned l = 0;
    while ((1u << l) < L) ++l;
    free(f->plan.tw_a); free(f->plan.tw_b);
    f->plan.kind = 1; f->plan.N1 = 1u << (l / 2); f->plan.N2 = L / f->plan.N1;
    f->plan.tw_a = sdo_spec_twiddles(f->plan.N1);
    f->plan.tw_b = sdo_spec_twiddles(f->plan.N2);
  }
  return 0;
}

void sdo_fac_free(sdo_fac *f)
{
  free(f->blk); free(f->fac); free(f->v);
  sdo_spec_plan_free(&f->plan);
  memset(f, 0, sizeof(*f));
}

void sdo_fac_magnitude(sdo_fac *f, const sdo_cpx *block, float *v, int twice)
{
  const unsigned L = f->L;
  unsigned i;
  sdo_cpx *X = (sdo_cpx *) malloc(sizeof(sdo_cpx) * L), *A = (sdo_cpx *) malloc(sizeof(sdo_cpx) * L);
  sdo_spec_forward(&f->plan, block, NULL, X);
  for (i = 0; i < L; ++i) { X[i].re = fmaf(X[i].re, X[i].re, X[i].im * X[i].im); X[i].im = 0.0f; }
  if (L <= 4096 && !twice) {
    memcpy(A, X, sizeof(sdo_cpx) * L);
    sdo_spec_inverse_stockham(&f->plan, A);
  } else {
    sdo_spec_forward(&f->plan, X, NULL, A);
  }
  for (i = 0; i < L / 2; ++i) v[i] = sqrtf(A[i].re * A[i].re + A[i].im * A[i].im);
  free(X); free(A);
}

void sdo_fac_acc_init(sdo_fac_acc *a)
{
  a->blocks = 0; a->pos = 0; a->count = 0; a->local = -INFINITY; a->power = 0.0f;
}

/* FC.2: lags of the window in ascending order, in tiles of 1024 from lo; a value above the running maximum of the
 * feed is a record (localMax, pos) and is left out of the power, every other value's square goes to its tile position;
 * each tile is summed by the fixed tree s[i] += s[i + h], h = 512 .. 1, and the tile sums are added to power in order.
 * FC.3: fac[l] += alpha (v[l] / max - fac[l]) with max including this block. */
void sdo_fac_update(sdo_fac *f, sdo_fac_acc *a, const float *v)
{
  float s[SDO_FAC_TILE];
  unsigned t0, i, h, l;
  for (t0 = f->lo; t0 < f->hi; t0 += SDO_FAC_TILE) {
    memset(s, 0, sizeof(s));
    for (i = 0; i < SDO_FAC_TILE && t0 + i < f->hi; ++i) {
      const float x = v[t0 + i];
      if (x > a->local) { a->local = x; a->pos = t0 + i; }
      else { s[i] = x * x; ++a->count; }
      if (x > f->max) f->max = x;
      if (x < f->min) f->min = x;
    }
    for (h = SDO_FAC_TILE / 2; h > 0; h >>= 1)
      for (i = 0; i < h; ++i) s[i] = s[i] + s[i + h];
    a->power = a->power + s[0];
  }
  for (l = 0; l < f->L / 2; ++l) {
    const float t = v[l] / f->max;
    f->fac[l] = f->fac[l] + f->alpha * (t - f->fac[l]);
  }
  ++a->blocks;
}

void sdo_fac_finish(const sdo_fac *f, const sdo_fac_acc *a, sdo_fac_status *st)
{
  st->blocks = a->blocks; st->peak_lag = a->pos; st->max = f->max; st->min = f->min;
  st->sigmas = 0.0f; st->marker = 0;
  if (a->blocks > 0 && !isinf(a->local) && a->count > 0) {
    st->sigmas = a->local / sqrtf(a->power / (float) a->count);
    st->marker = (double) st->sigmas > f->sigma;
  }
}

void sdo_fac_feed(sdo_fac *f, const sdo_cpx *x, unsigned n, sdo_fac_status *st)
{
  sdo_fac_acc a;
  sdo_fac_acc_init(&a);
  while (n > 0) {
    unsigned got = f->L - f->p;
    if (got > n) got = n;
    memcpy(f->blk + f->p, x, got * sizeof(sdo_cpx));
    f->p += got; x += got; n -= got;
    if (f->p == f->L) {
      f->p = 0;
      sdo_fac_magnitude(f, f->blk, f->v, 0);
      sdo_fac_update(f, &a, f->v);
    }
  }
  sdo_fac_finish(f, &a, st);
}
