/*
 * fac.h -- ORACLE (test infrastructure). The inspector's FAC tab (SPEC_FC.md): blocks of L soft symbols in, the
 * averaged, peak-marked autocorrelation out.  Built on its own (fac.mk) with the SPEC transforms of fft_spec.c.
 */
#ifndef SD_FAC_H
#define SD_FAC_H
#include "sd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

#define SDO_FAC_TILE 1024u
typedef struct { unsigned blocks, peak_lag; float max, min, sigmas; int marker; } sdo_fac_status;
typedef struct {
  unsigned L, lo, hi;          /* block size, lag window [lo, hi) */
  float alpha; double sigma;
  unsigned p;                  /* fill of the carried block */
  float max, min;              /* running extremes of v over the window (FC.2) */
  sdo_cpx *blk; float *fac, *v;
  sdo_spec_plan plan;          /* F.2 (L <= 4096) or F.3 (kind 1) */
} sdo_fac;
/* the per-feed accumulator of FC.2 / FC.4 */
typedef struct { unsigned blocks, pos, count; float local, power; } sdo_fac_acc;

int  sdo_fac_init(sdo_fac *f, unsigned L, float alpha, unsigned lo, unsigned hi, double sigma);
void sdo_fac_free(sdo_fac *f);
/* FC.1: v[l] = |A[l]|, l < L / 2, of one block.  twice = 1 runs the forward dataflow twice (|F_L(P)|) also for
 * L <= 4096, where the statement is the F.2 inverse (the identity of FC.1) */
void sdo_fac_magnitude(sdo_fac *f, const sdo_cpx *block, float *v, int twice);
/* FC.2 / FC.3 for one block's v; FC.4 closes a feed */
void sdo_fac_acc_init(sdo_fac_acc *a);
void sdo_fac_update(sdo_fac *f, sdo_fac_acc *a, const float *v);
void sdo_fac_finish(const sdo_fac *f, const sdo_fac_acc *a, sdo_fac_status *st);
/* one feed of n symbols: blocks, statistics, averaging and status */
void sdo_fac_feed(sdo_fac *f, const sdo_cpx *x, unsigned n, sdo_fac_status *st);

#ifdef __cplusplus
}
#endif
#endif
