/*
 * decimate.h -- ORACLE (test infrastructure). Source decimation (SPEC_L.md): taps sdo_taps_brickwall_lp(16 D + 1, 1/D),
 * output k = sum h_i x[kD - i].  Input in a SPEC Q format (the SDB_FORMAT_* order); the carry makes the output
 * independent of how the input is split into feeds.  Built on its own over libsdoracle.so (decimate.mk).
 */
#ifndef SD_DECIMATE_H
#define SD_DECIMATE_H
#include "sd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { SDO_FMT_F32 = 0, SDO_FMT_U8 = 1, SDO_FMT_S8 = 2, SDO_FMT_S16 = 3 };
#define SDO_DECIM_MAX 256
typedef struct {
  unsigned D, n;             /* decimation, taps (16 D + 1) */
  float   *h;
  sdo_cpx *hist;             /* the last 16 D input samples, oldest first */
  unsigned phase;            /* input samples fed so far, modulo D */
} sdo_decimate;
int    sdo_decimate_init(sdo_decimate *d, unsigned D);
void   sdo_decimate_free(sdo_decimate *d);
void   sdo_decimate_reset(sdo_decimate *d);
size_t sdo_decimate_feed(sdo_decimate *d, const void *x, int fmt, size_t m, sdo_cpx *y);   /* -> outputs written */

#ifdef __cplusplus
}
#endif
#endif
