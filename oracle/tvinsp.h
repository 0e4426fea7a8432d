/*
 * tvinsp.h -- ORACLE (test infrastructure). The inspector's Analog TV tab (SPEC_TI.md): a psk / fsk / ask inspector's
 * soft symbols converted as TVProcessorTab::feed converts them (TI.1, sdo_tv_feed_transform), one SPEC TV step each
 * (sdo_tv_feed of tvproc.c), and the first frame a feed completes posted as it stood when it completed (TI.3).  Built on
 * its own (tvinsp.mk).
 */
#ifndef SD_TVINSP_H
#define SD_TVINSP_H
#include "sd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* as sdb_tv_status: frames so far; the posted frame's number (1 = the first frame, 0 before any); frames the latest
 * feed completed; W, H; the estimates after the feed */
typedef struct {
  uint64_t frames, posted_no;
  uint32_t completed, width, height;
  float line_len, hsync_len, agc_gain;
} sdo_tvinsp_status;
typedef struct {
  sdo_tv *tv;
  int mode;                    /* sdo_tv_feed_transform: 0 modulus (ask), 1 argument (psk, fsk) */
  float k, dc;                 /* -1 with invert_sync, +1 otherwise; the value added */
  float *posted;               /* [H][W] */
  sdo_tvinsp_status st;
} sdo_tvinsp;

/* the tab on (class 0 psk, 1 fsk, 2 ask); -1 for another class or parameters sdo_tv_new refuses */
int  sdo_tvinsp_init(sdo_tvinsp *t, int insp_class, const sdo_tv_params *p, int invert_sync, float dc);
void sdo_tvinsp_free(sdo_tvinsp *t);
/* TI.4: from the next symbol on; -1 (nothing changed) when invalid or when the geometry would change */
int  sdo_tvinsp_set_params(sdo_tvinsp *t, const sdo_tv_params *p, int invert_sync, float dc);
/* TI.1-TI.3: one feed of n soft symbols */
void sdo_tvinsp_feed(sdo_tvinsp *t, const sdo_cpx *x, unsigned n);

#ifdef __cplusplus
}
#endif
#endif
