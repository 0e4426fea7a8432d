/*
 * snr.h -- ORACLE (test infrastructure). The inspector's SNR meter (SPEC_SN.md): a psk / fsk / ask inspector's soft
 * symbols binned into the decision-space histogram (SN.1), one SPEC Y.7 step per feed that brought symbols (SN.2, the
 * step of tasks.c), and the state rules of SN.3 / SN.4.  Built on its own (snr.mk).
 */
#ifndef SD_SNR_H
#define SD_SNR_H
#include "sd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { unsigned long long counted; unsigned steps, stepped; float sigma, snr, delta; } sdo_snr_status;
typedef struct {
  unsigned L, K, bps;          /* bins, comb teeth 2^bps (bps 0 read as 1), bits per symbol */
  int mode;                    /* SPEC D: SDO_DECIDE_ARGUMENT (psk, fsk) or SDO_DECIDE_MODULUS (ask) */
  unsigned *h;                 /* h[L] */
  float *model;                /* H[L] of the latest step (0 before the first) */
  sdo_snr_estimator est;       /* the Y.7 state: sigma, alpha, delta */
  sdo_snr_status st;
} sdo_snrm;

/* SN.3: switch the meter on (class 0 psk, 1 fsk, 2 ask); -1 for another class or L outside [16, 1024] */
int      sdo_snrm_init(sdo_snrm *m, int insp_class, unsigned L, unsigned bps, float sigma, float alpha);
void     sdo_snrm_free(sdo_snrm *m);
/* SN.1: the bin of one symbol, or L when it is not counted */
unsigned sdo_snrm_bin(int mode, unsigned L, sdo_cpx x);
/* SN.2: one feed of n soft symbols */
void     sdo_snrm_feed(sdo_snrm *m, const sdo_cpx *x, unsigned n);
/* SN.3: the reset (sigma only) */
void     sdo_snrm_reset(sdo_snrm *m, float sigma);
/* SN.4: a re-plan that keeps the class and L; same_cfg = the inspector configuration is unchanged field by field */
void     sdo_snrm_replan(sdo_snrm *m, int same_cfg, unsigned bps, float alpha);

#ifdef __cplusplus
}
#endif
#endif
