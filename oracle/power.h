/*
 * power.h -- ORACLE (test infrastructure). The power inspector (SPEC_PW.md): the RMS tool's raw-mode integration
 * (Default/RMSInspector/RMSInspector.cpp:538-560, 327-338).  p = re re + im im in binary32, widened to binary64 and
 * added with Kahan compensation; every M samples the mean acc / n, rounded to binary32, is one output.  The group
 * carries across feeds.  Built on its own (power.mk).
 */
#ifndef SD_POWER_H
#define SD_POWER_H
#include <stddef.h>
#include <stdint.h>
#include "sd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  uint64_t M;                /* samples per mean, >= 1 (power.integrate-samples; 0 is read as 1) */
  double   acc, c;           /* Kahan sum of the group and its compensation */
  uint64_t n;                /* samples in the group */
} sdo_power;
void   sdo_power_init(sdo_power *p, uint64_t M);
size_t sdo_power_feed(sdo_power *p, const sdo_cpx *x, size_t m, float *mean);   /* -> means written */

#ifdef __cplusplus
}
#endif
#endif
