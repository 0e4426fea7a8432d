/*
 * chtrack.h -- ORACLE (test infrastructure). Channel tracking across detector updates (SPEC_KT.md): the SPEC K lists of
 * successive updates (sdo_chdet_feed, chdetect.c) in, a table of at most 256 live tracks out.  Built on its own
 * (chtrack.mk).
 */
#ifndef SD_CHTRACK_H
#define SD_CHTRACK_H
#include "sd_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

#define SDO_CHTRACK_CAP 256u
typedef struct {
  unsigned a, b;               /* [a, b) in ascending-frequency bin order */
  float    s0;                 /* beta-smoothed peak level */
  unsigned id, age, present, misses;
} sdo_track;
typedef struct {
  float    beta;
  unsigned hold, count, next_id;
  unsigned long long dropped;
  sdo_track tr[SDO_CHTRACK_CAP];  /* live tracks, ascending (a, id) */
} sdo_chtrack;
void sdo_chtrack_init(sdo_chtrack *t, float beta, unsigned hold);
void sdo_chtrack_update(sdo_chtrack *t, const sdo_channel *det, unsigned nd);

#ifdef __cplusplus
}
#endif
#endif
