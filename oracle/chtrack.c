/* ORACLE (test infrastructure): SPEC KT, channel tracking across detector updates.  See chtrack.h. */
#include "chtrack.h"
#include <string.h>

/* KT (SPEC_KT.md): one tracking update over the K.4 list det[0 .. nd) of the same update, in ascending frequency.
 * The table stays in ascending (a, id); the caller skips updates of feeds without frames (KT.1). */
void sdo_chtrack_init(sdo_chtrack *t, float beta, unsigned hold)
{
  memset(t, 0, sizeof(*t));
  t->beta = beta; t->hold = hold; t->next_id = 1;
}

static int track_before(const sdo_track *x, const sdo_track *y)
{
  return x->a < y->a || (x->a == y->a && x->id < y->id);
}

void sdo_chtrack_update(sdo_chtrack *t, const sdo_channel *det, unsigned nd)
{
  int matched[SDO_CHTRACK_CAP];
  sdo_track next[SDO_CHTRACK_CAP];
  unsigned i, j, n = 0, live;
  int det_matched[SDO_CHTRACK_CAP];
  for (i = 0; i < t->count; ++i) matched[i] = 0;
  /* KT.3 / KT.4: detections in ascending frequency, each takes the unmatched track of largest overlap; the table is
   * in ascending (a, id), so the first of equal overlaps is the tie-break winner */
  for (j = 0; j < nd; ++j) {
    int best = -1;
    long best_ov = 0;
    for (i = 0; i < t->count; ++i) {
      const long lo = det[j].bin_lo > t->tr[i].a ? det[j].bin_lo : t->tr[i].a;
      const long hi = det[j].bin_hi < t->tr[i].b ? det[j].bin_hi : t->tr[i].b;
      if (matched[i] || hi - lo <= 0) continue;
      if (hi - lo > best_ov) { best_ov = hi - lo; best = (int) i; }
    }
    det_matched[j] = best >= 0;
    if (best >= 0) {
      sdo_track *r = &t->tr[best];
      matched[best] = 1;
      r->a = det[j].bin_lo; r->b = det[j].bin_hi;
      r->s0 = r->s0 + t->beta * (det[j].s0 - r->s0);
      r->age += 1; r->present += 1; r->misses = 0;
    }
  }
  /* KT.5: unmatched tracks age; removals before any insertion */
  for (i = 0; i < t->count; ++i) {
    sdo_track r = t->tr[i];
    if (!matched[i]) {
      r.age += 1; r.misses += 1;
      if (r.misses > t->hold) continue;
    }
    next[n++] = r;
  }
  live = n;
  /* KT.6: unmatched detections open tracks in ascending frequency while fewer than 256 are live */
  for (j = 0; j < nd; ++j) {
    if (det_matched[j]) continue;
    if (live == SDO_CHTRACK_CAP) { ++t->dropped; continue; }
    next[live].a = det[j].bin_lo; next[live].b = det[j].bin_hi; next[live].s0 = det[j].s0;
    next[live].id = t->next_id++;
    next[live].age = 1; next[live].present = 1; next[live].misses = 0;
    ++live;
  }
  /* KT.7: ascending (a, id), by insertion */
  for (i = 0; i < live; ++i) {
    sdo_track r = next[i];
    unsigned k = i;
    while (k > 0 && track_before(&r, &t->tr[k - 1])) { t->tr[k] = t->tr[k - 1]; --k; }
    t->tr[k] = r;
  }
  t->count = live;
}
