/*
 * tvinsp.c -- ORACLE (test infrastructure). The inspector's Analog TV tab, SPEC_TI.md.  The conversion is
 * sdo_tv_feed_transform and the step sdo_tv_feed, both of tvproc.c, called here and not copied.
 */
#include "tvinsp.h"
#include <stdlib.h>
#include <string.h>

static void tvinsp_estimates(sdo_tvinsp *t)
{
  sdo_tv_estimates(t->tv, &t->st.line_len, &t->st.hsync_len, &t->st.agc_gain);
  t->st.frames = sdo_tv_frames(t->tv);
}

int sdo_tvinsp_init(sdo_tvinsp *t, int insp_class, const sdo_tv_params *p, int invert_sync, float dc)
{
  int w, h;
  memset(t, 0, sizeof *t);
  if (insp_class < 0 || insp_class > 2 || !(t->tv = sdo_tv_new(p))) return -1;
  sdo_tv_geometry(t->tv, &w, &h);
  t->posted = calloc((size_t) w * h, sizeof(float));
  t->mode = insp_class == 2 ? 0 : 1;
  t->k = invert_sync ? -1.0f : 1.0f; t->dc = dc;
  t->st.width = (uint32_t) w; t->st.height = (uint32_t) h;
  tvinsp_estimates(t);
  return 0;
}

void sdo_tvinsp_free(sdo_tvinsp *t)
{
  sdo_tv_destroy(t->tv);
  free(t->posted);
  memset(t, 0, sizeof *t);
}

int sdo_tvinsp_set_params(sdo_tvinsp *t, const sdo_tv_params *p, int invert_sync, float dc)
{
  if (!sdo_tv_set_params(t->tv, p)) return -1;
  t->k = invert_sync ? -1.0f : 1.0f; t->dc = dc;
  return 0;
}

void sdo_tvinsp_feed(sdo_tvinsp *t, const sdo_cpx *x, unsigned n)
{
  unsigned i;
  t->st.completed = 0;
  for (i = 0; i < n; ++i) {
    float v;
    sdo_tv_feed_transform(x + i, 1, t->mode, t->k, t->dc, &v);                   /* TI.1 */
    if (sdo_tv_feed(t->tv, v) && ++t->st.completed == 1) {                        /* TI.3: the first, as it stands */
      const uint64_t f = sdo_tv_frames(t->tv);
      memcpy(t->posted, sdo_tv_frame(t->tv, f - 1), (size_t) t->st.width * t->st.height * sizeof(float));
      t->st.posted_no = f;
    }
  }
  tvinsp_estimates(t);
}
