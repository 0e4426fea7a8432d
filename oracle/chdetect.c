/* chdetect.c -- ORACLE (test infrastructure): channel detector on the main PSD, SPEC.md section K.
 *
 * What the reference shows: the analyzer is parameterised with detector_params.{alpha, beta, gamma, snr} and
 * channel_update_int (Suscan/AnalyzerParams.cpp:27-66: "spectrumAvgAlpha", "sAvgAlpha", "nAvgAlpha", "snr"), and
 * delivers MESSAGE_TYPE_CHANNEL lists of struct sigutils_channel {fc, f_lo, f_hi, bw, snr, S0, N0, ft}
 * (Suscan/Messages/ChannelMessage.cpp:25-70, include/Suscan/Channel.h:26-32) that this GUI discards
 * (Suscan/Analyzer.cpp:75-98); the scanner switches the detector off (Panoramic/Scanner.cpp:325-329).  The
 * algorithm itself is upstream (sigutils su_channel_detector) and NOT in the reference: what follows is THIS
 * project's definition (parity unpinned), chosen to be order-independent so that a parallel implementation can
 * be bit-identical: exponential averaging, an exact order statistic for the noise floor, threshold, runs.
 */
#include "sd_oracle.h"
#include <stdlib.h>
#include <string.h>

int sdo_chdet_init(sdo_chdet *d, unsigned n, float alpha, float gamma, float snr, unsigned min_bins)
{
  memset(d, 0, sizeof(*d));
  if (n < 16 || (n & (n - 1))) return -1;
  d->n = n; d->alpha = alpha; d->gamma = gamma; d->snr = snr; d->min_bins = min_bins < 1 ? 1 : min_bins;
  d->avg = (float *) calloc(n, sizeof(float));
  d->tmp = (float *) calloc(n, sizeof(float));
  return d->avg && d->tmp ? 0 : -1;
}

void sdo_chdet_free(sdo_chdet *d) { free(d->avg); free(d->tmp); memset(d, 0, sizeof(*d)); }

static int cmp_float(const void *a, const void *b)
{
  const float x = *(const float *) a, y = *(const float *) b;
  return (x > y) - (x < y);
}

/* K.1-K.4: `frames` PSD frames of n bins (linear power, DC at index 0), then one channel update.
 * Returns the number of channels written (ascending frequency), at most cap. */
unsigned sdo_chdet_feed(sdo_chdet *d, const float *psd, unsigned frames, sdo_channel *out, unsigned cap)
{
  const unsigned n = d->n, half = n / 2;
  unsigned f, k, count = 0, i, raw = 0;
  float n0_inst, thr;
  if (frames == 0) return 0;                   /* K.2: a feed without frames changes nothing */
  for (f = 0; f < frames; ++f) {
    const float *p = psd + (size_t) f * n;
    if (!d->primed) { memcpy(d->avg, p, n * sizeof(float)); d->primed = 1; }
    else for (k = 0; k < n; ++k) d->avg[k] = d->avg[k] + d->alpha * (p[k] - d->avg[k]);
  }
  if (!d->primed) return 0;
  /* K.2 noise floor: the (n/4)-th smallest averaged bin, smoothed with gamma */
  memcpy(d->tmp, d->avg, n * sizeof(float));
  qsort(d->tmp, n, sizeof(float), cmp_float);
  n0_inst = d->tmp[n / 4];
  if (!d->n0_primed) { d->n0 = n0_inst; d->n0_primed = 1; }
  else d->n0 = d->n0 + d->gamma * (n0_inst - d->n0);
  thr = d->n0 * d->snr;
  /* K.3 / K.4: runs of bins above the threshold in ascending frequency (index j = (k + n/2) mod n) */
  i = 0;
  while (i < n) {
    unsigned a, b;
    float s0 = 0.0f;
    if (!(d->avg[(i + half) & (n - 1)] > thr)) { ++i; continue; }
    a = i;
    while (i < n && d->avg[(i + half) & (n - 1)] > thr) {
      const float v = d->avg[(i + half) & (n - 1)];
      if (v > s0) s0 = v;
      ++i;
    }
    b = i;
    if (raw == SDO_CHDET_MAXRAW) break;       /* K.4: only the first MAXRAW raw runs are examined */
    ++raw;
    if (b - a >= d->min_bins) {
      if (count < cap) {
        out[count].bin_lo = a; out[count].bin_hi = b;
        out[count].s0 = s0; out[count].n0 = d->n0; out[count].snr = s0 / d->n0;
      }
      ++count;
    }
  }
  d->last_total = count;
  return count < cap ? count : cap;
}
