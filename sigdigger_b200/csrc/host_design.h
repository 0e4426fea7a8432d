// host_design.h -- host-side set-up arithmetic of the product (not on the hot path): window taps,
// channel geometry, shaping response, RRC / Butterworth design, AGC constants.  Double precision,
// rounded to float once.  Formulas are SPEC.md sections W, S.2, S.3, I, A; the reference-side call
// sites that fix the parameterisation are cited per function.  Independent of oracle/ (the oracle
// states the same SPEC separately in C).
#pragma once
#include <math.h>
#include <stdint.h>
#include <complex>
#include <vector>
#include "sdb_math.h"

namespace sdbh {

static const double kPi = 3.14159265358979323846;

// SU_CHANNEL_DETECTOR_WINDOW_* taps (include/Suscan/AnalyzerParams.h:37-43), symmetric form.
inline void window_fill(std::vector<float> &w, unsigned n, int type)
{
  w.resize(n);
  for (unsigned i = 0; i < n; ++i) {
    double x = n > 1 ? 2.0 * kPi * (double) i / (double) (n - 1) : 0.0, v;
    switch (type) {
      case 1: v = 0.54 - 0.46 * cos(x); break;
      case 2: v = 0.5 - 0.5 * cos(x); break;
      case 3: v = 1.0 - 1.93 * cos(x) + 1.29 * cos(2 * x) - 0.388 * cos(3 * x) + 0.028 * cos(4 * x); break;
      case 4: v = 0.35875 - 0.48829 * cos(x) + 0.14128 * cos(2 * x) - 0.01168 * cos(3 * x); break;
      default: v = 1.0; break;
    }
    w[i] = (float) v;
  }
}

// su_specttuner_open_channel geometry (params at Tasks/LPFTask.cpp:63-67).
inline void channel_geometry(unsigned ws, float f0, float bw, float guard, unsigned *center,
                             unsigned *size, unsigned *width)
{
  const double N = (double) ws;
  double krel = (double) guard * (double) bw / (2.0 * kPi);
  double c = 2.0 * floor((double) f0 / (4.0 * kPi) * N + 0.5);
  double m = ceil(krel * N - 1e-3);
  if (m < 4.0) m = 4.0;
  if (m > N) m = N;
  unsigned msz = (unsigned) m, sz = 1;
  while (sz < msz) sz <<= 1;
  if (sz > ws) sz = ws;
  unsigned w = (unsigned) ceil((double) msz / (double) guard - 1e-3);
  if (w > sz) w = sz;
  if (w < 2) w = 2;
  *center = ((unsigned) c) % ws;
  *size = sz;
  *width = w;
}

// k*h for the 2*halfw copied bins, ordered from bin -halfw to +halfw-1 (SPEC S.3).
inline void channel_weights(unsigned ws, unsigned halfw, std::vector<float> &kh)
{
  static const double c[4] = { 0.35875, 0.48829 / 2.0, 0.14128 / 2.0, 0.01168 / 2.0 };
  const float k = 1.0f / (float) ws;
  kh.resize(2 * halfw);
  for (unsigned i = 0; i < 2 * halfw; ++i) {
    int b = (int) i - (int) halfw;
    double acc = 0.0;
    if (2 * halfw >= ws) acc = 1.0;
    else
      for (int m = -3; m <= 3; ++m) {
        int q = b - m;
        if (q >= -(int) halfw && q < (int) halfw) acc += c[m < 0 ? -m : m];
      }
    kh[i] = k * (float) acc;
  }
}

inline void xfade_fill(unsigned size, std::vector<float> &w)
{
  w.resize(size);
  for (unsigned i = 0; i < size; ++i) {
    double s = sin(kPi * (double) i / (double) size);
    w[i] = (float) (s * s);
  }
}

inline void twiddle_fill(unsigned n, std::vector<float2> &tw)
{
  tw.resize(n);
  for (unsigned i = 0; i < n; ++i) {
    double a = 2.0 * kPi * (double) i / (double) n;
    tw[i].x = (float) cos(a);
    tw[i].y = (float) -sin(a);
  }
}

// su_iir_rrc_init(filt, n, T, beta) (Tasks/WaveSampler.cpp:74-80), Hamming-windowed (manual p.61).
inline void taps_rrc(std::vector<float> &h, unsigned n, float T, float beta)
{
  h.resize(n);
  const double b = beta, Td = T;
  for (unsigned i = 0; i < n; ++i) {
    double t = ((double) i - (double) n / 2.0) / Td;
    double f = 4.0 * b * t;
    double dem = kPi * t * (1.0 - f * f);
    double num = sin(kPi * t * (1.0 - b)) + 4.0 * b * t * cos(kPi * t * (1.0 + b));
    double v;
    if (fabs(t) < 1e-9) v = 1.0 - b + 4.0 * b / kPi;
    else if (fabs(dem) < 1e-9)
      v = b / sqrt(2.0) * ((1.0 + 2.0 / kPi) * sin(kPi / (4.0 * b)) + (1.0 - 2.0 / kPi) * cos(kPi / (4.0 * b)));
    else v = num / dem;
    v /= Td;
    if (n > 1) v *= 0.54 - 0.46 * cos(2.0 * kPi * (double) i / (double) (n - 1));
    h[i] = (float) v;
  }
}

// SPEC I.3 (su_taps_brickwall_lp_init): h_i = fc sinc(fc (i - floor(n / 2))) x Hamming, binary64 rounded once
inline void taps_brickwall_lp(float *h, unsigned n, float fc)
{
  for (unsigned i = 0; i < n; ++i) {
    const double t = (double) i - (double) (n >> 1);
    const double xx = kPi * (double) fc * t;
    double v = fabs(xx) < 1e-12 ? (double) fc : (double) fc * sin(xx) / xx;
    if (n > 1) v *= 0.54 - 0.46 * cos(2.0 * kPi * (double) i / (double) (n - 1));
    h[i] = (float) v;
  }
}

inline unsigned mf_span(float T)  // include/WaveSampler.h:29-30
{
  double s = ceil(6.0 * (double) T);
  if (s < 1.0) s = 1.0;
  if (s > 1024.0) s = 1024.0;
  return (unsigned) s;
}

// Butterworth low-pass by bilinear transform; fc relative to Nyquist. order <= 4 here.
inline bool butter_lp(unsigned order, float fc, float *b, float *a)
{
  if (order < 1 || order > 16 || !(fc > 0.0f) || !(fc < 1.0f)) return false;
  typedef std::complex<double> cd;
  cd pz[16], pa[17], pb[17], kden(1.0, 0.0);
  double warped = 4.0 * tan(kPi * (double) fc / 2.0);
  for (unsigned k = 0; k < order; ++k) {
    double th = kPi * (2.0 * k + order + 1.0) / (2.0 * order);
    cd s = warped * cd(cos(th), sin(th));
    pz[k] = (4.0 + s) / (4.0 - s);
    kden *= (4.0 - s);
  }
  double gain = pow(warped, (double) order) * (1.0 / kden).real();
  for (unsigned k = 0; k <= order; ++k) { pa[k] = 0; pb[k] = 0; }
  pa[0] = 1.0; pb[0] = 1.0;
  for (unsigned k = 0; k < order; ++k)
    for (unsigned j = k + 1; j >= 1; --j) {
      pa[j] = pa[j] - pz[k] * pa[j - 1];
      pb[j] = pb[j] + pb[j - 1];
    }
  for (unsigned k = 0; k <= order; ++k) {
    a[k] = (float) pa[k].real();
    b[k] = (float) (gain * pb[k].real());
  }
  return true;
}

inline float alpha_of(float t) { return (float) (1.0 - exp(-1.0 / (double) t)); }

struct AgcDesign {
  float knee, gain_slope, fixed_gain, far_, faf, sar, saf;
  unsigned hang_max, dl_size, mh_size;
};

// AGC constants as fractions of tau (Tasks/AGCTask.cpp:22-28; frac_scale 2 there, 1 in inspectors).
inline AgcDesign agc_from_tau(float tau, float frac_scale)
{
  AgcDesign d;
  const float rise = frac_scale * 3.9062e-1f;
  float fast_rise_t = tau * rise;
  float fast_fall_t = tau * (2.0f * rise);
  float slow_rise_t = tau * (10.0f * rise);
  float slow_fall_t = tau * (10.0f * (2.0f * rise));
  d.hang_max = (unsigned) (tau * (rise * 5.0f));
  d.dl_size = (unsigned) (tau * (rise * 10.0f));
  d.mh_size = (unsigned) (tau * (rise * 10.0f));
  if (d.dl_size < 1) d.dl_size = 1;
  if (d.mh_size < 1) d.mh_size = 1;
  if (d.dl_size > 4096) d.dl_size = 4096;
  if (d.mh_size > 4096) d.mh_size = 4096;
  d.knee = -100.0f;
  d.gain_slope = 6.0f * 1e-2f;
  d.fixed_gain = d_db_to_mag(d.knee * (d.gain_slope - 1.0f));
  d.far_ = alpha_of(fast_rise_t);
  d.faf = alpha_of(fast_fall_t);
  d.sar = alpha_of(slow_rise_t);
  d.saf = alpha_of(slow_fall_t);
  return d;
}

inline float clampf(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }

}  // namespace sdbh
