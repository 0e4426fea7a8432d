// sdb_tv_steps.h -- the analog-TV processor's per-sample recurrence (SPEC.md section TV), written once for
//   * device: k_tv_feed (tv_kernels.cu), one warp per processor, lane 0 runs this step;
//   * host:   su_tv_processor_feed of the sigutils-named shim (a per-sample call by ABI:
//             Default/GenericInspector/TVProcessorWorker.cpp:133).
// What it replaces: su_tv_processor_{new, feed, take_frame, set_params} of sigutils as the reference drives them
// (Default/GenericInspector/TVProcessorWorker.cpp:120-151, 186-239; parameter block filled at
// Default/GenericInspector/TVProcessorTab.cpp:549-597).  The algorithm is upstream's (not in the reference):
// SPEC TV is this project's statement of it -- comb filter, peak AGC, pulse filter, horizontal flywheel with slow /
// fast tracking, equalising-pulse vertical sync, sub-pixel raster.  Every expression is IEEE binary32 in source order
// (units compiled with -fmad=false / -ffp-contract=off), so host, device and oracle/tvproc.c agree bit for bit.
#pragma once
#include "sdb_internal.h"
#include "sdb_math.h"
#include <stdint.h>

#define SDB_TV_RING 4          // frame buffers per processor (completed frames are read from the ring)
#define SDB_TV_MAX_W 4096      // pixels per line the shared-memory line buffer holds
#define SDB_TV_MAX_H 4096

// derived, read-only while the processor runs (SPEC TV.1)
struct SdbTvCfg {
  int enable_sync, reverse, interlace, enable_agc, dominance, enable_comb, comb_reverse;
  int W, H, delay_len;
  unsigned vsync_trigger;
  float x_off, frame_spacing, hsync_len, vsync_len, line_len;
  float t_tol, g_tol, thr;                     // thr = 1 - l_tol
  float huge_err, max_err, min_err;
  float agc_alpha, pulse_alpha, hsync_len_alpha, line_len_alpha, fast_alpha, slow_alpha;
};

struct SdbTvState {
  unsigned long long ptr, sync_start, last_hsync, last_short;
  unsigned long long frames;                   // completed frames; the current one goes to ring slot frames % SDB_TV_RING
  int field_x, field_y, field_parity, field_lines, row;
  float field_x_dec;
  int delay_ptr;
  float agc_gain, agc_line_max, agc_accum; unsigned agc_lines;
  float pulse;
  int sync_found, have_last_hsync, slow_track;
  float est_hsync_len, est_line_len, ll_accum; unsigned ll_count;
  unsigned vsync_counter, lines_since_vsync;
};

enum { SDB_TV_LINE_DONE = 1, SDB_TV_FRAME_DONE = 2 };

SDB_HD int sdb_tv_row_of(const SdbTvCfg &c, int field_y, int parity)
{
  const int row = c.interlace ? 2 * field_y + (parity ^ (c.dominance ? 0 : 1)) : field_y;
  return row >= 0 && row < c.H ? row : -1;
}

SDB_HD void sdb_tv_state_init(const SdbTvCfg &c, SdbTvState &s)
{
  s.ptr = 0; s.sync_start = 0; s.last_hsync = 0; s.last_short = 0; s.frames = 0;
  s.field_x = 0; s.field_x_dec = 0.0f; s.field_y = 0; s.field_parity = 0;
  s.field_lines = c.interlace ? (c.H + 1) / 2 : c.H;
  s.row = sdb_tv_row_of(c, 0, 0);
  s.delay_ptr = 0;
  s.agc_gain = 1.0f; s.agc_line_max = 0.0f; s.agc_accum = 0.0f; s.agc_lines = 0;
  s.pulse = 0.0f; s.sync_found = 0; s.have_last_hsync = 0; s.slow_track = 0;
  s.est_hsync_len = c.hsync_len; s.est_line_len = c.line_len; s.ll_accum = 0.0f; s.ll_count = 0;
  s.vsync_counter = 0; s.lines_since_vsync = 0x7fffffffu;
}

SDB_HD void sdb_tv_set_xf(SdbTvState &s, float xf)
{
  const float fl = floorf(xf);
  s.field_x = (int) fl;
  s.field_x_dec = xf - fl;
}

// One input sample.  `delay` [delay_len] and `line` [W] are the processor's comb delay line and the row being drawn.
// Returns SDB_TV_LINE_DONE when the row is complete: the CALLER stores `line` as row *flush_row (if >= 0) of ring slot
// *flush_slot and clears it, before the next sample; | SDB_TV_FRAME_DONE when that row was the last of a frame.
SDB_HD int sdb_tv_step(const SdbTvCfg &c, SdbTvState &s, float *delay, float *line, float x, int *flush_row,
                       int *flush_slot)
{
  // ---- TV.2 comb filter over one line period
  if (c.enable_comb) {
    const float prev = delay[s.delay_ptr];
    delay[s.delay_ptr] = x;
    s.delay_ptr = s.delay_ptr + 1 == c.delay_len ? 0 : s.delay_ptr + 1;
    x = 0.5f * (c.comb_reverse ? x - prev : x + prev);
  }
  // ---- TV.3 peak AGC: the sync tip is the line's maximum
  if (x > s.agc_line_max) s.agc_line_max = x;
  const float xg = c.enable_agc ? s.agc_gain * x : x;
  // ---- TV.4 pulse filter
  s.pulse = s.pulse + c.pulse_alpha * (xg - s.pulse);
  // ---- TV.5 sync separator
  if (c.enable_sync) {
    const int up = s.pulse > c.thr;
    if (!s.sync_found) {
      if (up) { s.sync_found = 1; s.sync_start = s.ptr; }
    } else if (!up) {
      s.sync_found = 0;
      const float len = (float) (s.ptr - s.sync_start);
      if (fabsf(len - s.est_hsync_len) <= c.t_tol * s.est_hsync_len) {
        // line length from consecutive horizontal pulses
        if (s.have_last_hsync) {
          const float dl = (float) (s.sync_start - s.last_hsync);
          if (fabsf(dl - s.est_line_len) <= c.g_tol * s.est_line_len) { s.ll_accum = s.ll_accum + dl; s.ll_count += 1; }
        }
        s.have_last_hsync = 1; s.last_hsync = s.sync_start;
        // horizontal flywheel: the pulse centre belongs at hsync_len / 2 + x_off
        s.est_hsync_len = s.est_hsync_len + c.hsync_len_alpha * (len - s.est_hsync_len);
        float xf = (float) s.field_x + s.field_x_dec;
        const float L = s.est_line_len;
        float err = (0.5f * s.est_hsync_len + c.x_off) - (xf - 0.5f * len);
        if (err > 0.5f * L) err = err - L; else if (err < -0.5f * L) err = err + L;
        const float rel = fabsf(err) / L;
        if (rel > c.max_err) s.slow_track = 0; else if (rel < c.min_err) s.slow_track = 1;
        if (rel > c.huge_err) xf = xf + err;
        else xf = xf + (s.slow_track ? c.slow_alpha : c.fast_alpha) * err;
        if (xf < 0.0f) xf = xf + L;
        sdb_tv_set_xf(s, xf);
      } else {
        s.have_last_hsync = 0;
        if (fabsf(len - c.vsync_len) <= 2.0f * c.t_tol * c.vsync_len) {
          // equalising pulses come half a line apart; the vsync_trigger-th of a train ends the field
          const float age = (float) (s.sync_start - s.last_short);
          if (s.vsync_counter > 0 && fabsf(age - 0.5f * s.est_line_len) <= 2.0f * c.t_tol * s.est_line_len)
            s.vsync_counter += 1;
          else
            s.vsync_counter = 1;
          s.last_short = s.sync_start;
          if (s.vsync_counter == c.vsync_trigger && s.lines_since_vsync >= (unsigned) (s.field_lines / 2)) {
            s.lines_since_vsync = 0;
            // the field boundary is the end of this line.  Late in a field: end it here.  Early in a field (the
            // flywheel wrapped a line or so before the train said so): stay in it and restart its line count.
            const int early = s.field_y < s.field_lines / 2;
            if (c.interlace) {
              // a train whose trigger pulse sits mid-line precedes the second field
              const float pos = ((float) s.field_x + s.field_x_dec) - 0.5f * len;
              const int mid = fabsf(pos - 0.5f * s.est_line_len) < 0.25f * s.est_line_len;
              const int next = mid ? 1 : 0;
              s.field_parity = early ? next : next ^ 1;     // (late: swapped when this line ends)
              s.field_lines = s.field_parity == 0 ? (c.H + 1) / 2 : c.H / 2;
            }
            s.field_y = early ? -1 : s.field_lines - 1;
          }
        } else {
          s.vsync_counter = 0;                             // a broad pulse (or noise) ends the train
        }
      }
    }
  }
  // ---- TV.6 raster: the sample at x = n + d adds (1 - d) v to pixel n and starts pixel n + 1 with d v
  const float val = c.reverse ? xg : 1.0f - xg;
  {
    const int n = s.field_x; const float d = s.field_x_dec;
    if (n >= 0 && n < c.W) line[n] = line[n] + (1.0f - d) * val;
    if (n + 1 >= 0 && n + 1 < c.W) line[n + 1] = d * val;
  }
  s.field_x += 1;
  int flags = 0;
  float xf = (float) s.field_x + s.field_x_dec;
  if (xf >= s.est_line_len) {
    flags = SDB_TV_LINE_DONE;
    *flush_row = s.row; *flush_slot = (int) (s.frames % SDB_TV_RING);
    xf = xf - s.est_line_len;
    s.agc_accum = s.agc_accum + s.agc_line_max; s.agc_lines += 1; s.agc_line_max = 0.0f;
    if (s.lines_since_vsync < 0x7fffffffu) s.lines_since_vsync += 1;
    s.field_y += 1;
    if (s.field_y >= s.field_lines) {
      s.field_y = 0;
      if (c.enable_agc && s.agc_lines > 0 && s.agc_accum > 0.0f)
        s.agc_gain = s.agc_gain + c.agc_alpha * ((float) s.agc_lines / s.agc_accum - s.agc_gain);
      s.agc_accum = 0.0f; s.agc_lines = 0;
      if (s.ll_count > 0) {
        s.est_line_len = s.est_line_len + c.line_len_alpha * (s.ll_accum / (float) s.ll_count - s.est_line_len);
        s.ll_accum = 0.0f; s.ll_count = 0;
      }
      int frame_done = 1;
      if (c.interlace) {
        s.field_parity ^= 1;
        s.field_lines = s.field_parity == 0 ? (c.H + 1) / 2 : c.H / 2;
        frame_done = s.field_parity == 0;
      }
      if (frame_done) {
        flags |= SDB_TV_FRAME_DONE;
        s.frames += 1;
        xf = xf - c.frame_spacing * s.est_line_len;
      }
    }
    sdb_tv_set_xf(s, xf);
    s.row = sdb_tv_row_of(c, s.field_y, s.field_parity);
  }
  s.ptr += 1;
  return flags;
}

// ---- the engine's Analog TV tab (oracle/SPEC_TI.md; k_tv_insp in tv_kernels.cu).  One descriptor per channel with
// the TV on; its processors are chain0 + s (s < n_streams), each with its delay line, row, ring and posted frame at
// the channel's offset + s times their size.
struct SdbTvInspChan {
  SdbTvCfg c;
  uint32_t k, chain0;                 // channel (symbol row s * n_channels + k), first processor
  int32_t mode;                       // TI.1: 0 modulus (ask), 1 argument (psk, fsk), as k_tv_feed_transform
  float gain, dc;                     // TI.1: k = -1 (invert_sync) or +1, and dc
  size_t delay_off, line_off, ring_off, post_off;
};
struct SdbTvInspArgs {
  const SdbTvInspChan *chans; int n_chans, n_streams, n_channels; size_t smem;
  const float2 *soft; const uint32_t *counts; size_t sym_cap;
  SdbTvState *state; float *delay, *line, *ring, *post; sdb_tv_status *status;
};
cudaError_t sdb_launch_tv_insp(const SdbLaunchCtx &ctx, const SdbTvInspArgs &a);

// ---- host-side: validity and derived constants (SPEC TV.0 / TV.1).  P has the fields of sigutils_tv_processor_params
// (sdb_tv_params in the C-ABI, struct sigutils_tv_processor_params in <sigutils/tvproc.h>).
#include <math.h>
static inline float sdb_tv_alpha(float tau) { return 1.0f - expf(-1.0f / tau); }       // SU_SPLPF_ALPHA

template <class P> static inline bool sdb_tv_params_valid(const P &p)
{
  if (!(p.line_len >= 8.0f) || !(p.line_len < (float) SDB_TV_MAX_W + 1.0f)) return false;
  if (!(p.hsync_len >= 1.0f) || !(p.hsync_len < 0.5f * p.line_len) || !(p.vsync_len >= 1.0f)) return false;
  if (p.frame_lines < 2 || p.frame_lines > SDB_TV_MAX_H) return false;
  if (!(p.frame_spacing >= 0.0f && p.frame_spacing < 1.0f)) return false;
  if (!(p.t_tol > 0 && p.t_tol < 1) || !(p.l_tol > 0 && p.l_tol < 1) || !(p.g_tol > 0 && p.g_tol < 1)) return false;
  if (!(p.hsync_len_tau > 0) || !(p.line_len_tau > 0) || !(p.agc_tau > 0) || !(p.hsync_fast_track_tau > 0) ||
      !(p.hsync_slow_track_tau > 0))
    return false;
  return true;
}

template <class P> static inline void sdb_tv_derive(const P &p, SdbTvCfg &c)
{
  c.enable_sync = p.enable_sync != 0; c.reverse = p.reverse != 0; c.interlace = p.interlace != 0;
  c.enable_agc = p.enable_agc != 0; c.dominance = p.dominance != 0; c.enable_comb = p.enable_comb != 0;
  c.comb_reverse = p.comb_reverse != 0;
  c.W = (int) floorf(p.line_len); c.H = (int) p.frame_lines; c.delay_len = (int) ceilf(p.line_len);
  c.vsync_trigger = (unsigned) p.vsync_odd_trigger;
  c.x_off = p.x_off; c.frame_spacing = p.frame_spacing; c.hsync_len = p.hsync_len; c.vsync_len = p.vsync_len;
  c.line_len = p.line_len;
  c.t_tol = p.t_tol; c.g_tol = p.g_tol; c.thr = 1.0f - p.l_tol;
  c.huge_err = p.hsync_huge_err; c.max_err = p.hsync_max_err; c.min_err = p.hsync_min_err;
  float pt = p.hsync_len / 20.0f;
  if (pt < 1.0f) pt = 1.0f;
  c.agc_alpha = sdb_tv_alpha(p.agc_tau); c.pulse_alpha = sdb_tv_alpha(pt);
  c.hsync_len_alpha = sdb_tv_alpha(p.hsync_len_tau); c.line_len_alpha = sdb_tv_alpha(p.line_len_tau);
  c.fast_alpha = sdb_tv_alpha(p.hsync_fast_track_tau); c.slow_alpha = sdb_tv_alpha(p.hsync_slow_track_tau);
}

// the GUI's presets (su_tv_processor_params_pal / _ntsc, Default/GenericInspector/TVProcessorTab.cpp:629,633)
template <class P> static inline void sdb_tv_preset(P &p, float fs, bool pal)
{
  p.enable_sync = 1; p.reverse = 0; p.interlace = 1; p.enable_agc = 1; p.x_off = 0; p.dominance = 1;
  p.frame_spacing = 0; p.enable_comb = 1; p.comb_reverse = 0;
  p.t_tol = 1e-1f; p.l_tol = 1e-1f; p.g_tol = 1e-1f;
  p.hsync_huge_err = .25f; p.hsync_max_err = 1e-2f; p.hsync_min_err = .5e-2f;
  p.hsync_len_tau = 9.5f; p.line_len_tau = 1e3f; p.agc_tau = 1e-5f;
  p.hsync_fast_track_tau = 9.5f; p.hsync_slow_track_tau = 1e3f;
  if (pal) {
    p.frame_lines = 625; p.hsync_len = fs * 4e-6f; p.vsync_len = fs * 2e-6f; p.line_len = fs * 64e-6f;
    p.vsync_odd_trigger = 5;
  } else {
    p.frame_lines = 525; p.hsync_len = fs * 4.749e-6f; p.vsync_len = fs * 2.375e-6f; p.line_len = fs * 63.556e-6f;
    p.vsync_odd_trigger = 6;
  }
}
