"""Exact binary32 statement of the analog-TV processor, SPEC.md section TV.  TEST INFRASTRUCTURE ONLY.

Written from the SPEC text alone, independently of oracle/tvproc.c and of sdb_tv_steps.h (the step k_tv_feed runs on
the device and the <sigutils/tvproc.h> shim on the host).  The processor is a per-sample recurrence full of
discontinuities (the sync threshold, the tolerance windows, the `lines_since_vs` gate, `xf >= L`), so the statement
is exact: numpy binary32 scalars, one rounding per SPEC operation in the order written, no contraction; counters and
the sample counter are Python integers, and their differences are rounded once to binary32.  `α(τ)` is
`1 − exp(−1/τ)` with `exp` correctly rounded (binary64 `math.exp` of the binary32 quotient, rounded once), which SPEC
TV.1 allows in place of C's `expf`.

`TvStmt.hits` counts every branch of the step taken (BRANCHES, in the step's order), plus the two equality edges
EDGES, so that a scene can show which rules it exercised.

`mistake` plants one deliberate error, so that the tests can show the comparison would catch it:
    "t_tol_lt"            the horizontal window with < instead of <=
    "line_max_kept"       the line peak never reset at a line end
    "fs_pre_update"       the frame_spacing shift with the line length before that field's update
    "late_no_preswap"     a late trigger sets the announced parity directly, without the pre-swap
    "dominance_inverted"  the field row offset is parity xor dominance instead of parity xor !dominance
    "comb_sign"           the comb filter's sum and difference exchanged
    "no_xf_wrap"          no +L when the flywheel correction leaves xf < 0
    "gate_gt"             the lines_since_vs gate with > instead of >=
"""
import math
from collections import Counter

import numpy as np

F = np.float32
MISTAKES = ("t_tol_lt", "line_max_kept", "fs_pre_update", "late_no_preswap", "dominance_inverted", "comb_sign",
            "no_xf_wrap", "gate_gt")
RING = 4
MAX_W = MAX_H = 4096
SAT = 0x7FFFFFFF

BRANCHES = (
    "comb_sum", "comb_diff", "agc_peak", "agc_off",                        # TV.2, TV.3
    "sync_off", "rise", "fall",                                             # TV.5 edges
    "hsync", "ll_first", "ll_accept", "ll_reject",                          # horizontal pulse, line-length sample
    "err_wrap_hi", "err_wrap_lo", "to_fast", "to_slow", "huge_jump", "track_fast", "track_slow", "xf_wrap",
    "equalising", "eq_count", "eq_restart", "broad",                        # equalising train
    "trigger", "trigger_gated", "trigger_early", "trigger_late", "parity_mid", "parity_start",
    "raster_left", "raster_right",                                          # TV.6 pixels outside [0, W)
    "line_end", "row_off", "field_end", "agc_update", "agc_hold", "ll_update", "field_odd", "frame_end",
)
EDGES = ("t_tol_edge", "gate_edge")        # |len - est_hsync| == t_tol est_hsync; lines_since_vs == field_lines / 2

FIELDS = ("enable_sync", "reverse", "interlace", "enable_agc", "x_off", "dominance", "frame_lines", "frame_spacing",
          "enable_comb", "comb_reverse", "hsync_len", "vsync_len", "line_len", "vsync_odd_trigger", "t_tol", "l_tol",
          "g_tol", "hsync_huge_err", "hsync_max_err", "hsync_min_err", "hsync_len_tau", "line_len_tau", "agc_tau",
          "hsync_fast_track_tau", "hsync_slow_track_tau")
INTS = {"enable_sync", "reverse", "interlace", "enable_agc", "dominance", "frame_lines", "enable_comb", "comb_reverse",
        "vsync_odd_trigger"}


def params(p):
    """the parameter block as a dict of Python ints (switches, counts) and binary32 scalars"""
    get = p.get if isinstance(p, dict) else (lambda k: getattr(p, k))
    return {k: int(get(k)) if k in INTS else F(get(k)) for k in FIELDS}


def alpha(tau):
    """TV.1: 1 - exp(-1/tau), the quotient and the difference in binary32, exp correctly rounded"""
    q = F(-1.0) / F(tau)
    return F(1.0) - F(math.exp(float(q)))


def valid(p):
    """TV.0"""
    p = params(p)
    ok = F(8.0) <= p["line_len"] < F(MAX_W + 1)
    ok = ok and F(1.0) <= p["hsync_len"] < F(0.5) * p["line_len"] and p["vsync_len"] >= F(1.0)
    ok = ok and 2 <= p["frame_lines"] <= MAX_H and F(0.0) <= p["frame_spacing"] < F(1.0)
    ok = ok and all(F(0.0) < p[k] < F(1.0) for k in ("t_tol", "l_tol", "g_tol"))
    return bool(ok and all(p[k] > F(0.0) for k in ("hsync_len_tau", "line_len_tau", "agc_tau", "hsync_fast_track_tau",
                                                   "hsync_slow_track_tau")))


class TvStmt:
    def __init__(self, p, mistake=None):
        assert mistake is None or mistake in MISTAKES
        assert valid(p), "invalid parameters"
        self.mistake = mistake
        self.hits = Counter()
        self._derive(params(p))
        q = self.p
        # TV.1 geometry, fixed for the processor's life
        self.W, self.H, self.dlen = int(np.floor(q["line_len"])), q["frame_lines"], int(np.ceil(q["line_len"]))
        self.interlace = q["interlace"]
        self.ring = np.zeros((RING, self.H, self.W), F)
        self.dl = [F(0.0)] * self.dlen
        self.line = [F(0.0)] * self.W
        # initial state
        self.dp = 0
        self.ptr = 0
        self.gain, self.line_max, self.accum, self.agc_lines = F(1.0), F(0.0), F(0.0), 0
        self.pulse = F(0.0)
        self.sync, self.start = False, 0
        self.have_last, self.last_hsync, self.slow = False, 0, False
        self.est_hsync, self.est_line = q["hsync_len"], q["line_len"]
        self.ll_accum, self.ll_count = F(0.0), 0
        self.vs_count, self.last_short, self.lines_since = 0, 0, SAT
        self.xf_n, self.xf_d = 0, F(0.0)
        self.y, self.parity = 0, 0
        self.field_lines = (self.H + 1) // 2 if self.interlace else self.H
        self.row = self._row(0, 0)
        self.frames = 0

    def _derive(self, q):
        self.p = q
        pt = q["hsync_len"] / F(20.0)
        self.a_pulse = alpha(max(pt, F(1.0)))
        self.a_agc, self.a_hsync, self.a_line = alpha(q["agc_tau"]), alpha(q["hsync_len_tau"]), alpha(q["line_len_tau"])
        self.a_fast, self.a_slow = alpha(q["hsync_fast_track_tau"]), alpha(q["hsync_slow_track_tau"])
        self.thr = F(1.0) - q["l_tol"]

    def set_params(self, p):
        """live update: refused (False) if invalid or if it would change W, H, the delay length or interlacing"""
        if not valid(p):
            return False
        q = params(p)
        if (int(np.floor(q["line_len"])), q["frame_lines"], int(np.ceil(q["line_len"])), q["interlace"] != 0) != \
                (self.W, self.H, self.dlen, self.interlace != 0):
            return False
        self._derive(q)
        return True

    def _row(self, y, parity):
        if self.interlace:
            off = parity ^ (1 if self.p["dominance"] else 0) if self.mistake == "dominance_inverted" else \
                parity ^ (0 if self.p["dominance"] else 1)
            r = 2 * y + off
        else:
            r = y
        return r if 0 <= r < self.H else -1

    def _size(self, parity):
        return (self.H + 1) // 2 if parity == 0 else self.H // 2

    def _set_xf(self, xf):
        fl = np.floor(xf)
        self.xf_n, self.xf_d = int(fl), xf - fl

    # ---- one sample ---------------------------------------------------------------------------------------------
    def step(self, x):
        p, hit, m = self.p, self.hits, self.mistake
        half = F(0.5)
        # TV.2 comb
        if p["enable_comb"]:
            prev = self.dl[self.dp]
            self.dl[self.dp] = x
            self.dp = (self.dp + 1) % self.dlen
            diff = bool(p["comb_reverse"]) != (m == "comb_sign")
            hit["comb_diff" if diff else "comb_sum"] += 1
            x = half * (x - prev) if diff else half * (x + prev)
        # TV.3 peak AGC
        if x > self.line_max:
            hit["agc_peak"] += 1
            self.line_max = x
        if p["enable_agc"]:
            xg = self.gain * x
        else:
            hit["agc_off"] += 1
            xg = x
        # TV.4
        self.pulse = self.pulse + self.a_pulse * (xg - self.pulse)
        # TV.5
        if not p["enable_sync"]:
            hit["sync_off"] += 1
        elif not self.sync:
            if self.pulse > self.thr:
                hit["rise"] += 1
                self.sync, self.start = True, self.ptr
        elif not self.pulse > self.thr:
            hit["fall"] += 1
            self.sync = False
            self._pulse(F(self.ptr - self.start))
        self._raster(xg)
        self.ptr += 1

    def _pulse(self, ln):
        p, hit, m = self.p, self.hits, self.mistake
        half, two = F(0.5), F(2.0)
        dev, win = abs(ln - self.est_hsync), p["t_tol"] * self.est_hsync
        if dev == win:
            hit["t_tol_edge"] += 1
        if (dev < win) if m == "t_tol_lt" else (dev <= win):
            hit["hsync"] += 1
            if not self.have_last:
                hit["ll_first"] += 1
            else:
                dl = F(self.start - self.last_hsync)
                if abs(dl - self.est_line) <= p["g_tol"] * self.est_line:
                    hit["ll_accept"] += 1
                    self.ll_accum = self.ll_accum + dl
                    self.ll_count += 1
                else:
                    hit["ll_reject"] += 1
            self.have_last, self.last_hsync = True, self.start
            self.est_hsync = self.est_hsync + self.a_hsync * (ln - self.est_hsync)
            L = self.est_line
            xf = F(self.xf_n) + self.xf_d
            err = (half * self.est_hsync + p["x_off"]) - (xf - half * ln)
            if err > half * L:
                hit["err_wrap_hi"] += 1
                err = err - L
            elif err < -(half * L):
                hit["err_wrap_lo"] += 1
                err = err + L
            rel = abs(err) / L
            if rel > p["hsync_max_err"]:
                hit["to_fast"] += 1
                self.slow = False
            elif rel < p["hsync_min_err"]:
                hit["to_slow"] += 1
                self.slow = True
            if rel > p["hsync_huge_err"]:
                hit["huge_jump"] += 1
                xf = xf + err
            else:
                hit["track_slow" if self.slow else "track_fast"] += 1
                xf = xf + (self.a_slow if self.slow else self.a_fast) * err
            if xf < F(0.0) and m != "no_xf_wrap":
                hit["xf_wrap"] += 1
                xf = xf + L
            self._set_xf(xf)
            return
        self.have_last = False
        if abs(ln - p["vsync_len"]) > two * p["t_tol"] * p["vsync_len"]:
            hit["broad"] += 1
            self.vs_count = 0
            return
        hit["equalising"] += 1
        age = F(self.start - self.last_short)
        if self.vs_count > 0 and abs(age - half * self.est_line) <= two * p["t_tol"] * self.est_line:
            hit["eq_count"] += 1
            self.vs_count += 1
        else:
            hit["eq_restart"] += 1
            self.vs_count = 1
        self.last_short = self.start
        if self.vs_count != p["vsync_odd_trigger"]:
            return
        gate = self.field_lines // 2
        if not ((self.lines_since > gate) if m == "gate_gt" else (self.lines_since >= gate)):
            hit["trigger_gated"] += 1
            return
        hit["trigger"] += 1
        if self.lines_since == gate:
            hit["gate_edge"] += 1
        self.lines_since = 0
        early = self.y < self.field_lines // 2
        hit["trigger_early" if early else "trigger_late"] += 1
        if self.interlace:
            pos = (F(self.xf_n) + self.xf_d) - half * ln
            mid = abs(pos - half * self.est_line) < F(0.25) * self.est_line
            hit["parity_mid" if mid else "parity_start"] += 1
            nxt = 1 if mid else 0
            self.parity = nxt if early or m == "late_no_preswap" else nxt ^ 1
            self.field_lines = self._size(self.parity)
        self.y = -1 if early else self.field_lines - 1

    def _raster(self, xg):
        p, hit = self.p, self.hits
        v = xg if p["reverse"] else F(1.0) - xg
        n, d = self.xf_n, self.xf_d
        if 0 <= n < self.W:
            self.line[n] = self.line[n] + (F(1.0) - d) * v
        else:
            hit["raster_left" if n < 0 else "raster_right"] += 1
        if 0 <= n + 1 < self.W:
            self.line[n + 1] = d * v
        self.xf_n += 1
        xf = F(self.xf_n) + d
        if not xf >= self.est_line:
            return
        hit["line_end"] += 1
        if self.row >= 0:
            self.ring[self.frames % RING, self.row] = self.line
        else:
            hit["row_off"] += 1
        self.line = [F(0.0)] * self.W
        xf = xf - self.est_line
        self.accum = self.accum + self.line_max
        self.agc_lines += 1
        if self.mistake != "line_max_kept":
            self.line_max = F(0.0)
        if self.lines_since < SAT:
            self.lines_since += 1
        self.y += 1
        if self.y >= self.field_lines:
            hit["field_end"] += 1
            self.y = 0
            L_pre = self.est_line
            if p["enable_agc"] and self.agc_lines > 0 and self.accum > F(0.0):
                hit["agc_update"] += 1
                self.gain = self.gain + self.a_agc * (F(self.agc_lines) / self.accum - self.gain)
            elif p["enable_agc"]:
                hit["agc_hold"] += 1
            self.accum, self.agc_lines = F(0.0), 0
            if self.ll_count > 0:
                hit["ll_update"] += 1
                self.est_line = self.est_line + self.a_line * (self.ll_accum / F(self.ll_count) - self.est_line)
                self.ll_accum, self.ll_count = F(0.0), 0
            done = True
            if self.interlace:
                self.parity ^= 1
                self.field_lines = self._size(self.parity)
                done = self.parity == 0
            if done:
                hit["frame_end"] += 1
                self.frames += 1
                xf = xf - p["frame_spacing"] * (L_pre if self.mistake == "fs_pre_update" else self.est_line)
            else:
                hit["field_odd"] += 1
        self._set_xf(xf)
        self.row = self._row(self.y, self.parity)

    # ---- feeds and reads ------------------------------------------------------------------------------------------
    def feed(self, x):
        """the samples in order; returns the number of frames completed"""
        f0 = self.frames
        for v in np.ascontiguousarray(x, F):
            self.step(v)
        return self.frames - f0

    def frame(self, no):
        """frame `no` while readable: the last three completed (frames - 3 ... frames - 1) and the one in progress"""
        assert self.frames - RING < no <= self.frames, "frame no longer (or not yet) in the ring"
        return self.ring[no % RING].copy()

    def estimates(self):
        """(est_line, est_hsync, gain)"""
        return self.est_line, self.est_hsync, self.gain

    def state(self):
        return {"ptr": self.ptr, "frames": self.frames, "x": (self.xf_n, self.xf_d), "y": self.y, "parity": self.parity,
                "field_lines": self.field_lines, "row": self.row, "gain": self.gain, "est_line": self.est_line,
                "est_hsync": self.est_hsync, "pulse": self.pulse, "vs_count": self.vs_count,
                "lines_since_vs": self.lines_since, "slow": self.slow}
