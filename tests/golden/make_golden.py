#!/usr/bin/env python
"""Generates the fixtures under tests/golden/ (run from the repo root: `python tests/golden/make_golden.py`).

The reference repo ships no test vectors and its DSP lives in libraries that are absent (SURVEY.md section 0), so there
are two kinds of fixture, kept apart on purpose:

* `ref_*.npz` -- outputs of LITERAL Python transcriptions of the arithmetic that IS in /root/reference:
    - Panoramic/Scanner.cpp:56-256 (SpectrumView::feed, linear + histogram modes, interpolate, forgetting rule):
      transcription `_sview_literal` in tests/test_oracle.py;
    - Tasks/QuadDemodTask.cpp:44-60 (dst[0] = 0, dst[p] = i/pi * arg(x[p] conj(x[p-1]))) evaluated in float64;
    - Default/GenericInspector/FACTab.cpp:209-221 (FFT -> x conj(x) -> inverse FFT -> |.| of the first half) in float64;
    - the offline TimeWindow tasks (`ref_timewindow.npz`): Tasks/DelayedConjTask.cpp:58-100, Tasks/WaveSampler.cpp:96-175
      (manual sampler) and :222-292 (zero-crossing sampler, block by block) statement by statement in binary32 scalars,
      Tasks/HistogramFeeder.cpp:35-87 and Tasks/CarrierDetector.cpp:49-147 in float64 (numpy FFT, incl. the un-squared
      notch bins).
  These pin the oracle to the reference where the reference is specific.  Nothing here needs the reference at test time.
* `pin_*.json` -- SHA-256 of the ORACLE's own outputs on seeded inputs for the parts whose inner arithmetic is upstream
  (FFT dataflows, AGC / Costas / Gardner chains, channeliser, spectrum sources, channel detector).  They are NOT
  upstream golden vectors ("parity unpinned"); they freeze SPEC.md so that a change of the oracle -- against which the
  CUDA path is compared bit for bit -- cannot go unnoticed.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle_lib as O                      # noqa: E402
from sigdigger_b200 import synth            # noqa: E402
from test_oracle import _sview_literal      # noqa: E402


def sview_case():
    fmin, fmax, fftbw, psize = 100e6, 140e6, 2e6, 2048
    rng = np.random.default_rng(7)
    feeds = []
    for hop in range(60):
        feeds.append(((rng.random(psize).astype(np.float32) * 10 - 90), fmin + 0.5e6 + hop * 0.66e6, fftbw))
    feeds += feeds[10:30]
    feeds += feeds[10:30] * 4
    return fmin, fmax, fftbw, psize, feeds


def quad_case():
    rng = np.random.default_rng(11)
    n = 4096
    x = (np.exp(2j * np.pi * np.cumsum(0.05 + 0.02 * rng.standard_normal(n))) * (0.5 + rng.random(n))).astype(np.complex64)
    ref = np.zeros(n, np.complex128)
    xd = x.astype(np.complex128)
    ref[1:] = 1j / np.pi * np.angle(xd[1:] * np.conj(xd[:-1]))
    return x, ref


def fac_case():
    n = 4096
    s, _ = synth.psk_signal(n + 1, 8.0, order=4, seed=3)
    rng = np.random.default_rng(3)
    x = (0.3 * s + synth.awgn(n + 1, 1e-3, rng)).astype(np.complex64)
    fr = x[-1024:].astype(np.complex128)
    ref = np.abs(np.fft.ifft(np.abs(np.fft.fft(fr)) ** 2))[:512]      # FACTab: unnormalised inverse / N here
    return x, ref


# ---- literal transcriptions of the offline TimeWindow tasks (SPEC Y): binary32 scalars (np.float32) where the C++
# ---- uses SUFLOAT / SUCOMPLEX, Python floats where it uses qreal / double, same statement order.
F = np.float32


def _cmul_conj(ar, ai, br, bi):
    """(ar + i ai) * conj(br + i bi) the way std::complex<float> multiplies: four products, two sums"""
    return F(F(ar * br) + F(ai * bi)), F(F(ai * br) - F(ar * bi))


def delayed_conj_literal(x, delay):
    """Tasks/DelayedConjTask.cpp:58-100 (circular delay line == x[p - delay])"""
    y = np.zeros(len(x), np.complex64)
    line = [0j] * delay
    q = 0
    for p in range(len(x)):
        v = x[p]
        if p >= delay:
            prev = line[q]
            kinv = F(1.0 / (float(np.hypot(float(prev.real), float(prev.imag))) + 1e-3))
            tr, ti = F(kinv * F(v.real)), F(kinv * F(v.imag))
            yr, yi = _cmul_conj(tr, ti, F(prev.real), F(prev.imag))
            y[p] = complex(yr, yi)
        line[q] = v
        q = (q + 1) % delay
    return y


def sample_manual_literal(x, space, symbol_sync, symbol_count):
    """Tasks/WaveSampler.cpp:28-46 (delta, sampOffset), 96-175 (sampleManual), all work() blocks in sequence"""
    n = len(x)
    delta = n / symbol_count
    samp_offset = symbol_sync / delta
    delta_inv = F(F(1.0) / F(delta))
    out = []
    pr, pi = F(0), F(0)
    for p in range(int(symbol_count)):
        start = (p - samp_offset) * delta + symbol_sync
        end = start + delta
        i_start, i_end = int(np.floor(start)), int(np.ceil(end))
        t_start, t_end = F(1 - (start - i_start)), F(1 - (i_end - end))
        ar, ai = F(0), F(0)
        for i in range(i_start, i_end + 1):
            if 0 <= i < n:
                xr, xi = F(x[i].real), F(x[i].imag)
                if i == i_start:
                    xr, xi = F(t_start * xr), F(t_start * xi)
                elif i == i_end:
                    xr, xi = F(t_end * xr), F(t_end * xi)
            else:
                xr, xi = F(0), F(0)
            if space == "amplitude":
                dr, di = _cmul_conj(xr, xi, xr, xi)
            else:
                dr, di = _cmul_conj(xr, xi, pr, pi)
            ar, ai = F(ar + dr), F(ai + di)
            pr, pi = xr, xi
        if space == "amplitude":
            out.append(complex(np.sqrt(F(delta_inv * ar)), 0.0))
        else:
            out.append(complex(F(delta_inv * ar), F(delta_inv * ai)))
    return np.asarray(out, np.complex64)


def zero_crossing_literal(x, space, amplitude, threshold, zc_angle, bnor):
    """Tasks/WaveSampler.cpp:222-292, one call per 4096-sample block; prevVar / prevSample are the members'
    initial values in every call because the method never writes them back; lastZc is written back."""
    n = len(x)
    tr_, ti_ = F(threshold.real), F(threshold.imag)
    zr, zi = F(zc_angle.real), F(zc_angle.imag)
    thres = F(F(tr_ * tr_) + F(ti_ * ti_)) if amplitude else F(F(tr_ * zr) - F(ti_ * zi))
    bnor = F(bnor)
    out = []
    p = 0
    last_zc = 0
    while p < n:
        amount = min(n - p, 4096)
        last = p + amount >= n
        i = 0
        prev_var = F(-1)
        pr, pi = F(0), F(0)
        for _ in range(amount):
            xr, xi = F(x[p].real), F(x[p].imag)
            if space == "amplitude":
                var = F(F(xr * xr) + F(xi * xi)) if amplitude else F(F(xr * zr) - F(xi * zi))
                var = F(var - thres)
            elif space == "phase":
                var = F(np.arctan2(F(F(xr * zi) + F(xi * zr)), F(F(xr * zr) - F(xi * zi))))
            else:
                ir, ii = F(-xi), xr
                dr, di = _cmul_conj(ir, ii, pr, pi)
                var = F(np.arctan2(di, dr))
                pr, pi = xr, xi
            if (var > 0 or var < 0) or last:
                if F(var * prev_var) < 0 or last:
                    samples = p - last_zc
                    symbols = int(np.floor(float(F(F(samples) * bnor)) + 0.5))      # round(): value is >= 0
                    while symbols > 0 and i < 4096:
                        out.append(1 if var > 0 else 0)
                        i += 1
                        symbols -= 1
                    last_zc = p
                    prev_var = var
            p += 1
    return np.asarray(out, np.uint8)


def carrier_detect_literal(x, avg_rel_bw, dc_notch_rel_bw):
    """Tasks/CarrierDetector.cpp:49-147 in float64 with numpy's FFT, including the un-squared bins inside the notch"""
    n = len(x)
    alloc = 1
    while alloc < n:
        alloc <<= 1
    k = np.arange(n)
    a = 2 * np.pi * k / (n - 1)
    w = 0.35875 - 0.48829 * np.cos(a) + 0.14128 * np.cos(2 * a) - 0.01168 * np.cos(3 * a)
    buf = np.zeros(alloc, np.complex128)
    buf[:n] = x.astype(np.complex128) * w
    X = np.fft.fft(buf)
    notch = min(max(dc_notch_rel_bw, 0.0), 1.0)
    bins = int(alloc * avg_rel_bw) + 1
    delta = (bins - 1) // 2
    skip = int(.5 * notch * alloc)
    vals = X.copy()
    sl = slice(skip, alloc - skip)
    vals[sl] = np.abs(X[sl]) ** 2
    max_val, max_ndx = 0.0, 0
    region = vals[sl].real
    if len(region) and region.max() > 0:
        max_ndx = skip + int(np.argmax(region))
    start = max_ndx - delta
    acc = 0j
    for i in range(bins):
        j = (i + start) % alloc
        acc += vals[j].real * np.exp(1j * np.pi * (2.0 * j / alloc))
    return float(np.angle(acc))


def timewindow_case():
    rng = np.random.default_rng(17)
    n = 2 * 4096 + 1500
    noise = (0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))).astype(np.complex64)
    lvl = np.repeat(rng.integers(0, 2, n // 12 + 1), 12)[:n]
    ask = ((0.2 + 0.8 * lvl) * np.exp(0.3j)).astype(np.complex64) + noise
    psk = np.exp(0.7j * (2.0 * lvl - 1.0)).astype(np.complex64) + noise
    tone = (0.6 * np.exp(2j * np.pi * 0.0731 * np.arange(n))).astype(np.complex64) + noise
    return dict(ask=ask, psk=psk, tone=tone)


def timewindow_refs():
    c = timewindow_case()
    out = dict(c)
    out["dconj_7"] = delayed_conj_literal(c["tone"][:3000], 7)
    out["dconj_500"] = delayed_conj_literal(c["tone"][:3000], 500)
    for space, sig in (("amplitude", "ask"), ("phase", "psk"), ("frequency", "psk")):
        out["manual_" + space] = sample_manual_literal(c[sig][:6000], space, 5, 487.3)
    out["zc_amp_power"] = zero_crossing_literal(c["ask"], "amplitude", True, 0.6 + 0.1j, 1 + 0j, 1.0 / 12)
    out["zc_amp_proj"] = zero_crossing_literal(c["ask"], "amplitude", False, 0.55 + 0.2j, np.exp(-0.3j), 1.0 / 12)
    out["zc_phase"] = zero_crossing_literal(c["psk"], "phase", False, 0j, np.exp(0.1j), 1.0 / 12)
    out["zc_amp_fast"] = zero_crossing_literal(c["ask"], "amplitude", True, 0.6 + 0.1j, 1 + 0j, 1.0)
    xd = c["psk"].astype(np.complex128)
    out["hist_amplitude"] = np.abs(xd)
    out["hist_phase"] = np.angle(xd)
    out["hist_frequency"] = np.angle(xd[1:] * np.conj(xd[:-1]))
    out["carrier"] = np.array([carrier_detect_literal(c["tone"][:m], 0.004, nt)
                               for m, nt in ((4096, 0.0), (6000, 0.0), (9692, 0.02))])
    return out


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def pins():
    """seeded oracle outputs (see module docstring: self-pins, not upstream vectors)"""
    out = {}
    rng = np.random.default_rng(2026)
    z = (rng.standard_normal(65536) + 1j * rng.standard_normal(65536)).astype(np.complex64)
    out["spec_fft_65536"] = sha(O.spec_fft(z))
    out["spec_fft_4096_stockham"] = sha(O.spec_fft(z[:4096]))
    out["spec_fft_8192_fourstep"] = sha(O.spec_fft(z[:8192]))
    out["psd_bh_8192"] = sha(O.psd_frames(z[:8192 * 4], 8192, "blackmann_harris"))
    n, sps = 40000, 3.125
    s, _ = synth.psk_signal(n, sps, order=4, seed=5)
    x = (0.25 * synth.mix(s, 1e-4, 0.2) + synth.awgn(n, 10 ** (-45 / 20), np.random.default_rng(5))).astype(np.complex64)
    kw = dict(baud=1.0 / sps, costas_order=2, bits_per_symbol=2, loop_bw=2e-3, mf_type=1, mf_rolloff=0.35, clock_type=1,
              clock_gain=0.1)
    soft, hard = O.inspector_run(O.insp_config("psk", 1.0, **kw), x)
    out["psk_soft"], out["psk_hard"] = sha(soft), sha(hard)
    soft, hard = O.inspector_run(O.insp_config("psk", 1.0, eq_type=1, eq_rate=5e-3, **kw), x)
    out["psk_cma_soft"] = sha(soft)
    fs_, _ = synth.fsk_signal(30000, 5.0, h=1.0, seed=4)
    xf = (0.3 * fs_ + synth.awgn(30000, 10 ** (-35 / 20), np.random.default_rng(4))).astype(np.complex64)
    soft, hard = O.inspector_run(O.insp_config("fsk", 1.0, baud=0.2, bits_per_symbol=1, mf_type=1, clock_type=1,
                                               clock_gain=0.2), xf)
    out["fsk_soft"] = sha(soft)
    W = 8192
    xc = (z[:W * 8] * 0.05 + 0.4 * np.exp(2j * np.pi * 0.1251 * np.arange(W * 8))).astype(np.complex64)
    ch = O.specttuner_run(xc, W, [dict(f0=2 * np.pi * 0.125, bw=2 * np.pi / 32, guard=1.0)])[0]
    out["channeliser"] = sha(ch)
    out["spectsrc_cyclo"] = sha(O.spectsrc_frame("cyclo", 1024, ch))
    out["spectsrc_fac"] = sha(O.spectsrc_frame("fac", 1024, ch))
    d = O.ChannelDetector(8192, 0.25, 0.5, 6.0, 3)
    chans, total = d.feed(O.psd_frames(xc[:8192 * 4], 8192, "hann"))
    d.close()
    out["chdet"] = sha(np.array([(a, b) for a, b, *_ in chans], np.uint32))
    out["chdet_total"] = int(total)
    return out


def sview_cases():
    """SpectrumView runs of tests/test_ref.py -> [(fmin, fmax, fft_bandwidth, feeds)]; the third re-feeds the first"""
    fmin, fmax, fftbw, psize, feeds = sview_case()
    rng = np.random.default_rng(3)
    fmin2, fmax2 = 1.0e9, 1.0e9 + 65536 * 1000.0 * 40
    feeds2 = [((rng.random(512).astype(np.float32) * 10 - 80), fmin2 + (5 + 37.3 * h) * 40e3, 30e3) for h in range(200)]
    return [(fmin, fmax, fftbw, feeds), (fmin2, fmax2, feeds2[0][2], feeds2), (fmin - 10e6, fmax + 25e6, fftbw, None)]


def ref_task_input(n, seed):
    x, _ = synth.multi_carrier(n, 1.0, [("qpsk", 0.01, 0.1, -6.0, {})], noise_db=-40.0, seed=seed)
    return np.ascontiguousarray(x, np.complex64)


TV_CASES = ((False, 40), (True, 61))
SNR_CASES = ((1, 256), (2, 256), (3, 400))
CARRIER_CASES = ((5000, 0.0371, 0.0), (16384, -0.212, 0.0), (3000, 0.11, 0.05), (9000, -0.4, 0.02))


def snr_histograms(bps, length, rng):
    k = 1 << bps
    centres = (rng.integers(0, k, 200000) + 0.5) / k
    v = (centres + 0.03 * rng.standard_normal(200000)) % 1.0
    return np.bincount((v * length).astype(int) % length, minlength=length).astype(np.uint32)


def carrier_input(n, f0, rng):
    t = np.arange(n)
    return (np.exp(2j * np.pi * f0 * t) * (1 + 0.3 * np.cos(2 * np.pi * 0.001 * t))
            + 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) + 0.5).astype(np.complex64)


def compiled_reference():
    """Outputs of the reference's sources compiled into oracle/_ref/ (`make -C oracle ref`) on the inputs of
    tests/test_ref.py: SHA-256 of the bytes where that test compares bit for bit, arrays otherwise."""
    import ctypes as C
    import test_oracle_tv as T
    L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libsdref.so"))
    L2 = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libsdref_suscan.so"))
    L.ref_sview_new.restype = C.c_void_p
    L.ref_sview_read.restype = C.c_uint
    L.ref_sview_set_range.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_float]
    L.ref_sview_feed.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_ulong, C.c_double, C.c_int]
    L.ref_sview_feed_view.argtypes = [C.c_void_p, C.c_void_p]
    L.ref_sview_read.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.ref_wave_sampler.restype = C.c_long
    L.ref_wave_sampler.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int,
                                   C.c_float, C.c_float, C.c_float, C.c_float, C.c_size_t, C.c_double, C.c_void_p,
                                   C.c_void_p, C.c_size_t]
    L.ref_quad_demod.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.ref_delayed_conj.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_ulong]
    L.ref_averager.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_float, C.c_void_p]
    out = {}

    views = []
    for i, (fmin, fmax, fftbw, feeds) in enumerate(sview_cases()):
        v = C.c_void_p(L.ref_sview_new())
        L.ref_sview_set_range(v, C.c_double(fmin), C.c_double(fmax), C.c_double(fftbw), C.c_float(0.5))
        if feeds is None:
            L.ref_sview_feed_view(v, views[0])
        for psd, fc, bw in feeds or ():
            p = np.ascontiguousarray(psd, np.float32)
            L.ref_sview_feed(v, p.ctypes.data, None, C.c_ulong(len(p)), C.c_double(fc), 1)
        views.append(v)
        a = [np.zeros(65536, np.float32) for _ in range(3)]
        n = L.ref_sview_read(v, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data)
        out["sview%d_size" % i] = np.int64(n)
        out["sview%d_sha" % i] = np.array([sha(q[:n]) for q in a])

    c = timewindow_case()
    x = c["tone"][:5000]
    y = np.zeros_like(x)
    L.ref_quad_demod(x.ctypes.data, y.ctypes.data, C.c_size_t(len(x)))
    out["quad_demod"] = y
    for delay in (7, 500):
        x = c["tone"][:3000]
        y = np.zeros_like(x)
        L.ref_delayed_conj(x.ctypes.data, y.ctypes.data, C.c_size_t(len(x)), C.c_ulong(delay))
        out["delayed_conj_%d" % delay] = y
    for space, sig in (("amplitude", "ask"), ("phase", "psk"), ("frequency", "psk")):
        x = np.ascontiguousarray(c[sig][:6000])
        y = np.zeros(1024, np.complex64)
        n = L.ref_wave_sampler(x.ctypes.data, C.c_size_t(len(x)), 0, O.SPACE[space], C.c_double(1.0), C.c_double(0.1),
                               C.c_double(0.1), 0, C.c_float(0), C.c_float(0), C.c_float(1), C.c_float(0), C.c_size_t(5),
                               C.c_double(487.3), y.ctypes.data, None, C.c_size_t(1024))
        out["manual_" + space] = y[:n].copy()
    for i, (sig, space, amp, thr, zc, bnor) in enumerate(ZC_CASES):
        x = np.ascontiguousarray(c[sig])
        sym = np.zeros(len(x), np.uint8)
        n = L.ref_wave_sampler(x.ctypes.data, C.c_size_t(len(x)), 2, O.SPACE[space], C.c_double(1.0), C.c_double(bnor),
                               C.c_double(0.1), int(amp), C.c_float(thr.real), C.c_float(thr.imag), C.c_float(np.real(zc)),
                               C.c_float(np.imag(zc)), C.c_size_t(0), C.c_double(100.0), None, sym.ctypes.data,
                               C.c_size_t(len(x)))
        out["zero_crossing_%d" % i] = sym[:n].copy()
    x = np.ascontiguousarray(c["psk"])
    y = np.zeros(len(x), np.complex64)
    n = L.ref_wave_sampler(x.ctypes.data, C.c_size_t(len(x)), 1, O.SPACE["frequency"], C.c_double(1.0),
                           C.c_double(1.0 / 12), C.c_double(0.2), 0, C.c_float(0), C.c_float(0), C.c_float(1), C.c_float(0),
                           C.c_size_t(0), C.c_double(100.0), y.ctypes.data, None, C.c_size_t(len(x)))
    out["gardner_sha"] = np.array(sha(y[:n]))

    frames = averager_frames()
    for alpha in (0.25, 1.0):
        y = np.zeros(4096, np.float32)
        L.ref_averager(frames.ctypes.data, 7, 4096, C.c_float(alpha), y.ctypes.data)
        out["averager_%g_sha" % alpha] = np.array(sha(y))

    L.ref_tv_worker.restype = C.c_long
    L.ref_tv_worker.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                C.c_void_p]
    for interlace, lines in TV_CASES:
        x, _, _ = T.toy_signal(lines, interlace, frames=10)
        sp = T.toy_params(lines, interlace, 4, cls=T.ShimTvParams)
        W, H, cap, block = int(np.floor(T.LINE)), lines, 16, 7000
        y = np.zeros((cap, H, W), np.float32)
        w, h = C.c_int(), C.c_int()
        got = L.ref_tv_worker(C.byref(sp), x.ctypes.data, x.size, block, y.ctypes.data, cap, C.byref(w), C.byref(h))
        out["tv_%d_%d" % (interlace, lines)] = np.array([got, w.value, h.value], np.int64)
        out["tv_%d_%d_sha" % (interlace, lines)] = np.array(sha(y))

    L2.ref_suscan_psd_message.restype = C.c_long
    L2.ref_suscan_psd_message.argtypes = [C.c_void_p, C.c_ulong, C.c_double, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
    lin = psd_message_input()
    y = np.zeros(len(lin), np.float32)
    fc, rate = C.c_double(), C.c_uint()
    n = L2.ref_suscan_psd_message(lin.ctypes.data, len(lin), 433.92e6, 2000000, y.ctypes.data, C.byref(fc), C.byref(rate))
    out["psd_message"] = y[:n].copy()
    out["psd_message_meta"] = np.array([fc.value, rate.value])
    # Suscan/MQ.cpp, SamplesMessage, StatusMessage over libsuscan.so
    L2.ref_suscan_mq_samples.restype = C.c_long
    L2.ref_suscan_mq_samples.argtypes = [C.c_void_p, C.c_ulong, C.c_uint, C.c_void_p, C.c_void_p]
    L2.ref_suscan_status_message.argtypes = [C.c_int, C.c_char_p, C.c_char_p, C.c_size_t]
    x = mq_input()
    y = np.zeros_like(x)
    iid = C.c_uint()
    n = L2.ref_suscan_mq_samples(x.ctypes.data, x.size, 0xBEEF, y.ctypes.data, C.byref(iid))
    out["mq_samples"] = np.array([n, iid.value], np.int64)
    out["mq_samples_sha"] = np.array(sha(y))
    status = []
    for code, text in MQ_STATUS_CASES:
        buf = C.create_string_buffer(64)
        status += [str(L2.ref_suscan_status_message(code, text, buf, 64)), buf.value.decode()]
    out["status_messages"] = np.array(status)

    n = 2 * 4096 + 777
    x = ref_task_input(n, 5)
    y = np.zeros(n, np.complex64)
    for kind in (1, 2, 3):
        L.ref_task_costas.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float, C.c_float, C.c_int]
        assert L.ref_task_costas(x.ctypes.data, y.ctypes.data, n, C.c_float(10.0), C.c_float(2e-3), kind) == 0
        out["task_costas_%d_sha" % kind] = np.array(sha(y))
    L.ref_task_pll.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float]
    assert L.ref_task_pll(x.ctypes.data, y.ctypes.data, n, C.c_float(5e-3)) == 0
    out["task_pll_sha"] = np.array(sha(y))
    L.ref_task_agc.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float]
    assert L.ref_task_agc(x.ctypes.data, y.ctypes.data, n, C.c_float(20.0)) == 0
    out["task_agc_sha"] = np.array(sha(y))
    L.ref_task_xlate.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float, C.c_float]
    assert L.ref_task_xlate(x.ctypes.data, y.ctypes.data, n, C.c_float(0.0123), C.c_float(0.5)) == 0
    out["task_xlate_sha"] = np.array(sha(y))

    L.ref_task_histogram.restype = C.c_long
    L.ref_task_histogram.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t]
    n = 3 * 4096 + 55
    x = ref_task_input(n, 8)
    for space in (0, 1, 2):
        y = np.zeros(n, np.float32)
        k = L.ref_task_histogram(x.ctypes.data, n, space, y.ctypes.data, n)
        out["histogram_%d" % space] = y[:k].copy()

    L.ref_snr_estimator.argtypes = [C.c_uint, C.c_float, C.c_float, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p,
                                    C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(4)
    for bps, length in SNR_CASES:
        h = snr_histograms(bps, length, rng)
        feeds = 6
        hs = np.ascontiguousarray(np.tile(h, (feeds, 1)))
        sig, snr, model = np.zeros(feeds, np.float32), np.zeros(feeds, np.float32), np.zeros(length, np.float32)
        assert L.ref_snr_estimator(bps, C.c_float(0.5), C.c_float(0.0), hs.ctypes.data, length, feeds,
                                   sig.ctypes.data, snr.ctypes.data, model.ctypes.data) == length
        out["snr_%d_%d" % (bps, length)] = np.concatenate([sig, snr, model])

    L.ref_carrier_detect.restype = C.c_float
    L.ref_carrier_detect.argtypes = [C.c_void_p, C.c_size_t, C.c_double, C.c_double]
    rng = np.random.default_rng(12)
    peaks = []
    for n, f0, notch in CARRIER_CASES:
        x = carrier_input(n, f0, rng)
        peaks.append(L.ref_carrier_detect(x.ctypes.data, n, 0.01, notch))
    out["carrier_detect"] = np.array(peaks, np.float32)
    return out


ZC_CASES = [("ask", "amplitude", True, 0.6 + 0.1j, 1 + 0j, 1.0 / 12),
            ("ask", "amplitude", False, 0.55 + 0.2j, np.exp(-0.3j), 1.0 / 12),
            ("psk", "phase", False, 0j, np.exp(0.1j), 1.0 / 12), ("ask", "amplitude", True, 0.6 + 0.1j, 1 + 0j, 1.0)]
LPF_N, LPF_SEED, LPF_BW = 5 * 4096 + 300, 9, 0.2


MQ_STATUS_CASES = ((-1, b"source failed to start"), (0, None))


def mq_input():
    rng = np.random.default_rng(22)
    return (rng.standard_normal(1000) + 1j * rng.standard_normal(1000)).astype(np.complex64)


def averager_frames():
    return np.random.default_rng(9).random((7, 4096)).astype(np.float32) * 40 - 100


def psd_message_input():
    rng = np.random.default_rng(21)
    n = 8192
    lin = (rng.standard_normal(n) ** 2 * 10.0 ** rng.uniform(-9, 1, n)).astype(np.float32)
    lin[:4] = [0.0, 1e-12, 1.0, 123.5]
    return lin


def compiled_reference_gpu():
    """Tasks/LPFTask.cpp of oracle/_ref/ over the GPU tuner of <sigutils/specttuner.h>: SHA-256 of its output."""
    import ctypes as C
    R = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libsdref.so"))
    R.ref_task_lpf.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_float]
    x = ref_task_input(LPF_N, LPF_SEED)
    y = np.zeros(LPF_N, np.complex64)
    assert R.ref_task_lpf(x.ctypes.data, y.ctypes.data, LPF_N, C.c_float(LPF_BW)) == 0
    return {"task_lpf_sha": sha(y)}


def main():
    if "--compiled-reference" in sys.argv:
        np.savez_compressed(os.path.join(HERE, "ref_compiled.npz"), **compiled_reference())
        print("wrote ref_compiled.npz")
        return
    if "--compiled-reference-gpu" in sys.argv:
        json.dump(compiled_reference_gpu(), open(os.path.join(HERE, "ref_compiled_gpu.json"), "w"), indent=1)
        print("wrote ref_compiled_gpu.json")
        return
    fmin, fmax, fftbw, psize, feeds = sview_case()
    psd, acc, cnt, size = _sview_literal(fmin, fmax, feeds)
    np.savez_compressed(os.path.join(HERE, "ref_spectrumview.npz"), psd=psd, count=cnt, size=size)
    x, ref = quad_case()
    np.savez_compressed(os.path.join(HERE, "ref_quad_demod.npz"), x=x, y=ref)
    x, ref = fac_case()
    np.savez_compressed(os.path.join(HERE, "ref_fac.npz"), x=x, fac=ref)
    np.savez_compressed(os.path.join(HERE, "ref_timewindow.npz"), **timewindow_refs())
    json.dump(pins(), open(os.path.join(HERE, "pin_oracle.json"), "w"), indent=1, sort_keys=True)
    print("wrote", sorted(os.listdir(HERE)))


if __name__ == "__main__":
    main()
