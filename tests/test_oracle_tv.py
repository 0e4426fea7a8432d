"""CPU: analog-TV processor (SPEC TV; SURVEY 8(f) rank 4).  The recurrence is upstream's (sigutils, not in the
reference, no vectors): what pins the oracle is the exact statement of tests/tv_stmt.py (tests/test_tv_stmt.py) and
behaviour -- it locks on a synthetic composite signal with a fractional line length, follows the vertical intervals,
recovers the picture -- and the reference-shaped worker loop
(tests/shim/reference_tu.cpp: TVProcessorWorker::work over <sigutils/tvproc.h>, whose per-sample entry point runs the
GPU kernel's own step on the host) is held to the oracle bit for bit.  GPU batch: tests/test_gpu_tv.py."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as OL
import shim_build as SB
from sigdigger_b200 import synth

LINE, HSYNC, SHORT = 400.37, 30.0, 15.0


class ShimTvParams(C.Structure):
    """struct sigutils_tv_processor_params (include/sigutils/tvproc.h): SUBOOL = int, SUSCOUNT = uint64"""
    _fields_ = [("enable_sync", C.c_int), ("reverse", C.c_int), ("interlace", C.c_int), ("enable_agc", C.c_int),
                ("x_off", C.c_float), ("dominance", C.c_int), ("frame_lines", C.c_uint64),
                ("frame_spacing", C.c_float), ("enable_comb", C.c_int), ("comb_reverse", C.c_int),
                ("hsync_len", C.c_float), ("vsync_len", C.c_float), ("line_len", C.c_float),
                ("vsync_odd_trigger", C.c_uint64), ("t_tol", C.c_float), ("l_tol", C.c_float), ("g_tol", C.c_float),
                ("hsync_huge_err", C.c_float), ("hsync_max_err", C.c_float), ("hsync_min_err", C.c_float),
                ("hsync_len_tau", C.c_float), ("line_len_tau", C.c_float), ("agc_tau", C.c_float),
                ("hsync_fast_track_tau", C.c_float), ("hsync_slow_track_tau", C.c_float)]


def tv_lib():
    L = OL.lib()
    L.sdo_tv_new.restype = C.c_void_p
    L.sdo_tv_new.argtypes = [C.c_void_p]
    L.sdo_tv_destroy.argtypes = [C.c_void_p]
    L.sdo_tv_set_params.argtypes = [C.c_void_p, C.c_void_p]
    L.sdo_tv_feed_bulk.restype = C.c_size_t
    L.sdo_tv_feed_bulk.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.sdo_tv_frames.restype = C.c_uint64
    L.sdo_tv_frames.argtypes = [C.c_void_p]
    L.sdo_tv_frame.restype = C.POINTER(C.c_float)
    L.sdo_tv_frame.argtypes = [C.c_void_p, C.c_uint64]
    L.sdo_tv_estimates.argtypes = [C.c_void_p] + [C.POINTER(C.c_float)] * 3
    L.sdo_tv_params_pal.argtypes = [C.c_void_p, C.c_float]
    L.sdo_tv_params_ntsc.argtypes = [C.c_void_p, C.c_float]
    L.sdo_tv_feed_transform.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_float, C.c_float, C.c_void_p]
    return L


def toy_params(lines, interlace, trigger, cls=OL.TvParams, comb=False):
    p = OL.TvParams()
    tv_lib().sdo_tv_params_pal(C.byref(p), 1e6)
    p.line_len, p.hsync_len, p.vsync_len = LINE, HSYNC, SHORT
    p.frame_lines, p.interlace, p.vsync_odd_trigger, p.enable_comb = lines, int(interlace), trigger, int(comb)
    if cls is OL.TvParams:
        return p
    q = cls()
    for name, _ in OL.TvParams._fields_:
        setattr(q, name, getattr(p, name))
    return q


def toy_signal(lines, interlace, frames=40, start=17.3, amp=0.5, noise=0.002, seed=3):
    rng = np.random.default_rng(seed)
    pic = rng.random((lines, 16)).repeat(4, axis=1)
    x, act = synth.tv_composite(LINE, HSYNC, SHORT, lines, interlace, frames, pic, amp=amp, noise=noise, seed=seed)
    return np.ascontiguousarray(x[int(LINE * start):]), pic, act       # start mid-frame: forces acquisition


class OracleTv:
    def __init__(self, p):
        self.L = tv_lib()
        self.h = self.L.sdo_tv_new(C.byref(p))
        self.W, self.H = int(np.floor(p.line_len)), int(p.frame_lines)

    def feed(self, x):
        x = np.ascontiguousarray(x, np.float32)
        return int(self.L.sdo_tv_feed_bulk(self.h, x.ctypes.data, x.size))

    @property
    def frames(self):
        return int(self.L.sdo_tv_frames(self.h))

    def frame(self, no):
        return np.ctypeslib.as_array(self.L.sdo_tv_frame(self.h, no), shape=(self.H, self.W)).copy()

    def estimates(self):
        a, b, g = C.c_float(), C.c_float(), C.c_float()
        self.L.sdo_tv_estimates(self.h, C.byref(a), C.byref(b), C.byref(g))
        return a.value, b.value, g.value

    def close(self):
        if self.h:
            self.L.sdo_tv_destroy(self.h)
            self.h = None


def line_map(frame, pic, act):
    """for every decoded row: the transmitted line it matches best and the correlation, at the one horizontal shift
    (the sync separator's group delay, a pixel or two) that suits the whole frame best"""
    H, W = frame.shape
    a0, a1 = act
    c0, c1 = int(a0) + 6, int(a1) - 6
    best = None
    for shift in range(-3, 4):
        cols = np.clip(((np.arange(W) + shift - a0) / (a1 - a0) * pic.shape[1]).astype(int), 0, pic.shape[1] - 1)
        exp = 1.0 - (0.65 - 0.55 * pic[:, cols])             # 1 - x with the tip at 1
        fz = frame[:, c0:c1] - frame[:, c0:c1].mean(axis=1, keepdims=True)
        ez = exp[:, c0:c1] - exp[:, c0:c1].mean(axis=1, keepdims=True)
        fn, en = np.linalg.norm(fz, axis=1), np.linalg.norm(ez, axis=1)
        cc = (fz @ ez.T) / np.maximum(np.outer(fn, en), 1e-12)            # [row][line]
        out = [(int(np.argmax(cc[r])), float(cc[r].max())) if fn[r] > 1e-6 else (-1, 0.0) for r in range(H)]
        score = sum(c for _, c in out)
        if best is None or score > best[0]:
            best = (score, out)
    return best[1]


def test_locks_on_progressive_signal(oracle):
    lines = 40
    x, pic, act = toy_signal(lines, False)
    t = OracleTv(toy_params(lines, False, 4))
    n = t.feed(x)
    est_line, est_hsync, gain = t.estimates()
    assert n == t.frames and 38 <= n <= 40
    assert abs(est_line - LINE) < 2e-3                       # line length tracked to 1e-5 relative
    assert abs(gain - 2.0) < 0.05                            # sync tip (amp 0.5) brought to 1
    m1, m2 = line_map(t.frame(n - 2), pic, act), line_map(t.frame(n - 1), pic, act)
    assert all(a == b for (a, ca), (b, cb) in zip(m1, m2) if ca > 0.9 and cb > 0.9)      # vertically locked
    good = [(r, l) for r, (l, c) in enumerate(m2) if c > 0.9]
    assert len(good) >= lines - 9                            # everything outside the 7.5-line vertical interval
    assert len({l - r for r, l in good}) == 1                # one constant vertical offset
    t.close()


@pytest.mark.parametrize("trigger", [4, 5])
def test_locks_on_interlaced_signal(oracle, trigger):
    lines = 61
    x, pic, act = toy_signal(lines, True, frames=64)
    t = OracleTv(toy_params(lines, True, trigger))
    n = t.feed(x)
    assert 60 <= n <= 63
    m, mp = line_map(t.frame(n - 1), pic, act), line_map(t.frame(n - 2), pic, act)
    assert all(a == b for (a, ca), (b, cb) in zip(m, mp) if ca > 0.9 and cb > 0.9)      # vertically locked
    even = [(r, l) for r, (l, c) in enumerate(m) if c > 0.9 and r % 2 == 0]
    odd = [(r, l) for r, (l, c) in enumerate(m) if c > 0.9 and r % 2 == 1]
    assert len(even) >= 20 and len(odd) >= 20
    # each field fills every other row with consecutive lines; the fields are half a frame apart
    assert len({2 * l - r for r, l in even}) == 1 and len({2 * l - r for r, l in odd}) == 1
    de, do = (2 * even[0][1] - even[0][0]), (2 * odd[0][1] - odd[0][0])
    assert abs(abs(de - do) - lines) <= 2
    t.close()


def test_follows_a_line_rate_offset_and_agc_step(oracle):
    lines = 40
    p = toy_params(lines, False, 4)
    p.line_len = LINE * 1.004                                # the processor starts 0.4 % off
    p.line_len_tau = 10.0                                    # fields (the preset's 1e3 takes minutes of video)
    rng = np.random.default_rng(1)
    pic = rng.random((lines, 16)).repeat(4, axis=1)
    x, act = synth.tv_composite(LINE, HSYNC, SHORT, lines, False, 120, pic, amp=0.25, noise=0.001)
    t = OracleTv(p)
    t.feed(x)
    est_line, _, gain = t.estimates()
    assert abs(est_line - LINE) < 0.05 and abs(gain - 4.0) < 0.1
    t.close()


def test_invalid_parameters_and_live_update(oracle):
    L = tv_lib()
    p = toy_params(40, False, 4)
    bad = toy_params(40, False, 4)
    bad.hsync_len = 0.4                                      # sample rate too low for this standard
    assert not L.sdo_tv_new(C.byref(bad))
    t = OracleTv(p)
    q = toy_params(40, False, 4)
    q.l_tol = 0.2
    assert L.sdo_tv_set_params(t.h, C.byref(q)) == 1
    q.frame_lines = 50
    assert L.sdo_tv_set_params(t.h, C.byref(q)) == 0         # geometry is fixed while running
    t.close()
    pal, ntsc = OL.TvParams(), OL.TvParams()
    L.sdo_tv_params_pal(C.byref(pal), 8e6)
    L.sdo_tv_params_ntsc(C.byref(ntsc), 8e6)
    assert pal.frame_lines == 625 and abs(pal.line_len - 512.0) < 1e-3 and pal.vsync_odd_trigger == 5
    assert ntsc.frame_lines == 525 and abs(ntsc.line_len - 508.448) < 1e-2 and ntsc.vsync_odd_trigger == 6


def test_feed_transform_matches_the_reference_expression(oracle):
    """TVProcessorTab::feed (Default/GenericInspector/TVProcessorTab.cpp:601-620)"""
    L = tv_lib()
    rng = np.random.default_rng(2)
    x = (rng.standard_normal(4096) + 1j * rng.standard_normal(4096)).astype(np.complex64)
    out = np.empty(x.size, np.float32)
    L.sdo_tv_feed_transform(x.ctypes.data, x.size, 0, -1.0, 0.25, out.ctypes.data)
    assert np.allclose(out, -np.abs(x) + 0.25, rtol=2e-7, atol=1e-7)
    L.sdo_tv_feed_transform(x.ctypes.data, x.size, 1, 1.0, -0.1, out.ctypes.data)
    assert np.allclose(out, np.angle(x) / np.pi - 0.1, rtol=0, atol=3e-7)


@pytest.mark.parametrize("interlace,lines,comb", [(False, 40, False), (True, 61, True)])
def test_reference_shaped_worker_over_the_shim_is_bit_identical(oracle, interlace, lines, comb):
    """TVProcessorWorker::work (reference-shaped, tests/shim/reference_tu.cpp) over <sigutils/tvproc.h>: every frame
    the display receives equals the oracle's frame of the same number, bit for bit."""
    tu = SB.reference_tu()
    x, pic, act = toy_signal(lines, interlace, frames=12)
    sp = toy_params(lines, interlace, 4, cls=ShimTvParams, comb=comb)
    W, H = int(np.floor(LINE)), lines
    cap = 16
    out = np.zeros((cap, H, W), np.float32)
    w, h = C.c_int(), C.c_int()
    block = 5000
    got = tu.tu_tv_worker(C.byref(sp), x.ctypes.data, x.size, block, out.ctypes.data, cap, C.byref(w), C.byref(h))
    assert got > 0 and (w.value, h.value) == (W, H)
    # the worker hands out at most one frame per work() call -- the first completed in the block, copied at completion
    # time.  Replay the blocks on the oracle in 64-sample steps; a frame's rows are final once it completes, so reading
    # frame f0 right after its completion gives the picture the worker copied.
    t = OracleTv(toy_params(lines, interlace, 4, comb=comb))
    k = 0
    for p0 in range(0, x.size, block):
        blk = x[p0:p0 + block]
        sent = False
        for pos in range(0, blk.size, 64):
            f0 = t.frames
            t.feed(blk[pos:pos + 64])
            if t.frames > f0 and not sent:
                assert np.array_equal(out[k].view(np.uint32), t.frame(f0).view(np.uint32))
                k += 1
                sent = True
    assert k == got
    t.close()


def test_c_abi_presets_equal_the_oracle_presets(oracle):
    """sdb_tv_params_pal / _ntsc (host-only entry points of the C-ABI) fill the same block as the oracle's presets and
    as the shim's su_tv_processor_params_* (modulo the shim's wider integer fields)."""
    import sigdigger_b200 as sdb
    L, T = sdb.load_library(), tv_lib()
    for name in ("pal", "ntsc"):
        for fs in (8e6, 13.5e6):
            a, b = sdb.TvParams(), OL.TvParams()
            getattr(L, "sdb_tv_params_" + name)(C.byref(a), fs)
            getattr(T, "sdo_tv_params_" + name)(C.byref(b), fs)
            assert bytes(a) == bytes(b)
    su = C.CDLL(sdb.LIB_PATH.replace("libsigdigger_b200.so", "libsigutils.so"))
    s = ShimTvParams()
    su.su_tv_processor_params_pal.argtypes = [C.c_void_p, C.c_float]
    su.su_tv_processor_params_pal(C.byref(s), 8e6)
    b = OL.TvParams()
    T.sdo_tv_params_pal(C.byref(b), 8e6)
    assert all(getattr(s, n) == getattr(b, n) for n, _ in OL.TvParams._fields_)


def test_free_running_raster_reverse_and_comb(oracle):
    """SPEC TV.2 / TV.6 without the sync separator: the raster free-runs at line_len, `reverse` shows x instead of
    1 - x (the sub-pixel weights of a pixel sum to one), and the comb filter removes a component that alternates from
    line to line (what it is there for: the chroma sub-carrier of a composite signal)."""
    lines = 20
    p = toy_params(lines, False, 4)
    p.enable_sync, p.enable_agc, p.line_len = 0, 0, 64.0                # integer line length: pixels = samples
    n = 64 * lines * 3
    rng = np.random.default_rng(7)
    x = rng.uniform(0.1, 0.9, n).astype(np.float32)
    t = OracleTv(p)
    assert t.feed(x) == 3                                               # exactly one frame per 64 * 20 samples
    f0 = t.frame(0)
    assert np.array_equal(f0.ravel(), (np.float32(1.0) - x[:64 * lines]))    # d = 0: pixel n = 1 - x[n]
    t.close()
    p.reverse = 1
    t = OracleTv(p)
    t.feed(x)
    assert np.array_equal(t.frame(0).ravel(), x[:64 * lines])
    t.close()
    # fractional line length: every pixel is the (1 - d, d) blend of two consecutive samples
    p.reverse, p.line_len = 0, 64.5
    t = OracleTv(p)
    t.feed(x)
    row1 = t.frame(0)[1]                # 65 samples went into the first line; sample 65 lands at x = 0.5 of the second
    want = 1.0 - (0.5 * x[65:65 + 63].astype(np.float64) + 0.5 * x[66:66 + 63])      # pixel k = (v[64 + k] + v[65 + k]) / 2
    assert np.max(np.abs(row1[1:64] - want)) < 1e-6
    t.close()
    # comb: luma repeats line after line, "chroma" flips sign every line -> (x + previous line) / 2 keeps the luma
    p.line_len, p.enable_comb, p.comb_reverse = 64.0, 1, 0
    luma = np.tile(rng.uniform(0.2, 0.6, 64), lines * 2)
    chroma = 0.2 * np.tile(np.concatenate([np.ones(64), -np.ones(64)]), lines)
    t = OracleTv(p)
    t.feed((luma + chroma).astype(np.float32))
    fr = t.frame(1)                                                     # past the first (unfilled delay line) frame
    assert np.max(np.abs((1.0 - fr[3]) - luma[:64])) < 1e-6
    p.comb_reverse = 1                                                  # the other output of the comb: the chroma
    t2 = OracleTv(p)
    t2.feed((luma + chroma).astype(np.float32))
    assert np.max(np.abs(np.abs(1.0 - t2.frame(1)[3]) - 0.2)) < 1e-6
    t.close()
    t2.close()
