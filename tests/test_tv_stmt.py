"""CPU: the analog-TV processor held to tests/tv_stmt.py, the exact binary32 statement of SPEC TV written from the SPEC
text alone.  For every scene of SCENES (a composite signal from synth.tv_composite plus edits, a parameter block, a
split into feeds and live parameter changes between them):
  * the oracle (oracle/tvproc.c) equals the statement bit for bit after every feed: every frame of the readable window
    (the last three completed and the one in progress), the frame count and the estimates;
  * the step k_tv_feed runs, on the host through the <sigutils/tvproc.h> shim (sdb_tv_step on the caller's thread),
    equals the oracle bit for bit after every feed: the frame su_tv_processor_take_frame returns, the frame count and
    the estimates -- for the long scenes and the presets at full size too, which the statement is too slow for;
  * the statement reached every branch the scene names, and every branch of the step is named by some scene.
Each planted mistake of the statement (tv_stmt.MISTAKES) changes the outcome of the scene named for it.
GPU batch: tests/test_gpu_tv.py runs the same scenes through k_tv_feed."""
import ctypes as C
import math
import os
from dataclasses import dataclass, field

import numpy as np
import pytest

import oracle_lib as OL
import test_oracle_tv as T
import tv_stmt as S
from sigdigger_b200 import synth

LINE, HSYNC, SHORT = T.LINE, T.HSYNC, T.SHORT


def base(lines=20, interlace=False, trigger=4, **kw):
    """the PAL preset with the toy geometry of tests/test_oracle_tv.py, as a dict"""
    o = T.toy_params(lines, interlace, trigger)
    d = {k: getattr(o, k) for k, _ in OL.TvParams._fields_}
    d.update(kw)
    return d


def composite(lines=20, interlace=False, frames=3, start=3.3, amp=0.5, noise=0.002, seed=3, line=LINE, hsync=HSYNC,
              short=SHORT, n_eq=5):
    rng = np.random.default_rng(seed)
    pic = rng.random((lines, 16)).repeat(4, axis=1)
    x, _ = synth.tv_composite(line, hsync, short, lines, interlace, frames, pic, amp=amp, noise=noise, seed=seed,
                              n_eq=n_eq)
    return np.ascontiguousarray(x[int(line * start):])


def pulse_starts(lines, frames, start, line=LINE):
    """sample index (in the cut signal) of every line's horizontal pulse"""
    k = np.arange(lines * frames + 1)
    s = np.ceil(k * line).astype(np.int64) - int(line * start)
    return s[s >= 0]


def drop_and_spurious(v):
    """hsync pulses 30-33 removed (blanking), two spurious pulses mid-line"""
    x = composite(frames=3, start=3.3, amp=0.95, seed=3 + v)
    st = pulse_starts(20, 3, 3.3)
    for s in st[30:34]:
        x[s:s + int(HSYNC) + 1] = np.float32(0.7 * 0.95)
    for s in st[40:42]:
        m = s + 200
        x[m:m + int(HSYNC)] = np.float32(0.95)
    return x


def broken_train(v):
    """the second equalising pulse of the second frame's train removed: the count restarts, that frame's trigger is
    missed"""
    x = composite(frames=3, start=3.3, amp=0.95, seed=3 + v)
    s0 = int(math.ceil(20 * LINE)) - int(LINE * 3.3) + int(math.ceil(LINE / 2))
    x[s0:s0 + int(SHORT) + 1] = np.float32(0.7 * 0.95)
    return x


def amp_step(v):
    """sync tip 0.5, then 0.25 from the middle on"""
    x = composite(frames=5, start=3.3, seed=3 + v)
    x[x.size // 2:] *= np.float32(0.5)
    return x


def dropout(v):
    """two fields and a half of silence in the middle: one whole field without a peak"""
    x = composite(frames=5, start=3.3, amp=0.95, seed=3 + v)
    a = x.size // 3
    x[a:a + int(2.5 * 20 * LINE)] = 0.0
    return x


@dataclass
class Scene:
    name: str
    params: dict
    signal: object                                  # variant -> float32 samples (variant 0 is the statement's)
    branches: tuple = ()
    feeds: list = field(default_factory=list)       # [(samples, parameter changes before this feed)], rest last
    long: bool = False                              # oracle and shim only: too long for the statement


def _sig(**kw):
    """a composite scene whose variant v differs in its picture and noise"""
    return lambda v: composite(**{**kw, "seed": 3 + v})


COMMON = ("rise", "fall", "hsync", "line_end", "field_end", "frame_end", "raster_right", "agc_peak")

SCENES = [
    Scene("acquire", base(), _sig(frames=3, start=3.3),
          COMMON + ("huge_jump", "err_wrap_lo", "to_fast", "to_slow", "track_slow", "ll_first", "ll_accept",
                    "ll_update", "equalising", "eq_count", "eq_restart", "broad", "trigger", "trigger_gated",
                    "trigger_early", "agc_update")),
    Scene("acquire_late", base(lines=40), _sig(lines=40, frames=3, start=17.3),
          COMMON + ("huge_jump", "trigger_late", "trigger_gated")),
    Scene("fast_slow", base(), _sig(frames=3, start=0.1, amp=0.95, noise=0.012),
          COMMON + ("to_fast", "to_slow", "track_fast", "track_slow")),
    Scene("x_off_neg", base(x_off=-50.0), _sig(frames=3, start=3.8, amp=0.95),
          COMMON + ("huge_jump", "xf_wrap", "err_wrap_lo")),
    Scene("x_off_pos", base(x_off=250.0), _sig(frames=3, start=3.95, amp=0.95),
          COMMON + ("huge_jump", "err_wrap_hi")),
    Scene("line_rate", base(line_len=np.float32(LINE * 1.004), line_len_tau=10.0), _sig(frames=6, start=3.3),
          COMMON + ("ll_accept", "ll_update")),
    Scene("dropped_spurious", base(), drop_and_spurious,
          COMMON + ("ll_reject", "huge_jump", "to_fast")),
    Scene("broken_train", base(), broken_train, COMMON + ("eq_restart", "eq_count", "broad")),
    Scene("agc_step", base(), amp_step, COMMON + ("agc_update",)),
    Scene("agc_off", base(enable_agc=0), _sig(frames=3, amp=0.95), COMMON + ("agc_off",)),
    Scene("dropout", base(), dropout, COMMON + ("agc_hold",)),
    Scene("interlaced_odd", base(lines=41, interlace=True),
          _sig(lines=41, interlace=True, frames=4, start=5.3, amp=0.95),
          COMMON + ("parity_mid", "parity_start", "field_odd", "trigger_late", "trigger_early")),
    Scene("interlaced_even", base(lines=40, interlace=True, trigger=5),
          _sig(lines=40, interlace=True, frames=4, start=2.6, amp=0.95),
          COMMON + ("parity_mid", "parity_start", "trigger_late")),
    Scene("h2", base(lines=2, interlace=True), _sig(lines=21, interlace=True, frames=2, amp=0.95),
          COMMON + ("field_odd", "trigger")),
    Scene("dominance0", base(lines=39, interlace=True, dominance=0),
          _sig(lines=41, interlace=True, frames=3, start=5.3, amp=0.95), COMMON + ("field_odd", "row_off")),
    Scene("reverse", base(reverse=1), _sig(frames=3), COMMON),
    Scene("comb", base(enable_comb=1), _sig(frames=3), COMMON + ("comb_sum",)),
    Scene("comb_reverse", base(enable_comb=1, comb_reverse=1, enable_sync=0, enable_agc=0), _sig(frames=3),
          ("comb_diff", "sync_off")),
    Scene("frame_spacing", base(frame_spacing=0.375, line_len=np.float32(LINE * 1.004), line_len_tau=10.0),
          _sig(frames=5, start=3.3, amp=0.95), COMMON + ("raster_left", "ll_update")),
    Scene("free_running", base(enable_sync=0), _sig(frames=3), ("sync_off", "line_end", "frame_end")),
    Scene("line_int", base(line_len=400.0), _sig(frames=3, line=400.0), COMMON),
    Scene("line_8", base(lines=20, line_len=8.0, hsync_len=2.0, vsync_len=1.0),
          _sig(frames=6, start=0.5, line=8.0, hsync=2.0, short=1.0, amp=0.95), ("line_end", "frame_end")),
    Scene("line_8_5", base(lines=20, line_len=8.5, hsync_len=2.0, vsync_len=1.0),
          _sig(frames=6, start=0.5, line=8.5, hsync=2.0, short=1.0, amp=0.95), ("line_end", "frame_end")),
    Scene("line_4096", base(lines=12, line_len=4096.0, hsync_len=300.0, vsync_len=150.0),
          _sig(lines=12, frames=3, start=0.5, line=4096.0, hsync=300.0, short=150.0, amp=0.95), COMMON),
    Scene("tall_odd", base(lines=2049, interlace=True, line_len=16.5, hsync_len=4.0, vsync_len=2.0),
          _sig(lines=2049, interlace=True, frames=3, start=0.5, line=16.5, hsync=4.0, short=2.0, amp=0.95),
          ("line_end", "frame_end", "field_odd")),
    Scene("line_4096_5", base(lines=12, line_len=4096.5, hsync_len=300.0, vsync_len=150.0),
          _sig(lines=12, frames=3, start=0.5, line=4096.5, hsync=300.0, short=150.0, amp=0.95), COMMON),
]


def preset(standard, frames, v):
    """the preset's own geometry at 8 MS/s; NTSC's trigger is the sixth pulse, so its trains have six"""
    q = _struct(preset_params(standard))
    rng = np.random.default_rng(5 + v)
    pic = rng.random((q.frame_lines, 32)).repeat(4, axis=1)
    x, _ = synth.tv_composite(q.line_len, q.hsync_len, q.vsync_len, q.frame_lines, True, frames, pic, amp=0.6,
                              noise=0.003, seed=5 + v, n_eq=q.vsync_odd_trigger)
    return np.ascontiguousarray(x[int(q.line_len * (17.3 + 3.1 * v)):])


def preset_params(standard):
    q = OL.TvParams()
    getattr(T.tv_lib(), "sdo_tv_params_" + standard)(C.byref(q), 8e6)
    return {k: getattr(q, k) for k, _ in OL.TvParams._fields_}


def _struct(d, cls=OL.TvParams):
    q = cls()
    for k, _ in OL.TvParams._fields_:
        setattr(q, k, d[k])
    return q


LIVE = [(8000, {}), (8000, {"reverse": 1}), (8000, {"reverse": 0, "enable_agc": 0}),
        (8000, {"enable_agc": 1, "dominance": 0}), (8000, {"dominance": 1, "enable_comb": 1}),
        (8000, {"enable_comb": 0}), (8000, {"enable_comb": 1}),          # back on: the delay line is stale
        (8000, {"comb_reverse": 1}), (8000, {"comb_reverse": 0, "enable_sync": 0}),
        (8000, {"enable_sync": 1, "x_off": 20.0}), (20000, {"frame_spacing": 0.25}),
        (None, {"x_off": 0.0, "frame_spacing": 0.0, "vsync_odd_trigger": 5})]

SCENES += [
    Scene("t_tol_edge", base(hsync_len=32.0, t_tol=0.125), _sig(frames=2, amp=0.95), COMMON + ("t_tol_edge",)),
    Scene("gate_edge", base(lines=21, interlace=True),                   # trains 7.5 lines long in 10-line fields
          _sig(lines=21, interlace=True, frames=4, amp=0.95), COMMON + ("gate_edge",)),
    Scene("live_switches", base(lines=41, interlace=True), _sig(lines=41, interlace=True, frames=9, amp=0.95),
          COMMON + ("comb_sum", "comb_diff", "agc_off", "sync_off", "field_odd", "raster_left"), LIVE),
    Scene("pal", preset_params("pal"), lambda v: preset("pal", 4, v), long=True),
    Scene("ntsc", preset_params("ntsc"), lambda v: preset("ntsc", 4, v), long=True),
    Scene("interlaced_long", base(lines=61, interlace=True),
          _sig(lines=61, interlace=True, frames=24, start=17.3, amp=0.5), long=True),
]
BY_NAME = {s.name: s for s in SCENES}
MISTAKE_SCENE = {"t_tol_lt": "t_tol_edge", "line_max_kept": "agc_step", "fs_pre_update": "frame_spacing",
                 "late_no_preswap": "interlaced_odd", "dominance_inverted": "interlaced_odd", "comb_sign": "comb",
                 "no_xf_wrap": "x_off_neg", "gate_gt": "gate_edge"}


def plan(scene, n):
    """[(length, parameter changes before it)] over n samples: the scene's own feeds, else three uneven feeds"""
    feeds = scene.feeds or [(n // 3 + 17, {}), (n // 3 - 5, {}), (None, {})]
    out, pos = [], 0
    for k, ch in feeds:
        k = n - pos if k is None else min(k, n - pos)
        out.append((k, ch))
        pos += k
    return out


def readable(frames):
    return range(max(0, frames - 3), frames + 1)


def run_stmt(scene, x, mistake=None):
    """[(frames, {frame no: picture}, estimates)] after every feed, and the statement (for its branch counters)"""
    p = dict(scene.params)
    s = S.TvStmt(p, mistake=mistake)
    out, pos = [], 0
    for k, ch in plan(scene, x.size):
        if ch:
            p.update(ch)
            assert s.set_params(p)
        s.feed(x[pos:pos + k])
        pos += k
        out.append((s.frames, {f: s.frame(f) for f in readable(s.frames)}, s.estimates()))
    return out, s


def run_oracle(scene, x):
    p = dict(scene.params)
    t = T.OracleTv(_struct(p))
    out, pos = [], 0
    try:
        for k, ch in plan(scene, x.size):
            if ch:
                p.update(ch)
                assert T.tv_lib().sdo_tv_set_params(t.h, C.byref(_struct(p))) == 1
            t.feed(x[pos:pos + k])
            pos += k
            out.append((t.frames, {f: t.frame(f) for f in readable(t.frames)}, tuple(map(np.float32, t.estimates()))))
    finally:
        t.close()
    return out


class _FrameBuf(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("buffer", C.POINTER(C.c_float)), ("next", C.c_void_p)]


def shim():
    import sigdigger_b200 as sdb
    su = C.CDLL(sdb.LIB_PATH.replace("libsigdigger_b200.so", "libsigutils.so"))
    su.su_tv_processor_new.restype = C.c_void_p
    su.su_tv_processor_new.argtypes = [C.c_void_p]
    su.su_tv_processor_set_params.argtypes = [C.c_void_p, C.c_void_p]
    su.su_tv_processor_feed.argtypes = [C.c_void_p, C.c_float]
    su.su_tv_processor_take_frame.restype = C.POINTER(_FrameBuf)
    su.su_tv_processor_take_frame.argtypes = [C.c_void_p]
    su.su_tv_processor_return_frame.argtypes = [C.c_void_p, C.POINTER(_FrameBuf)]
    su.su_tv_processor_destroy.argtypes = [C.c_void_p]
    su.sdb_shim_tv_estimates.argtypes = [C.c_void_p] + [C.POINTER(C.c_float)] * 3 + [C.POINTER(C.c_ulonglong)]
    return su


def run_shim(scene, x):
    """[(frames, the frame take_frame returns (or None), estimates)] after every feed, su_tv_processor_* per sample"""
    su = shim()
    p = dict(scene.params)
    h = su.su_tv_processor_new(C.byref(_struct(p, T.ShimTvParams)))
    assert h
    feed = su.su_tv_processor_feed
    out, pos = [], 0
    try:
        for k, ch in plan(scene, x.size):
            if ch:
                p.update(ch)
                assert su.su_tv_processor_set_params(h, C.byref(_struct(p, T.ShimTvParams)))
            for v in x[pos:pos + k].tolist():
                feed(h, v)
            pos += k
            a, b, g, n = C.c_float(), C.c_float(), C.c_float(), C.c_ulonglong()
            su.sdb_shim_tv_estimates(h, C.byref(a), C.byref(b), C.byref(g), C.byref(n))
            f = su.su_tv_processor_take_frame(h)
            pic = None
            if f:
                fb = f.contents
                pic = np.ctypeslib.as_array(fb.buffer, shape=(fb.height, fb.width)).copy()
                su.su_tv_processor_return_frame(h, f)
            out.append((n.value, pic, (np.float32(a.value), np.float32(b.value), np.float32(g.value))))
    finally:
        su.su_tv_processor_destroy(h)
    return out


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def same(ra, rb):
    """two per-feed runs agree bit for bit: counts, every readable frame, estimates"""
    return all(fa == fb and fa_.keys() == fb_.keys() and all(np.array_equal(bits(fa_[k]), bits(fb_[k])) for k in fa_)
               and np.array_equal(bits(ea), bits(eb)) for (fa, fa_, ea), (fb, fb_, eb) in zip(ra, rb))


SHORT_SCENES = [s.name for s in SCENES if not s.long]


@pytest.mark.parametrize("name", SHORT_SCENES)
def test_oracle_equals_statement(oracle, name):
    scene = BY_NAME[name]
    x = scene.signal(0)
    ref = run_oracle(scene, x)
    got, st = run_stmt(scene, x)
    assert ref[-1][0] >= 1, "the scene completes no frame"
    for i, ((fa, fa_, ea), (fb, fb_, eb)) in enumerate(zip(ref, got)):
        assert fa == fb, (i, fa, fb)
        for f in fa_:
            assert np.array_equal(bits(fa_[f]), bits(fb_[f])), (i, f)
        assert np.array_equal(bits(ea), bits(eb)), (i, ea, eb)
    missing = [b for b in scene.branches if not st.hits[b]]
    assert not missing, missing


@pytest.mark.parametrize("name", [s.name for s in SCENES])
def test_shim_step_equals_oracle(oracle, name):
    """sdb_tv_step, the step k_tv_feed runs, on the host through <sigutils/tvproc.h>"""
    scene = BY_NAME[name]
    x = scene.signal(0)
    ref = run_oracle(scene, x)
    got = run_shim(scene, x)
    assert ref[-1][0] >= (2 if scene.long else 1)
    for i, ((fa, fa_, ea), (fb, pic, eb)) in enumerate(zip(ref, got)):
        assert fa == fb, (i, fa, fb)
        assert (pic is None) == (fa == 0)
        if fa:
            assert np.array_equal(bits(fa_[fa - 1]), bits(pic)), (i, fa)
        assert np.array_equal(bits(ea), bits(eb)), (i, ea, eb)


def test_every_branch_of_the_step_is_named_by_a_scene():
    named = set().union(*(s.branches for s in SCENES))
    assert set(S.BRANCHES) | set(S.EDGES) == named, sorted((set(S.BRANCHES) | set(S.EDGES)) ^ named)


@pytest.mark.parametrize("mistake", S.MISTAKES)
def test_planted_mistake_is_caught(mistake):
    assert set(MISTAKE_SCENE) == set(S.MISTAKES)
    scene = BY_NAME[MISTAKE_SCENE[mistake]]
    x = scene.signal(0)
    good, _ = run_stmt(scene, x)
    bad, _ = run_stmt(scene, x, mistake=mistake)
    assert not same(good, bad), mistake


def test_alpha_agrees_with_c_expf():
    """SPEC TV.1: the statement's correctly rounded exp gives C's expf result on every tau the scenes use"""
    libm = C.CDLL(None)
    libm.expf.restype = C.c_float
    libm.expf.argtypes = [C.c_float]
    taus = set()
    for s in SCENES:
        p = s.params
        taus |= {float(np.float32(p[k])) for k in ("agc_tau", "hsync_len_tau", "line_len_tau", "hsync_fast_track_tau",
                                                    "hsync_slow_track_tau")}
        taus.add(float(max(np.float32(p["hsync_len"]) / np.float32(20.0), np.float32(1.0))))
    taus |= {5.0, 0.5, 1.5, 2.0, 3.0}
    for tau in sorted(taus):
        c = np.float32(1.0) - np.float32(libm.expf(float(np.float32(-1.0) / np.float32(tau))))
        assert bits(S.alpha(tau)) == bits(c), tau


def test_statement_imports_nothing_from_the_implementations():
    src = open(os.path.join(os.path.dirname(__file__), "tv_stmt.py")).read()
    for word in ("oracle", "sigdigger_b200", "ctypes", "shim"):
        assert not any(line.startswith(("import", "from")) and word in line for line in src.splitlines()), word


def test_invalid_parameters_refused_alike(oracle):
    """TV.0 validity and the live update's fixed geometry: the statement, the oracle and the shim agree"""
    su = shim()
    good = base()
    cases = [dict(line_len=7.99), dict(line_len=4097.0), dict(line_len=4096.99), dict(line_len=8.0),
             dict(hsync_len=0.99), dict(hsync_len=200.2), dict(vsync_len=0.5), dict(frame_lines=1),
             dict(frame_lines=4097), dict(frame_spacing=1.0), dict(frame_spacing=-0.1), dict(t_tol=1.0),
             dict(l_tol=0.0), dict(agc_tau=0.0)]
    for ch in cases:
        d = {**good, **ch}
        ok = T.tv_lib().sdo_tv_new(C.byref(_struct(d)))
        if ok:
            T.tv_lib().sdo_tv_destroy(ok)
        sh = su.su_tv_processor_new(C.byref(_struct(d, T.ShimTvParams)))
        if sh:
            su.su_tv_processor_destroy(sh)
        assert S.valid(d) == bool(ok) == bool(sh), ch
    s = S.TvStmt(good)
    for ch, want in ((dict(line_len=LINE + 0.5), True), (dict(line_len=LINE + 1), False), (dict(frame_lines=21), False),
                     (dict(interlace=1), False), (dict(line_len=400.0), False), (dict(enable_sync=0), True)):
        assert s.set_params({**good, **ch}) == want, ch
