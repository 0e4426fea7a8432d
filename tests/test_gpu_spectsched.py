"""Scheduled inspector spectra and baud estimates (oracle/SPEC_US.md) on the GPU: every emission bit-identical to the
oracle over the engine's own channel stream, whatever the feed split, beside legacy channels and inspectors, across
re-plans, and through the analyzer."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from sigdigger_b200 import synth
import shim_build as SB
from spectsched_stmt import reference, same, schedule

pytestmark = pytest.mark.gpu

ESTS = ("baud-fac", "baud-nonlinear")
W, S = 4096, 3


def _capture(n, seed, f=0.1):
    xs = []
    for s in range(S):
        rng = np.random.default_rng(seed + s)
        sig, _ = synth.psk_signal(n, 16.0, order=4, seed=seed + s)
        xs.append(0.3 * synth.mix(sig, f + 1e-5 * s, 0.2 * s) + synth.awgn(n, 1e-3, rng))
    return np.stack(xs).astype(np.complex64)


def _engine(sdb, size, kind, ns, I, max_hops, f=0.1, fmt="f32", extra=None):
    e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=max_hops * W // 2, input_format=fmt)
    h = e.open_channel(2 * np.pi * f, 2 * np.pi * size / W, 1.0)
    assert e.channel_info(h).size == size
    if kind:
        e.set_spectrum_source(h, kind, ns)
    for est in ESTS:
        e.set_estimator(h, est)
    if I:
        e.set_spectrum_interval(h, I)
    if extra:
        extra(e)
    e.commit()
    return e, h


def _feed(e, x, fmt):
    if fmt == "device":
        import torch
        e.feed(torch.from_numpy(np.ascontiguousarray(x)).cuda())
    else:
        e.feed(x)


def _run(sdb, size, kind, ns, I, split, x, fmt="f32"):
    """feeds of `split` hops; -> (emissions per stream [(t_j, (spectrum, fac, nonlinear))], channel stream per stream,
    emissions per feed)"""
    e, h = _engine(sdb, size, kind, ns, I, max(split), fmt="u8" if fmt == "u8" else "f32")
    em, chan, counts = [[] for _ in range(S)], [[] for _ in range(S)], []
    pos = 0
    for hops in split:
        n = hops * W // 2
        _feed(e, x[:, pos:pos + n], fmt)
        pos += n
        spectra, ends = e.read_spectra(h)
        ests = [e.read_estimates(h, est) for est in ESTS]
        counts.append(len(ends))
        last, sizes = e.read_spectrum(h)                  # the per-feed read gives the feed's last emission
        assert np.all(sizes == (spectra.shape[2] if len(ends) else 0))
        for s in range(S):
            chan[s].append(e.read_channel(s, h))
            if len(ends):
                assert np.array_equal(last[s, :spectra.shape[2]], spectra[s, -1])
            for j, t in enumerate(ends):
                em[s].append((int(t), [spectra[s, j]] + [v[s, j] if ok[s, j] else None for v, ok in ests]))
    e.close()
    return em, [np.concatenate(c) for c in chan], counts


def _oracle_fn(oracle, kind, ns, fs_ch):
    def fn(c):
        return [oracle.spectsrc_frame(kind, ns, c)] + [oracle.estimate_baud(est, ns, fs_ch, c) for est in ESTS]
    return fn


CASES = {   # channel size: (kind, Ns, I, hops of two feed splits)
    4: ("psd", 64, 20, ([9, 3, 17, 1, 30, 8, 12], [1, 40, 1, 1, 37])),
    8: ("cyclo", 64, 37, ([5, 5, 5, 5, 25, 5], [13, 7, 2, 28])),
    64: ("fac", 256, 300, ([3, 11, 2, 9, 15], [20, 20])),
    1024: ("abstimediff", 4096, 3000, ([7, 2, 5, 1, 3, 6, 4, 2], [1, 3, 7, 7, 7, 5])),
}


@pytest.mark.parametrize("size", sorted(CASES))
@pytest.mark.parametrize("fmt", ["f32", "device", "u8"])
def test_engine_against_oracle(sdb, oracle, size, fmt):
    """Two feed splits of the same input: both bit-identical to the oracle at every t_j over the engine's own channel
    stream, and so to each other."""
    kind, ns, I, splits = CASES[size]
    assert sum(splits[0]) == sum(splits[1])
    n = sum(splits[0]) * W // 2
    x = _capture(n, seed=size)
    if fmt == "u8":
        x = np.stack([np.clip(np.round(x.real * 300 + 127.5), 0, 255), np.clip(np.round(x.imag * 300 + 127.5), 0, 255)],
                     axis=-1).astype(np.uint8)
    fs_ch = np.float32(size / W)
    results = []
    for split in splits:
        em, chan, counts = _run(sdb, size, kind, ns, I, split, x, fmt)
        for s in range(S):
            want = reference(chan[s], ns, I, _oracle_fn(oracle, kind, ns, fs_ch))
            assert len(want) >= 3
            assert same(em[s], want), (size, fmt, split, s)
        results.append((em, counts))
    assert same(sum(results[0][0], []), sum(results[1][0], []))
    if size <= 8:
        assert 0 in results[0][1] and max(results[0][1]) >= 2     # narrow: feeds without and with several emissions


def test_tie_to_legacy_per_feed(sdb, oracle):
    """I = the samples of every feed: each feed emits once, at its end, the legacy U.1 spectrum and estimates of the
    same feed (the first feed has one hop more: its first hop only primes the history)."""
    size, ns, H = 1024, 1024, 4
    I = H * size // 2
    split = [H + 1] + [H] * 5
    x = _capture(sum(split) * W // 2, seed=3)
    eng = {}
    for name, iv in (("legacy", 0), ("sched", I)):
        eng[name] = _engine(sdb, size, "exp_2", ns, iv, H + 1)
    pos = 0
    for k, hops in enumerate(split):
        n = hops * W // 2
        for e, _ in eng.values():
            e.feed(x[:, pos:pos + n])
        pos += n
        (el, hl), (es, hs) = eng["legacy"], eng["sched"]
        leg, sizes = el.read_spectrum(hl)
        spectra, ends = es.read_spectra(hs)
        assert list(ends) == [(k + 1) * I] and np.all(sizes == ns)
        assert np.array_equal(spectra[:, 0].view(np.uint32), leg.view(np.uint32))
        for est in ESTS:
            v, ok = el.read_estimate(hl, est)
            vs, oks = es.read_estimates(hs, est)
            assert np.array_equal(ok, oks[:, 0]) and np.array_equal(v[ok == 1].view(np.uint32),
                                                                     vs[:, 0][ok == 1].view(np.uint32))


def test_mixed_plan_leaves_the_rest_unchanged(sdb):
    """Legacy spectrum channels and inspector symbols are bit-identical with and without scheduled channels beside
    them."""
    hops, feeds = 8, 4
    x = _capture(hops * feeds * W // 2, seed=9, f=0.2)

    def build(with_sched):
        e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=hops * W // 2)
        a = e.open_channel(2 * np.pi * 0.2, 2 * np.pi * 64 / W, 1.0)
        e.set_spectrum_source(a, "psd", 256)
        e.set_estimator(a, "baud-nonlinear")
        b = e.open_channel(2 * np.pi * 0.2, 2 * np.pi * 128 / W, 1.0)
        e.set_inspector(b, "psk")
        if with_sched:
            for f, sz in ((0.3, 4), (0.25, 256)):
                c = e.open_channel(2 * np.pi * f, 2 * np.pi * sz / W, 1.0)
                e.set_spectrum_source(c, "cyclo", 1024)
                e.set_estimator(c, "baud-fac")
                e.set_spectrum_interval(c, 700)
        e.commit()
        return e, a, b

    (e0, a0, b0), (e1, a1, b1) = build(False), build(True)
    n = hops * W // 2
    for k in range(feeds):
        for e in (e0, e1):
            e.feed(x[:, k * n:(k + 1) * n])
        for (p, q) in ((e0.read_spectrum(a0), e1.read_spectrum(a1)),
                       (e0.read_estimate(a0, "baud-nonlinear"), e1.read_estimate(a1, "baud-nonlinear"))):
            assert all(np.array_equal(u, v) for u, v in zip(p, q))
        for s in range(S):
            for u, v in zip(e0.read_symbols(s, b0), e1.read_symbols(s, b1)):
                assert np.array_equal(u, v)


def _migrate(sdb, dst, src, old_of_new):
    L = sdb.load_library()
    sdb._check(L.sdb_engine_migrate_map(dst._h, src._h, (C.c_int32 * len(old_of_new))(*old_of_new), len(old_of_new)))


def test_migration_carries_and_retune_restarts(sdb, oracle):
    """An unrelated inspector opens and closes mid-stream and the kind switches psd -> cyclo: the scheduled channel's
    emissions equal those of an engine that never re-planned (same t_j, frames over the same stream).  A retuned
    channel restarts at t = 0."""
    size, ns, I, hops = 64, 512, 200, 6
    n = hops * W // 2
    x = _capture(9 * n, seed=17)
    fs_ch = np.float32(size / W)

    def make(kind, with_other, f=0.1):
        def extra(e):
            if with_other:
                o = e.open_channel(2 * np.pi * 0.3, 2 * np.pi * 16 / W, 1.0)
                e.set_inspector(o, "raw")
        return _engine(sdb, size, kind, ns, I, hops, f=f, extra=extra)

    ref, hr = make("psd", False)
    stages = [("psd", False, [0]), ("psd", True, [0]), ("cyclo", False, [0, -1])]   # engine per 3 feeds
    cur, hc, got, chan = None, None, [], []
    for k in range(9):
        if k % 3 == 0:
            kind, other, _ = stages[k // 3]
            nxt, hn = make(kind, other)
            if cur is not None:
                _migrate(sdb, nxt, cur, [0, -1] if other else [0])
                cur.close()
            cur, hc = nxt, hn
        xs = x[:, k * n:(k + 1) * n]
        ref.feed(xs)
        cur.feed(xs)
        spectra, ends = cur.read_spectra(hc)
        chan.append(ref.read_channel(0, hr))
        assert np.array_equal(cur.read_channel(0, hc), chan[-1])
        kind = stages[k // 3][0]
        got += [(int(t), [spectra[0, j]]) for j, t in enumerate(ends)]
        rs, rends = ref.read_spectra(hr)
        assert list(rends) == list(ends)
        if kind == "psd":
            assert np.array_equal(spectra.view(np.uint32), rs.view(np.uint32))
    c = np.concatenate(chan)
    psd = [(t, [oracle.spectsrc_frame("psd", ns, c[:t])]) for t, _ in got if t <= 6 * hops * size // 2 - size // 2]
    cyc = [(t, [oracle.spectsrc_frame("cyclo", ns, c[:t])]) for t, _ in got if t > 6 * hops * size // 2 - size // 2]
    assert len(cyc) >= 3 and same(got, psd + cyc)
    # retune: the channel moves; its count starts again, so over four feeds (768 samples) it emits once, at 600, over
    # its new samples (a carried count, 1 696, would have emitted at 1 800, 2 000, 2 200 and 2 400)
    moved, hm = make("psd", False, f=0.15)
    _migrate(sdb, moved, cur, [0])
    em, c0 = [], []
    for k in range(4):
        moved.feed(x[:, k * n:(k + 1) * n])
        spectra, ends = moved.read_spectra(hm)
        c0.append(moved.read_channel(0, hm))
        em += [(int(t), [spectra[0, j]]) for j, t in enumerate(ends)]
    c0 = np.concatenate(c0)
    assert len(c0) == 4 * hops * size // 2 and [t for t, _ in em] == [600]
    assert same(em, [(600, [oracle.spectsrc_frame("psd", ns, c0[:600])])])
    for e in (ref, cur, moved):
        e.close()


def test_interval_change_across_migration(sdb, oracle):
    """SPEC US.5 on the GPU: I = 1000 for three feeds, then a re-planned engine with I = 300 that carries the count and
    the ring.  The emissions equal the statement's (the engine's ring model, tests/spectsched_stmt.py) over the same
    channel samples and feed boundaries, including the point it skips because its frame reaches before the samples
    the old interval kept."""
    size, ns, hops = 64, 256, 6
    n = hops * W // 2
    x = _capture(7 * n, seed=41)
    fs_ch = np.float32(size / W)
    old, ho = _engine(sdb, size, "psd", ns, 1000, hops)
    feeds, got = [], []
    for k in range(7):
        if k == 3:
            new, hn = _engine(sdb, size, "psd", ns, 300, hops)
            _migrate(sdb, new, old, [0])
            old.close()
            old, ho = new, hn
        old.feed(x[:, k * n:(k + 1) * n])
        spectra, ends = old.read_spectra(ho)
        ests = [old.read_estimates(ho, est) for est in ESTS]
        feeds.append(old.read_channel(0, ho))
        got += [(int(t), [spectra[0, j]] + [v[0, j] if ok[0, j] else None for v, ok in ests]) for j, t in enumerate(ends)]
    old.close()
    fn = _oracle_fn(oracle, "psd", ns, fs_ch)
    a, st = schedule(feeds[:3], ns, 1000, fn)
    b, _ = schedule(feeds[3:], ns, 300, fn, state=st)
    want = [x for g in a + b for x in g]
    # the switch at t = 3 * 192 - 32 = 544: 600 needs samples from 343 on, but I = 1000 kept none of them
    assert 600 not in [t for t, _ in want] and 900 in [t for t, _ in want]
    assert same(got, want)
    # every emitted frame is still the whole-stream frame
    c = np.concatenate(feeds)
    assert same(want, [(t, fn(c[:t])) for t, _ in want])


def test_refusals_have_messages(sdb):
    L = sdb.load_library()
    e = sdb.Engine(n_streams=1, psd_size=0, st_window_size=W, max_feed=8 * W // 2)
    h = e.open_channel(1.0, 2 * np.pi * 512 / W, 1.0)
    assert L.sdb_engine_set_spectrum_interval(e._h, h, 100) == -1
    assert "without a spectrum source or estimator" in sdb.last_error()
    e.set_spectrum_source(h, "psd", 1024)
    e.set_spectrum_interval(h, 7)          # 8 hops x 512 samples / 7 > 256 emissions per feed
    with pytest.raises(sdb.SdbError, match="at most 256"):
        e.commit()
    e2 = sdb.Engine(n_streams=1, psd_size=0, st_window_size=W, max_feed=8 * W // 2)
    h2 = e2.open_channel(1.0, 2 * np.pi * 512 / W, 1.0)
    g = e2.open_channel(2.0, 2 * np.pi * 64 / W, 1.0)
    e2.set_spectrum_source(h2, "psd", 1024)
    e2.set_spectrum_source(g, "psd", 1024)
    e2.set_spectrum_interval(h2, 8)        # exactly 256
    e2.commit()
    assert L.sdb_engine_set_spectrum_interval(e2._h, h2, 100) == -1 and "committed" in sdb.last_error()
    out, ends = np.zeros(4096, np.float32), np.zeros(4, np.uint64)
    assert L.sdb_engine_read_spectra(e2._h, g, out.ctypes.data, ends.ctypes.data, 1) == -1
    assert "no spectrum interval" in sdb.last_error()
    e3 = sdb.Engine(n_streams=1, psd_size=0, st_window_size=W, max_feed=8 * W // 2)
    h3 = e3.open_channel(1.0, 2 * np.pi * 512 / W, 1.0)
    e3.set_estimator(h3, "baud-fac")
    assert L.sdb_engine_set_spectrum_interval(e3._h, h3, (1 << 62) + 1) == -1 and "at most 2^62" in sdb.last_error()
    e3.close()
    e.close()
    e2.close()


# ---------------------------------------------------------------------------------------------- analyzer
def _analyzer_run(sdb, x, fs, N, per_block, upd, channels):
    from sigdigger_b200.analyzer import Analyzer
    import threading
    started = threading.Event()
    pos = [0]

    def read(priv, dst, maxn):
        started.wait(30)
        take = min(maxn, len(x) - pos[0])
        if take > 0:
            C.memmove(dst, x.ctypes.data + 8 * pos[0], 8 * take)
            pos[0] += take
        return take

    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=1.0, read=read, read_size=per_block,
                 spectrum_update_int=upd)
    assert a.read(5000)[0] == "SOURCE_INFO"
    req = 1
    for h, (cls, fc, bw, spect) in enumerate(channels):
        a.open(cls, fc, bw, req_id=req)
        a.set_inspector_id(h, 100 + h, req_id=req + 1)
        if spect:
            a.set_spectrum_source(h, sdb.SPECTSRC[spect], req_id=req + 2)
        req += 3
    started.set()
    msgs = []
    while True:
        name, m = a.read(60000)
        assert name != "TIMEOUT"
        msgs.append((name, m))
        if name in ("EOS", "READ_ERROR", "HALT"):
            break
    a.close()
    return msgs


def test_analyzer_schedule(sdb, oracle):
    """A narrow channel that posts no SPECTRUM per block posts, at spectrum_update_int = 0.1, exactly the 4096-point
    spectra of the points j I >= 4097, equal to the oracle over a "raw" inspector's samples of the same channel; a wide
    channel posts at the 100 ms cadence instead of once per block."""
    N, fs, blocks = 8192, 1.0e6, 72
    per_block = 8 * N                                            # 65.5 ms a block, 16 channeliser hops
    n = blocks * per_block
    x, _ = synth.multi_carrier(n, fs, [("qpsk", 0.1 * fs, fs / 400, -10.0, {}), ("qpsk", -0.2 * fs, fs / 16, -10.0, {})],
                               noise_db=-40.0, seed=4)
    x = np.ascontiguousarray(x, np.complex64)
    # 6 bins: an 8-bin channel, 64 samples a block (too few for the smallest per-block frame, 64 + 1)
    narrow = [("raw", 0.1 * fs, 6 * fs / N, None), ("psk", 0.1 * fs, 6 * fs / N, "psd")]
    wide = [("psk", -0.2 * fs, fs / 8, "psd")]
    spect = lambda msgs, iid: [m for name, m in msgs if name == "INSPECTOR" and m["kind"] == "SPECTRUM"
                               and m["spectrum"] is not None and m["inspector_id"] == iid]
    assert spect(_analyzer_run(sdb, x, fs, N, per_block, 0.0, narrow), 101) == []
    msgs = _analyzer_run(sdb, x, fs, N, per_block, 0.1, narrow + wide)
    raw = np.concatenate([m["samples"] for name, m in msgs if name == "SAMPLES" and m["inspector_id"] == 100])
    got = spect(msgs, 101)
    fs_ch = float(got[0]["equiv_fs"])
    I = max(1, int(np.floor(0.1 * fs_ch + 0.5)))
    want = [t for t in range(I, len(raw) + 1, I) if t >= 4097]
    assert len(want) >= 2 and len(got) == len(want)
    for m, t in zip(got, want):
        ref = oracle.spectsrc_frame("psd", 4096, raw[:t])
        assert len(m["spectrum"]) == 4096 and np.array_equal(np.asarray(m["spectrum"]).view(np.uint32),
                                                            ref.view(np.uint32))
    w = spect(msgs, 102)
    secs = blocks * per_block / fs
    assert abs(len(w) - secs / 0.1) <= 1.5 and len(w) < blocks


def test_analyzer_interval_too_short_for_the_block(sdb):
    """An interval shorter than a block allows (1 us: 125 samples of a 125 kHz channel would be 262 emissions in a
    65 ms block) is raised to ceil(samples per block / 256): the session runs to EOS, posting 256 spectra a block.
    Infinite and negative intervals are refused with a message."""
    from sigdigger_b200.analyzer import Analyzer
    N, fs, blocks = 8192, 1.0e6, 4
    per_block = 8 * N
    x, _ = synth.multi_carrier(blocks * per_block, fs, [("qpsk", -0.2 * fs, fs / 16, -10.0, {})], noise_db=-40.0,
                               seed=8)
    x = np.ascontiguousarray(x, np.complex64)
    msgs = _analyzer_run(sdb, x, fs, N, per_block, 1e-6, [("raw", -0.2 * fs, fs / 8, None),
                                                           ("psk", -0.2 * fs, fs / 8, "psd")])
    assert msgs[-1][0] == "EOS"
    got = [m for name, m in msgs if name == "INSPECTOR" and m["kind"] == "SPECTRUM" and m["spectrum"] is not None]
    # 1024-bin channel: 16 hops x 512 = 8192 samples a block, so I = 32; T channel samples (those of the raw
    # inspector on the same channel) emit at every multiple of 32 from 4128 (the first >= 4097) on
    T = sum(len(m["samples"]) for name, m in msgs if name == "SAMPLES" and m["inspector_id"] == 100)
    assert T >= 2 * 8192 and len(got) == T // 32 - 4096 // 32 and all(len(m["spectrum"]) == 4096 for m in got)
    for bad in (math.inf, -1.0, math.nan):
        with pytest.raises(sdb.SdbError, match="spectrum_update_int"):
            Analyzer(fs, window_size=N, data=x, read_size=per_block, spectrum_update_int=bad)


def test_shim_session_posts_on_the_gui_period(sdb, oracle):
    """Through libsuscan.so (the GUI's only path; the shim sets the 100 ms period): a narrow channel that gets no
    per-block spectrum posts the 4096-point spectra of the points j I >= 4097, equal to the oracle over a "raw"
    inspector's samples of the same channel, and a wide channel posts every 100 ms instead of every block."""
    so = os.path.join(SB.build_dir(), "libspectschedtu.so")
    libdir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sigdigger_b200")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-I", os.path.join(os.path.dirname(libdir), "include"),
                    os.path.join(os.path.dirname(libdir), "tests", "shim", "spectsched_tu.cpp"), "-o", so, "-L", libdir,
                    "-lsuscan", "-lsigutils", "-Wl,-rpath," + libdir, "-lpthread"], check=True)
    tu = C.CDLL(so)
    tu.tu_spectrum_session.restype = C.c_int
    tu.tu_spectrum_session.argtypes = [C.c_void_p, C.c_size_t, C.c_uint, C.c_uint, C.c_size_t, C.c_double, C.c_double,
                                       C.c_double, C.c_double, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                       C.c_void_p, C.c_void_p]
    N, fs, blocks = 8192, 1000000, 72
    per_block = 8 * N
    n = blocks * per_block
    x, _ = synth.multi_carrier(n, float(fs), [("qpsk", 0.1 * fs, fs / 400, -10.0, {}),
                                              ("qpsk", -0.2 * fs, fs / 16, -10.0, {})], noise_db=-40.0, seed=4)
    x = np.ascontiguousarray(x, np.complex64)
    raw = np.zeros(blocks * 64, np.complex64)
    narrow = np.zeros((16, 4096), np.float32)
    counts, sizes = np.zeros(3, np.uint64), np.zeros(2, np.int64)
    rc = tu.tu_spectrum_session(x.ctypes.data, n, fs, N, per_block, 0.1 * fs, 6.0 * fs / N, -0.2 * fs, fs / 8.0,
                                raw.ctypes.data, len(raw), narrow.ctypes.data, len(narrow), counts.ctypes.data,
                                sizes.ctypes.data)
    assert rc == 0, rc
    raw = raw[:int(counts[0])]
    fs_ch = fs * 8 / N                                    # 6 bins -> an 8-bin channel, 64 samples a block
    I = max(1, int(math.floor(0.1 * fs_ch + 0.5)))
    want = [t for t in range(I, len(raw) + 1, I) if t >= 4097]
    assert len(want) >= 2 and int(counts[1]) == len(want) and sizes[0] == 4096
    for k, t in enumerate(want):
        ref = oracle.spectsrc_frame("psd", 4096, raw[:t])
        assert np.array_equal(narrow[k].view(np.uint32), ref.view(np.uint32)), k
    secs = n / fs
    assert sizes[1] == 4096 and abs(int(counts[2]) - secs / 0.1) <= 1.5 and int(counts[2]) < blocks
