"""-m gpu: the inspector's Analog TV tab inside the engine (oracle/SPEC_TI.md, k_tv_insp).  After every feed, each
stream's posted frame and status are bit-identical to the oracle tab (oracle/tvinsp.c) fed the same engine's soft
symbols (read back with sdb_engine_read_symbols), for psk, fsk and ask inspectors beside channels with the TV off, over
several streams, ragged feeds and feeds without symbols; a feed that completes more frames than the ring holds posts
its first; the processor's state does not depend on how the symbols were split into feeds; live parameter changes take
effect at the next feed and a geometry change is refused; a re-plan keeps or restarts the processor as TI.5 says; a
tab that is off changes nothing; a composite-video AM carrier read by an ask inspector locks and gives its picture; the
analyzer acknowledges, refuses and posts frames after each block's SAMPLES."""
import ctypes as C

import numpy as np
import pytest

import tvinsp_oracle as TO

pytestmark = pytest.mark.gpu

W = 8192
NP = 4096


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _signal(S, n, seed):
    rng = np.random.default_rng(seed)
    x = 0.3 * (rng.standard_normal((S, n)) + 1j * rng.standard_normal((S, n)))
    t = np.arange(n)
    for f in (0.3, 1.1, 1.9, 2.6, 3.4, 4.3):           # a carrier in every channel
        x = x + 0.5 * np.exp(1j * (f * t + rng.uniform(0, 6)))
    return x.astype(np.complex64)


def _tv(sdb, line_len=40.3, lines=8, **kw):
    """a small picture in symbols: frame_lines x line_len, non-interlaced, no comb"""
    q = dict(line_len=line_len, hsync_len=3.0, vsync_len=1.5, frame_lines=lines, interlace=0, enable_comb=0,
             vsync_odd_trigger=4)
    q.update(kw)
    return sdb.tv_params("pal", 1e6, **q)


def _inspector(e, h, cls, **extra):
    rate = e.channel_rate(h)
    if cls == "psk":
        cfg = dict(baud=rate / 4, costas_order=2, bits_per_symbol=2, loop_bw=rate * 2e-3, mf_type=1, mf_rolloff=0.35,
                   clock_type=1, clock_gain=0.1)
    else:
        cfg = dict(baud=rate / 4, bits_per_symbol=1, clock_type=1, clock_gain=0.1)
    cfg.update(extra)
    e.set_inspector(h, cls, **cfg)


def _engine(sdb, S, max_feed, chans):
    """chans: [(f0, class, tv kwargs of set_tv or None, extra inspector fields)]"""
    e = sdb.Engine(n_streams=S, psd_size=NP, psd_window="hann", st_window_size=W, max_feed=max_feed, samp_rate=1.0)
    hs = []
    for f0, cls, tv, extra in chans:
        h = e.open_channel(f0, 2 * np.pi * 0.05, 1.0)
        _inspector(e, h, cls, **extra)
        if tv is not None:
            e.set_tv(h, **tv)
        hs.append(h)
    e.commit()
    return e, hs


def _check(e, h, tabs, S):
    """the channel's processors after the latest feed against the oracle fed the same soft symbols; -> completed"""
    frames, st = e.read_tv(h)
    done = []
    for s in range(S):
        soft, _ = e.read_symbols(s, h)
        o = tabs[s]
        o.feed(soft)
        got = TO.Status(st[s].frames, st[s].posted_no, st[s].completed, st[s].width, st[s].height, st[s].line_len,
                        st[s].hsync_len, st[s].agc_gain)
        assert got.key() == o.status.key(), (h, s, got.key(), o.status.key())
        if o.status.posted_no:
            assert np.array_equal(_bits(frames[s]), _bits(o.posted)), (h, s)
        done.append(st[s].completed)
    return done


def _plan(sdb):
    return [(0.3, "psk", dict(params=_tv(sdb), dc=0.1), {}), (1.1, "psk", None, {}),
            (1.9, "fsk", dict(params=_tv(sdb, 33.7, 6), invert=True, dc=-0.2), {}),
            (2.6, "ask", dict(params=_tv(sdb, 52.0, 10), dc=0.05), {}), (3.4, "ask", None, {})]


def _tabs(sdb, cls, tv, S):
    return [TO.Tab(cls, tv["params"], tv.get("invert", False), tv.get("dc", 0.0)) for _ in range(S)]


def test_bit_identical_per_feed(sdb):
    S = 3
    plan = _plan(sdb)
    e, hs = _engine(sdb, S, 16 * W, plan)
    tabs = {h: _tabs(sdb, cls, tv, S) for h, (_, cls, tv, _) in zip(hs, plan) if tv is not None}
    x = _signal(S, 80 * W, 1)
    e.timing(True)
    pos, seen = 0, set()
    units = [0.5, 1, 16, 3, 0.5, 16, 7, 16, 0.5, 5]     # half a window: a feed without channel samples
    for u in units:
        n = int(u * W)
        e.feed(x[:, pos:pos + n])
        pos += n
        for h in tabs:
            seen.update(_check(e, h, tabs[h], S))
    assert 0 in seen and 1 in seen and max(seen) > 4, seen          # including more than the ring holds
    avg, n = e.kernel_time("tv")
    assert n == len(units)


def test_more_frames_than_the_ring_posts_the_first(sdb):
    """one feed completes 7 or more frames: the posted frame is the feed's first, which the ring no longer holds"""
    S = 2
    tv = dict(params=_tv(sdb, 12.0, 2), dc=0.0)                  # 24 symbols per frame
    e, hs = _engine(sdb, S, 16 * W, [(1.1, "psk", tv, {})])
    tabs = _tabs(sdb, "psk", tv, S)
    x = _signal(S, 16 * W, 2)
    e.feed(x)
    done = _check(e, hs[0], tabs, S)
    assert min(done) > 4 * 4, done
    _, st = e.read_tv(hs[0])
    assert all(q.posted_no == q.frames - q.completed + 1 for q in st)


def test_feed_splits_give_the_same_processor(sdb):
    S = 2
    plan = [(1.1, "psk", dict(params=_tv(sdb), invert=True), {}), (2.6, "ask", dict(params=_tv(sdb, 52.0, 10)), {})]
    x = _signal(S, 48 * W, 3)
    out = []
    for units in ([16, 16, 16], [1, 3, 0.5, 12.5, 7, 8, 16]):
        e, hs = _engine(sdb, S, 16 * W, plan)
        tabs = {h: _tabs(sdb, cls, tv, S) for h, (_, cls, tv, _) in zip(hs, plan)}
        pos = 0
        for u in units:
            n = int(u * W)
            e.feed(x[:, pos:pos + n])
            pos += n
            for h in hs:
                _check(e, h, tabs[h], S)
        out.append([[q.frames, float(q.line_len), float(q.agc_gain)] for h in hs for q in e.read_tv(h)[1]])
        out[-1].append([t.status.frames for h in hs for t in tabs[h]])
    assert out[0] == out[1]
    assert out[0][0][0] > 0


def test_live_parameters(sdb):
    S = 2
    tv = dict(params=_tv(sdb), dc=0.1)
    e, hs = _engine(sdb, S, 16 * W, [(1.9, "fsk", tv, {})])
    h = hs[0]
    tabs = _tabs(sdb, "fsk", tv, S)
    x = _signal(S, 40 * W, 4)
    pos = 0
    changes = {1: dict(params=_tv(sdb, enable_agc=0, t_tol=0.15), invert=True, dc=0.3),
               3: dict(params=_tv(sdb, reverse=1), dc=-0.1)}
    for i, u in enumerate((8, 5, 8, 3, 8)):
        if i in changes:
            c = changes[i]
            e.set_tv_params(h, **c)
            for o in tabs:
                assert o.set_params(c["params"], c.get("invert", False), c.get("dc", 0.0))
        e.feed(x[:, pos:pos + u * W])
        pos += u * W
        _check(e, h, tabs, S)
    for bad in (_tv(sdb, lines=9), _tv(sdb, line_len=41.3), _tv(sdb, interlace=1)):
        with pytest.raises(sdb.SdbError, match="geometry"):
            e.set_tv_params(h, params=bad)
    with pytest.raises(sdb.SdbError, match="invalid"):
        e.set_tv_params(h, params=_tv(sdb, hsync_len=30.0))
    e.feed(x[:, pos:pos + 8 * W])
    _check(e, h, tabs, S)                                         # the refusals changed nothing


@pytest.mark.parametrize("change", ["keep", "config", "retune", "class", "geometry"])
def test_migration(sdb, change):
    S = 2
    x = _signal(S, 60 * W, 5)
    tv = dict(params=_tv(sdb), dc=0.1)
    e1, hs = _engine(sdb, S, 8 * W, [(1.1, "psk", tv, {})])
    twin, _ = _engine(sdb, S, 8 * W, [(1.1, "psk", tv, {})])      # never re-planned
    tabs = _tabs(sdb, "psk", tv, S)
    pos = 0
    for u in (8, 3):
        e1.feed(x[:, pos:pos + u * W])
        twin.feed(x[:, pos:pos + u * W])
        pos += u * W
        _check(e1, hs[0], tabs, S)
    f0, cls, extra, tv2 = 1.1, "psk", {}, dict(tv, invert=True, dc=0.2)
    if change == "keep":
        tv2 = tv
    elif change == "config":
        extra = dict(clock_gain=0.2)
    elif change == "retune":
        f0 = 1.13
    elif change == "class":
        cls = "fsk"
    elif change == "geometry":
        tv2 = dict(params=_tv(sdb, lines=10))
    e2, hs2 = _engine(sdb, S, 8 * W, [(f0, cls, tv2, extra)])
    assert e2._L.sdb_engine_migrate_map(e2._h, e1._h, (C.c_int32 * 1)(0), 1) == 0, sdb.last_error()
    if change in ("class", "geometry"):
        tabs = _tabs(sdb, cls, tv2, S)
        assert all(q.frames == 0 for q in e2.read_tv(hs2[0])[1])
    else:
        for o in tabs:
            assert o.set_params(tv2["params"], tv2.get("invert", False), tv2.get("dc", 0.0))
        assert [q.frames for q in e2.read_tv(hs2[0])[1]] == [t.status.frames for t in tabs]
    for u in (8, 5, 8):
        e2.feed(x[:, pos:pos + u * W])
        twin.feed(x[:, pos:pos + u * W])
        pos += u * W
        _check(e2, hs2[0], tabs, S)
        if change == "keep":
            a, b = e2.read_tv(hs2[0]), twin.read_tv(0)
            assert np.array_equal(_bits(a[0]), _bits(b[0]))
            assert [TO.Status(*[getattr(q, f) for f, _ in TO.Status._fields_]).key() for q in a[1]] == \
                [TO.Status(*[getattr(q, f) for f, _ in TO.Status._fields_]).key() for q in b[1]]


def test_tv_off_changes_nothing(sdb):
    S = 2
    plan = [(0.3, "psk", None, {}), (1.9, "fsk", None, {}), (2.6, "ask", None, {})]
    e0, hs = _engine(sdb, S, 16 * W, plan)
    e1 = sdb.Engine(n_streams=S, psd_size=NP, psd_window="hann", st_window_size=W, max_feed=16 * W, samp_rate=1.0)
    for f0, cls, _, extra in plan:
        h = e1.open_channel(f0, 2 * np.pi * 0.05, 1.0)
        _inspector(e1, h, cls, **extra)
        e1.set_tv(h, params=_tv(sdb))
        e1.set_tv(h, enabled=False)
    e1.commit()
    e2, _ = _engine(sdb, S, 16 * W, [(0.3, "psk", None, {}), (1.9, "fsk", dict(params=_tv(sdb)), {}),
                                     (2.6, "ask", None, {})])
    x = _signal(S, 40 * W, 6)
    pos = 0
    for u in (1, 16, 0.5, 7, 16):
        n = int(u * W)
        l0, l1, l2 = e0.launches, e1.launches, e2.launches
        for e in (e0, e1, e2):
            e.feed(x[:, pos:pos + n])
        pos += n
        assert e1.launches - l1 == e0.launches - l0
        assert e2.launches - l2 == e0.launches - l0 + 1             # one k_tv_insp per feed
        for e in (e1, e2):
            assert np.array_equal(_bits(e0.read_psd()), _bits(e.read_psd()))
            for h in hs:
                for s in range(S):
                    assert np.array_equal(_bits(e0.read_channel(s, h)), _bits(e.read_channel(s, h)))
                    a, b = e0.read_symbols(s, h), e.read_symbols(s, h)
                    assert np.array_equal(_bits(a[0]), _bits(b[0])) and np.array_equal(a[1], b[1])
    assert e1.kernel_time("tv")[1] == 0


def test_refusals(sdb):
    e = sdb.Engine(n_streams=1, psd_size=NP, psd_window="hann", st_window_size=W, max_feed=W, samp_rate=1.0)
    hp = e.open_channel(0.5, 2 * np.pi * 0.05, 1.0)
    _inspector(e, hp, "psk")
    others = []
    for f0, cls in ((1.5, "raw"), (2.5, "power"), (3.5, "audio")):
        h = e.open_channel(f0, 2 * np.pi * 0.05, 1.0)
        e.set_inspector(h, cls)
        others.append(h)
    for h in others:
        with pytest.raises(sdb.SdbError, match="psk, fsk or ask"):
            e.set_tv(h, params=_tv(sdb))
    for bad in (_tv(sdb, line_len=4.0), _tv(sdb, hsync_len=30.0), _tv(sdb, lines=1), _tv(sdb, t_tol=0.0)):
        with pytest.raises(sdb.SdbError, match="invalid"):
            e.set_tv(hp, params=bad)
    with pytest.raises(sdb.SdbError, match="invalid"):
        e.set_tv(hp)                        # PAL at the symbol rate of a normalised-rate engine: far too short
    with pytest.raises(sdb.SdbError, match="wrong handle"):
        e.set_tv(7, params=_tv(sdb))
    with pytest.raises(sdb.SdbError, match="not committed"):
        e.set_tv_params(hp, params=_tv(sdb))
    e.set_tv(hp, params=_tv(sdb))
    e.commit()
    with pytest.raises(sdb.SdbError, match="already committed"):
        e.set_tv(hp, params=_tv(sdb))
    with pytest.raises(sdb.SdbError, match="not on"):
        e.read_tv(others[0])
    with pytest.raises(sdb.SdbError, match="not on"):
        e.set_tv_params(others[0], params=_tv(sdb))
    _, st = e.read_tv(hp)
    assert (st[0].frames, st[0].posted_no, st[0].completed, st[0].width, st[0].height) == (0, 0, 0, 40, 8)


def _composite_am(sdb, L_sym, r, lines, frames, seed):
    """composite video (sync tips high) over `lines` x L_sym symbols at a channel rate r, as the envelope of a carrier
    at the engine's input rate 1: -> (x, picture, (act0, act1) in symbols)"""
    from sigdigger_b200 import synth
    rng = np.random.default_rng(seed)
    pic = rng.random((lines, 8)).repeat(4, axis=1)
    c, (a0, a1) = synth.tv_composite(L_sym / r, 7.5 / r, 3.75 / r, lines, False, frames, pic, amp=1.0, seed=seed)
    return c, pic, (a0 * r, a1 * r)


def test_end_to_end_composite_am(sdb):
    """A composite-video picture AM-modulated onto a carrier, read by an ask inspector at one sample per symbol: the
    processor locks (line_len within 0.5 % of the transmitted 100.37 symbols) and the posted frame correlates with the
    transmitted picture (> 0.8, at the best row and column alignment), bit-identical to the oracle throughout."""
    S, L_sym, lines, f_c = 1, 100.37, 20, 1.1
    e = sdb.Engine(n_streams=S, psd_size=NP, psd_window="hann", st_window_size=W, max_feed=16 * W, samp_rate=1.0)
    h = e.open_channel(f_c, 2 * np.pi * 0.05, 1.0)
    r = e.channel_rate(h)
    e.set_inspector(h, "ask", baud=r, clock_type=0, mf_type=0, agc_enabled=0, bits_per_symbol=1)
    tvp = sdb.tv_params("pal", 1e6, line_len=L_sym, hsync_len=7.5, vsync_len=3.75, frame_lines=lines, interlace=0,
                        enable_comb=0, vsync_odd_trigger=4)
    e.set_tv(h, params=tvp)
    e.commit()
    c, pic, (a0, a1) = _composite_am(sdb, L_sym, r, lines, 12, 7)
    t = np.arange(c.size)
    rng = np.random.default_rng(8)
    x = (0.2 + 0.6 * c) * np.exp(1j * f_c * t) + 1e-3 * (rng.standard_normal(c.size) + 1j * rng.standard_normal(c.size))
    x = x.astype(np.complex64)[None, :]
    tab = [TO.Tab("ask", tvp)]
    best, posted = 0.0, 0
    for pos in range(0, (x.shape[1] // (4 * W)) * 4 * W, 4 * W):
        e.feed(x[:, pos:pos + 4 * W])
        _check(e, h, tab, S)
        frames, st = e.read_tv(h)
        if st[0].completed and st[0].frames >= 3:
            posted += 1
            assert abs(st[0].line_len - L_sym) < 0.005 * L_sym, st[0].line_len
            best = max(best, _match(frames[0], pic, a0, a1))
    assert posted >= 1
    assert best > 0.8, best


def _match(frame, pic, a0, a1, first=8):
    """the largest correlation of the frame's active columns with the picture lines from `first` on (the lines before
    carry the vertical interval), over every row shift and small column shifts"""
    H, Wd = frame.shape
    cols = np.arange(int(np.ceil(a0)) + 2, int(a1) - 2)
    ref = pic[first:, np.clip(((cols - a0) / (a1 - a0) * pic.shape[1]).astype(int), 0, pic.shape[1] - 1)]
    best = -1.0
    for dy in range(H):
        for dx in range(-4, 5):
            cc = np.clip(cols + dx, 0, Wd - 1)
            a = np.roll(frame, -dy, axis=0)[first:, cc].ravel()
            b = ref.ravel()
            if a.std() > 0:
                best = max(best, float(np.corrcoef(a, b)[0, 1]))
    return best


def test_analyzer_tv_messages_follow_the_samples(sdb):
    """Through an analyzer session: every block whose feed completed a frame posts, after its SAMPLES and after its SNR
    message, one TV message whose frame and status equal the oracle tab fed that block's SAMPLES; requests are
    acknowledged or refused (WRONG_KIND, WRONG_HANDLE, WRONG_OBJECT); a change that keeps the geometry applies from the
    next block without a re-plan; after "off" no TV message follows."""
    from sigdigger_b200.analyzer import Analyzer
    from test_gpu_fac import _Stepper
    N, fs, blocks = 8192, 1.0e6, 16
    per_block = 4 * N
    x = _signal(1, blocks * per_block, 9)[0]
    src = _Stepper(x)
    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=1.0, read=src.read, read_size=per_block)
    assert a.read(5000)[0] == "SOURCE_INFO"
    src.park(1)
    a.open("psk", 0.1 * fs, fs / 16, req_id=1)                       # handle 0
    a.open("raw", 0.3 * fs, fs / 32, req_id=2)                       # handle 1
    a.set_inspector_id(0, 10, req_id=20)
    a.set_inspector_id(1, 11, req_id=21)
    src.release(1)
    src.park(2)
    cfg = sdb.InspectorConfig()
    assert a._L.sdb_analyzer_get_inspector_config(a._h, 0, C.byref(cfg)) == 0
    cfg.clock_running = 1
    cfg.baud = cfg.fs / 4
    a.set_inspector_config(0, cfg, req_id=30)
    p1 = _tv(sdb)
    a.set_snr(0, 0.25, bins=64, req_id=39)
    a.set_tv(0, p1, dc=0.1, req_id=40)
    a.set_tv(1, p1, req_id=41)
    a.set_tv(0, _tv(sdb, line_len=2.0), req_id=42)
    a.set_tv(9, p1, req_id=43)
    src.release(5)
    src.park(6)
    p2 = _tv(sdb, reverse=1)
    a.set_tv(0, p2, invert=True, dc=0.2, req_id=44)                 # same geometry: live
    src.release(9)
    src.park(10)
    a.set_tv(0, None, req_id=45)                                     # off
    src.release(10**6)
    msgs = []
    while True:
        name, m = a.read(60000)
        assert name != "TIMEOUT"
        msgs.append((name, m))
        if name in ("EOS", "READ_ERROR", "HALT"):
            break
    a.close()
    assert msgs[-1][0] == "EOS"
    replies = {m["req_id"]: m for name, m in msgs if name == "INSPECTOR" and m["req_id"]}
    assert replies[40]["kind"] == "TV" and replies[44]["kind"] == "TV" and replies[45]["kind"] == "TV"
    assert replies[41]["kind"] == "WRONG_KIND" and replies[42]["kind"] == "WRONG_OBJECT"
    assert replies[43]["kind"] == "WRONG_HANDLE"
    tab, pending, posted, on, off_seen, snr_seen = None, [], 0, False, False, False
    for name, m in msgs:
        if name == "INSPECTOR" and m["req_id"] == 40:
            tab, on = TO.Tab("psk", p1, False, 0.1), True
        elif name == "INSPECTOR" and m["req_id"] == 44:
            if pending:                                          # blocks before the change, that completed no frame
                tab.feed(np.concatenate(pending))
                pending = []
            assert tab.set_params(p2, True, 0.2)
        elif name == "INSPECTOR" and m["req_id"] == 45:
            off_seen = True
        elif name == "SAMPLES" and m["inspector_id"] == 10:
            if on:
                pending.append(m["samples"])
            snr_seen = False
        elif name == "INSPECTOR" and m["kind"] == "SNR" and m["req_id"] == 0:
            snr_seen = True
        elif name == "INSPECTOR" and m["kind"] == "TV" and m["req_id"] == 0:
            assert not off_seen, "a TV message after the tab was turned off"
            assert pending and snr_seen, "a TV message before the block's SAMPLES or SNR message"
            tab.feed(np.concatenate(pending))
            pending = []
            q = m["tv"]
            got = TO.Status(q["frames"], q["posted_no"], q["completed"], q["width"], q["height"], q["line_len"],
                            q["hsync_len"], q["agc_gain"])
            assert got.key() == tab.status.key(), (got.key(), tab.status.key())
            assert np.array_equal(_bits(m["frame"]), _bits(tab.posted))
            posted += 1
    assert off_seen and posted >= 3, posted
