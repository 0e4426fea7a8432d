"""-m gpu: the inspector's SNR meter (oracle/SPEC_SN.md).  The engine's histograms, models and status are bit-identical
to the oracle meter fed the same engine's soft symbols (read back with sdb_engine_read_symbols), for psk, fsk and ask
inspectors over several streams, ragged feeds and feeds without symbols; the counts do not depend on how the symbols
were split into feeds; a re-plan keeps or restarts the meter as SN.4 says; a meter that is off changes nothing; the
analyzer acknowledges, refuses and posts the meter's data after each block's SAMPLES."""
import numpy as np
import pytest

import snr_oracle

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
        x = x + 0.5 * np.exp(1j * (f / (2 * np.pi) * 2 * np.pi * t + rng.uniform(0, 6)))
    return x.astype(np.complex64)


def _inspector(e, h, cls, bps, **extra):
    rate = e.channel_rate(h)
    if cls == "psk":
        cfg = dict(baud=rate / 4, costas_order=min(max(bps, 1), 3), bits_per_symbol=bps, loop_bw=rate * 2e-3,
                   mf_type=1, mf_rolloff=0.35, clock_type=1, clock_gain=0.1)
    else:
        cfg = dict(baud=rate / 4, bits_per_symbol=bps, clock_type=1, clock_gain=0.1)
    cfg.update(extra)
    e.set_inspector(h, cls, **cfg)


def _engine(sdb, S, max_feed, chans):
    """chans: [(f0, class, bps, snr kwargs or None, extra inspector fields)]"""
    e = sdb.Engine(n_streams=S, psd_size=NP, psd_window="hann", st_window_size=W, max_feed=max_feed, samp_rate=1.0)
    hs = []
    for f0, cls, bps, snr, extra in chans:
        h = e.open_channel(f0, 2 * np.pi * 0.05, 1.0)
        if cls in ("psk", "fsk", "ask"):
            _inspector(e, h, cls, bps, **extra)
        else:
            e.set_inspector(h, cls)
        if snr is not None:
            e.set_snr(h, **snr)
        hs.append(h)
    e.commit()
    return e, hs


def _check(e, h, meters, S):
    """the channel's meters of the latest feed against the oracle fed the same soft symbols"""
    hist, model, st = e.read_snr(h)
    for s in range(S):
        soft, _ = e.read_symbols(s, h)
        o = meters[s]
        o.feed(soft)
        assert np.array_equal(hist[s], o.h), (h, s)
        assert np.array_equal(_bits(model[s]), _bits(o.model)), (h, s)
        got = snr_oracle.Status(st[s].counted, st[s].steps, st[s].stepped, st[s].sigma, st[s].snr, st[s].delta)
        assert got.key() == o.status.key(), (h, s, got.key(), o.status.key())
    return sum(x.stepped for x in st)


PLAN = [(0.3, "psk", 1, dict(bins=16), {}), (1.1, "psk", 2, dict(bins=256), {}), (1.9, "psk", 3, dict(bins=1024), {}),
        (2.6, "fsk", 1, dict(bins=100, sigma=0.5, alpha=0.3), {}), (3.4, "ask", 2, dict(bins=256), {}),
        (4.3, "ask", 0, dict(bins=64), {})]


def test_bit_identical_per_feed(sdb):
    S = 3
    e, hs = _engine(sdb, S, 16 * W, PLAN)
    meters = {}
    for h, (_, cls, bps, snr, _) in zip(hs, PLAN):
        K = 1 << max(bps, 1)
        meters[h] = [snr_oracle.Meter(cls, snr["bins"], bps, snr.get("sigma", 1.0), snr.get("alpha", 1.0 / K))
                     for _ in range(S)]
    x = _signal(S, 80 * W, 1)
    e.timing(True)
    pos, steps, idle = 0, 0, 0
    units = [0.5, 1, 16, 3, 0.5, 16, 7, 16, 0.5, 5]     # half a window: a feed without channel samples
    for u in units:
        n = int(u * W)
        e.feed(x[:, pos:pos + n])
        pos += n
        for h in hs:
            k = _check(e, h, meters[h], S)
            steps += k
            idle += S - k
    assert steps > 0 and idle > 0
    avg, n = e.kernel_time("snr")
    assert n == len(units)


def test_counts_do_not_depend_on_the_feed_split(sdb):
    S = 2
    plan = [(1.1, "psk", 2, dict(bins=256), {}), (3.4, "ask", 1, dict(bins=128), {})]
    x = _signal(S, 48 * W, 2)
    out = []
    for units in ([16, 16, 16], [1, 3, 0.5, 12.5, 7, 8, 16]):
        e, hs = _engine(sdb, S, 16 * W, plan)
        pos = 0
        for u in units:
            n = int(u * W)
            e.feed(x[:, pos:pos + n])
            pos += n
        out.append([e.read_snr(h)[0] for h in hs])
    for a, b in zip(*out):
        assert np.array_equal(a, b)
        assert a.sum() > 0


def _migrate(sdb, dst, src):
    assert dst._L.sdb_engine_migrate(dst._h, src._h) == 0, sdb.last_error()


@pytest.mark.parametrize("change", ["keep", "alpha", "config", "bps", "bins", "class"])
def test_migration_and_reset(sdb, change):
    S = 2
    x = _signal(S, 60 * W, 3)
    p1 = (1.1, "psk", 2, dict(bins=256, sigma=1.0, alpha=0.25), {})
    e1, hs = _engine(sdb, S, 8 * W, [p1])
    h = hs[0]
    meters = [snr_oracle.Meter("psk", 256, 2, 1.0, 0.25) for _ in range(S)]
    pos = 0
    for u in (8, 3):
        e1.feed(x[:, pos:pos + u * W]); pos += u * W
        _check(e1, h, meters, S)
    e1.reset_snr(h, 0.5)                              # SN.3: sigma only, h kept, from the next feed
    for o in meters:
        o.reset(0.5)
    e1.feed(x[:, pos:pos + 4 * W]); pos += 4 * W
    _check(e1, h, meters, S)
    f0, cls, bps, snr, extra = p1
    snr = dict(snr)
    if change == "alpha":
        snr["alpha"] = 0.1
    elif change == "config":
        extra = dict(clock_gain=0.2)
    elif change == "bps":
        bps = 3
    elif change == "bins":
        snr["bins"] = 512
    elif change == "class":
        cls, bps = "fsk", 2
    e2, hs2 = _engine(sdb, S, 8 * W, [(f0, cls, bps, snr, extra)])
    _migrate(sdb, e2, e1)
    if change in ("keep", "alpha", "config", "bps"):
        for o in meters:
            o.replan(change in ("keep", "alpha"), bps, snr["alpha"])
    else:
        meters = [snr_oracle.Meter(cls, snr["bins"], bps, snr["sigma"], snr["alpha"]) for _ in range(S)]
    hist, _, st = e2.read_snr(hs2[0])
    assert (hist.sum() > 0) == (change in ("keep", "alpha"))
    for s in range(S):
        assert st[s].sigma == np.float32(meters[s].status.sigma)
    for u in (8, 5, 8):
        e2.feed(x[:, pos:pos + u * W]); pos += u * W
        _check(e2, hs2[0], meters, S)


def test_meter_off_changes_nothing(sdb):
    S = 2
    plan = [(0.3, "psk", 2, None, {}), (2.6, "fsk", 1, None, {}), (3.4, "ask", 1, None, {})]
    e0, hs = _engine(sdb, S, 16 * W, plan)
    e1 = sdb.Engine(n_streams=S, psd_size=NP, psd_window="hann", st_window_size=W, max_feed=16 * W, samp_rate=1.0)
    for f0, cls, bps, _, extra in plan:
        h = e1.open_channel(f0, 2 * np.pi * 0.05, 1.0)
        _inspector(e1, h, cls, bps, **extra)
        e1.set_snr(h, bins=256)
        e1.set_snr(h, enabled=False)
    e1.commit()
    e2, _ = _engine(sdb, S, 16 * W, [(f0, c, b, dict(bins=128), x) for f0, c, b, _, x in plan])
    x = _signal(S, 40 * W, 4)
    pos = 0
    for u in (1, 16, 0.5, 7, 16):
        n = int(u * W)
        l0, l1, l2 = e0.launches, e1.launches, e2.launches
        for e in (e0, e1, e2):
            e.feed(x[:, pos:pos + n])
        pos += n
        assert e1.launches - l1 == e0.launches - l0
        assert e2.launches - l2 == e0.launches - l0 + 1             # one k_snr per feed
        for e in (e1, e2):
            assert np.array_equal(_bits(e0.read_psd()), _bits(e.read_psd()))
            for h in hs:
                for s in range(S):
                    assert np.array_equal(_bits(e0.read_channel(s, h)), _bits(e.read_channel(s, h)))
                    a, b = e0.read_symbols(s, h), e.read_symbols(s, h)
                    assert np.array_equal(_bits(a[0]), _bits(b[0])) and np.array_equal(a[1], b[1])
    avg, n = e1.kernel_time("snr")
    assert n == 0


def test_refusals(sdb):
    e = sdb.Engine(n_streams=1, psd_size=NP, psd_window="hann", st_window_size=W, max_feed=W, samp_rate=1.0)
    hp = e.open_channel(0.5, 2 * np.pi * 0.05, 1.0)
    _inspector(e, hp, "psk", 2)
    hr = e.open_channel(1.5, 2 * np.pi * 0.05, 1.0)
    e.set_inspector(hr, "raw")
    hw = e.open_channel(2.5, 2 * np.pi * 0.05, 1.0)
    e.set_inspector(hw, "power")
    ha = e.open_channel(3.5, 2 * np.pi * 0.05, 1.0)
    e.set_inspector(ha, "audio")

    def refused(h, msg, **kw):
        with pytest.raises(sdb.SdbError, match=msg):
            e.set_snr(h, **kw)

    for L in (0, 15, 1025, 4096):
        refused(hp, "bins must be in \\[16, 1024\\]", bins=L)
    for h in (hr, hw, ha):
        refused(h, "psk, fsk or ask", bins=256)
    for v in (0.0, -1.0, float("nan"), float("inf")):
        refused(hp, "sigma", sigma=v)
        refused(hp, "alpha", alpha=v)
    refused(7, "wrong handle")
    e.set_snr(hp, bins=256)
    e.commit()
    with pytest.raises(sdb.SdbError, match="already committed"):
        e.set_snr(hp, bins=256)
    with pytest.raises(sdb.SdbError, match="not on"):
        e.read_snr(hr)
    with pytest.raises(sdb.SdbError, match="not on"):
        e.reset_snr(hr, 1.0)
    with pytest.raises(sdb.SdbError, match="wrong handle"):
        e.reset_snr(9, 1.0)
    for v in (0.0, float("nan")):
        with pytest.raises(sdb.SdbError, match="sigma"):
            e.reset_snr(hp, v)


def test_analyzer_snr_messages_follow_the_samples(sdb):
    """Through an analyzer session: every block in which the meter stepped posts, after its SAMPLES, one SNR message
    whose model, histogram and status equal the oracle meter fed that block's SAMPLES as one feed, across a reset and a
    re-plan that opens another inspector mid-stream; requests are acknowledged or refused with the engine's rules, and
    the payload equals what the engine reads."""
    import ctypes as C

    from sigdigger_b200.analyzer import Analyzer
    from test_gpu_fac import _Stepper
    N, fs, blocks = 8192, 1.0e6, 14
    per_block = 4 * N
    x = _signal(1, blocks * per_block, 5)[0]
    src = _Stepper(x)
    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=1.0, read=src.read, read_size=per_block)
    assert a.read(5000)[0] == "SOURCE_INFO"
    src.park(1)
    a.open("psk", 0.1 * fs, fs / 16, req_id=1)                       # handle 0
    a.open("ask", -0.2 * fs, fs / 16, req_id=2)                      # handle 1
    a.open("raw", 0.3 * fs, fs / 32, req_id=3)                       # handle 2
    for h, iid in ((0, 10), (1, 11), (2, 12)):
        a.set_inspector_id(h, iid, req_id=20 + h)
    src.release(1)
    src.park(2)
    for h in (0, 1):
        cfg = sdb.InspectorConfig()
        assert a._L.sdb_analyzer_get_inspector_config(a._h, h, C.byref(cfg)) == 0
        cfg.clock_running = 1
        cfg.baud = cfg.fs / 4
        a.set_inspector_config(h, cfg, req_id=30 + h)
    a.set_snr(0, 0.25, bins=256, req_id=40)
    a.set_snr(1, 0.5, bins=100, sigma=0.7, req_id=41)
    a.set_snr(2, 0.5, req_id=42)
    a.set_snr(0, 0.25, bins=2000, req_id=43)
    a.reset_snr(2, 1.0, req_id=44)
    a.set_snr(9, 0.25, req_id=45)
    src.release(5)
    src.park(6)
    a.reset_snr(0, 0.6, req_id=46)
    src.release(7)
    src.park(8)
    a.open("fsk", 0.4 * fs, fs / 16, req_id=4)                       # a re-plan mid-stream: the meters carry on
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
    assert replies[40]["kind"] == "SNR" and replies[41]["kind"] == "SNR" and replies[46]["kind"] == "SNR"
    assert replies[42]["kind"] == "WRONG_KIND" and replies[43]["kind"] == "WRONG_OBJECT"
    assert replies[44]["kind"] == "WRONG_OBJECT" and replies[45]["kind"] == "WRONG_HANDLE"
    meters = {10: snr_oracle.Meter("psk", 256, 2, 1.0, 0.25), 11: snr_oracle.Meter("ask", 100, 1, 0.7, 0.5)}
    pending, posted, seen_reset = {10: [], 11: []}, {10: 0, 11: 0}, False
    on = set()                                   # the meter counts from the block after its acknowledgement
    for name, m in msgs:
        if name == "INSPECTOR" and m["req_id"] in (40, 41):
            on.add(10 if m["req_id"] == 40 else 11)
        if name == "INSPECTOR" and m["req_id"] == 46:
            seen_reset = True
            meters[10].reset(0.6)
        if name == "SAMPLES" and m["inspector_id"] in on:
            pending[m["inspector_id"]].append(m["samples"])
        elif name == "INSPECTOR" and m["kind"] == "SNR" and m["spectrum"] is not None:
            iid = m["inspector_id"]
            assert pending[iid], "an SNR message without the block's SAMPLES before it"
            o = meters[iid]
            o.feed(np.concatenate(pending[iid]))
            pending[iid] = []
            q = m["snr"]
            got = snr_oracle.Status(q["counted"], q["steps"], q["stepped"], q["sigma"], q["snr"], q["delta"])
            assert got.key() == o.status.key(), (iid, got.key(), o.status.key())
            assert np.array_equal(_bits(m["spectrum"]), _bits(o.model))
            assert np.array_equal(m["histogram"], o.h)
            posted[iid] += 1
    assert seen_reset
    assert all(not v for v in pending.values()), "a block's SNR message is missing"
    assert posted[10] >= 6 and posted[11] >= 6, posted
