"""-m gpu: the inspector's FAC tab (oracle/SPEC_FC.md).  The engine's fac, max, min, peak lag, sigmas, marker and block
count are bit-identical to the oracle fed the same engine's soft symbols, at every block size from 512 to 2^19, over
ragged feeds, feeds without symbols and feeds that complete many blocks; the FAC leaves every other output of a plan
unchanged; a re-plan keeps or restarts it as the header says; and every refusal says why."""
import numpy as np
import pytest

import fac_oracle

pytestmark = pytest.mark.gpu

W = 8192
NP = 4096
SIZES = [1 << m for m in range(9, 20)]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _signal(S, n, seed, period=2999):
    """a repeating segment in noise: symbol streams with a period for the FAC to find"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(S):
        seg = rng.standard_normal(period) + 1j * rng.standard_normal(period)
        x = 0.3 * np.resize(seg, n) + 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
        out.append(x.astype(np.complex64))
    return np.stack(out)


def _psk(e, h):
    rate = e.channel_rate(h)
    e.set_inspector(h, "psk", baud=rate / 2, costas_order=2, bits_per_symbol=2, loop_bw=rate * 2e-3, mf_type=1,
                    mf_rolloff=0.35, clock_type=1, clock_gain=0.1)


def _engine(sdb, S, max_feed, chans):
    """chans: [(f0, bw fraction, class, fac kwargs or None)]"""
    e = sdb.Engine(n_streams=S, psd_size=NP, psd_window="hann", st_window_size=W, max_feed=max_feed, samp_rate=1.0)
    hs = []
    for f0, frac, cls, fac in chans:
        h = e.open_channel(f0, 2 * np.pi * frac, 1.0)
        if cls in ("psk", "fsk", "ask"):
            rate = e.channel_rate(h)
            if cls == "psk":
                _psk(e, h)
            else:
                e.set_inspector(h, cls, baud=rate / 4, bits_per_symbol=1, clock_type=1, clock_gain=0.1)
        elif cls == "power":
            e.set_inspector(h, "power", power_integrate_samples=64)
        elif cls == "audio":
            e.set_inspector(h, "audio")                  # the class defaults
        if fac is not None:
            e.set_fac(h, **fac)
        hs.append(h)
    e.commit()
    return e, hs


def _check(e, hs, oracles, S):
    """every FAC chain of the latest feed against its oracle fed the same soft symbols"""
    blocks = 0
    for h in hs:
        if h not in oracles:
            continue
        fac, st = e.read_fac(h)
        for s in range(S):
            soft, _ = e.read_symbols(s, h)
            o = oracles[h][s]
            ref = o.feed(soft)
            b32 = lambda v: int(np.float32(v).view(np.uint32))     # noqa: E731
            got = (st[s].blocks, st[s].peak_lag, b32(st[s].max), b32(st[s].min), b32(st[s].sigmas), st[s].marker)
            assert got == ref.key(), (h, s, o.L, got, ref.key())
            assert np.array_equal(_bits(fac[s]), _bits(o.fac)), (h, s, o.L)
            blocks += st[s].blocks
    return blocks


def test_every_size_bit_identical(sdb):
    S = 2
    chans = []
    for i, L in enumerate(SIZES):
        lags = [None, (1, L // 2), (3, min(L // 2, 2500))][i % 3]
        alpha = [1.0, 0.5, 0.25][i % 3]
        chans.append((0.3 + 0.5 * i, 0.4 if L >= 1 << 17 else 0.1, "psk",
                      dict(size=L, alpha=alpha, lags=lags, sigma=3.0)))
    units = [0.5, 1, 120, 7, 200, 33, 200]          # in W-sample feeds; the first has no channel samples
    e, hs = _engine(sdb, S, 200 * W, chans)
    oracles = {h: [fac_oracle.Fac(c[3]["size"], c[3]["alpha"], c[3]["lags"], 3.0) for _ in range(S)]
               for h, c in zip(hs, chans)}
    x = _signal(S, int(sum(units) * W), 1)
    e.timing(True)
    pos, total, markers = 0, {}, 0
    for u in units:
        n = int(u * W)
        launches = e.launches
        e.feed(x[:, pos:pos + n])
        pos += n
        _check(e, hs, oracles, S)
        for h in hs:
            _, st = e.read_fac(h)
            total[h] = total.get(h, 0) + st[0].blocks
            markers += sum(s.marker for s in st)
        assert e.launches > launches
    # every size completed at least one block, the small ones many in one feed
    assert all(total[h] >= 1 for h in hs), total
    assert total[hs[0]] > 100
    assert markers > 0
    avg, n = e.kernel_time("fac")
    assert n == len(units)


def test_mixed_plan_leaves_other_outputs_unchanged(sdb):
    S = 2
    plan = [(0.4, 0.05, "psk", dict(size=1024, alpha=0.5, lags=(2, 512))), (1.1, 0.02, "fsk", None),
            (1.9, 0.01, "power", None), (2.6, 0.01, "audio", None), (3.4, 0.08, "ask", dict(size=16384)),
            (4.3, 0.05, "psk", None)]
    off = [(f0, frac, cls, None) for f0, frac, cls, _ in plan]
    e1, hs = _engine(sdb, S, 16 * W, plan)
    e0, _ = _engine(sdb, S, 16 * W, off)
    oracles = {h: [fac_oracle.Fac(c[3]["size"], c[3].get("alpha", 1.0), c[3].get("lags"), 5.0) for _ in range(S)]
               for h, c in zip(hs, plan) if c[3] is not None}
    x = _signal(S, 60 * W, 2)
    pos = 0
    for u in [1, 16, 3, 16, 8, 16]:
        n = u * W
        l0, l1 = e0.launches, e1.launches
        e0.feed(x[:, pos:pos + n]); e1.feed(x[:, pos:pos + n])
        pos += n
        assert np.array_equal(_bits(e0.read_psd()), _bits(e1.read_psd()))
        for h in hs:
            for s in range(S):
                assert np.array_equal(_bits(e0.read_channel(s, h)), _bits(e1.read_channel(s, h)))
                a, b = e0.read_symbols(s, h), e1.read_symbols(s, h)
                assert np.array_equal(_bits(a[0]), _bits(b[0])) and np.array_equal(a[1], b[1])
        _check(e1, hs, oracles, S)
        assert e1.launches - l1 > e0.launches - l0


def _migrate(sdb, dst, src):
    assert dst._L.sdb_engine_migrate(dst._h, src._h) == 0, sdb.last_error()


@pytest.mark.parametrize("change", ["keep", "alpha_window", "size", "rate"])
def test_migration(sdb, change):
    S = 2
    x = _signal(S, 40 * W, 3)
    fac = dict(size=2048, alpha=0.5, lags=None, sigma=5.0)
    e1, hs = _engine(sdb, S, 8 * W, [(0.7, 0.05, "psk", fac)])
    h = hs[0]
    orc = [fac_oracle.Fac(2048, 0.5, None, 5.0) for _ in range(S)]
    pos = 0
    for u in (8, 3):
        e1.feed(x[:, pos:pos + u * W]); pos += u * W
        _check(e1, hs, {h: orc}, S)
    fac2, bw = dict(fac), 0.05
    if change == "alpha_window":
        fac2.update(alpha=0.25, lags=(5, 700), sigma=2.0)
    elif change == "size":
        fac2.update(size=4096)
    elif change == "rate":
        bw = 0.1
    e2, hs2 = _engine(sdb, S, 8 * W, [(0.7, bw, "psk", fac2)])
    _migrate(sdb, e2, e1)
    if change in ("keep", "alpha_window"):
        for o in orc:                       # the tab keeps its state and takes the new parameters
            o.f.alpha, o.f.sigma = np.float32(fac2["alpha"]), fac2["sigma"]
            o.f.lo, o.f.hi = fac2["lags"] if fac2["lags"] else (0, 1024)
    else:
        orc = [fac_oracle.Fac(fac2["size"], fac2["alpha"], fac2["lags"], fac2["sigma"]) for _ in range(S)]
    for u in (8, 5, 8):
        e2.feed(x[:, pos:pos + u * W]); pos += u * W
        _check(e2, hs2, {hs2[0]: orc}, S)


def test_refusals(sdb):
    e = sdb.Engine(n_streams=1, psd_size=NP, psd_window="hann", st_window_size=W, max_feed=W, samp_rate=1.0)
    hp = e.open_channel(0.5, 2 * np.pi * 0.05, 1.0)
    _psk(e, hp)
    hr = e.open_channel(1.5, 2 * np.pi * 0.05, 1.0)
    e.set_inspector(hr, "raw")
    hw = e.open_channel(2.5, 2 * np.pi * 0.05, 1.0)
    e.set_inspector(hw, "power")

    def refused(h, msg, **kw):
        with pytest.raises(sdb.SdbError, match=msg):
            e.set_fac(h, **kw)

    for L in (256, 1000, 1 << 20):
        refused(hp, "power of two in \\[512, 2\\^19\\]", size=L)
    refused(hr, "psk, fsk or ask", size=1024)
    refused(hw, "psk, fsk or ask", size=1024)
    for a in (-0.1, 1.5, float("nan")):
        refused(hp, "alpha", size=1024, alpha=a)
    for lags in ((10, 10), (20, 10), (0, 513)):
        refused(hp, "lag window", size=1024, lags=lags)
    refused(hp, "sigma", size=1024, sigma=float("nan"))
    refused(7, "wrong handle", size=1024)
    e.set_fac(hp, size=1024)
    e.commit()
    with pytest.raises(sdb.SdbError, match="FAC is not enabled"):
        e.read_fac(hr)
    with pytest.raises(sdb.SdbError, match="wrong handle"):
        e.read_fac(9)
    with pytest.raises(sdb.SdbError, match="already committed"):
        e.set_fac(hp, size=1024)


class _Stepper:
    """In-memory source read block by block: read call k parks until the test allows it, so that requests sent while
    the worker is parked in call k take effect from block k + 1."""

    def __init__(self, x):
        import threading
        self.x, self.pos, self.calls, self.allowed = x, 0, 0, 0
        self.cv = threading.Condition()

    def read(self, priv, dst, maxn):
        import ctypes as C
        with self.cv:
            self.calls += 1
            self.cv.notify_all()
            self.cv.wait_for(lambda: self.calls <= self.allowed, timeout=60)
        take = min(maxn, len(self.x) - self.pos)
        if take > 0:
            C.memmove(dst, self.x.ctypes.data + 8 * self.pos, 8 * take)
            self.pos += take
        return take

    def park(self, k):
        with self.cv:
            assert self.cv.wait_for(lambda: self.calls >= k, timeout=60)

    def release(self, k):
        with self.cv:
            self.allowed = k
            self.cv.notify_all()


def test_analyzer_fac_messages_follow_the_samples(sdb):
    """Through an analyzer session: every block that completes a FAC block posts, after its SAMPLES, one FAC message
    whose fac and status equal the FAC of those very symbols (the oracle fed the SAMPLES batches, which the engine
    tests above hold the engine to), across a re-plan that opens another inspector mid-stream; each request is
    acknowledged, and refused on a raw inspector (WRONG_KIND) or with a size the engine refuses (WRONG_OBJECT)."""
    import ctypes as C
    from sigdigger_b200.analyzer import Analyzer
    N, fs, blocks = 8192, 1.0e6, 14
    per_block = 4 * N
    x = _signal(1, blocks * per_block, 5)[0]
    src = _Stepper(x)
    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=1.0, read=src.read, read_size=per_block)
    assert a.read(5000)[0] == "SOURCE_INFO"
    src.park(1)
    a.open("psk", 0.1 * fs, fs / 16, req_id=1)                       # handle 0
    a.open("fsk", -0.2 * fs, fs / 16, req_id=2)                      # handle 1
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
    a.set_fac(0, size=1024, alpha=0.5, lags=(2, 512), sigma=2.0, req_id=40)
    a.set_fac(1, size=2048, req_id=41)
    a.set_fac(2, size=1024, req_id=42)
    a.set_fac(0, size=1000, req_id=43)
    src.release(6)
    src.park(7)
    a.open("ask", 0.4 * fs, fs / 16, req_id=4)                       # a re-plan mid-stream: the FAC state carries
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
    assert replies[40]["kind"] == "FAC" and replies[41]["kind"] == "FAC"
    assert replies[42]["kind"] == "WRONG_KIND" and replies[43]["kind"] == "WRONG_OBJECT"
    oracles = {10: fac_oracle.Fac(1024, 0.5, (2, 512), 2.0), 11: fac_oracle.Fac(2048)}
    expect, posted = {}, {10: 0, 11: 0}
    for name, m in msgs:
        if name == "SAMPLES" and m["inspector_id"] in oracles:
            iid = m["inspector_id"]
            assert expect.get(iid) is None, "a block's FAC message is missing"
            st = oracles[iid].feed(m["samples"])
            expect[iid] = st if st.blocks else None
        elif name == "INSPECTOR" and m["kind"] == "FAC" and m["spectrum"] is not None:
            iid = m["inspector_id"]
            st = expect.pop(iid, None)
            assert st is not None, "a FAC message without a completed block before it"
            f = m["fac"]
            b32 = lambda v: int(np.float32(v).view(np.uint32))     # noqa: E731
            got = (f["blocks"], f["peak_lag"], b32(f["max"]), b32(f["min"]), b32(f["sigmas"]), f["marker"])
            assert got == st.key(), (iid, got, st.key())
            assert np.array_equal(_bits(m["spectrum"]), _bits(oracles[iid].fac))
            posted[iid] += 1
    assert all(v is None for v in expect.values())
    assert posted[10] >= 4 and posted[11] >= 2, posted
