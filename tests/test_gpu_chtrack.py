"""Channel tracking across detector updates (oracle/SPEC_KT.md): the engine's k_chtrack against the oracle's
sdo_chtrack_update, bit for bit (ranges, S0, ids, age, present, misses, dropped), fed with the oracle's own SPEC K
lists of the engine's PSD; on both detector paths, the PSD stream, a u8 feed under DC removal and a dB-averaged PSD;
the beta = 1 / hold = 0 property, launch counts, refusals, migration and the analyzer's CHANNEL messages."""
import numpy as np
import pytest

import chdet_stmt as cs
import chtrack_oracle as co
import chtrack_stmt as kt

pytestmark = pytest.mark.gpu


def _tones(N, frames, S, tones, seed, sigma=0.01):
    """[S, frames * N] complex64: per frame, noise plus tones [(bin, amplitude)] exactly on bins (periodic per frame)."""
    rng = np.random.default_rng(seed)
    out = np.empty((S, frames, N), np.complex64)
    for s in range(S):
        for f in range(frames):
            X = np.zeros(N, np.complex128)
            for b, amp in tones(s, f):
                X[int(b) % N] += amp * N * np.exp(2j * np.pi * rng.random())
            out[s, f] = np.fft.ifft(X) + (rng.standard_normal(N) + 1j * rng.standard_normal(N)) * (sigma / np.sqrt(2))
    return out.reshape(S, frames * N)


def _bursty(N, frames, feeds, S, seed):
    """Per feed: a steady carrier, a bursty one (off every third feed), one that drifts by a bin, a pair that merges
    into one run at high level and splits at low level, and a weak one near the threshold; levels vary per feed."""
    w = max(1, N // 512)

    def tones(s, f):
        g = f // frames
        out = [(N // 8 + s, 0.02 * (1 + 0.1 * (g % 3)))]
        if g % 3 != 1:
            out.append((-N // 4, 0.05 * (1 + g % 2)))
        out.append((N // 3 + g % 2, 0.01))
        amp = 0.08 if g % 2 else 0.004
        out += [(-N // 3, amp), (-N // 3 + 3 * w + 4, amp)]
        out.append((3 * N // 8, 0.0012 * (1 + 0.5 * ((g + s) % 2))))
        return out
    return _tones(N, frames * feeds, S, tones, seed)


def _check(e, N, S, trackers, dets, where):
    """After a feed: feed the oracle's K list of the engine's PSD to the oracle tracker and compare every stream."""
    psd = e.read_psd()
    for s in range(S):
        ref, _ = dets[s].feed(psd[s])
        trackers[s].update([(a, b, np.float32(s0)) for a, b, s0, _n0, _snr in ref])
        got, tot, dropped = e.read_tracked_channels(s, center_freq=1.0e6)
        keys = [(g.bin_lo, g.bin_hi, int(np.float32(g.S0).view(np.uint32)), g.id, g.age, g.present, g.misses)
                for g in got]
        assert keys == trackers[s].keys(), where + (s,)
        assert tot == len(got) and dropped == trackers[s].dropped, where + (s,)
        n0 = np.float32(dets[s].d.n0)
        for g in got:
            assert np.float32(g.N0).view(np.uint32) == n0.view(np.uint32)
            assert np.float32(g.snr).view(np.uint32) == np.float32(np.float32(g.S0) / n0).view(np.uint32)
            assert (g.f_lo, g.f_hi, g.fc, g.bw) == cs.frequencies(g.bin_lo, g.bin_hi, N, e.samp_rate, 1.0e6)


def _run(sdb, oracle, kw, prm, beta, hold, feeds, S, N, setup=None):
    e = sdb.Engine(**kw)
    if setup:
        setup(e)
    e.set_channel_detector(beta=beta, **prm)
    e.set_channel_tracking(hold)
    e.commit()
    dets = [oracle.ChannelDetector(N, prm["alpha"], prm["gamma"], prm["snr"], prm["min_bins"]) for _ in range(S)]
    trackers = [co.Tracker(beta, hold) for _ in range(S)]
    try:
        for i, x in enumerate(feeds):
            e.feed(x)
            _check(e, N, S, trackers, dets, (N, beta, hold, i))
    finally:
        for d in dets:
            d.close()
    return e, trackers


PRM = dict(alpha=1.0, gamma=0.5, snr=40.0, min_bins=2)      # alpha = 1: a carrier that stops leaves the list


@pytest.mark.parametrize("N", [512, 16384, 65536, 131072])
@pytest.mark.parametrize("beta,hold", [(0.5, 1), (0.01, 7), (1.0, 0)])
def test_tracks_bit_identical_to_oracle(sdb, oracle, N, beta, hold):
    """Both detector paths (k_chdet_avg + k_chdet_find at 512 and 131072, k_chdet_fused at 16384 and 65536), 3
    streams, 8 feeds of a bursty scene: every track of every stream equals the oracle's after every feed."""
    S, frames, nf = 3, 2, 8
    x = _bursty(N, frames, nf, S, seed=N % 97)
    kw = dict(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=N * frames, samp_rate=2.0e6)
    e, trackers = _run(sdb, oracle, kw, PRM, beta, hold, [x[:, i * N * frames:(i + 1) * N * frames] for i in range(nf)],
                       S, N)
    # the scene reaches what it is for: several tracks, some in hold or re-opened when hold allows
    assert all(t.next_id > 3 for t in trackers)
    if hold:
        assert any(k[6] > 0 for t in trackers for k in t.keys())
    e.close()


def test_tracks_on_the_psd_stream_u8_dc_and_db_average(sdb, oracle):
    """The detector on the engine's second stream (open channels at 16384 points), a u8 feed with DC removal, and
    SHIFT_DB confined to the frame-averaged output: tracks bit-identical to the oracle."""
    N, S, frames, nf = 16384, 3, 2, 6
    x = _bursty(N, frames, nf, S, seed=11)
    feeds = [x[:, i * N * frames:(i + 1) * N * frames] for i in range(nf)]

    def chans(e):
        for f0 in (0.11, 1 - 0.27):
            e.open_channel(2 * np.pi * f0, 2 * np.pi * 0.02)
    kw = dict(n_streams=S, psd_size=N, st_window_size=N, max_feed=N * frames, samp_rate=2.0e6)
    _run(sdb, oracle, kw, PRM, 0.25, 2, feeds, S, N, setup=chans)[0].close()
    raw = [np.stack([np.clip(np.rint(f.real * 400 + 140), 0, 255), np.clip(np.rint(f.imag * 400 + 121), 0, 255)],
                    axis=-1).astype(np.uint8) for f in feeds]
    kw = dict(n_streams=S, psd_size=4096, max_feed=4096 * 8, samp_rate=2.0e6, input_format="u8",
              flags=sdb.FLAG_DC_REMOVE)
    _run(sdb, oracle, kw, dict(PRM, snr=8.0), 0.25, 2, [r[:, :4096 * 8] for r in raw], S, 4096)[0].close()
    kw = dict(n_streams=S, psd_size=N, max_feed=N * frames, samp_rate=2.0e6, psd_average=2,
              flags=sdb.FLAG_PSD_SHIFT_DB)
    _run(sdb, oracle, kw, PRM, 0.5, 1, feeds, S, N)[0].close()


def test_cap_and_dropped(sdb, oracle):
    """260 carriers, then 260 others while the first 256 are in hold: the table stays at 256, the new detections are
    counted in dropped, and the first return to their ids."""
    N, S = 16384, 2
    first = [(-8000 + 30 * i, 0.01) for i in range(260)]
    second = [(-7985 + 30 * i, 0.01) for i in range(260)]
    plan = [first, second, second, first, []]
    x = _tones(N, len(plan), S, lambda s, f: plan[f], seed=3)
    kw = dict(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=N, samp_rate=2.0e6)
    prm = dict(alpha=1.0, gamma=1.0, snr=40.0, min_bins=2)
    e, trackers = _run(sdb, oracle, kw, prm, 0.5, 2, [x[:, i * N:(i + 1) * N] for i in range(len(plan))], S, N)
    got, tot, dropped = e.read_tracked_channels(0)
    assert tot == len(got) == 256 and dropped >= 256
    assert all(t.next_id == 257 for t in trackers)
    assert e.read_all_tracked_channels([0.0, 1.0e6])[1][1] == trackers[1].dropped
    e.close()


def test_beta1_hold0_is_the_detector_list(sdb):
    """beta = 1, hold = 0: the tracked ranges are sdb_engine_read_channels' list, and S0 its peaks where the
    difference of KT.4 is exact (Sterbenz), feed after feed, on both detector paths."""
    for N in (512, 16384):
        S, frames, nf = 2, 2, 6
        x = _bursty(N, frames, nf, S, seed=5)
        e = sdb.Engine(n_streams=S, psd_size=N, max_feed=N * frames, samp_rate=2.0e6)
        e.set_channel_detector(beta=1.0, **PRM)
        e.set_channel_tracking(0)
        e.commit()
        prev = [dict() for _ in range(S)]
        for i in range(nf):
            e.feed(x[:, i * N * frames:(i + 1) * N * frames])
            for s in range(S):
                det, tot = e.read_channels(s)
                got, gtot, dropped = e.read_tracked_channels(s)
                assert [(g.bin_lo, g.bin_hi) for g in got] == [(d.bin_lo, d.bin_hi) for d in det]
                assert gtot == len(det) and dropped == 0
                for g, d in zip(got, det):
                    old = prev[s].get(g.id)
                    s0d = np.float32(d.S0)
                    want = s0d if old is None else np.float32(old + np.float32(s0d - old))
                    assert np.float32(g.S0) == want
                    if old is None or old / 2 <= s0d <= 2 * old:
                        assert np.float32(g.S0).view(np.uint32) == s0d.view(np.uint32)
                    assert g.N0 == d.N0 and g.misses == 0
                prev[s] = {g.id: np.float32(g.S0) for g in got}
        e.close()


def test_launches_and_timing_family(sdb):
    """Tracking off: the launches of the parent (no chan_track span); on: one k_chtrack per feed, on both paths."""
    for N in (512, 16384):
        x = _bursty(N, 2, 3, 2, seed=1)
        counts = []
        for track in (False, True):
            e = sdb.Engine(n_streams=2, psd_size=N, max_feed=2 * N, samp_rate=2.0e6)
            e.set_channel_detector(beta=0.5, **PRM)
            if track:
                e.set_channel_tracking(3)
            e.commit()
            e.timing(True)
            for i in range(3):
                e.feed(x[:, i * 2 * N:(i + 1) * 2 * N])
            e.sync()
            counts.append(e.launches)
            assert e.kernel_time("chan_track")[1] == (3 if track else 0)
            e.close()
        assert counts[1] - counts[0] == 3


def test_refusals(sdb):
    SdbError = sdb.SdbError
    e = sdb.Engine(n_streams=1, psd_size=1024, max_feed=1024)
    with pytest.raises(SdbError, match="needs the channel detector"):
        e.set_channel_tracking(1)
    e.set_channel_detector(beta=0.5, **PRM)
    with pytest.raises(SdbError, match="at most 65535"):
        e.set_channel_tracking(65536)
    e.set_channel_tracking(65535)
    e.commit()
    with pytest.raises(SdbError, match="already committed"):
        e.set_channel_tracking(1)
    e.close()
    for beta in (0.0, -0.5, 1.5, float("nan")):
        e = sdb.Engine(n_streams=1, psd_size=1024, max_feed=1024)
        e.set_channel_detector(beta=beta, **PRM)
        e.set_channel_tracking(1)
        with pytest.raises(SdbError, match=r"beta in \(0, 1\]"):
            e.commit()
        e.close()
    e = sdb.Engine(n_streams=1, psd_size=1024, max_feed=1024)
    e.set_channel_detector(beta=0.0, **PRM)           # beta is not checked while tracking is off
    e.commit()
    with pytest.raises(SdbError, match="channel tracking not enabled"):
        e.read_tracked_channels(0)
    with pytest.raises(SdbError, match="channel tracking not enabled"):
        e.read_all_tracked_channels([0.0])
    e.close()


def test_migration_restarts_tracks(sdb, oracle):
    """sdb_engine_migrate does not carry the detector, so the tracks restart with it: ids begin again at 1."""
    N, S, frames = 4096, 2, 2
    x = _bursty(N, frames, 6, S, seed=9)
    kw = dict(n_streams=S, psd_size=N, max_feed=N * frames, samp_rate=2.0e6)
    a, _ = _run(sdb, oracle, kw, PRM, 0.5, 2, [x[:, i * N * frames:(i + 1) * N * frames] for i in range(3)], S, N)
    assert max(g.id for g in a.read_tracked_channels(0)[0]) > 3
    b = sdb.Engine(**kw)
    b.set_channel_detector(beta=0.5, **PRM)
    b.set_channel_tracking(2)
    b.commit()
    assert b._L.sdb_engine_migrate(b._h, a._h) == 0
    dets = [oracle.ChannelDetector(N, PRM["alpha"], PRM["gamma"], PRM["snr"], PRM["min_bins"]) for _ in range(S)]
    trackers = [co.Tracker(0.5, 2) for _ in range(S)]
    for i in range(3, 6):
        b.feed(x[:, i * N * frames:(i + 1) * N * frames])
        _check(b, N, S, trackers, dets, ("migrated", i))
    got = b.read_tracked_channels(0)[0]
    assert sorted(g.id for g in got)[0] == 1 and max(g.age for g in got) <= 3
    for d in dets:
        d.close()
    a.close()
    b.close()


def _analyzer_channels(sdb, x, fs, N, per_block, hold_int, beta):
    from sigdigger_b200.analyzer import Analyzer
    a = Analyzer(fs, window_size=N, window="blackmann_harris", psd_update_int=1.0, data=x, read_size=per_block,
                 channel_update_int=per_block / fs, alpha=1.0, beta=beta, gamma=0.5, snr=40.0, freq=433e6,
                 channel_hold_int=hold_int)
    lists = []
    while True:
        name, m = a.read(20000)
        assert name != "TIMEOUT"
        if name == "CHANNEL":
            lists.append(m["channels"])
        elif name in ("EOS", "READ_ERROR", "HALT"):
            break
    a.close()
    assert name == "EOS"
    return lists


def test_analyzer_channel_messages_keep_bursty_carriers(sdb):
    """channel_hold_int: a carrier that drops out for one block stays one entry with the same id through the gap
    (hold = 2 blocks), age and present grow, and S0 is the statement's beta-smoothed level of the untracked lists;
    channel_hold_int = 0 posts the untracked lists unchanged."""
    from sigdigger_b200.analyzer import Analyzer
    N, fs, blocks = 8192, 1.0e6, 8
    per_block = 4 * N
    x = _bursty(N, 4, blocks, 1, seed=21)[0]
    plain = _analyzer_channels(sdb, x, fs, N, per_block, 0.0, 0.25)
    tracked = _analyzer_channels(sdb, x, fs, N, per_block, 2 * per_block / fs, 0.25)
    assert len(plain) == len(tracked) == blocks
    assert all("id" not in c for lst in plain for c in lst)
    t = kt.Tracker(0.25, 2)
    df = fs / N
    for lst, got in zip(plain, tracked):
        dets = [(int(round((c["f_lo"] - 433e6) / df + N / 2)), int(round((c["f_hi"] - 433e6) / df + N / 2)),
                 np.float32(c["S0"])) for c in lst]
        t.update(dets)
        assert [(c["id"], c["age"], c["present"], c["misses"]) for c in got] == \
            [(k.id, k.age, k.present, k.misses) for k in t.tracks]
        assert [np.float32(c["S0"]) for c in got] == [k.S0 for k in t.tracks]
    # the bursty carrier (off in blocks 1, 4, 7) is one track throughout, present in 5 of 8 updates
    bursty = [c for c in tracked[-1] if abs(c["fc"] - (433e6 - fs / 4)) < 4 * df]
    assert len(bursty) == 1
    assert bursty[0]["age"] == blocks and bursty[0]["present"] == 5 and bursty[0]["misses"] == 1
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(sdb.SdbError, match="channel_hold_int"):
            a = Analyzer(fs, window_size=N, data=x, read_size=per_block, channel_update_int=0.01, channel_hold_int=bad)
            a.close()
