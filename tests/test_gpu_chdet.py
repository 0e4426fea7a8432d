"""Channel detector (SPEC K, SURVEY.md 8(f) rank 3): CUDA path through the C-ABI against the oracle, bit-exact
(bin ranges, levels, noise floor), engine-integrated on the engine's own PSD and stand-alone on arbitrary spectra."""
import numpy as np
import pytest

import chdet_stmt as cs
from sigdigger_b200 import synth

pytestmark = pytest.mark.gpu


def _scene(S, N, frames, seed):
    """S streams: noise + a few carriers of different widths."""
    n = N * frames
    rng = np.random.default_rng(seed)
    xs = []
    truth = []
    for s in range(S):
        x = synth.awgn(n, 0.01, rng)
        tr = []
        for f, sps, amp in ((0.11 + 0.01 * s, 16.0, 0.3), (-0.27, 64.0, 0.2), (0.40, 8.0, 0.25)):
            sig, _ = synth.psk_signal(n, sps, order=4, seed=seed + 7 * s + int(sps))
            x = x + amp * synth.mix(sig, f, 0.1)
            tr.append((f, 1.0 / sps))
        xs.append(x)
        truth.append(tr)
    return np.stack(xs).astype(np.complex64), truth


def _same(got, ref):
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        assert (g.bin_lo, g.bin_hi) == (r[0], r[1])
        for a, b in ((g.S0, r[2]), (g.N0, r[3]), (g.snr, r[4])):
            assert np.float32(a).view(np.uint32) == np.float32(b).view(np.uint32)


@pytest.mark.parametrize("N", [4096, 65536])
def test_engine_channel_detector_bit_exact(sdb, oracle, N):
    S, frames, feeds = 3, 4, 3
    x, truth = _scene(S, N, frames * feeds, seed=N % 97)
    e = sdb.Engine(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=N * frames)
    kw = dict(alpha=0.25, gamma=0.5, snr=8.0, min_bins=max(2, N // 2048))
    e.set_channel_detector(beta=0.1, **kw)
    e.commit()
    dets = [oracle.ChannelDetector(N, kw["alpha"], kw["gamma"], kw["snr"], kw["min_bins"]) for _ in range(S)]
    for f in range(feeds):
        e.feed(x[:, f * N * frames:(f + 1) * N * frames])
        psd = e.read_psd()
        for s in range(S):
            ref, rtot = dets[s].feed(psd[s])
            got, tot = e.read_channels(s)
            assert tot == rtot
            _same(got, ref)
    # after averaging the three carriers are found where they were put, roughly as wide as their symbol rate
    got, _ = e.read_channels(0, center_freq=100e6)
    for f, baud in truth[0]:
        hit = [c for c in got if c.f_lo - 100e6 <= f <= c.f_hi - 100e6]
        assert len(hit) == 1, (f, [(c.f_lo, c.f_hi) for c in got])
        assert 0.7 * baud < hit[0].bw < 2.5 * baud
        assert hit[0].fc == pytest.approx(0.5 * (hit[0].f_lo + hit[0].f_hi))
        assert hit[0].snr > 8.0
    for d in dets:
        d.close()


def test_standalone_detector_edges_caps_and_noise(sdb, oracle):
    import torch
    N, S = 8192, 4
    rng = np.random.default_rng(3)
    psd = rng.exponential(1.0, (S, 2, N)).astype(np.float32)
    psd[0, :, :] += 0.0
    psd[1, :, N // 2 - 40:N // 2 + 7] += 50.0          # touches both array edges in shifted order (around index N/2)
    psd[2, :, 0:30] += 40.0
    psd[2, :, N - 25:] += 40.0                          # straddles DC in unshifted order = one run in shifted order
    psd[3, :, ::3] += 30.0                              # thousands of 1-bin runs: all rejected by min_bins
    d = sdb.ChannelDetector(N, S, alpha=0.5, gamma=1.0, snr=6.0, min_bins=3)
    dets = [oracle.ChannelDetector(N, 0.5, 1.0, 6.0, 3) for _ in range(S)]
    t = torch.from_numpy(psd).cuda()
    for rep in range(2):
        d.feed(t)
        for s in range(S):
            ref, rtot = dets[s].feed(psd[s])
            got, tot = d.read(s, samp_rate=1.0)
            assert tot == rtot
            _same(got, ref)
    got, _ = d.read(2)
    assert any(c.bin_lo <= N // 2 - 25 and c.bin_hi >= N // 2 + 30 for c in got)
    got1, _ = d.read(1)
    assert got1 and got1[0].bin_lo == 0 and got1[-1].bin_hi == N      # runs clipped at the band edges, not merged
    got3, _ = d.read(3)
    assert all(c.bin_hi - c.bin_lo >= 3 for c in got3)               # min_bins removed the 1- and 2-bin runs
    d.close()
    for o in dets:
        o.close()


def test_many_channels_cap(sdb, oracle):
    import torch
    N = 16384
    psd = np.full((1, 1, N), 1.0, np.float32)
    for i in range(400):                                 # 400 carriers of 8 bins: more than the 256-entry report cap
        psd[0, 0, 20 + 40 * i:28 + 40 * i] = 100.0
    d = sdb.ChannelDetector(N, 1, alpha=1.0, gamma=1.0, snr=4.0, min_bins=2)
    d.feed(torch.from_numpy(psd).cuda())
    got, tot = d.read(0)
    o = oracle.ChannelDetector(N, 1.0, 1.0, 4.0, 2)
    ref, rtot = o.feed(psd[0])
    assert tot == rtot == 400 and len(got) == len(ref) == 256
    _same(got, ref)
    d.close()
    o.close()


# ---- every accepted size, both kernel paths, against the oracle and the statement of SPEC K (tests/chdet_stmt.py) --
SIZES = [1 << k for k in range(4, 21)]


def _same_all(got, tot, ref, rtot, stmt, stot, where):
    """GPU list == oracle list == statement list, bit for bit, with equal totals; frequencies as K.4 in binary64"""
    assert tot == rtot == stot, where
    _same(got, ref)
    assert [(g.bin_lo, g.bin_hi) + tuple(int(np.float32(v).view(np.uint32)) for v in (g.S0, g.N0, g.snr))
            for g in got] == [c.key() for c in stmt], where


def _check_freqs(got, N, samp_rate, center):
    for g in got:
        assert (g.f_lo, g.f_hi, g.fc, g.bw) == cs.frequencies(g.bin_lo, g.bin_hi, N, samp_rate, center)


@pytest.mark.parametrize("N", SIZES)
def test_standalone_detector_every_size(sdb, oracle, N):
    """Every N = 16 ... 2^20 with 3 streams (k_chdet_avg + k_chdet_find below 2048 and above 65536, k_chdet_fused
    between), over every scene of tests/chdet_stmt.py, feed after feed: a zero-frame feed through the C-ABI changes
    nothing."""
    import ctypes as C
    import torch
    S = 3
    L = sdb.load_library()
    dummy = torch.zeros(1, device="cuda")
    for name, prm, feeds in cs.scenes(N, streams=S, seed=1):
        if N > 1 << 16 and name.startswith("noise_carriers") and prm["alpha"] != prm["gamma"]:
            continue                                       # the alpha / gamma grid's diagonal above 65536 bins
        d = sdb.ChannelDetector(N, S, **prm)
        dets = [oracle.ChannelDetector(N, prm["alpha"], prm["gamma"], prm["snr"], prm["min_bins"]) for _ in range(S)]
        stmts = [cs.Detector(N, **prm) for _ in range(S)]
        try:
            for i, f in enumerate(feeds):
                where = (N, name, i)
                if f.shape[1] == 0:
                    before = [d.read(s) for s in range(S)]
                    assert L.sdb_chdet_feed_device(d._h, C.c_void_p(dummy.data_ptr()), 0, N) == 0
                    for s in range(S):
                        got, tot = d.read(s)
                        assert tot == before[s][1] and [(g.bin_lo, g.bin_hi, g.S0, g.N0) for g in got] == \
                            [(g.bin_lo, g.bin_hi, g.S0, g.N0) for g in before[s][0]], where
                        stmts[s].feed(f[s])
                        assert dets[s].feed(f[s])[0] == []
                    continue
                d.feed(torch.from_numpy(f).cuda())
                for s in range(S):
                    ref, rtot = dets[s].feed(f[s])
                    stmt, stot = stmts[s].feed(f[s])
                    got, tot = d.read(s, samp_rate=2.0e6, center_freq=433.0e6)
                    _same_all(got, tot, ref, rtot, stmt, stot, where + (s,))
                    _check_freqs(got, N, 2.0e6, 433.0e6)
        finally:
            d.close()
            for o in dets:
                o.close()


def _engine_vs_oracle(oracle, e, N, S, feeds, prm):
    """Feeds one chunk at a time; after each, the engine's lists == oracle == statement on the engine's own PSD."""
    dets = [cs.Detector(N, **prm) for _ in range(S)]
    odets = [oracle.ChannelDetector(N, prm["alpha"], prm["gamma"], prm["snr"], prm["min_bins"]) for _ in range(S)]
    try:
        for i, x in enumerate(feeds):
            e.feed(x)
            psd = e.read_psd()
            for s in range(S):
                ref, rtot = odets[s].feed(psd[s])
                stmt, stot = dets[s].feed(psd[s])
                got, tot = e.read_channels(s, center_freq=1.0e6)
                _same_all(got, tot, ref, rtot, stmt, stot, (N, i, s))
                _check_freqs(got, N, e.samp_rate, 1.0e6)
    finally:
        for o in odets:
            o.close()


def _detector_launches(sdb, kw, prm, x):
    """launches the detector adds to one feed"""
    counts = []
    for with_det in (False, True):
        e = sdb.Engine(**kw)
        if with_det:
            e.set_channel_detector(beta=0.1, **prm)
        e.commit()
        e.feed(x)
        counts.append(e.launches)
        e.close()
    return counts[1] - counts[0]


@pytest.mark.parametrize("N", [512, 16384, 131072])
def test_engine_detector_both_paths(sdb, oracle, N):
    """The engine's detector at a two-kernel size below (512) and above (131072) the fused range and in it (16384):
    lists bit-identical to the oracle and the statement on the engine's PSD, three feeds, 3 streams; the launch count
    shows which path ran (2 launches: k_chdet_avg + k_chdet_find, 1: k_chdet_fused)."""
    S, frames = 3, 3
    x, _ = _scene(S, N, frames * 3, seed=N % 89)
    prm = dict(alpha=0.25, gamma=0.5, snr=6.0, min_bins=max(1, N // 4096))
    kw = dict(n_streams=S, psd_size=N, psd_window="blackmann_harris", max_feed=N * frames, samp_rate=2.0e6)
    assert _detector_launches(sdb, kw, prm, x[:, :N * frames]) == (1 if 2048 <= N <= 65536 else 2)
    e = sdb.Engine(**kw)
    e.set_channel_detector(beta=0.1, **prm)
    e.commit()
    _engine_vs_oracle(oracle, e, N, S, [x[:, f * N * frames:(f + 1) * N * frames] for f in range(3)], prm)
    e.close()


def test_engine_detector_on_the_psd_stream(sdb, oracle):
    """16384-point PSD with a 16384-point channeliser and open channels: the stream-group schedule runs the PSD and
    the detector on the engine's second stream while the channeliser runs on the main one.  Lists bit-identical to
    the oracle and the statement, feed after feed."""
    N, S, frames = 16384, 3, 4
    x, _ = _scene(S, N, frames * 3, seed=5)
    prm = dict(alpha=0.5, gamma=0.25, snr=6.0, min_bins=4)
    e = sdb.Engine(n_streams=S, psd_size=N, st_window_size=N, max_feed=N * frames, samp_rate=2.0e6)
    for f0 in (0.11, 1 - 0.27):
        e.open_channel(2 * np.pi * f0, 2 * np.pi * 0.02)
    e.set_channel_detector(beta=0.1, **prm)
    e.commit()
    _engine_vs_oracle(oracle, e, N, S, [x[:, f * N * frames:(f + 1) * N * frames] for f in range(3)], prm)
    assert e.read_channels(0)[1] >= 3                       # the three carriers of the scene are found
    e.close()


def test_engine_detector_u8_dc_remove(sdb, oracle):
    """A u8 feed with DC removal: the detector sees the corrected PSD the engine emits."""
    N, S, frames = 4096, 3, 4
    x, _ = _scene(S, N, frames * 3, seed=17)
    raw = np.stack([np.clip(np.rint(x.real * 100 + 140), 0, 255), np.clip(np.rint(x.imag * 100 + 121), 0, 255)],
                   axis=-1).astype(np.uint8)
    prm = dict(alpha=0.25, gamma=0.5, snr=6.0, min_bins=2)
    e = sdb.Engine(n_streams=S, psd_size=N, max_feed=N * frames, samp_rate=2.0e6, input_format="u8",
                   flags=sdb.FLAG_DC_REMOVE)
    e.set_channel_detector(beta=0.1, **prm)
    e.commit()
    _engine_vs_oracle(oracle, e, N, S, [raw[:, f * N * frames:(f + 1) * N * frames] for f in range(3)], prm)
    e.close()


def test_engine_detector_with_averaged_db_psd(sdb, oracle):
    """psd_average = 3 with SHIFT_DB: the means are emitted in dB, the per-frame PSD stays linear and is what the
    detector averages."""
    N, S, frames = 8192, 3, 4
    x, _ = _scene(S, N, frames * 3, seed=29)
    prm = dict(alpha=0.25, gamma=0.5, snr=6.0, min_bins=2)
    e = sdb.Engine(n_streams=S, psd_size=N, max_feed=N * frames, samp_rate=2.0e6, psd_average=3,
                   flags=sdb.FLAG_PSD_SHIFT_DB)
    e.set_channel_detector(beta=0.1, **prm)
    e.commit()
    _engine_vs_oracle(oracle, e, N, S, [x[:, f * N * frames:(f + 1) * N * frames] for f in range(3)], prm)
    assert np.all(e.read_psd() >= 0) and np.any(e.read_psd_average() < 0)      # linear frames, dB means
    e.close()
