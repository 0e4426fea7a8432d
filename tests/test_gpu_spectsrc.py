"""Inspector spectrum sources and baud estimators (SPEC U, SURVEY.md 8(f) rank 1): the CUDA path through the C-ABI
against the oracle on the channel samples the engine itself produced (bit-exact), over several streams and feeds."""
import numpy as np
import pytest

import spectsrc_f64 as sf
from sigdigger_b200 import synth

pytestmark = pytest.mark.gpu

KINDS = ["psd", "cyclo", "fmspect", "timediff", "abstimediff", "exp_2", "exp_4", "exp_8", "fac"]


def _capture(S, n, sps_in, seed):
    xs = []
    for s in range(S):
        sig, _ = synth.psk_signal(n, sps_in, order=4, seed=seed + s)
        rng = np.random.default_rng(seed + s)
        xs.append(0.3 * synth.mix(sig, 0.1 + 1e-4 * s, 0.2 * s) + synth.awgn(n, 1e-3, rng))
    return np.stack(xs).astype(np.complex64)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("ns", [256, 4096])
def test_spectrum_source_bit_exact(sdb, oracle, kind, ns):
    W, hops, S = 8192, 48, 3
    n = W // 2 * hops
    x = _capture(S, n, 64.0, seed=11)                     # 1/64 baud at the input rate
    e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=n)
    h = e.open_channel(2 * np.pi * 0.1, 2 * np.pi * 4 / 64.0, 1.0)   # decimation 16 -> 4 samples per symbol
    e.set_spectrum_source(h, kind, ns)
    e.commit()
    for lo, hi in ((0, n // 2), (n // 2, n)):              # two feeds: the frame is the tail of each feed's output
        e.feed(x[:, lo:hi])
        got, sizes = e.read_spectrum(h)
        for s in range(S):
            chan = e.read_channel(s, h)
            ref = oracle.spectsrc_frame(kind, ns, chan)
            if ref is None:
                assert sizes[s] == 0
                continue
            assert sizes[s] == len(ref) == (ns // 2 if kind == "fac" else ns)
            assert np.array_equal(got[s, :len(ref)].view(np.uint32), ref.view(np.uint32)), (kind, ns, s)


def test_short_feed_emits_nothing(sdb, oracle):
    W, S = 4096, 2
    n = W // 2 * 4
    x = _capture(S, n, 32.0, seed=5)
    e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=n)
    h = e.open_channel(2 * np.pi * 0.1, 2 * np.pi * 4 / 32.0, 1.0)
    e.set_spectrum_source(h, "psd", 4096)
    e.set_estimator(h, "baud-nonlinear")
    e.commit()
    e.feed(x)
    _, sizes = e.read_spectrum(h)
    vals, valid = e.read_estimate(h, "baud-nonlinear")
    assert not sizes.any() and not valid.any()


@pytest.mark.parametrize("ns", [1024, 4096])
def test_baud_estimators_bit_exact_and_right(sdb, oracle, ns):
    W, hops, S = 8192, 24, 4
    n = W // 2 * hops
    x = _capture(S, n, 64.0, seed=23)
    e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=n)
    h = e.open_channel(2 * np.pi * 0.1, 2 * np.pi * 8 / 64.0, 1.0)   # decimation 8 -> 8 samples per symbol
    e.set_spectrum_source(h, "abstimediff", ns)
    e.set_estimator(h, "baud-fac")
    e.set_estimator(h, "baud-nonlinear")
    e.commit()
    e.feed(x)
    fs_ch = e.channel_rate(h)
    true_baud = e.samp_rate / 64.0
    for est in ("baud-fac", "baud-nonlinear"):
        vals, valid = e.read_estimate(h, est)
        for s in range(S):
            ref = oracle.estimate_baud(est, ns, fs_ch, e.read_channel(s, h))
            assert (ref is not None) == bool(valid[s])
            assert ref is not None
            assert np.float32(ref).view(np.uint32) == vals[s].view(np.uint32), (est, s, ref, vals[s])
            # baud-fac resolves whole lags only (8 +- 1 samples per symbol here); the spectral line is sharp
            tol = 0.15 if est == "baud-fac" else 0.02
            assert abs(vals[s] - true_baud) / true_baud < tol, (est, vals[s], true_baud)


def test_registry_names_and_errors(sdb):
    L = sdb.load_library()
    assert [L.sdb_spectsrc_name(i).decode() for i in range(10)] == [
        "none", "psd", "cyclo", "fmspect", "timediff", "abstimediff", "exp_2", "exp_4", "exp_8", "fac"]
    assert [L.sdb_estimator_name(i).decode() for i in range(2)] == ["baud-fac", "baud-nonlinear"]
    assert L.sdb_spectsrc_name(10) is None
    e = sdb.Engine(n_streams=1, psd_size=0, st_window_size=4096, max_feed=8192)
    h = e.open_channel(1.0, 0.2, 1.0)
    assert L.sdb_engine_set_spectrum_source(e._h, h, 1, 1000) == -1      # not a power of two
    assert L.sdb_engine_set_spectrum_source(e._h, h, 42, 1024) == -1
    assert L.sdb_engine_set_spectrum_source(e._h, h + 1, 1, 1024) == -1   # wrong handle
    assert L.sdb_engine_set_estimator(e._h, h, 7, 1) == -1
    e.commit()
    assert L.sdb_engine_set_spectrum_source(e._h, h, 1, 1024) == -1      # after commit


# ---- every size and kind, many channels in one launch, the U.1 boundary, zeros; against the oracle and the float64
# ---- statement of SPEC U (tests/spectsrc_f64.py)
def _within_statement(kind, ns, chan, got):
    err = np.abs(got.astype(np.float64) - sf.spectrum(kind, ns, chan))
    bound = sf.spectrum_bound(kind, ns, chan)
    assert np.all(err <= bound), (kind, ns, float(np.max(err - bound)))


def _estimate_agrees(est, ns, fs, chan, val, valid):
    """value and validity equal the statement's wherever its margin clears twice the bound"""
    fn = sf.baud_fac if est == "baud-fac" else sf.baud_nonlinear
    want, margin = fn(ns, fs, chan)
    bound = sf.acf_bound(ns, chan) if est == "baud-fac" else \
        float(np.max(sf.spectrum_bound("abstimediff", ns, chan)[sf.KMIN:ns // 2]))
    if margin > 2 * bound:
        assert bool(valid) == (want is not None) and (want is None or np.float32(want) == val), (est, ns, want, val)


def _check_channel(e, oracle, h, kind, ns, ests, S):
    got, sizes = e.read_spectrum(h) if kind != "none" else (None, None)
    fs_ch = e.channel_rate(h)
    for s in range(S):
        chan = e.read_channel(s, h)
        if kind != "none":
            ref = oracle.spectsrc_frame(kind, ns, chan)
            assert sizes[s] == (0 if ref is None else len(ref)), (kind, ns, s)
            if ref is not None:
                assert np.array_equal(got[s, :len(ref)].view(np.uint32), ref.view(np.uint32)), (kind, ns, s)
                _within_statement(kind, ns, chan, got[s, :len(ref)])
        for est in ests:
            vals, valid = e.read_estimate(h, est)
            ref = oracle.estimate_baud(est, ns, fs_ch, chan)
            assert (ref is not None) == bool(valid[s]), (est, ns, s)
            if ref is not None:
                assert np.float32(ref).view(np.uint32) == vals[s].view(np.uint32), (est, ns, s)
                _estimate_agrees(est, ns, np.float32(fs_ch), chan, vals[s], valid[s])


def _multi_capture(S, n, freqs, sps_in, seed):
    xs = []
    for s in range(S):
        rng = np.random.default_rng(seed + s)
        x = synth.awgn(n, 1e-3, rng)
        for i, f in enumerate(freqs):
            sig, _ = synth.psk_signal(n, sps_in, order=4, seed=seed + 13 * s + i)
            x = x + 0.2 * synth.mix(sig, f, 0.3 * i)
        xs.append(x)
    return np.stack(xs).astype(np.complex64)


@pytest.mark.parametrize("ns", sf.SIZES)
def test_every_kind_at_every_size(sdb, oracle, ns):
    """One channel per kind, all at this Ns, 3 streams, two feeds: bit-identical to the oracle on the channel samples
    the engine produced, within the bound of the float64 statement."""
    W, hops, S = 8192, 48, 3
    n = W // 2 * hops
    freqs = [0.05 + 0.1 * i for i in range(len(KINDS))]
    x = _multi_capture(S, n, freqs, 64.0, seed=ns)
    e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=n)
    hs = []
    for kind, f in zip(KINDS, freqs):
        h = e.open_channel(2 * np.pi * f, 2 * np.pi * 4 / 64.0, 1.0)
        e.set_spectrum_source(h, kind, ns)
        hs.append(h)
    e.commit()
    for lo, hi in ((0, n // 2), (n // 2, n)):
        e.feed(x[:, lo:hi])
        for h, kind in zip(hs, KINDS):
            _check_channel(e, oracle, h, kind, ns, (), S)


def test_many_channels_in_one_launch(sdb, oracle):
    """Channels of different sizes, kinds and Ns in one engine (one k_spectsrc launch sized for the largest): a
    64-point source beside a 4096-point one, a precise channel, an estimator-only channel at the default Ns of 1024,
    and a channel with nothing.  Every spectrum and estimate is the oracle's on that channel's own samples."""
    W, hops, S = 8192, 48, 3
    n = W // 2 * hops
    plan = [  # (f0, bw in cycles per sample, precise, kind, ns, estimators)
        (0.05, 1 / 256.0, False, "psd", 64, ()),
        (0.15, 1 / 8.0, False, "cyclo", 4096, ("baud-nonlinear",)),
        (0.40, 1 / 32.0, True, "fac", 256, ()),
        (0.55, 4 / 64.0, False, "none", 1024, ("baud-fac", "baud-nonlinear")),
        (0.70, 1 / 16.0, False, "none", None, ()),
        (0.85, 1 / 64.0, False, "exp_4", 128, ("baud-fac",)),
    ]
    x = _multi_capture(S, n, [p[0] for p in plan], 64.0, seed=77)
    L = sdb.load_library()
    e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=n)
    hs = []
    for f0, bw, precise, kind, ns, ests in plan:
        h = e.open_channel(2 * np.pi * f0, 2 * np.pi * bw, 1.0, precise=precise)
        if kind != "none":
            e.set_spectrum_source(h, kind, ns)
        for est in ests:
            e.set_estimator(h, est)
        hs.append(h)
    assert len({e.channel_info(h).size for h in hs}) >= 4
    e.commit()
    for lo, hi in ((0, n // 2), (n // 2, n)):
        e.feed(x[:, lo:hi])
        for h, (f0, bw, precise, kind, ns, ests) in zip(hs, plan):
            if kind == "none":                               # no spectrum source: nothing to read
                buf, sizes = np.zeros((S, 4096), np.float32), np.zeros(S, np.uint32)
                assert L.sdb_engine_read_spectrum(e._h, h, buf.ctypes.data, sizes.ctypes.data) == -1
            if ns is None:
                continue
            _check_channel(e, oracle, h, kind, ns, ests, S)
    e.close()


@pytest.mark.parametrize("ns", [64, 1024])
def test_u1_boundary_geometry(sdb, oracle, ns):
    """4-bin channels (2 samples per hop): a first feed of ns / 2 channelised hops gives exactly Ns channel samples
    and emits nothing (sizes 0, estimators invalid); one hop more gives Ns + 2, the smallest count this geometry
    reaches that emits (the CPU tests cover Ns + 1 itself)."""
    W, S = 256, 3
    for n_ch in (ns, ns + 2):
        n = (W // 2) * (n_ch // 2 + 1)                       # the first feed's first hop only primes the history
        x = _capture(S, n, 8.0, seed=n_ch)
        e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=n)
        h = e.open_channel(2 * np.pi * 0.1, 2 * np.pi * 2 / W, 1.0)
        assert e.channel_info(h).size == 4
        e.set_spectrum_source(h, "timediff", ns)
        e.set_estimator(h, "baud-fac")
        e.set_estimator(h, "baud-nonlinear")
        e.commit()
        e.feed(x)
        assert len(e.read_channel(0, h)) == n_ch
        _, sizes = e.read_spectrum(h)
        _, valid = e.read_estimate(h, "baud-fac")
        _, valid2 = e.read_estimate(h, "baud-nonlinear")
        if n_ch == ns:
            assert not sizes.any() and not valid.any() and not valid2.any()
        else:
            assert np.all(sizes == ns)
        _check_channel(e, oracle, h, "timediff", ns, ("baud-fac", "baud-nonlinear"), S)
        e.close()


def test_all_zero_input(sdb, oracle):
    """Zeros in: every kind's spectrum is exactly 0 and both estimators are invalid."""
    W, hops, S = 4096, 16, 3
    n = W // 2 * hops
    e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=n)
    hs = []
    for i, kind in enumerate(KINDS):
        h = e.open_channel(2 * np.pi * (0.05 + 0.1 * i), 2 * np.pi / 16.0, 1.0)
        e.set_spectrum_source(h, kind, 256)
        e.set_estimator(h, "baud-fac")
        e.set_estimator(h, "baud-nonlinear")
        hs.append(h)
    e.commit()
    e.feed(np.zeros((S, n), np.complex64))
    for h, kind in zip(hs, KINDS):
        got, sizes = e.read_spectrum(h)
        assert np.all(sizes == (128 if kind == "fac" else 256)) and not got.any(), kind
        for est in ("baud-fac", "baud-nonlinear"):
            assert not e.read_estimate(h, est)[1].any()
        _check_channel(e, oracle, h, kind, 256, ("baud-fac", "baud-nonlinear"), S)
    e.close()


@pytest.mark.parametrize("ns", [64, 256, 4096])
def test_estimators_known_baud(sdb, oracle, ns):
    """Both estimators at Ns = 64, 256, 4096 on QPSK at 8 channel samples per symbol: bit-identical to the oracle and
    equal to the statement where its margin is clear (how close they come to the baud is test_baud_estimators_bit_
    exact_and_right's business: 8 symbols in a 64-point frame say little about it)."""
    W, hops, S = 8192, 48, 3
    n = W // 2 * hops
    x = _capture(S, n, 64.0, seed=ns + 1)
    e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=n)
    h = e.open_channel(2 * np.pi * 0.1, 2 * np.pi * 8 / 64.0, 1.0)   # decimation 8 -> 8 samples per symbol
    e.set_spectrum_source(h, "abstimediff", ns)
    e.set_estimator(h, "baud-fac")
    e.set_estimator(h, "baud-nonlinear")
    e.commit()
    e.feed(x)
    _check_channel(e, oracle, h, "abstimediff", ns, ("baud-fac", "baud-nonlinear"), S)
    assert e.read_estimate(h, "baud-nonlinear")[1].all()
    e.close()
