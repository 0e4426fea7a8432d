"""-m gpu: the frame-group stages of the main PSD through the engine and the analyzer: the frame-averaged PSD (SPEC A,
oracle/SPEC_A.md) and the peak detectors (SPEC PK, oracle/SPEC_PK.md).

The statement of A.2 is `group_means` below: a float32 loop over frames, vectorised over bins, that adds each frame in
order to the running sum and divides once per group (no np.sum, which adds pairwise).  The statement of PK.2 is
tests/psd_peak_stmt.py.  Every comparison applies a statement to the same engine's per-frame linear PSD, so it is bit
for bit (NaN-aware where PK.2 allows a NaN)."""
import ctypes as C

import numpy as np
import pytest
import torch

from psd_peak_stmt import group_peaks, same
from sigdigger_b200 import synth
from test_gpu_analyzer import Gate

pytestmark = pytest.mark.gpu

# the engine field of each stage, which is also the name of its timing family
FIELD = {"mean": "psd_average", "peak": "psd_peak"}


def group_means(psd, A, acc=None, cnt=0):
    """SPEC A.2 over psd [S, F, N] float32 -> (means [S, groups, N], acc, cnt) with the partial group carried"""
    S, F, N = psd.shape
    acc = np.zeros((S, N), np.float32) if acc is None else acc
    out = []
    for f in range(F):
        acc = (acc + psd[:, f]).astype(np.float32)
        cnt += 1
        if cnt == A:
            out.append((acc / np.float32(A)).astype(np.float32))
            acc, cnt = np.zeros((S, N), np.float32), 0
    means = np.stack(out, axis=1) if out else np.zeros((S, 0, N), np.float32)
    return means, acc, cnt


def _signal(S, n, seed):
    """a different scene in every stream"""
    xs = [synth.multi_carrier(n, 1.0, [("qpsk", 0.11 + 0.07 * s, 1 / 64., -12.0 - 3 * s, {}),
                                       ("fsk", -0.23 + 0.05 * s, 1 / 96., -18.0, {})],
                              noise_db=-40.0 + 2 * s, seed=seed + s)[0] for s in range(S)]
    return np.ascontiguousarray(np.stack(xs).astype(np.complex64))


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _db(sdb, lin):
    """sdb_psd_shift_db_device over [S, groups, N] linear group outputs"""
    S, G, N = lin.shape
    t = torch.from_numpy(np.ascontiguousarray(lin)).cuda()
    out = torch.empty_like(t)
    if lin.size:
        sdb.psd_shift_db(t.data_ptr(), out.data_ptr(), S * G, N)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _outputs(e, stage):
    """the group outputs of the engine's latest feed: (means,) or (maxima, minima)"""
    return (e.read_psd_average(),) if stage == "mean" else e.read_psd_peak()


def _groups(e, stage):
    return e.psd_average_frames if stage == "mean" else e.psd_peak_groups()


def _stmt(frames, stage, G):
    """the statement's group outputs over frames [S, F, N], as _outputs gives them"""
    return (group_means(frames, G)[0],) if stage == "mean" else group_peaks(frames, G)[:2]


# N = 512: one CTA per frame; 8192 / 32768: the F.5 two-kernel transforms (with a channel of the same window, the PSD
# runs on its own stream beside the channeliser); 65536: the cluster transform; 131072: the Stockham four-step
@pytest.mark.parametrize("N", [512, 8192, 32768, 65536, 131072])
def test_means_bit_identical_to_statement(sdb, N):
    S, F, feeds = 3, 4, 3
    n = F * N
    x = _signal(S, feeds * n, N % 97)
    chan = N in (8192, 32768)

    def engine(A, flags=0):
        e = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=n, flags=flags, psd_average=A)
        if chan:
            e.open_channel(2 * np.pi * 0.11, 2 * np.pi * 0.02, 1.0)
        e.commit()
        return e

    ref = engine(0)
    frames = []
    for i in range(feeds):
        ref.feed(x[:, i * n:(i + 1) * n])
        frames.append(ref.read_psd())
    frames = np.concatenate(frames, axis=1)
    assert ref.psd_average_frames == 0 and not ref.psd_average_device_ptr
    for A in (2, 3, 7, 10):                                   # 10: more than one feed's 4 frames
        for flags in ((0, sdb.FLAG_PSD_SHIFT_DB) if A == 3 else (0,)):
            e = engine(A, flags)
            got, acc, cnt = [], None, 0
            for i in range(feeds):
                e.feed(x[:, i * n:(i + 1) * n])
                # the per-frame PSD stays linear and equals an engine's without averaging
                assert np.array_equal(_bits(e.read_psd()), _bits(frames[:, i * F:(i + 1) * F]))
                want, acc, cnt = group_means(frames[:, i * F:(i + 1) * F], A, acc, cnt)
                assert e.psd_average_frames == want.shape[1]
                m = e.read_psd_average()
                if flags:
                    want = _db(sdb, want)
                assert np.array_equal(_bits(m), _bits(want)), (A, flags, i)
                got.append(m)
            assert sum(g.shape[1] for g in got) == (feeds * F) // A
            e.close()
    ref.close()


@pytest.mark.parametrize("N", [512, 8192, 32768, 65536, 131072])
def test_peaks_bit_identical_to_statement(sdb, N):
    S, F, feeds = 3, 4, 3
    n = F * N
    x = _signal(S, feeds * n, N % 89)
    chan = N in (8192, 32768)

    def engine(P, flags=0, A=0):
        e = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=n, flags=flags, psd_average=A, psd_peak=P)
        if chan:
            e.open_channel(2 * np.pi * 0.11, 2 * np.pi * 0.02, 1.0)
        e.commit()
        return e

    ref, avg = engine(0), engine(0, A=2)
    frames, means = [], []
    for i in range(feeds):
        ref.feed(x[:, i * n:(i + 1) * n]); frames.append(ref.read_psd())
        avg.feed(x[:, i * n:(i + 1) * n]); means.append(avg.read_psd_average())
    assert ref.psd_peak_groups() == 0 and not ref.psd_peak_device_ptr(0) and not ref.psd_peak_device_ptr(1)
    for P in (2, 3, 7, 10):                                   # 10: more than one feed's 4 frames
        arms = [(0, 0)] + ([(sdb.FLAG_PSD_SHIFT_DB, 0), (0, 2)] if P == 3 else [])
        for flags, A in arms:
            e = engine(P, flags, A)
            carry, total = None, 0
            for i in range(feeds):
                e.feed(x[:, i * n:(i + 1) * n])
                # the per-frame PSD stays linear and equals an engine's without peak detection
                assert np.array_equal(_bits(e.read_psd()), _bits(frames[i]))
                want_mx, want_mn, carry = group_peaks(frames[i], P, carry)
                assert e.psd_peak_groups() == want_mx.shape[1]
                mx, mn = e.read_psd_peak()
                if flags:
                    want_mx, want_mn = _db(sdb, want_mx), _db(sdb, want_mn)
                assert np.array_equal(_bits(mx), _bits(want_mx)) and np.array_equal(_bits(mn), _bits(want_mn)), \
                    (P, flags, A, i)
                if A:                                         # averaging beside it: the averaging-only engine's means
                    assert np.array_equal(_bits(e.read_psd_average()), _bits(means[i]))
                total += mx.shape[1]
            assert total == (feeds * F) // P
            e.close()
    ref.close(); avg.close()


def test_burst_in_one_frame_per_group(sdb):
    """A tone gated into one frame of each group of P: every max holds it at its single-frame level, every min is the
    noise floor there, and the mean of the same group is about 10 log10(P) dB below the max."""
    N, P, G = 4096, 8, 6
    fs = 1.0
    rng = np.random.default_rng(12)
    x = ((rng.standard_normal(G * P * N) + 1j * rng.standard_normal(G * P * N)) * 1e-3).astype(np.complex64)
    k = 700                                                   # a bin-centred tone
    t = np.arange(N)
    for g in range(G):
        f = g * P + (3 * g) % P                               # a different frame of each group
        x[f * N:(f + 1) * N] += np.exp(2j * np.pi * k * t / N).astype(np.complex64)
    e = sdb.Engine(n_streams=1, psd_size=N, psd_window="hann", max_feed=G * P * N, samp_rate=fs, psd_average=P,
                   psd_peak=P)
    e.commit()
    e.feed(x.reshape(1, -1))
    frames = e.read_psd()
    mx, mn = e.read_psd_peak()
    mean = e.read_psd_average()
    assert mx.shape == mn.shape == mean.shape == (1, G, N)
    for g in range(G):
        f = g * P + (3 * g) % P
        assert mx[0, g, k] == frames[0, f, k]                 # the burst frame's own value
        assert 10 * np.log10(mx[0, g, k] / frames[0, f, k - 40]) > 60
        assert 10 * np.log10(mx[0, g, k] / mn[0, g, k]) > 60  # absent from the min
        down = 10 * np.log10(mx[0, g, k] / mean[0, g, k])
        assert abs(down - 10 * np.log10(P)) < 0.05, down
    want_mx, want_mn, _ = group_peaks(frames, P)
    assert same(mx, want_mx) and same(mn, want_mn)
    e.close()


def test_non_finite_input(sdb):
    """NaN and inf input samples in single frames make those frames' spectra non-finite; the extremes follow PK.2:
    NaN ignored, also as a group's first frame; a group of NaN frames gives NaN."""
    N, P, F = 1024, 3, 15
    x = _signal(1, F * N, 7)
    x[0, 5 * N + 17] = np.nan                                 # group 1: last frame
    x[0, 6 * N + 100] = np.complex64(np.inf)                  # group 2: first frame
    for f in (9, 10, 11):                                     # group 3: every frame
        x[0, f * N + 3] = np.nan
    e = sdb.Engine(n_streams=1, psd_size=N, psd_window="hann", max_feed=F * N, psd_peak=P)
    e.commit()
    e.feed(x)
    frames = e.read_psd()
    assert np.isnan(frames[0, 5]).any() and not np.isfinite(frames[0, 6]).all() and np.isnan(frames[0, 9:12]).all()
    mx, mn = e.read_psd_peak()
    want_mx, want_mn, _ = group_peaks(frames, P)
    assert same(mx, want_mx) and same(mn, want_mn)
    assert np.isnan(mx[0, 3]).all() and np.isnan(mn[0, 3]).all()
    assert not np.isnan(mn[0, 1]).any() and not np.isnan(mn[0, 2]).any()
    e.close()


@pytest.mark.parametrize("stage", ["mean", "peak"])
def test_feed_split_independence(sdb, stage):
    """Ragged host and device feeds of u8 IQ give the group outputs of one feed of the same samples."""
    S, N, G = 2, 1024, 5
    split = [3, 7, 1, 9, 4]                                   # frames per feed: 24 in all, 4 groups
    total = sum(split) * N
    rng = np.random.default_rng(6)
    x = rng.integers(0, 256, size=(S, total, 2), dtype=np.uint8)
    one = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=total, input_format="u8",
                     **{FIELD[stage]: G})
    one.commit()
    one.feed(x)
    want = _outputs(one, stage)
    assert want[0].shape == (S, sum(split) // G, N)
    e = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=max(split) * N, input_format="u8",
                   **{FIELD[stage]: G})
    e.commit()
    got, pos = [], 0
    for i, f in enumerate(split):
        part = np.ascontiguousarray(x[:, pos:pos + f * N])
        if i % 2:
            d = torch.from_numpy(part.reshape(S, -1)).cuda()
            e.feed_device_ptr(d.data_ptr(), f * N, f * N)
            e.sync()
        else:
            e.feed(part)
        got.append(_outputs(e, stage))
        pos += f * N
    for w, ref in enumerate(want):
        assert np.array_equal(_bits(np.concatenate([g[w] for g in got], axis=1)), _bits(ref))
    one.close(); e.close()


def _migrating_engine(sdb, S, N, n, stage, G, bws):
    e = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=n, **{FIELD[stage]: G})
    for f0, bw in bws:
        e.open_channel(2 * np.pi * f0, 2 * np.pi * bw, 1.0)
    e.commit()
    return e


@pytest.mark.parametrize("stage", ["mean", "peak"])
def test_migration_keeps_partial_group(sdb, stage):
    """An engine re-planned mid-group through migrate_map (one channel added) gives the group outputs of an engine
    that never re-planned; a re-plan to another group size starts an empty group."""
    S, N, G, F = 2, 8192, 4, 3
    n = F * N
    x = _signal(S, 6 * n, 3)
    L = sdb.load_library()
    chans = [(0.11, 0.02)]
    steady = _migrating_engine(sdb, S, N, n, stage, G, chans)
    first = _migrating_engine(sdb, S, N, n, stage, G, chans)
    ref, got = [], []
    for i in range(3):                                       # 9 frames: 2 groups, 1 frame carried
        steady.feed(x[:, i * n:(i + 1) * n]); ref.append(_outputs(steady, stage))
        first.feed(x[:, i * n:(i + 1) * n]); got.append(_outputs(first, stage))
    second = _migrating_engine(sdb, S, N, n, stage, G, chans + [(0.31, 0.01)])
    other_g = _migrating_engine(sdb, S, N, n, stage, 3, chans)
    sdb._check(L.sdb_engine_migrate_map(second._h, first._h, (C.c_int32 * 2)(0, -1), 2))
    sdb._check(L.sdb_engine_migrate_map(other_g._h, first._h, (C.c_int32 * 1)(0), 1))
    for i in range(3, 6):
        steady.feed(x[:, i * n:(i + 1) * n]); ref.append(_outputs(steady, stage))
        second.feed(x[:, i * n:(i + 1) * n]); got.append(_outputs(second, stage))
        other_g.feed(x[:, i * n:(i + 1) * n])
        if i == 3:
            assert _groups(other_g, stage) == 1
            for o, w in zip(_outputs(other_g, stage), _stmt(steady.read_psd(), stage, 3)):
                assert np.array_equal(_bits(o), _bits(w))
    for w in range(len(ref[0])):
        assert np.array_equal(_bits(np.concatenate([g[w] for g in got], axis=1)),
                              _bits(np.concatenate([r[w] for r in ref], axis=1)))
    assert sum(r[0].shape[1] for r in ref) == 6 * F // G
    for e in (steady, first, second, other_g):
        e.close()


@pytest.mark.parametrize("stage", ["mean", "peak"])
def test_detector_beside_db(sdb, stage):
    """Channel detector + SHIFT_DB + a group stage in one engine: the channel lists of a detector-only engine, a linear
    per-frame PSD, and the group outputs (not the frames) in dB.  Without a group stage the detector still refuses
    SHIFT_DB."""
    S, N, F = 2, 8192, 4
    n = F * N
    x = _signal(S, 4 * n, 9)
    both = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=n, flags=sdb.FLAG_PSD_SHIFT_DB,
                      **{FIELD[stage]: 4})
    alone = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=n)
    for e in (both, alone):
        e.set_channel_detector(alpha=0.2, gamma=0.5, snr=4.0, min_bins=2)
        e.commit()
    fields = lambda c: (c.fc, c.f_lo, c.f_hi, c.bw, c.snr, c.S0, c.N0, c.bin_lo, c.bin_hi)
    found = 0
    for i in range(4):
        both.feed(x[:, i * n:(i + 1) * n]); alone.feed(x[:, i * n:(i + 1) * n])
        for s in range(S):
            a, ta = both.read_channels(s)
            b, tb = alone.read_channels(s)
            assert ta == tb and [fields(c) for c in a] == [fields(c) for c in b]
            found += len(a)
        lin = alone.read_psd()
        assert np.array_equal(_bits(both.read_psd()), _bits(lin))
        for o, want in zip(_outputs(both, stage), _stmt(lin, stage, 4)):
            assert o.shape == (S, 1, N) and np.array_equal(_bits(o), _bits(_db(sdb, want)))
            assert np.allclose(o, 10 * np.log10(np.fft.fftshift(want, axes=2) + 1e-8), atol=1e-3)
    assert found > 0
    db_only = sdb.Engine(n_streams=1, psd_size=N, max_feed=n, flags=sdb.FLAG_PSD_SHIFT_DB)
    with pytest.raises(sdb.SdbError, match="needs a linear PSD"):
        db_only.set_channel_detector()
    both.close(); alone.close(); db_only.close()


@pytest.mark.parametrize("stage", ["mean", "peak"])
def test_limits_and_accessors(sdb, stage):
    """A group size > 65536 and a group stage without a main PSD are refused at commit with a message; with 0 or 1 the
    engine issues the launches it issues without the field, the reads refuse, the accessors are empty and the stage's
    timing family records nothing; otherwise one more launch per feed, which the family counts.  The means' read takes
    no NULL destination, the extremes' read either one NULL."""
    field = FIELD[stage]
    e = sdb.Engine(n_streams=1, psd_size=1024, max_feed=1024, **{field: 65537})
    with pytest.raises(sdb.SdbError, match=f"{field} must be at most 65536, got 65537"):
        e.commit()
    e.close()
    e = sdb.Engine(n_streams=1, psd_size=0, st_window_size=1024, max_feed=1024, **{field: 2})
    with pytest.raises(sdb.SdbError, match=f"{field} needs the main PSD"):
        e.commit()
    e.close()
    x = _signal(1, 4096, 1)
    for G, extra in ((0, 0), (1, 0), (65536, 2)):
        e = sdb.Engine(n_streams=1, psd_size=1024, max_feed=4096, **{field: G})
        e.commit()
        e.timing(True)
        e.feed(x); e.feed(x)
        assert e.launches == 2 + extra                        # the 1024-point PSD is one launch a feed
        assert e.kernel_time(field)[1] == extra
        assert _groups(e, stage) == 0
        ptrs = [e.psd_average_device_ptr] if stage == "mean" else [e.psd_peak_device_ptr(0), e.psd_peak_device_ptr(1)]
        if G < 2:
            assert not any(ptrs)
            if stage == "mean":
                with pytest.raises(sdb.SdbError, match="PSD averaging not enabled"):
                    e.read_psd_average(np.empty((1, 1, 1024), np.float32))
            else:
                with pytest.raises(sdb.SdbError, match="PSD peak detection not enabled"):
                    e.read_psd_peak()
        else:
            assert all(ptrs) and all(o.shape == (1, 0, 1024) for o in _outputs(e, stage))
        e.close()
    e = sdb.Engine(n_streams=1, psd_size=1024, max_feed=4096, **{field: 2})
    e.commit()
    e.feed(x)
    if stage == "mean":
        with pytest.raises(sdb.SdbError, match="null argument"):
            sdb._check(e._L.sdb_engine_read_psd_average(e._h, None, 1 << 20))
    else:
        mx, mn = e.read_psd_peak()
        only = np.zeros_like(mn)
        sdb._check(e._L.sdb_engine_read_psd_peak(e._h, None, only.ctypes.data, only.size))
        assert np.array_equal(_bits(only), _bits(mn))
    e.close()


# ---- analyzer: fs = 2^20 Hz makes every frame duration and psd_update_int below exact in binary32 -------------------

def _engine_frames(sdb, x, N, fs):
    e = sdb.Engine(n_streams=1, psd_size=N, psd_window="hann", max_feed=len(x), samp_rate=fs)
    e.commit()
    e.feed(x.reshape(1, -1))
    f = e.read_psd()
    e.close()
    return f


def _drain(a):
    msgs = []
    while True:
        name, m = a.read(30000)
        assert name != "TIMEOUT"
        msgs.append((name, m))
        if name in ("EOS", "READ_ERROR", "HALT"):
            return msgs


def _psd(msgs):
    return [m for name, m in msgs if name == "PSD"]


def _check_posts(msgs, frames, posted, G, N, D, fs, first_frame=0):
    """PSD messages == the SPEC A means ("mean"), SPEC PK maxima ("pos_peak") or minima ("neg_peak") of frames from
    first_frame on, time-stamped at each group's first sample"""
    f = frames[:, first_frame:]
    want = group_means(f, G)[0] if posted == "mean" else group_peaks(f, G)[1 if posted == "neg_peak" else 0]
    assert len(msgs) == want.shape[1]
    for j, m in enumerate(msgs):
        assert np.array_equal(_bits(m["psd"]), _bits(want[0, j])), j
        assert m["samp_rate"] == np.float32(fs / D)
        assert abs(m["timestamp"] - (first_frame + j * G) * N * D / fs) < 1.5e-6


def _tone(n, fs, seed):
    x, _ = synth.multi_carrier(n, fs, [("qpsk", 0.1 * fs, fs / 64, -10.0, {})], noise_db=-45.0, seed=seed)
    return x.astype(np.complex64)


@pytest.mark.parametrize("D", [1, 2])
@pytest.mark.parametrize("posted", ["mean", "pos_peak", "neg_peak"])
def test_analyzer_posts(sdb, D, posted):
    """psd_update_int = 5 frames: one PSD message per 5 frames, their mean, maximum or minimum, stamped at the first
    sample of its group; at D = 2 the frames are those of the decimated stream and the stamps stay in source time.
    psd_average is set beside the detectors too: a detector takes precedence."""
    from sigdigger_b200.analyzer import Analyzer
    N, fs, G, per_block, blocks = 4096, 2.0 ** 20, 5, 4096 * 6, 7
    x = _tone(blocks * per_block * D, fs, 21)
    if D > 1:
        dec = sdb.Decimator(D, max_feed=len(x))
        dec.feed(x.reshape(1, -1))
        xd = dec.read()[0]
        dec.close()
    else:
        xd = x
    frames = _engine_frames(sdb, xd, N, fs / D)
    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=G * N / (fs / D), data=x, read_size=per_block,
                 decimation=D, psd_average=1, psd_detector=0 if posted == "mean" else posted)
    msgs = _drain(a)
    a.close()
    assert msgs[-1][0] == "EOS"
    _check_posts(_psd(msgs), frames, posted, G, N, D, fs)


def _gated(x, fs, N, per_block, **kw):
    from sigdigger_b200.analyzer import Analyzer
    gate, pos = Gate(), [0]

    def read(priv, dst, maxn):
        gate.wait(30)
        take = min(maxn, len(x) - pos[0])
        if take > 0:
            C.memmove(dst, x.ctypes.data + 8 * pos[0], 8 * take)
            pos[0] += take
        return take

    a = Analyzer(fs, window_size=N, window="hann", read=read, read_size=per_block, **kw)
    assert a.read(5000)[0] == "SOURCE_INFO"
    assert gate.parked.wait(10)
    return a, gate


@pytest.mark.parametrize("posted", ["mean", "pos_peak"])
def test_analyzer_inspector_open_keeps_the_group(sdb, posted):
    """Opening an inspector after the first block (a re-plan that migrates) leaves the PSD messages unchanged."""
    N, fs, G, per_block, blocks = 4096, 2.0 ** 20, 4, 4096 * 6, 6
    x = _tone(blocks * per_block, fs, 8)
    kw = dict(psd_average=1) if posted == "mean" else dict(psd_detector=posted)
    runs = []
    for open_one in (False, True):
        a, gate = _gated(x, fs, N, per_block, psd_update_int=G * N / fs, **kw)
        if open_one:
            a.open("psk", 0.1 * fs, fs / 16, req_id=1)
        gate.set()
        msgs = _drain(a)
        a.close()
        assert msgs[-1][0] == "EOS"
        runs.append(msgs)
    assert any(name == "INSPECTOR" for name, _ in runs[1])
    _check_posts(_psd(runs[0]), _engine_frames(sdb, x, N, fs), posted, G, N, 1, fs)
    assert [(_bits(m["psd"]).tobytes(), m["timestamp"]) for m in _psd(runs[0])] == \
           [(_bits(m["psd"]).tobytes(), m["timestamp"]) for m in _psd(runs[1])]


def test_analyzer_set_params_changes_a(sdb):
    """SET_PARAMS after the first block changes A from 4 to 3: the first block's 6 frames give one mean (2 frames
    carried), the re-plan drops the carry, and the means of A = 3 start at frame 6.  PARAMS echoes psd_average."""
    N, fs, per_block, blocks = 4096, 2.0 ** 20, 4096 * 6, 5
    x = _tone(blocks * per_block, fs, 4)
    a, gate = _gated(x, fs, N, per_block, psd_update_int=4 * N / fs, psd_average=1)
    a.set_params(req_id=3, psd_update_int=3 * N / fs)
    gate.set()
    msgs = _drain(a)
    a.close()
    assert msgs[-1][0] == "EOS"
    params = [m for name, m in msgs if name == "PARAMS"]
    assert len(params) == 1 and params[0]["psd_average"] == 1
    frames = _engine_frames(sdb, x, N, fs)
    psd = _psd(msgs)
    _check_posts(psd[:1], frames[:, :6], "mean", 4, N, 1, fs)
    _check_posts(psd[1:], frames, "mean", 3, N, 1, fs, first_frame=6)


def test_analyzer_without_averaging_posts_frames(sdb):
    """psd_average = 0: one engine frame per psd_update_int, as the per-frame PSD path posts them."""
    from sigdigger_b200.analyzer import Analyzer
    N, fs, per_block, blocks = 4096, 2.0 ** 20, 4096 * 6, 5
    x = _tone(blocks * per_block, fs, 6)
    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=4 * N / fs, data=x, read_size=per_block)
    msgs = _drain(a)
    a.close()
    frames = _engine_frames(sdb, x, N, fs)
    psd = _psd(msgs)
    assert len(psd) == blocks * 6 // 4
    for j, m in enumerate(psd):
        f = 4 * j + 3                                          # the credit reaches the interval at every 4th frame
        assert np.array_equal(_bits(m["psd"]), _bits(frames[0, f]))
        assert abs(m["timestamp"] - f * N / fs) < 1.5e-6


@pytest.mark.parametrize("change", ["P", "detector_on", "pos_to_neg"])
def test_analyzer_set_params(sdb, change):
    """SET_PARAMS after the first block (6 frames: one group of 4 posted, 2 frames carried):
    - P: 4 -> 3 drops the carry; the groups of P = 3 start at frame 6;
    - detector_on: means of 4 -> maxima of 4 drops the averaging carry; the maxima start at frame 6;
    - pos_to_neg: the same P keeps the carry; the minima continue at frame 4.
    PARAMS echoes psd_detector and psd_average as given."""
    N, fs, per_block, blocks = 4096, 2.0 ** 20, 4096 * 6, 5
    x = _tone(blocks * per_block, fs, 4)
    start = dict(psd_average=1) if change == "detector_on" else dict(psd_detector="pos_peak")
    a, gate = _gated(x, fs, N, per_block, psd_update_int=4 * N / fs, **start)
    if change == "P":
        a.set_params(req_id=3, psd_update_int=3 * N / fs)
    elif change == "detector_on":
        a.set_params(req_id=3, psd_detector="pos_peak")
    else:
        a.set_params(req_id=3, psd_detector="neg_peak")
    gate.set()
    msgs = _drain(a)
    a.close()
    assert msgs[-1][0] == "EOS"
    params = [m for name, m in msgs if name == "PARAMS"]
    assert len(params) == 1
    frames = _engine_frames(sdb, x, N, fs)
    psd = _psd(msgs)
    if change == "P":
        assert params[0]["psd_detector"] == 1 and params[0]["psd_average"] == 0
        _check_posts(psd[:1], frames[:, :6], "pos_peak", 4, N, 1, fs)
        _check_posts(psd[1:], frames, "pos_peak", 3, N, 1, fs, first_frame=6)
    elif change == "detector_on":
        assert params[0]["psd_detector"] == 1 and params[0]["psd_average"] == 1
        want, _, _ = group_means(frames[:, :6], 4)
        assert len(psd) >= 1 and np.array_equal(_bits(psd[0]["psd"]), _bits(want[0, 0]))
        _check_posts(psd[1:], frames, "pos_peak", 4, N, 1, fs, first_frame=6)
    else:
        assert params[0]["psd_detector"] == 2
        _check_posts(psd[:1], frames[:, :6], "pos_peak", 4, N, 1, fs)
        _check_posts(psd[1:], frames, "neg_peak", 4, N, 1, fs, first_frame=4)


@pytest.mark.parametrize("average", [0, 1])
def test_analyzer_default_detector_unchanged(sdb, average):
    """psd_detector = 0 given explicitly: one engine frame per psd_update_int, or the means with psd_average."""
    from sigdigger_b200.analyzer import Analyzer
    N, fs, per_block, blocks = 4096, 2.0 ** 20, 4096 * 6, 5
    x = _tone(blocks * per_block, fs, 6)
    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=4 * N / fs, data=x, read_size=per_block,
                 psd_average=average, psd_detector=0)
    msgs = _drain(a)
    a.close()
    frames = _engine_frames(sdb, x, N, fs)
    psd = _psd(msgs)
    if average:
        want, _, _ = group_means(frames, 4)
        assert len(psd) == want.shape[1]
        for j, m in enumerate(psd):
            assert np.array_equal(_bits(m["psd"]), _bits(want[0, j]))
            assert abs(m["timestamp"] - 4 * j * N / fs) < 1.5e-6
    else:
        assert len(psd) == blocks * 6 // 4
        for j, m in enumerate(psd):
            f = 4 * j + 3                                      # the credit reaches the interval at every 4th frame
            assert np.array_equal(_bits(m["psd"]), _bits(frames[0, f]))
            assert abs(m["timestamp"] - f * N / fs) < 1.5e-6


def test_analyzer_refuses_unknown_detector(sdb):
    from sigdigger_b200.analyzer import Analyzer
    x = _tone(4096 * 4, 2.0 ** 20, 1)
    with pytest.raises(sdb.SdbError, match="psd_detector must be"):
        Analyzer(2.0 ** 20, window_size=4096, data=x, psd_detector=3)
    a = Analyzer(2.0 ** 20, window_size=4096, data=x, read_size=4096 * 4)
    for bad in (-1, 3):
        with pytest.raises(sdb.SdbError, match="set_params_async rejected"):
            a.set_params(psd_detector=bad)
    assert a.params.psd_detector == 0
    _drain(a)
    a.close()
