"""-m gpu: the frame-averaged main PSD (SPEC A, oracle/SPEC_A.md) through the engine and the analyzer.

The statement of A.2 is `group_means` below: a float32 loop over frames, vectorised over bins, that adds each frame in
order to the running sum and divides once per group (no np.sum, which adds pairwise).  It is applied to the same
engine's per-frame linear PSD, so every comparison is bit for bit."""
import ctypes as C

import numpy as np
import pytest
import torch

from sigdigger_b200 import synth
from test_gpu_analyzer import Gate

pytestmark = pytest.mark.gpu


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
    xs = [synth.multi_carrier(n, 1.0, [("qpsk", 0.11 + 0.07 * s, 1 / 64., -12.0, {}), ("fsk", -0.23, 1 / 96., -18.0, {})],
                              noise_db=-40.0, seed=seed + s)[0] for s in range(S)]
    return np.ascontiguousarray(np.stack(xs).astype(np.complex64))


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


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
                    lin = torch.from_numpy(np.ascontiguousarray(want)).cuda()
                    db = torch.empty_like(lin)
                    if want.size:
                        sdb.psd_shift_db(lin.data_ptr(), db.data_ptr(), S * want.shape[1], N)
                    torch.cuda.synchronize()
                    want = db.cpu().numpy()
                assert np.array_equal(_bits(m), _bits(want)), (A, flags, i)
                got.append(m)
            assert sum(g.shape[1] for g in got) == (feeds * F) // A
            e.close()
    ref.close()


def test_feed_split_independence(sdb):
    """Ragged host and device feeds of u8 IQ give the means of one feed of the same samples."""
    S, N, A = 2, 1024, 5
    split = [3, 7, 1, 9, 4]                                   # frames per feed: 24 in all, 4 means
    total = sum(split) * N
    rng = np.random.default_rng(5)
    x = rng.integers(0, 256, size=(S, total, 2), dtype=np.uint8)
    one = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=total, input_format="u8", psd_average=A)
    one.commit()
    one.feed(x)
    want = one.read_psd_average()
    assert want.shape == (S, sum(split) // A, N)
    e = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=max(split) * N, input_format="u8",
                   psd_average=A)
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
        got.append(e.read_psd_average())
        pos += f * N
    assert np.array_equal(_bits(np.concatenate(got, axis=1)), _bits(want))
    one.close(); e.close()


def _migrating_engine(sdb, S, N, n, A, bws):
    e = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=n, psd_average=A)
    for f0, bw in bws:
        e.open_channel(2 * np.pi * f0, 2 * np.pi * bw, 1.0)
    e.commit()
    return e


def test_migration_keeps_partial_group(sdb):
    """An engine re-planned mid-group through migrate_map (one channel added) gives the means of an engine that never
    re-planned; a re-plan to another A starts an empty group."""
    S, N, A, F = 2, 8192, 4, 3
    n = F * N
    x = _signal(S, 6 * n, 3)
    L = sdb.load_library()
    chans = [(0.11, 0.02)]
    steady = _migrating_engine(sdb, S, N, n, A, chans)
    first = _migrating_engine(sdb, S, N, n, A, chans)
    ref, got = [], []
    for i in range(3):                                       # 9 frames: 2 means, 1 frame carried
        steady.feed(x[:, i * n:(i + 1) * n]); ref.append(steady.read_psd_average())
        first.feed(x[:, i * n:(i + 1) * n]); got.append(first.read_psd_average())
    second = _migrating_engine(sdb, S, N, n, A, chans + [(0.31, 0.01)])
    other_a = _migrating_engine(sdb, S, N, n, 3, chans)
    sdb._check(L.sdb_engine_migrate_map(second._h, first._h, (C.c_int32 * 2)(0, -1), 2))
    sdb._check(L.sdb_engine_migrate_map(other_a._h, first._h, (C.c_int32 * 1)(0), 1))
    frames = []
    for i in range(3, 6):
        steady.feed(x[:, i * n:(i + 1) * n]); ref.append(steady.read_psd_average())
        second.feed(x[:, i * n:(i + 1) * n]); got.append(second.read_psd_average())
        frames.append(steady.read_psd())
        other_a.feed(x[:, i * n:(i + 1) * n])
        if i == 3:
            assert other_a.psd_average_frames == 1
            want, _, _ = group_means(frames[0], 3)
            assert np.array_equal(_bits(other_a.read_psd_average()), _bits(want))
    assert np.array_equal(_bits(np.concatenate(got, axis=1)), _bits(np.concatenate(ref, axis=1)))
    assert sum(r.shape[1] for r in ref) == 6 * F // A
    for e in (steady, first, second, other_a):
        e.close()


def test_detector_beside_db_means(sdb):
    """Channel detector + SHIFT_DB + averaging in one engine: the channel lists of a detector-only engine, and the
    flag turns the means (not the frames) into dB.  Without averaging the detector still refuses SHIFT_DB."""
    S, N, F = 2, 8192, 4
    n = F * N
    x = _signal(S, 4 * n, 9)
    both = sdb.Engine(n_streams=S, psd_size=N, psd_window="hann", max_feed=n, flags=sdb.FLAG_PSD_SHIFT_DB,
                      psd_average=4)
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
        m = both.read_psd_average()
        want, _, _ = group_means(lin, 4)
        assert m.shape == (S, 1, N) and np.allclose(m, 10 * np.log10(np.fft.fftshift(want, axes=2) + 1e-8), atol=1e-3)
    assert found > 0
    db_only = sdb.Engine(n_streams=1, psd_size=N, max_feed=n, flags=sdb.FLAG_PSD_SHIFT_DB)
    with pytest.raises(sdb.SdbError, match="needs a linear PSD"):
        db_only.set_channel_detector()
    both.close(); alone.close(); db_only.close()


def test_limits_and_accessors(sdb):
    """A > 65536 and averaging without a main PSD are refused at commit with a message; without averaging the reads
    refuse, the accessors are empty and the psd_average timing family records no launch."""
    e = sdb.Engine(n_streams=1, psd_size=1024, max_feed=1024, psd_average=65537)
    with pytest.raises(sdb.SdbError, match="psd_average must be at most 65536, got 65537"):
        e.commit()
    e.close()
    e = sdb.Engine(n_streams=1, psd_size=0, st_window_size=1024, max_feed=1024, psd_average=2)
    with pytest.raises(sdb.SdbError, match="psd_average needs the main PSD"):
        e.commit()
    e.close()
    x = _signal(1, 4096, 1)
    for A, launches in ((0, 0), (1, 0), (65536, 2)):
        e = sdb.Engine(n_streams=1, psd_size=1024, max_feed=4096, psd_average=A)
        e.commit()
        e.timing(True)
        e.feed(x); e.feed(x)
        assert e.kernel_time("psd_average")[1] == launches
        assert e.psd_average_frames == 0
        if A < 2:
            assert not e.psd_average_device_ptr
            with pytest.raises(sdb.SdbError, match="PSD averaging not enabled"):
                e.read_psd_average(np.empty((1, 1, 1024), np.float32))
        else:
            assert e.psd_average_device_ptr and e.read_psd_average().shape == (1, 0, 1024)
        e.close()


# ---- analyzer: fs = 2^20 Hz makes every frame duration and psd_update_int below exact in binary32 -------------------------------------------------------------------------------------------------------

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


def _check_means(msgs, frames, A, N, D, fs, first_frame=0, t0=0.0):
    """PSD messages == SPEC A means of frames (first_frame onwards), time-stamped at each group's first sample"""
    want, _, _ = group_means(frames[:, first_frame:], A)
    assert len(msgs) == want.shape[1]
    for j, m in enumerate(msgs):
        assert np.array_equal(_bits(m["psd"]), _bits(want[0, j])), j
        assert m["samp_rate"] == np.float32(fs / D)
        assert abs(m["timestamp"] - (t0 + (first_frame + j * A) * N * D / fs)) < 1.5e-6


@pytest.mark.parametrize("D", [1, 2])
def test_analyzer_posts_means(sdb, D):
    """psd_update_int = 5 frames: one PSD message per 5 frames, the mean of the engine's frames, stamped at the first
    sample of its group; at D = 2 the frames are those of the decimated stream and the stamps stay in source time."""
    from sigdigger_b200.analyzer import Analyzer
    N, fs, A, per_block, blocks = 4096, 2.0 ** 20, 5, 4096 * 6, 7
    x, _ = synth.multi_carrier(blocks * per_block * D, fs, [("qpsk", 0.1 * fs, fs / 64, -10.0, {})], noise_db=-45.0,
                               seed=21)
    x = x.astype(np.complex64)
    if D > 1:
        dec = sdb.Decimator(D, max_feed=len(x))
        dec.feed(x.reshape(1, -1))
        xd = dec.read()[0]
        dec.close()
    else:
        xd = x
    frames = _engine_frames(sdb, xd, N, fs / D)
    a = Analyzer(fs, window_size=N, window="hann", psd_update_int=A * N / (fs / D), data=x, read_size=per_block,
                 decimation=D, psd_average=1)
    msgs = _drain(a)
    a.close()
    assert msgs[-1][0] == "EOS"
    _check_means(_psd(msgs), frames, A, N, D, fs)


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


def test_analyzer_inspector_open_keeps_the_group(sdb):
    """Opening an inspector after the first block (a re-plan that migrates) leaves the PSD messages unchanged."""
    N, fs, A, per_block, blocks = 4096, 2.0 ** 20, 4, 4096 * 6, 6
    x, _ = synth.multi_carrier(blocks * per_block, fs, [("qpsk", 0.1 * fs, fs / 64, -10.0, {})], noise_db=-45.0, seed=8)
    x = x.astype(np.complex64)
    runs = []
    for open_one in (False, True):
        a, gate = _gated(x, fs, N, per_block, psd_update_int=A * N / fs, psd_average=1)
        if open_one:
            a.open("psk", 0.1 * fs, fs / 16, req_id=1)
        gate.set()
        msgs = _drain(a)
        a.close()
        assert msgs[-1][0] == "EOS"
        runs.append(msgs)
    assert any(name == "INSPECTOR" for name, _ in runs[1])
    _check_means(_psd(runs[0]), _engine_frames(sdb, x, N, fs), A, N, 1, fs)
    assert [(_bits(m["psd"]).tobytes(), m["timestamp"]) for m in _psd(runs[0])] == \
           [(_bits(m["psd"]).tobytes(), m["timestamp"]) for m in _psd(runs[1])]


def test_analyzer_set_params_changes_a(sdb):
    """SET_PARAMS after the first block changes A from 4 to 3: the first block's 6 frames give one mean (2 frames
    carried), the re-plan drops the carry, and the means of A = 3 start at frame 6.  PARAMS echoes psd_average."""
    N, fs, per_block, blocks = 4096, 2.0 ** 20, 4096 * 6, 5
    x, _ = synth.multi_carrier(blocks * per_block, fs, [("qpsk", 0.1 * fs, fs / 64, -10.0, {})], noise_db=-45.0, seed=4)
    x = x.astype(np.complex64)
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
    _check_means(psd[:1], frames[:, :6], 4, N, 1, fs)
    _check_means(psd[1:], frames, 3, N, 1, fs, first_frame=6)


def test_analyzer_without_averaging_posts_frames(sdb):
    """psd_average = 0: one engine frame per psd_update_int, as the per-frame PSD path posts them."""
    from sigdigger_b200.analyzer import Analyzer
    N, fs, per_block, blocks = 4096, 2.0 ** 20, 4096 * 6, 5
    x, _ = synth.multi_carrier(blocks * per_block, fs, [("qpsk", 0.1 * fs, fs / 64, -10.0, {})], noise_db=-45.0, seed=6)
    x = x.astype(np.complex64)
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
