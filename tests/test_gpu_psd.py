"""-m gpu: the main PSD at every accepted size (16 ... 2^20 points) on all four transform paths.  Every case feeds two
streams with different content in two feeds; the output must be bit-identical to the CPU oracle (oracle.psd_frames,
the SPEC transform) and within SPEC T of the float64 statement of SPEC W / P / Q / R / M.6 (tests/psd_f64.py), which
shares no code with the oracle or the kernels.

Paths by size (make_plan in engine.cu): 16 ... 4096 k_small_psd (one CTA per frame; 32-thread CTAs with idle lanes
below 128 points, a radix-2 tail at odd log sizes), 8192 / 16384 / 32768 SPEC F.5 (k_cols16T + k_rows256), 65536
the cluster kernel k_fft65536, 2^17 ... 2^20 the generic four-step (k_pass_a + k_pass_b) through scratch chunks of
64 MB: 64, 32, 16 and 8 windows."""
import numpy as np
import pytest
import torch

import parity
import psd_f64 as pf
import st_f64 as st
from test_gpu_channeliser import _check as check_channels
from test_psd_f64 import IMPULSE_AMPS, WINDOWED, assert_impulse, impulse_frames, tone_noise

pytestmark = pytest.mark.gpu

SIZES = [1 << k for k in range(4, 21)]
S = 2


def _engine(sdb, N, kind, max_feed, **kw):
    """A PSD-only engine.  The channeliser window is at least 64 points even with no channel open, so a 16- or
    32-point PSD gets a 64-point one; max_feed is rounded up to what both sizes accept."""
    W = max(N, 64)
    unit = max(N, W // 2)
    e = sdb.Engine(n_streams=S, psd_size=N, psd_window=kind, st_window_size=W,
                   max_feed=-(-max_feed // unit) * unit, **kw)
    e.commit()
    return e


def _feed(e, blocks):
    """Feed each block ([S, n] or [S, n, 2]) and read its PSD -> [S, frames, N] over all blocks."""
    out = []
    for b in blocks:
        e.feed(b)
        out.append(e.read_psd().copy())
    e.close()
    return np.concatenate(out, axis=1)


def _split(x, frames, N):
    """[S, n, ...] -> the blocks of frames[0] N, frames[1] N, ... samples"""
    cut = np.cumsum([0] + [f * N for f in frames])
    return [np.ascontiguousarray(x[:, a:b]) for a, b in zip(cut[:-1], cut[1:])]


def _signal(n, N):
    """Two streams: noise plus a tone, with different seeds, tone frequencies and levels."""
    return np.stack([tone_noise(n, seed=N % 101 + 7 * s, f=0.1234 + 0.2311 * s, amp=0.5 + 0.3 * s,
                                noise=0.3 - 0.1 * s) for s in range(S)])


def _frames(N):
    """frames per stream in the first and second feed"""
    return (2, 3) if N <= 4096 else ((1, 2) if N <= 65536 else (1, 1))


def _assert_psd(oracle, got, xs, N, kind, f64=True):
    """got [S, frames, N]: bit-identical to the oracle on the float32 samples xs [S, n] and (f64) within T of the
    float64 statement; returns the worst tolerance ratio."""
    worst = 0.0
    for s in range(S):
        ref = oracle.psd_frames(xs[s], N, kind)
        assert got[s].shape == ref.shape, (got[s].shape, ref.shape)
        assert np.array_equal(got[s].view(np.uint32), ref.view(np.uint32)), \
            "N %d %s stream %d: not bit-identical to the oracle (%.2f x T)" % (N, kind, s, parity.psd_err_ratio(got[s], ref))
        if not f64:
            continue
        r = parity.psd_err_ratio(got[s], pf.psd(xs[s], N, kind))
        assert r <= 1.0, "N %d %s stream %d: worst bin at %.2f x T of the float64 statement" % (N, kind, s, r)
        worst = max(worst, r)
    return worst


def _tol_T(P):
    """SPEC T's tolerance for each bin of the float64 PSD frames P [..., N]"""
    M = P.mean(axis=-1, keepdims=True)
    Pmax = P.max(axis=-1, keepdims=True)
    return (parity.PSD_RTOL * P + parity.PSD_FLOOR * np.sqrt(P * M) + parity.PSD_LINE * np.sqrt(P * Pmax)
            + 1e-11 * M)


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", SIZES)
def test_every_size_every_window(sdb, oracle, N):
    """(a) every accepted size with all five windows"""
    fr = _frames(N)
    x = _signal(N * sum(fr), N)
    for kind in pf.KINDS:
        got = _feed(_engine(sdb, N, kind, N * max(fr)), _split(x, fr, N))
        _assert_psd(oracle, got, x, N, kind)


@pytest.mark.parametrize("N", SIZES)
def test_impulse_probe(sdb, oracle, N):
    """(b) frames holding one impulse a delta[n - p] at p in {0, 1, N/3, N/2 - 1, N/2, N - 2, N - 1} give
    |a|^2 w[p]^2 / N in every bin, w from the float64 formula: within 2e-6, and exactly zero where the tap is zero.
    This holds the window table itself to SPEC W, which the bit-exact comparison with the oracle cannot do when
    oracle/ and host_design.h make the same mistake."""
    amps = [IMPULSE_AMPS, IMPULSE_AMPS[1:] + IMPULSE_AMPS[:1]]
    xs, ps = zip(*[impulse_frames(N, a) for a in amps])
    x = np.stack(xs)
    fr = (3, len(ps[0]) - 3)
    for kind in WINDOWED:
        got = _feed(_engine(sdb, N, kind, N * max(fr)), _split(x, fr, N))
        _assert_psd(oracle, got, x, N, kind, f64=False)     # T is relative to the frame: zero for a zero tap
        for s in range(S):
            assert_impulse(got[s], N, kind, ps[s], amps[s])


@pytest.mark.parametrize("N", [16, 2048, 8192, 65536, 1 << 17, 1 << 20])
def test_shift_db_every_path(sdb, oracle, N):
    """(c) the SHIFT_DB epilogue of every path: bin k lands at (k + N/2) mod N; the output is bit-identical to
    sdb_psd_shift_db_device over the same engine's linear PSD; and every value lies within the bound that SPEC T and
    M.3 give for 10 log10(P + 1e-8): 4.343 tol_T(P) / (P + 1e-8) + 1.5e-6 |dB| + one float32 ulp."""
    fr = _frames(N)
    x = _signal(N * sum(fr), N)
    kind = "blackmann_harris"
    lin = _feed(_engine(sdb, N, kind, N * max(fr)), _split(x, fr, N))
    _assert_psd(oracle, lin, x, N, kind)
    db = _feed(_engine(sdb, N, kind, N * max(fr), flags=sdb.FLAG_PSD_SHIFT_DB), _split(x, fr, N))
    # the device pass over the linear frames
    d_lin = torch.from_numpy(np.ascontiguousarray(lin)).cuda()
    d_db = torch.empty_like(d_lin)
    sdb.psd_shift_db(d_lin.data_ptr(), d_db.data_ptr(), S * lin.shape[1], N)
    torch.cuda.synchronize()
    assert np.array_equal(db.view(np.uint32), d_db.cpu().numpy().view(np.uint32))
    for s in range(S):
        P = pf.psd(x[s], N, kind)
        want = pf.shift_db(P)
        for f in range(P.shape[0]):
            k = int(np.argmax(lin[s, f]))
            assert int(np.argmax(db[s, f])) == (k + N // 2) % N, (N, s, f)
        bound = (4.343 * np.roll(_tol_T(P), N // 2, axis=-1) / (np.roll(P, N // 2, axis=-1) + 1e-8)
                 + 1.5e-6 * np.abs(want) + np.spacing(np.abs(want).astype(np.float32)))
        err = np.abs(db[s].astype(np.float64) - want)
        assert np.all(err <= bound), "N %d stream %d: dB error %.3g x the bound" % (N, s, float(np.max(err / bound)))


# ------------------------------------------------------------------------------------------------------------------
FORMATS = ["f32", "u8", "s8", "s16"]
PATH_SIZES = [64, 2048, 8192, 65536, 1 << 18]


def _raw(fmt, n, seed):
    """[S, n] complex64 (f32) or [S, n, 2] native codes: noise plus a tone per stream, inside full scale"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    iq = []
    for s in range(S):
        z = 0.25 * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) + 0.4 * np.exp(2j * np.pi * (0.07 + 0.3 * s) * t)
        iq.append(np.stack([z.real, z.imag], axis=-1))
    iq = np.clip(np.stack(iq), -0.999, 0.999)
    if fmt == "f32":
        return (iq[..., 0] + 1j * iq[..., 1]).astype(np.complex64)
    if fmt == "u8":
        return np.rint(iq * 128.0 + 128.0).astype(np.uint8)
    if fmt == "s8":
        return np.rint(iq * 128.0).astype(np.int8)
    return np.rint(iq * 32768.0).astype(np.int16)


@pytest.mark.parametrize("N", PATH_SIZES)
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("iq_reverse", [False, True])
def test_input_formats(sdb, oracle, N, fmt, iq_reverse):
    """(d) every sample format with and without FLAG_IQ_REVERSE, one size per path: the oracle and the float64
    statement are fed the samples converted exactly as SPEC Q says"""
    fr = _frames(N)
    raw = _raw(fmt, N * sum(fr), seed=N % 89 + len(fmt))
    xc = pf.convert(raw, fmt, iq_reverse)
    flags = sdb.FLAG_IQ_REVERSE if iq_reverse else 0
    got = _feed(_engine(sdb, N, "hann", N * max(fr), input_format=fmt, flags=flags), _split(raw, fr, N))
    _assert_psd(oracle, got, xc, N, "hann")


@pytest.mark.parametrize("N,fmt", list(zip(PATH_SIZES, ["f32", "u8", "s8", "s16", "f32"])))
def test_device_feed_with_row_stride(sdb, oracle, N, fmt):
    """(d) device feeds whose stream rows lie stride > n samples apart (feed_device_ptr); the gaps hold values that
    would show in the PSD if they were read (NaN for float32, full-scale codes otherwise)"""
    fr = _frames(N)
    raw = _raw(fmt, N * sum(fr), seed=N % 83)
    xc = pf.convert(raw, fmt)
    e = _engine(sdb, N, "flat_top", N * max(fr), input_format=fmt)
    out = []
    for b in _split(raw, fr, N):
        n = b.shape[1]
        stride = n + 48
        pad = np.empty((S, stride) + b.shape[2:], b.dtype)
        if fmt == "f32":
            pad[:] = np.complex64(complex(np.nan, np.nan))
        else:
            pad[:] = np.iinfo(b.dtype).max
        pad[:, :n] = b
        d = torch.from_numpy(pad.view(np.uint8).reshape(S, -1)).cuda()
        e.feed_device_ptr(d.data_ptr(), stride, n)
        e.sync()
        out.append(e.read_psd().copy())
        del d
    e.close()
    _assert_psd(oracle, np.concatenate(out, axis=1), xc, N, "flat_top")


# ------------------------------------------------------------------------------------------------------------------
DC_FEEDS = {16: [48, 80, 336, 1040], 64: [64, 192, 320, 1088]}


@pytest.mark.parametrize("N", [16, 64])
@pytest.mark.parametrize("fmt", ["u8", "s16"])
def test_dc_removal(sdb, oracle, N, fmt):
    """(e) SPEC R before the PSD: feeds shorter than one 256-sample run, with a partial last run and over several runs;
    a different DC offset in each stream.  The PSD must be the oracle's PSD of the float64 statement's corrected
    samples, bit for bit."""
    fs = 1000.0
    feeds = DC_FEEDS[N]
    n = sum(feeds)
    rng = np.random.default_rng(N + len(fmt))
    t = np.arange(n)
    iq = []
    for s, dc in enumerate([0.3 - 0.2j, -0.25 + 0.35j]):
        z = dc + 0.1 * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) + 0.2 * np.exp(2j * np.pi * (0.19 + 0.4 * s) * t)
        iq.append(np.stack([z.real, z.imag], axis=-1))
    iq = np.clip(np.stack(iq), -0.999, 0.999)
    raw = np.rint(iq * 128.0 + 128.0).astype(np.uint8) if fmt == "u8" else np.rint(iq * 32768.0).astype(np.int16)
    xc = pf.convert(raw, fmt)
    cut = np.cumsum([0] + feeds)
    blocks = [np.ascontiguousarray(raw[:, a:b]) for a, b in zip(cut[:-1], cut[1:])]
    corrected = np.stack([np.concatenate(pf.dc_remove([xc[s, a:b] for a, b in zip(cut[:-1], cut[1:])], fs))
                          for s in range(S)])
    e = _engine(sdb, N, "hann", max(feeds), input_format=fmt, flags=sdb.FLAG_DC_REMOVE, samp_rate=fs)
    got = _feed(e, blocks)
    _assert_psd(oracle, got, corrected, N, "hann")
    # the estimate converges on each stream's own offset: the last frame's DC bin is far below the first's
    for s in range(S):
        assert got[s, -1, 0] < 0.2 * got[s, 0, 0], (s, got[s, -1, 0], got[s, 0, 0])


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,fr,kind", [(1 << 18, (17, 3), "flat_top"), (1 << 19, (9, 2), "hamming"),
                                       (1 << 20, (5, 1), "blackmann_harris")])
def test_generic_path_chunk_crossings(sdb, oracle, N, fr, kind):
    """(f) the generic four-step runs S x frames windows through scratch chunks of 64 MB / (8 N) = 32, 16 and 8
    windows: the first feed needs more than one chunk (the last one partial), the second fewer than one"""
    chunk = (64 << 20) // (8 * N)
    assert S * fr[0] > chunk and S * fr[0] % chunk
    x = _signal(N * sum(fr), N)
    got = _feed(_engine(sdb, N, kind, N * max(fr)), _split(x, fr, N))
    _assert_psd(oracle, got, x, N, kind)


def test_psd_and_channeliser_stream_groups(sdb, oracle):
    """(f) psd_size == st_window_size == 2^18 with channels open: the PSD and the channeliser run as two stream chains
    over groups of G = 32 // (frames + windows per stream) = 2 streams, so three streams end in a partial group in
    both feeds.  PSD bit-identical to the oracle and within T of the float64 statement; channels bit-identical to the
    oracle and within tolerance of st_f64."""
    W, n_streams = 1 << 18, 3
    chans = [c for c in st.edge_channels(W) if st.geometry(W, c["f0"], c["bw"], c["guard"])[1] <= 16384]
    feeds = [4 * W, 4 * W]
    x = np.stack([st.signal(sum(feeds), chans, seed=70 + s, noise=0.03 * (s + 1)) for s in range(n_streams)])
    x[1] = x[1][::-1]
    e = sdb.Engine(n_streams=n_streams, psd_size=W, psd_window="hann", st_window_size=W, max_feed=max(feeds))
    hs = [e.open_channel(c["f0"], c["bw"], c["guard"], c.get("precise", False)) for c in chans]
    e.commit()
    psd, acc, off = [], [[[] for _ in hs] for _ in range(n_streams)], 0
    for m in feeds:
        e.feed(x[:, off:off + m])
        off += m
        psd.append(e.read_psd().copy())
        for s in range(n_streams):
            for i, h in enumerate(hs):
                acc[s][i].append(e.read_channel(s, h))
    infos = [e.channel_info(h) for h in hs]
    e.close()
    psd = np.concatenate(psd, axis=1)
    for s in range(n_streams):
        ref = oracle.psd_frames(x[s], W, "hann")
        assert np.array_equal(psd[s].view(np.uint32), ref.view(np.uint32)), s
        parity.assert_psd_close(psd[s], pf.psd(x[s], W, "hann"))
    got = [[np.concatenate(a) for a in acc_s] for acc_s in acc]
    check_channels(oracle, x, W, chans, got, infos)
