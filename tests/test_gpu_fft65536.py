"""-m gpu: the fused 65536-point transform (one thread-block cluster per window, PSD frames and channeliser windows
of a feed in one launch) against the CPU oracle, bit for bit: several streams, the first feed (no channeliser
window 0) and later ones, engines with one kind of window or both, a 65536-point PSD beside an 8192-point
channeliser, and 8 / 16-bit input with I/Q reversal and DC removal."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 65536
CHANS = [dict(f0=2 * np.pi * 0.125, bw=2 * np.pi * 0.03, guard=1.0),
         dict(f0=2 * np.pi * 0.0007, bw=2 * np.pi * 0.02, guard=1.0),          # wraps around DC
         dict(f0=2 * np.pi * 0.3301, bw=2 * np.pi * 0.004, guard=2.0, precise=True)]


def _signal(S, n, seed):
    rng = np.random.default_rng(seed)
    x = 0.05 * (rng.standard_normal((S, n)) + 1j * rng.standard_normal((S, n)))
    t = np.arange(n)
    for s in range(S):                                  # a different tone per stream: a misplaced window shows
        x[s] += 0.4 * np.exp(2j * np.pi * (0.125 + 1e-4 * s) * t) + 0.2 * np.exp(2j * np.pi * (0.33 - 1e-4 * s) * t)
    return x.astype(np.complex64)


def _run(sdb, feeds, S, psd_size, W, chans, window="hann", **kw):
    """Feed the blocks in turn; returns (PSD frames [S, F, psd_size] or None, channel samples [S][channel])."""
    e = sdb.Engine(n_streams=S, psd_size=psd_size, psd_window=window, st_window_size=W,
                   max_feed=max(b.shape[1] for b in feeds), **kw)
    hs = [e.open_channel(c["f0"], c["bw"], c["guard"], c.get("precise", False)) for c in chans]
    e.commit()
    psd, ch = [], [[[] for _ in hs] for _ in range(S)]
    for b in feeds:
        e.feed(b)
        if psd_size:
            psd.append(e.read_psd().copy())
        for s in range(S):
            for i, h in enumerate(hs):
                ch[s][i].append(e.read_channel(s, h))
    cat = lambda a: np.concatenate(a) if a else np.zeros(0, np.complex64)
    return (np.concatenate(psd, axis=1) if psd_size else None), [[cat(a) for a in c] for c in ch]


def _check(oracle, x, psd, ch, psd_size, W, chans, window="hann"):
    """x: [S, n] complex64, exactly the samples the transforms saw."""
    for s in range(x.shape[0]):
        if psd_size:
            ref = oracle.psd_frames(x[s], psd_size, window)
            assert np.array_equal(psd[s].view(np.uint32), ref.view(np.uint32)), "stream %d: PSD" % s
        if chans:
            for i, r in enumerate(oracle.specttuner_run(x[s], W, chans)):
                assert len(ch[s][i]) == len(r) and len(r) > 0, (s, i, len(ch[s][i]), len(r))
                assert np.array_equal(ch[s][i].view(np.uint32), r.view(np.uint32)), "stream %d channel %d" % (s, i)


def _split(x, sizes):
    out, off = [], 0
    for m in sizes:
        out.append(x[:, off:off + m])
        off += m
    return out


@pytest.mark.parametrize("S", [1, 5, 133])
def test_psd_and_channeliser_in_one_launch(sdb, oracle, S):
    """psd_size == st_window_size == 65536: first feed (PSD frame 0, channeliser window 1), then a feed with
    channeliser window 0 and two PSD frames."""
    x = _signal(S, 3 * N, seed=S)
    chans = CHANS if S < 100 else CHANS[:1]
    psd, ch = _run(sdb, _split(x, [N, 2 * N]), S, N, 0, chans)
    _check(oracle, x, psd, ch, N, N, chans)


def test_psd_only(sdb, oracle):
    S = 3
    x = _signal(S, 4 * N, seed=11)
    psd, ch = _run(sdb, _split(x, [N, 3 * N]), S, N, 0, [], window="blackmann_harris")
    _check(oracle, x, psd, ch, N, N, [], window="blackmann_harris")


def test_channeliser_only(sdb, oracle):
    """No PSD: the first feed of half a window forms no window at all, later feeds odd and even counts."""
    S = 3
    x = _signal(S, 4 * N, seed=12)
    psd, ch = _run(sdb, _split(x, [N // 2, N, 3 * N // 2, N]), S, 0, N, CHANS)
    _check(oracle, x, psd, ch, 0, N, CHANS)


def test_psd_65536_beside_channeliser_8192(sdb, oracle):
    """The PSD frames take the fused kernel, the 8192-point channeliser windows the two-kernel path."""
    S = 3
    x = _signal(S, 3 * N, seed=13)
    psd, ch = _run(sdb, _split(x, [N, 2 * N]), S, N, 8192, CHANS)
    _check(oracle, x, psd, ch, N, 8192, CHANS)


def _dc_oracle(oracle, blocks, fs):
    L = oracle.lib()
    c = (C.c_float * 2)(0.0, 0.0)
    out = []
    for b in blocks:
        b = np.ascontiguousarray(b, np.complex64)
        y = np.empty_like(b)
        alpha = np.float32(1.0 - np.exp(-len(b) / (fs * 0.1)))
        L.sdo_dc_remove(c, oracle.ptr(b), oracle.ptr(y), C.c_size_t(len(b)), C.c_float(float(alpha)))
        out.append(y)
    return np.concatenate(out)


@pytest.mark.parametrize("fmt", ["s16", "u8"])
@pytest.mark.parametrize("dc", [False, True])
def test_native_format_iq_reverse(sdb, oracle, fmt, dc):
    """8 / 16-bit samples converted and I/Q-swapped in the transform's load (or, with DC removal, in the DC pass)."""
    S, fs = 2, 1.0e6
    sizes = [N, 2 * N]
    xf = _signal(S, sum(sizes), seed=14) + np.complex64(0.05 - 0.03j)
    iq = np.stack([xf.real, xf.imag], axis=-1)
    if fmt == "u8":
        q = np.clip(np.rint(iq * 128.0 + 128.0), 0, 255).astype(np.uint8)
        back = (q.astype(np.float32) - 128.0) / 128.0
    else:
        q = np.clip(np.rint(iq * 32768.0), -32768, 32767).astype(np.int16)
        back = q.astype(np.float32) / 32768.0
    x = (back[..., 1] + 1j * back[..., 0]).astype(np.complex64)      # (Q, I): what the transforms must see
    flags = sdb.FLAG_IQ_REVERSE | (sdb.FLAG_DC_REMOVE if dc else 0)
    feeds = []
    off = 0
    for m in sizes:
        feeds.append(q[:, off:off + m])
        off += m
    psd, ch = _run(sdb, feeds, S, N, 0, CHANS, input_format=fmt, flags=flags, samp_rate=fs)
    if dc:
        x = np.stack([_dc_oracle(oracle, [x[s, :N], x[s, N:]], fs) for s in range(S)])
    _check(oracle, x, psd, ch, N, N, CHANS)
