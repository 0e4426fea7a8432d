"""-m gpu: the channeliser at every window size, channel size and band edge.  Every channel's samples must be
bit-identical to the CPU oracle, within tolerance of the float64 statement of SPEC S (tests/st_f64.py), and
(half windows fed - 1) x size / 2 long.

Inverse-side kernels by channel size (sdb_launch_chan_ifft_group): 4 ... 256 k_chan_ifft<1> (CTAs of at least one
warp, so channels below 128 points leave threads idle), 512 ... 4096 k_chan_ifft16 (P = 8 / 4 / 2 / 1 hops per round,
the last round of a feed partial), 8192 k_chan_ifft<2>, 16384 k_chan_ifft<4>.  Forward side by window: <= 4096 and
131072 ... 1048576 the generic four-step, 8192 / 16384 / 32768 SPEC F.5 (bins compacted through the ka mask), 65536 the
fused cluster kernel."""
import numpy as np
import pytest

import parity
import st_f64 as st

pytestmark = pytest.mark.gpu

MAX_SIZE = 16384          # largest channel the engine opens


def _run(sdb, x, W, chans, feeds):
    """x: [S, n] complex64, fed in blocks of `feeds` samples -> (samples [S][channel], channel infos)."""
    S = x.shape[0]
    assert sum(feeds) == x.shape[1]
    e = sdb.Engine(n_streams=S, psd_size=0, st_window_size=W, max_feed=max(feeds))
    hs = [e.open_channel(c["f0"], c["bw"], c["guard"], c.get("precise", False)) for c in chans]
    e.commit()
    acc = [[[] for _ in hs] for _ in range(S)]
    off = 0
    for m in feeds:
        e.feed(x[:, off:off + m])
        off += m
        for s in range(S):
            for i, h in enumerate(hs):
                acc[s][i].append(e.read_channel(s, h))
    infos = [e.channel_info(h) for h in hs]
    e.close()
    return [[np.concatenate(a) for a in acc_s] for acc_s in acc], infos


def _check(oracle, x, W, chans, got, infos):
    half_windows = x.shape[1] // (W // 2)
    for s in range(x.shape[0]):
        ref = oracle.specttuner_run(x[s], W, chans)
        X = st.spectra(x[s], W)
        x_rms = float(np.sqrt(np.mean(np.abs(x[s].astype(np.complex128)) ** 2)))
        for i, (c, info) in enumerate(zip(chans, infos)):
            center, size, width = st.geometry(W, c["f0"], c["bw"], c["guard"])
            assert (info.center, info.size, info.width) == (center, size, width), (W, c)
            g, r = got[s][i], ref[i]
            assert len(g) == len(r) == (half_windows - 1) * size // 2, (W, s, c, len(g), len(r))
            assert np.array_equal(g.view(np.uint32), r.view(np.uint32)), \
                "W %d stream %d channel %d (size %d): not bit-identical to the oracle, max |d| = %g" % (
                    W, s, i, size, float(np.max(np.abs(g - r))) if len(g) else 0.0)
            f64 = st.channel(x[s], W, c["f0"], c["bw"], c["guard"], c.get("precise", False), X=X)
            parity.assert_channel_close(g, f64, x_rms, W / size)


def _sized(W, sizes, precise=()):
    """One channel per size, spread over the band (guard 1, bw 3/4 of the size: S.2 rounds it up to exactly that
    size)."""
    out = []
    for k, sz in enumerate(sizes):
        f0 = st.f32((0.037 + 0.071 * k) % 1.0 * st.TWO_PI)
        out.append(dict(f0=f0, bw=st.f32(st.TWO_PI * 0.75 * sz / W), guard=1.0, precise=sz in precise))
    return out


# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [64, 256, 1024, 4096, 8192, 16384, 32768, 65536, 131072, 262144, 524288, 1048576])
def test_band_edges_every_window(sdb, oracle, W):
    """DC, centres wrapping to 0, channels straddling DC from each side, full band (W <= 16384), minimum width,
    odd widths, overlapping channels, `precise` with both residual signs and a wrapped centre.  The first feed is
    three half windows (two transforms), the second the rest: the tails and LO phases carry across."""
    chans = [c for c in st.edge_channels(W) if st.geometry(W, c["f0"], c["bw"], c["guard"])[1] <= MAX_SIZE]
    half = 24 if W <= 4096 else (10 if W <= 65536 else 6)
    x = st.signal(W // 2 * half, chans, seed=W % 97)[None, :]
    feeds = [W // 2 * 3, W // 2 * (half - 3)]
    got, infos = _run(sdb, x, W, chans, feeds)
    _check(oracle, x, W, chans, got, infos)


@pytest.mark.parametrize("W", [16384, 32768, 65536])
def test_every_channel_size(sdb, oracle, W):
    """Every power of two from 4 to 16384 in one engine (every kernel of the inverse side at once); 64, 1024, 8192
    and 16384 as `precise` channels."""
    sizes = [1 << k for k in range(2, 15) if (1 << k) <= W]
    chans = _sized(W, sizes, precise=(64, 1024, 8192, 16384))
    half = 8 if W < 65536 else 6
    x = st.signal(W // 2 * half, chans, seed=W % 89)[None, :]
    got, infos = _run(sdb, x, W, chans, [W // 2 * 2, W // 2 * (half - 2)])
    assert sorted(i.size for i in infos) == sizes
    _check(oracle, x, W, chans, got, infos)


def test_full_band_size_16384(sdb, oracle):
    """A full-band channel at W = 16384 and a 20 %-wide one at W = 65536 are both 16384-point channels."""
    for W, chans in [(16384, [dict(f0=0.0, bw=st.f32(st.TWO_PI), guard=1.0),
                              dict(f0=st.f32(st.TWO_PI * 0.3), bw=st.f32(st.TWO_PI), guard=1.0, precise=True)]),
                     (65536, [dict(f0=st.f32(st.TWO_PI * 0.2), bw=st.f32(st.TWO_PI * 0.2), guard=1.0),
                              dict(f0=st.f32(st.TWO_PI * 0.9), bw=st.f32(st.TWO_PI * 0.2), guard=1.0, precise=True)])]:
        x = st.signal(W // 2 * 6, chans, seed=3)[None, :]
        got, infos = _run(sdb, x, W, chans, [W, W * 2])
        assert all(i.size == MAX_SIZE for i in infos)
        _check(oracle, x, W, chans, got, infos)


def test_ifft16_partial_rounds_three_streams(sdb, oracle):
    """k_chan_ifft16 transforms P = 4096 / size hops per round.  Feeds of 3, 5, 9 and 1 windows give sizes 512 (P = 8),
    1024 (P = 4) and 2048 (P = 2) a last round with fewer hops than P and one of P + 1 hops.  Three streams with
    different content."""
    W, S = 8192, 3
    chans = _sized(W, [512, 1024, 2048, 4096]) + _sized(W, [512, 1024, 2048], precise=(512, 1024, 2048))[::-1]
    windows = [3, 5, 9, 1]                                  # per feed; the first feed also primes the first half
    feeds = [W // 2 * (windows[0] + 1)] + [W // 2 * w for w in windows[1:]]
    x = np.stack([st.signal(sum(feeds), chans, seed=40 + s, noise=0.03 * (s + 1)) for s in range(S)])
    x[1] = x[1][::-1]                                       # a different spectrum in every stream
    got, infos = _run(sdb, x, W, chans, feeds)
    _check(oracle, x, W, chans, got, infos)


@pytest.mark.parametrize("W,ka_shift", [(8192, 5), (16384, 6), (32768, 7), (65536, 8)])
def test_narrow_channel_in_one_ka_group(sdb, oracle, W, ka_shift):
    """A single narrow channel whose bins all fall in one ka group: the row pass of the forward transform computes
    only the groups the mask names."""
    center = (5 << ka_shift) + (1 << (ka_shift - 1))
    chans = [dict(f0=st.f32(st.TWO_PI * center / W), bw=st.f32(st.TWO_PI * 6 / W), guard=1.0)]
    c, size, width = st.geometry(W, chans[0]["f0"], chans[0]["bw"], 1.0)
    assert {((c + b) % W) >> ka_shift & 15 for b in range(-(width // 2), width // 2)} == {5}
    x = st.signal(W // 2 * 8, chans, seed=ka_shift)[None, :]
    got, infos = _run(sdb, x, W, chans, [W // 2 * 3, W // 2 * 5])
    _check(oracle, x, W, chans, got, infos)


def test_size_limit(sdb, oracle):
    """A channel wider than 16384 bins is refused with its reason; the engine stays usable."""
    W = 65536
    e = sdb.Engine(n_streams=1, psd_size=0, st_window_size=W, max_feed=W * 2)
    with pytest.raises(sdb.SdbError, match="channel size > 16384"):
        e.open_channel(st.f32(st.TWO_PI * 0.5), st.f32(st.TWO_PI * 0.3), 1.0)     # size 32768
    chans = [dict(f0=st.f32(st.TWO_PI * 0.5), bw=st.f32(st.TWO_PI * 0.2), guard=1.0)]
    h = e.open_channel(chans[0]["f0"], chans[0]["bw"], 1.0)
    assert h == 0
    e.commit()
    x = st.signal(W * 2, chans, seed=9)[None, :]
    e.feed(x)
    got = [[e.read_channel(0, h)]]
    infos = [e.channel_info(h)]
    e.close()
    _check(oracle, x, W, chans, got, infos)


# the windows of one feed counted here are those of its single stream; each case names the count and the PSD size
LIMIT_CASES = [(128, 65535, 0), (128, 65535, 4096), (128, 65536, 0), (128, 65536, 4096), (64, 65536, 0),
               (64, 65536, 4096), (64, 131072, 0), (64, 131072, 4096), (64, 131073, 0), (64, 131071, 4096)]


def _limit_feeds(W, windows, psd_size):
    """Feeds (samples) whose first or second one holds exactly `windows` forward transforms.  The first feed also
    primes the first half window; with a 4096-point PSD every feed is a multiple of 4096 samples, so a count arrives
    in the first feed (4096 k / hop - 1 windows) or in the second (4096 k / hop)."""
    hop = W // 2
    unit = max(hop, psd_size)
    if (windows + 1) * hop % unit == 0:
        return [(windows + 1) * hop, unit]
    assert windows * hop % unit == 0, (W, windows, psd_size)
    return [unit, windows * hop]


@pytest.mark.parametrize("W,windows,psd_size", LIMIT_CASES)
def test_small_window_feeds_past_the_grid_y_limit(sdb, oracle, W, windows, psd_size):
    """64- and 128-point windows run on the generic four-step, whose scratch chunk is sized in bytes (64 MB: 131072
    or 65536 such windows) while both of its kernels put the window on grid.y, limited to 65535.  Feeds of 65535,
    65536, 131071, 131072 and 131073 windows, with no PSD and next to a 4096-point PSD (which takes the small-PSD path,
    so the channeliser owns the scratch): every channel bit-identical to the oracle and within tolerance of st_f64."""
    chans = [st.edge_channels(W)[i] for i in (0, 3, 11)]           # plain, straddling DC, `precise`
    feeds = _limit_feeds(W, windows, psd_size)
    x = st.signal(sum(feeds), chans, seed=windows % 61)[None, :]
    e = sdb.Engine(n_streams=1, psd_size=psd_size, psd_window="hann", st_window_size=W, max_feed=max(feeds))
    hs = [e.open_channel(c["f0"], c["bw"], c["guard"], c.get("precise", False)) for c in chans]
    e.commit()
    acc, off, psd = [[] for _ in hs], 0, []
    for m in feeds:
        e.feed(x[:, off:off + m])
        off += m
        for i, h in enumerate(hs):
            acc[i].append(e.read_channel(0, h))
        if psd_size:
            psd.append(e.read_psd()[0].copy())
    infos = [e.channel_info(h) for h in hs]
    e.close()
    assert windows in (feeds[0] // (W // 2) - 1, feeds[1] // (W // 2))
    _check(oracle, x, W, chans, [[np.concatenate(a) for a in acc]], infos)
    if psd_size:
        ref = oracle.psd_frames(x[0], psd_size, "hann")
        assert np.array_equal(np.concatenate(psd).view(np.uint32), ref.view(np.uint32))
