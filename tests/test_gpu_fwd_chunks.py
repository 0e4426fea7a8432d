"""-m gpu: forward transforms that run through the four-step scratch in several chunks, bit for bit against the CPU
oracle (psd_frames, specttuner_run).

Every case feeds, in one feed, more windows of an N-point transform than any scratch chunk the engine can size for
it.  That bound is the larger of sms * 65536 / N (the SPEC F.5 rule: 512 KB of windows per SM) and 64 MB / (8 N)
(the rule for every other size), with sms the device's multiprocessor count.  Each case feeds twice, so the
channeliser history and the channel tails carry across feeds, and every stream gets different content."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CHANS = [dict(f0=2 * np.pi * 0.125, bw=2 * np.pi * 0.03, guard=1.0),
         dict(f0=2 * np.pi * 0.0007, bw=2 * np.pi * 0.02, guard=1.0),          # wraps around DC
         dict(f0=2 * np.pi * 0.3301, bw=2 * np.pi * 0.004, guard=2.0, precise=True)]


def _bound(N):
    """Windows in the largest scratch chunk the engine can size for an N-point transform."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return max(sms * 65536 // N, (64 << 20) // (8 * N))


def _prime_above(v):
    p = v + 1
    while any(p % d == 0 for d in range(2, int(p ** 0.5) + 1)):
        p += 1
    return p


def _signal(S, n, seed):
    """[S, n] complex64: noise and two tones, different in every stream."""
    rng = np.random.default_rng(seed)
    x = 0.05 * (rng.standard_normal((S, n)) + 1j * rng.standard_normal((S, n)))
    t = np.arange(n)
    for s in range(S):
        x[s] += 0.4 * np.exp(2j * np.pi * (0.125 + 1e-4 * s) * t) + 0.2 * np.exp(2j * np.pi * (0.33 - 1e-4 * s) * t)
    return x.astype(np.complex64)


def _run_check(sdb, oracle, x, feeds, psd_size, W, chans, window="hann"):
    """Feed x [S, n] in blocks of `feeds` samples and compare every PSD frame and channel sample with the oracle."""
    S = x.shape[0]
    assert sum(feeds) == x.shape[1]
    e = sdb.Engine(n_streams=S, psd_size=psd_size, psd_window=window, st_window_size=W, max_feed=max(feeds))
    hs = [e.open_channel(c["f0"], c["bw"], c["guard"], c.get("precise", False)) for c in chans]
    e.commit()
    psd, ch = [], [[[] for _ in hs] for _ in range(S)]
    off = 0
    for m in feeds:
        e.feed(x[:, off:off + m])
        off += m
        if psd_size:
            psd.append(e.read_psd().copy())
        for s in range(S):
            for i, h in enumerate(hs):
                ch[s][i].append(e.read_channel(s, h))
    e.close()
    for s in range(S):
        if psd_size:
            got = np.concatenate([p[s] for p in psd])
            ref = oracle.psd_frames(x[s], psd_size, window)
            assert got.shape == ref.shape, (s, got.shape, ref.shape)
            assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), "stream %d: PSD" % s
        for i, r in enumerate(oracle.specttuner_run(x[s], W, chans) if chans else []):
            got = np.concatenate(ch[s][i])
            assert len(got) == len(r) and len(r) > 0, (s, i, len(got), len(r))
            assert np.array_equal(got.view(np.uint32), r.view(np.uint32)), "stream %d channel %d" % (s, i)


def test_psd_and_channeliser_stream_groups_32768(sdb, oracle):
    """psd_size == st_window_size == 32768: the PSD frames and channeliser windows of a group of streams run side by
    side, each in its part of the scratch.  The second feed holds 3 PSD frames and 6 channeliser windows per stream;
    S is a prime with S * 9 above the bound, so the streams need at least two groups and the last one is partial."""
    N = 32768
    windows = 3 + 6
    S = _prime_above(_bound(N) // windows)
    assert S * windows > _bound(N)
    feeds = [2 * N, 3 * N]
    x = _signal(S, sum(feeds), seed=21)
    _run_check(sdb, oracle, x, feeds, N, N, CHANS)


def test_psd_only_8192_partial_last_chunk(sdb, oracle):
    """8192-point PSD frames only (SPEC F.5): an odd number of frames in the second feed, so every chunk size the
    engine can pick (an even number of windows) leaves a partial last chunk."""
    N, S = 8192, 3
    frames = _bound(N) // S + 1
    frames += 1 - frames % 2
    assert S * frames > _bound(N) and (S * frames) % 2 == 1
    feeds = [5 * N, frames * N]
    x = _signal(S, sum(feeds), seed=22)
    _run_check(sdb, oracle, x, feeds, N, 0, [], window="blackmann_harris")


def test_stockham_psd_131072_channeliser_4096(sdb, oracle):
    """131072-point PSD frames beside 4096-point channeliser windows: both take the generic four-step path through a
    scratch sized for the larger transform, and both cross chunks in the second feed."""
    Np, W, S = 131072, 4096, 3
    frames = _bound(Np) // S + 1
    assert S * frames > _bound(Np) and S * (frames * Np // (W // 2)) > _bound(W)
    feeds = [Np, frames * Np]
    x = _signal(S, sum(feeds), seed=23)
    _run_check(sdb, oracle, x, feeds, Np, W, CHANS)
