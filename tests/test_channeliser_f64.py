"""The CPU oracle's channeliser (oracle/specttuner.c) against the float64 statement of SPEC S (tests/st_f64.py).

The GPU channeliser is held bit for bit to the oracle; these tests hold the oracle to the SPEC, so that a mistake
shared by both sides -- a sideband bin in the wrong slot, the wrong half of the previous hop in the cross-fade, a
wrong weight at the band edge, a wrong `precise` residual -- cannot pass unnoticed.  Known-answer tests keep the
float64 statement itself honest."""
import numpy as np
import pytest

import parity
import st_f64 as st

WINDOWS = [64, 256, 1024, 4096, 8192, 16384, 32768, 65536]


def _hops(N):
    return 24 if N <= 1024 else (12 if N <= 8192 else 6)


@pytest.mark.parametrize("N", WINDOWS)
def test_oracle_matches_f64_statement(oracle, N):
    chans = st.edge_channels(N)
    hops = _hops(N)
    x = st.signal(N // 2 * hops, chans, seed=N % 101)
    x_rms = float(np.sqrt(np.mean(np.abs(x.astype(np.complex128)) ** 2)))
    got = oracle.specttuner_run(x, N, chans)
    for c, g in zip(chans, got):
        center, size, width = st.geometry(N, c["f0"], c["bw"], c["guard"])
        assert (center, size, width) == oracle.channel_geometry(N, c["f0"], c["bw"], c["guard"]), c
        ref = st.channel(x, N, c["f0"], c["bw"], c["guard"], c.get("precise", False))
        assert len(g) == len(ref) == (hops - 1) * size // 2, (c, len(g), len(ref))
        parity.assert_channel_close(g, ref, x_rms, N / size)


def test_edge_geometry(oracle):
    """The edge set really reaches the edges it names, at every window."""
    for N in WINDOWS:
        g = [st.geometry(N, c["f0"], c["bw"], c["guard"]) for c in st.edge_channels(N)]
        assert g[2][0] == 0                                   # centre wrapped to bin 0
        assert g[5][1] == N and g[5][2] == N                  # full band
        assert g[6][2] == 2                                   # minimum width
        assert g[3][0] > N // 2 and g[3][0] + g[3][2] // 2 > N    # above DC, reaching across it
        assert g[4][0] < g[4][2] // 2                          # below DC, reaching across it
        assert abs(g[9][0] - g[0][0]) < g[0][2] // 2          # overlapping channels
        r = [st.lo_omega(N, c["f0"], gg[0], gg[1]) for c, gg in zip(st.edge_channels(N)[10:], g[10:])]
        assert r[0] > 0 and r[1] < 0 and r[2] < 0             # residual signs of the precise channels
    assert any(g[2] % 2 for N in WINDOWS for g in [st.geometry(N, c["f0"], c["bw"], c["guard"])
                                                   for c in st.edge_channels(N)])     # some odd width


@pytest.mark.parametrize("N", [64, 4096])
def test_f64_statement_tone_known_answer(oracle, N):
    """A tone on bin center + j comes out as A exp(2 pi i j t / size) -- frequency j D / N per channel sample, unity
    gain -- once the first half window has passed, for every pass-band bin j (h = 1 three bins in from the edges)."""
    f0, bw = st.f32(2 * np.pi * 0.25), st.f32(2 * np.pi * 0.2)
    center, size, width = st.geometry(N, f0, bw, 1.0)
    halfw, hs, hops = width // 2, size // 2, 8
    t = np.arange(N // 2 * hops)
    for j in sorted({-halfw + 3, -1, 0, 1, min(halfw // 2, halfw - 4), halfw - 4}):
        A = 0.5 * np.exp(0.3j)
        x = A * np.exp(2j * np.pi * (center + j) * t / N)
        y = st.channel(x, N, f0, bw, 1.0)
        assert len(y) == (hops - 1) * hs
        tt = np.arange(hs, len(y))
        np.testing.assert_allclose(y[hs:], A * np.exp(2j * np.pi * j * tt / size), rtol=0, atol=1e-10)
        # and the oracle on the float32 tone
        yo = oracle.specttuner_run(x.astype(np.complex64), N, [dict(f0=f0, bw=bw, guard=1.0)])[0]
        assert np.max(np.abs(yo[hs:] - y[hs:])) < 2e-6


def test_f64_statement_precise_known_answer(oracle):
    """`precise` on a tone at f0 on an odd bin, one bin off the even centre: the LO takes the residual out and leaves
    the constant A (up to the drift of the float32 phase accumulator)."""
    N, hops = 4096, 16
    t = np.arange(N // 2 * hops)
    signs = set()
    for k in (601, 1003, 2047, N - 1):                     # N - 1: the centre wraps to bin 0
        f0 = st.f32(2 * np.pi * k / N)
        center, size, _ = st.geometry(N, f0, st.f32(2 * np.pi * 0.01), 2.0)
        r = k - (center if center else N)
        assert abs(r) == 1
        signs.add(r)
        A = 0.4 * np.exp(-1.1j)
        x = A * np.exp(1j * f0 * t)
        y = st.channel(x, N, f0, st.f32(2 * np.pi * 0.01), 2.0, precise=True)
        yn = st.channel(x, N, f0, st.f32(2 * np.pi * 0.01), 2.0)
        phi = st.lo_phases(st.lo_omega(N, f0, center, size), len(y)).astype(np.float64)
        np.testing.assert_allclose(y, yn * np.exp(-1j * phi), rtol=0, atol=1e-14)
        hs = size // 2
        # the residual is r bins: omega = 2 pi r / size per channel sample (up to the float32 rounding of f0, times
        # the decimation); phi accumulates it in float32
        assert abs(float(st.lo_omega(N, f0, center, size)) - 2 * np.pi * r / size) < 1e-5
        assert np.max(np.abs(y[hs:] - A)) < 2e-3 * abs(A)
        yo = oracle.specttuner_run(x.astype(np.complex64), N,
                                   [dict(f0=f0, bw=st.f32(2 * np.pi * 0.01), guard=2.0, precise=True)])[0]
        parity.assert_channel_close(yo, y, abs(A), N / size)
    assert signs == {1, -1}


def test_f64_statement_weights():
    """S.3 weights: unity inside, the 7-tap Blackman-Harris roll-off over the last 3 + 4 bins of each edge, k = 1/N,
    and h = 1 without a roll-off for a channel spanning the band."""
    N, halfw = 4096, 20
    kh = st.weights(N, halfw) * N
    assert np.all(np.abs(kh[3:-3] - 1.0) < 1e-15)             # bins -halfw + 3 .. halfw - 4
    assert abs(kh[2] - (1.0 - st.BH_C[3])) < 1e-15 and abs(kh[-3] - (1.0 - st.BH_C[3])) < 1e-15
    assert abs(kh[0] - sum(st.BH_C)) < 1e-15                  # bin -halfw: only m = -3 .. 0 land inside
    np.testing.assert_allclose(kh, kh[::-1], rtol=0, atol=1e-15)   # h[b] = h[-1 - b]
    assert np.all(st.weights(64, 32) == 1.0 / 64)


@pytest.mark.parametrize("N,chunks", [(64, [1, 7, 32, 100]), (4096, [1000, 777, 2048, 6000])])
def test_oracle_length_and_chunked_feeding(oracle, N, chunks):
    """The output length is (half windows - 1) size / 2 whatever the feed sizes, and feeding in chunks gives the
    same samples bit for bit."""
    chans = st.edge_channels(N)
    for half_windows in (2, 3, 9):
        n = N // 2 * half_windows
        x = st.signal(n, chans, seed=half_windows)
        whole = oracle.specttuner_run(x, N, chans)
        for c, y in zip(chans, whole):
            assert len(y) == (half_windows - 1) * st.geometry(N, c["f0"], c["bw"], c["guard"])[1] // 2
        for ch in chunks:
            part = oracle.specttuner_run(x, N, chans, chunk=ch)
            for a, b in zip(whole, part):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), ch
    assert len(oracle.specttuner_run(np.zeros(N - 1, np.complex64), N, chans)[0]) == 0
