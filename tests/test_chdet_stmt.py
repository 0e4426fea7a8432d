"""The CPU oracle's channel detector (oracle/chdetect.c) against the exact statement of SPEC K (tests/chdet_stmt.py).

The CUDA detector is held bit for bit to the oracle; these tests hold the oracle to the SPEC at every N = 16 ... 2^20
over multi-feed scenes at the edges of K (ties at the quartile, zero noise floors, band edges, the 8192-run and
256-channel caps, alpha and gamma at 0 and 1, zero-frame feeds), and show that a statement with one deliberate
mistake is rejected by a named scene."""
import numpy as np
import pytest

import chdet_stmt as cs

SIZES = [1 << k for k in range(4, 21)]

# deliberate mistake -> (scene, N) that must catch it
MISTAKE_CASES = {
    "rank": ("noise_carriers_a0.25_g0.25", 1024),
    "ge": ("constant_snr1", 1024),
    "no_shift": ("edges_dc", 1024),
    "wrap": ("edges_dc", 1024),
    "no_cap": ("alternating", 1 << 15),
}


def oracle_keys(ref):
    return [(a, b) + tuple(int(np.float32(v).view(np.uint32)) for v in (s0, n0, snr)) for a, b, s0, n0, snr in ref]


def run_scene(oracle, N, prm, feeds, mistake=None):
    """Feeds one scene (stream 0) to the oracle and to the statement; returns the list of feeds where they differ
    (empty = bit-identical lists, totals and noise floors)."""
    o = oracle.ChannelDetector(N, prm["alpha"], prm["gamma"], prm["snr"], prm["min_bins"])
    st = cs.Detector(N, prm["alpha"], prm["gamma"], prm["snr"], prm["min_bins"], mistake=mistake)
    bad = []
    try:
        for i, f in enumerate(feeds):
            frames = f[0]
            n0_before = o.d.n0
            ref, rtot = o.feed(frames)
            got, tot = st.feed(frames)
            if len(frames) == 0:
                # K.2: nothing changes -- the oracle returns no list and keeps its total and noise floor
                assert ref == [] and rtot == tot and o.d.n0 == n0_before
                continue
            if tot != rtot or [c.key() for c in got] != oracle_keys(ref) or \
                    np.float32(o.d.n0).view(np.uint32) != np.float32(st.n0).view(np.uint32):
                bad.append(i)
    finally:
        o.close()
    return bad


@pytest.mark.parametrize("N", SIZES)
def test_oracle_equals_statement(oracle, N):
    """Every scene at every size: bins, S0, N0, snr and the total before the cap, bit for bit, feed after feed."""
    for name, prm, feeds in cs.scenes(N):
        assert run_scene(oracle, N, prm, feeds) == [], (N, name)


@pytest.mark.parametrize("mistake", cs.MISTAKES)
def test_statement_mistakes_are_caught(oracle, mistake):
    """Each planted mistake makes its named scene disagree with the oracle, which the correct statement matches."""
    name, N = MISTAKE_CASES[mistake]
    scene = {n: (p, f) for n, p, f in cs.scenes(N)}
    prm, feeds = scene[name]
    assert run_scene(oracle, N, prm, feeds) == []
    assert run_scene(oracle, N, prm, feeds, mistake=mistake) != [], (mistake, name, N)


def test_scene_edges_hold():
    """The scenes reach what they are named for (checked on the statement, which equals the oracle above)."""
    def last(N, name):
        prm, feeds = {n: (p, f) for n, p, f in cs.scenes(N)}[name]
        d = cs.Detector(N, **prm)
        for f in feeds:
            d.feed(f[0])
        return d
    N = 1 << 15
    d = last(N, "alternating")
    assert d.total == cs.MAXRAW and len(d.channels) == cs.CAP
    assert cs.Detector(N, 1.0, 1.0, 100.0, 1, mistake="no_cap").feed(
        {n: f for n, _, f in cs.scenes(N)}["alternating"][0][0])[1] == N // 2
    d = last(1024, "many_channels")
    assert cs.CAP < d.total < 1024 // 3 and all(c.bin_hi - c.bin_lo >= 2 for c in d.channels)
    for N in (16, 1024):
        d = last(N, "edges_dc")
        assert d.channels[0].bin_lo == 0 and d.channels[-1].bin_hi == N       # clipped at both edges
        assert any(c.bin_lo < N // 2 <= c.bin_hi for c in d.channels)         # one run across DC
        d = last(N, "zero_floor")
        assert d.n0 == 0 and d.channels and all(np.isinf(c.snr) for c in d.channels)
        d = last(N, "all_zero")
        assert d.n0 == 0 and d.total == 0
        assert last(N, "constant_snr1").total == 0
        d = last(N, "constant_snr_half")
        assert [(c.bin_lo, c.bin_hi, c.snr) for c in d.channels] == [(0, N, 1.0)]
        d = last(N, "tied_quartile")
        assert d.n0 == 1.0
        d = last(N, "one_bin_runs")
        assert d.total == N // 4 and all(c.bin_hi - c.bin_lo == 1 for c in d.channels[:d.total])


def test_statement_known_answers():
    """Hand-checked lists at N = 16: runs in frequency order, S0 the run's maximum, N0 the 4th smallest value, snr
    S0 / N0 in binary32; the first feed primes both averages; gamma smooths the floor; frequencies in binary64."""
    N = 16
    p = np.arange(1, N + 1, dtype=np.float32)          # avg[k] = k + 1, but avg[3] = 40: N0 = 6, T = 12
    p[3] = 40.0
    d = cs.Detector(N, alpha=0.5, gamma=0.5, snr=2.0, min_bins=1)
    got, tot = d.feed(p)
    # frequency order j = (k + 8) mod 16: k = 12 ... 15 (13 ... 16 > 12) lie at j = 4 ... 7, k = 3 at j = 11
    assert [(c.bin_lo, c.bin_hi, float(c.S0)) for c in got] == [(4, 8, 16.0), (11, 12, 40.0)] and tot == 2
    assert got[0].N0 == 6.0 and got[0].snr == np.float32(16.0) / np.float32(6.0)
    got, _ = d.feed(np.zeros((1, N), np.float32))      # avg halves: N0_inst = 3, N0 = 4.5, T = 9
    assert d.n0 == np.float32(4.5) and [(c.bin_lo, c.bin_hi, float(c.S0)) for c in got] == [(11, 12, 20.0)]
    assert d.feed(np.zeros((0, N), np.float32)) == (got, 1) and d.n0 == np.float32(4.5)
    f_lo, f_hi, fc, bw = cs.frequencies(0, N, N, 2.0e6, 100e6)
    assert (f_lo, f_hi, fc, bw) == (99e6, 101e6, 100e6, 2e6)
    assert cs.frequencies(9, 10, N, 16.0, 0.0) == (1.0, 2.0, 1.5, 1.0)
